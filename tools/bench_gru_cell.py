"""``GRUCell`` against ``torch.nn.GRUCell`` and against ``GRU`` called with T = 1, at I = 64, H = 256 and B in {1, 32, 512}.

Paths: ``GRUCell`` at bf16x3, bf16 and fp32; nn.GRUCell on CUDA at torch defaults (fp32) and with TF32 allowed; ``GRU(x[:, None],
hx)`` at bf16x3 and fp32 (``GRU`` refuses ``hx`` at bf16, so it has no stepping path there).  Cases, each with ``hx`` given:
  * step_forward: one no_grad step;
  * step_forward_backward: one step with grad, backward of a fixed random gradient of h';
  * loop128_forward_backward: 128 steps feeding h' back, a loss on every step, one backward through all of them.
Per path and case: ms per call from CUDA events over windows of at least --window seconds, --repeats windows each, paths in
rotating order (median, min, max), and the peak ``torch.cuda.max_memory_allocated`` of one call.  Per path: the one-step
output's rel-L2 error against float64 nn.GRUCell on the CPU.  The card's name, power limit and maximum SM clock are read in
the same run.

    python tools/bench_gru_cell.py [--out DIR] [--window 0.5] [--repeats 5]      (writes DIR/bench_gru_cell.json)"""
import argparse
import json
import os
import sys

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from financial_market_data_analysis_b200 import GRU, GRUCell   # noqa: E402
from bench_gru import peak_bytes                               # noqa: E402
from bench_lengths import card, time_window                    # noqa: E402

I, H, BATCHES, LOOP = 64, 256, (1, 32, 512), 128


class _Tf32(nn.Module):
    """nn.GRUCell with TF32 allowed for its matmuls during the call only."""

    def __init__(self, cell):
        super().__init__()
        self.cell = cell

    def forward(self, x, h):
        was = torch.backends.cuda.matmul.allow_tf32
        torch.backends.cuda.matmul.allow_tf32 = True
        try:
            return self.cell(x, h)
        finally:
            torch.backends.cuda.matmul.allow_tf32 = was


class _Step(nn.Module):
    """GRU called with T = 1: h' = GRU(x[:, None], h[None])."""

    def __init__(self, gru):
        super().__init__()
        self.gru = gru

    def forward(self, x, h):
        return self.gru(x[:, None], h[None])[1][0]


def paths():
    torch.manual_seed(0)
    ref = nn.GRUCell(I, H).cuda()
    sd = ref.state_dict()
    tf = nn.GRUCell(I, H).cuda()
    tf.load_state_dict(sd)
    out = {"torch_fp32": ref, "torch_tf32": _Tf32(tf)}
    for prec in ("bf16x3", "bf16", "fp32"):
        m = GRUCell(I, H, precision=prec).cuda()
        m.load_state_dict(sd)
        out[f"cell_{prec}"] = m
    for prec in ("bf16x3", "fp32"):
        g = GRU(I, H, 1, batch_first=True, precision=prec).cuda()
        g.load_state_dict({k + "_l0": v for k, v in sd.items()})
        out[f"gru_t1_{prec}"] = _Step(g)
    return out


def measure(calls, window, repeats):
    per = {}
    for name, fn in calls.items():
        time_window(fn, 3)
        per[name] = max(1, int(window * 1e3 / time_window(fn, 3)) + 1)
    samples = {name: [] for name in calls}
    names = list(calls)
    for r in range(repeats):
        for name in names[r % len(names):] + names[:r % len(names)]:
            samples[name].append(time_window(calls[name], per[name]))
    out = {}
    for name, s in samples.items():
        s = sorted(s)
        out[name] = {"ms_median": s[len(s) // 2], "ms_min": s[0], "ms_max": s[-1], "calls_per_window": per[name], "windows": len(s)}
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--out", default="bench_gru_cell_out")
    ap.add_argument("--window", type=float, default=0.5, help="seconds of work per timed window")
    ap.add_argument("--repeats", type=int, default=5, help="timed windows per path")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_gru_cell needs a CUDA device (an H100); there is nothing to measure without one")
    info = {"card": card(), "torch": torch.__version__, "shape": dict(I=I, H=H, loop_steps=LOOP), "window_s": a.window,
            "repeats": a.repeats, "batches": {}}
    mods = paths()
    for B in BATCHES:
        g = torch.Generator().manual_seed(B)
        x, h = torch.randn(B, I, generator=g), 0.5 * torch.randn(B, H, generator=g)
        xs = 0.5 * torch.randn(LOOP, B, I, generator=g)
        dy, w = torch.randn(B, H, generator=g), torch.randn(LOOP, B, H, generator=g)
        ref = nn.GRUCell(I, H).double()
        ref.load_state_dict({k: v.double().cpu() for k, v in mods["torch_fp32"].state_dict().items()})
        with torch.no_grad():
            want = ref(x.double(), h.double())
        x, h, xs, dy, w = x.cuda(), h.cuda(), xs.cuda(), dy.cuda(), w.cuda()

        def fwd(m):
            with torch.no_grad():
                return m(x, h)

        def step(m):
            xi, hi = x.clone().requires_grad_(), h.clone().requires_grad_()
            m(xi, hi).backward(dy)

        def loop(m):
            hc, loss = h, 0.0
            for t in range(LOOP):
                hc = m(xs[t], hc)
                loss = loss + (hc * w[t]).sum()
            loss.backward()

        err = {n: float((fwd(m).double().cpu() - want).norm() / want.norm()) for n, m in mods.items()}
        cases = {}
        for case, fn in (("step_forward", fwd), ("step_forward_backward", step), ("loop128_forward_backward", loop)):
            calls = {n: (lambda m=m: fn(m)) for n, m in mods.items()}
            res = measure(calls, a.window, a.repeats)
            for n, m in mods.items():
                m.zero_grad(set_to_none=True)
                res[n]["peak_bytes"] = peak_bytes(calls[n])
            cases[case] = res
        info["batches"][str(B)] = {"output_rel_l2_vs_fp64": err, **cases}
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "bench_gru_cell.json"), "w") as f:
        json.dump(info, f, indent=1)
    print(json.dumps(info))


if __name__ == "__main__":
    main()
