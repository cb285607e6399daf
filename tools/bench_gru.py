"""``GRU`` against ``torch.nn.GRU`` at configs[1]'s recurrence (B512 T128 F64 H256 L2, bidirectional, batch_first): forward +
backward (a fixed random gradient of the output and of h_n through ``torch.autograd.backward``) and the ``no_grad``
forward, for ``GRU`` at bf16x3 and bf16 and for nn.GRU on cuDNN in fp32 (torch defaults) and in bf16.

Per path: ms per call from CUDA events over windows of at least --window seconds, --repeats windows each, paths in
rotating order (median, min, max), sequences/s of the median, the peak ``torch.cuda.max_memory_allocated`` of one call, and
the output's rel-L2 against cuDNN fp32 in the same run.  The card's name, power limit and maximum SM clock are read in the
same run.

    python tools/bench_gru.py [--out DIR] [--window 0.5] [--repeats 7]      (writes DIR/bench_gru.json)"""
import argparse
import json
import os
import sys

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from financial_market_data_analysis_b200 import GRU   # noqa: E402
from bench_lengths import card, time_window           # noqa: E402

B, T, F, H, L = 512, 128, 64, 256, 2


def paths():
    """name -> (module, input dtype)."""
    torch.manual_seed(0)
    ref = nn.GRU(F, H, L, batch_first=True, bidirectional=True).cuda()
    sd = ref.state_dict()
    out = {"cudnn_fp32": (ref, torch.float32), "cudnn_bf16": (nn.GRU(F, H, L, batch_first=True, bidirectional=True).cuda().to(torch.bfloat16), torch.bfloat16)}
    out["cudnn_bf16"][0].load_state_dict({k: v.to(torch.bfloat16) for k, v in sd.items()})
    for prec in ("bf16x3", "bf16"):
        m = GRU(F, H, L, batch_first=True, bidirectional=True, precision=prec).cuda()
        m.load_state_dict(sd)
        out[prec] = (m, torch.float32)
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
        out[name] = {"ms_median": s[len(s) // 2], "ms_min": s[0], "ms_max": s[-1], "seq_per_s": B * 1e3 / s[len(s) // 2],
                     "calls_per_window": per[name], "windows": len(s)}
    return out


def peak_bytes(fn):
    """Peak bytes allocated beyond what was allocated before one call (on a fresh module: its workspaces included)."""
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--out", default="bench_gru_out")
    ap.add_argument("--window", type=float, default=0.5, help="seconds of work per timed window")
    ap.add_argument("--repeats", type=int, default=7, help="timed windows per path")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_gru needs a CUDA device (an H100); there is nothing to measure without one")
    g = torch.Generator().manual_seed(1)
    x = torch.randn(B, T, F, generator=g).cuda()
    dy, dhn = torch.randn(B, T, 2 * H, generator=g).cuda(), torch.randn(2 * L, B, H, generator=g).cuda()

    def train(m, dt):
        xi = x.to(dt).requires_grad_()
        y, hn = m(xi)
        torch.autograd.backward((y, hn), (dy.to(dt), dhn.to(dt)))

    def infer(m, dt):
        with torch.no_grad():
            return m(x.to(dt))

    peaks = {}
    for kind, fn in (("no_grad_forward", lambda m, dt: infer(m, dt)), ("forward_backward", lambda m, dt: train(m, dt))):
        fresh = paths()
        peaks[kind] = {n: peak_bytes(lambda m=m, dt=dt: fn(m, dt)) for n, (m, dt) in fresh.items()}
        del fresh
        torch.cuda.empty_cache()
    mods = paths()

    train_calls = {n: (lambda m=m, dt=dt: train(m, dt)) for n, (m, dt) in mods.items()}
    infer_calls = {n: (lambda m=m, dt=dt: infer(m, dt)) for n, (m, dt) in mods.items()}
    with torch.no_grad():
        ref_y = mods["cudnn_fp32"][0](x)[0].double()
    err = {n: float((infer(m, dt)[0].double() - ref_y).norm() / ref_y.norm()) for n, (m, dt) in mods.items()}
    info = {"card": card(), "torch": torch.__version__, "cudnn": torch.backends.cudnn.version(),
            "shape": dict(B=B, T=T, F=F, H=H, L=L, bidirectional=True, batch_first=True), "window_s": a.window,
            "repeats": a.repeats, "output_rel_l2_vs_cudnn_fp32": err,
            "forward_backward": measure(train_calls, a.window, a.repeats), "no_grad_forward": measure(infer_calls, a.window, a.repeats),
            "peak_bytes": peaks}
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "bench_gru.json"), "w") as f:
        json.dump(info, f, indent=1)
    print(json.dumps(info))


if __name__ == "__main__":
    main()
