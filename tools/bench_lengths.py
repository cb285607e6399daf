"""What per-sequence lengths cost: the configs[1] bf16x3 train step (B512 T128 F64 H256 L2, bidirectional, CE loss, Adam,
CUDA graph) and ``BiGRU.infer`` in three cases, alternating in one run: ``lengths=None``, every length equal to T (the
masked kernels doing no masking), and mixed lengths drawn uniformly from [T/2, T] (a CPU tensor, as a caller passes them).

Per case: ms per call from CUDA events over windows of at least --window seconds, --repeats windows each, cases in rotating
order (median, min, max reported), and the median's overhead against ``lengths=None``.  The card's name, power limit and
maximum SM clock are read in the same run.

    python tools/bench_lengths.py [--out DIR] [--window 0.5] [--repeats 7]      (writes DIR/bench_lengths.json)"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from financial_market_data_analysis_b200 import BiGRU   # noqa: E402

B, T, F, H, L, C = 512, 128, 64, 256, 2, 3


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    line = q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else ""
    name, power, clock = ([s.strip() for s in line.split(",")] + ["", "", ""])[:3]
    return {"name": name or torch.cuda.get_device_name(), "power_limit": power or "unknown", "max_sm_clock": clock or "unknown"}


def time_window(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / n


def model():
    torch.manual_seed(0)
    m = BiGRU(H, F, C, L, 50, 0.0, False, True, precision="bf16x3").cuda()
    m.add_loss_fn(nn.CrossEntropyLoss())
    m.add_optimizer(torch.optim.Adam(m.parameters(), lr=1e-3))
    m.train()
    return m


def measure(calls, window, repeats):
    """calls: name -> zero-argument callable.  Median / min / max ms per call of each, the names in rotating order."""
    per = {}
    for name, fn in calls.items():
        time_window(fn, 3)                                   # warm-up: plans, workspaces, graph capture
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
    base = out["none"]["ms_median"]
    for name in out:
        out[name]["overhead_vs_none"] = out[name]["ms_median"] / base - 1.0
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--out", default="bench_lengths_out")
    ap.add_argument("--window", type=float, default=0.5, help="seconds of work per timed window")
    ap.add_argument("--repeats", type=int, default=7, help="timed windows per case")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lengths needs a CUDA device (an H100); there is nothing to measure without one")
    g = torch.Generator().manual_seed(1)
    x = torch.randn(B, T, F, generator=g).cuda()
    tgt = torch.randint(0, C, (B,), generator=g).cuda()
    cases = {"none": None, "all_T": torch.full((B,), T, dtype=torch.int64),
             "mixed": torch.randint(T // 2, T + 1, (B,), generator=g)}
    models = {name: model() for name in cases}
    train = {name: (lambda m=models[name], n=n: m.train_step(x, tgt, lengths=n)) for name, n in cases.items()}
    infer = {name: (lambda m=models[name], n=n: m.infer(x, lengths=n)) for name, n in cases.items()}
    info = {"card": card(), "torch": torch.__version__, "shape": dict(B=B, T=T, F=F, H=H, L=L, C=C, bidirectional=True),
            "precision": "bf16x3", "window_s": a.window, "repeats": a.repeats,
            "mixed_lengths": {"min": int(cases["mixed"].min()), "max": int(cases["mixed"].max()),
                              "mean": float(cases["mixed"].float().mean())},
            "train_step": measure(train, a.window, a.repeats), "infer": measure(infer, a.window, a.repeats)}
    info["train_step_graphed"] = {name: len(m._graphs) == 1 for name, m in models.items()}
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "bench_lengths.json"), "w") as f:
        json.dump(info, f, indent=1)
    print(json.dumps(info))


if __name__ == "__main__":
    main()
