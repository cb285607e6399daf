"""What the optimizer setup costs the configs[1] bf16x3 train step (B512 T128 F64 H256 L2, bidirectional, 3 classes): three
cases, alternating in one run.

  adam_const         torch.optim.Adam, constant lr, CrossEntropyLoss (the setup bench.py measures)
  adam_cosine        torch.optim.Adam under CosineAnnealingLR, scheduler.step() after every train step
  adamw2_cosine      torch.optim.AdamW with two groups (biases without weight decay) under the same schedule

Each case runs ``BiGRU.train_step`` when the package fuses its setup (``can_fuse_step()``) and ``_generic_step`` (autograd,
clip_grad_norm_, torch's optimizer) when it does not, and reports which one ran.  The package is imported from
``--pkg-root``, so that the same script measures two checkouts, one process each.

Per case: ms per step from a host clock around windows of --steps steps that end in a device synchronise (a step that
captures a CUDA graph synchronises on the host, which events alone would hide), --repeats windows in rotating order
(median, min, max); the CUDA graphs captured over the whole run; and the memory the case adds at its peak, measured in a
pass of its own before the timed windows.  The card's name, power limit and maximum SM clock are read in the same run.

    python tools/bench_fused_optim.py --pkg-root DIR [--label NAME] [--out DIR] [--steps 20] [--repeats 7]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch
import torch.nn as nn

B, T, F, H, L, C = 512, 128, 64, 256, 2, 3
CASES = ("adam_const", "adam_cosine", "adamw2_cosine")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    line = q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else ""
    name, power, clock = ([s.strip() for s in line.split(",")] + ["", "", ""])[:3]
    return {"name": name or torch.cuda.get_device_name(), "power_limit": power or "unknown", "max_sm_clock": clock or "unknown"}


class Case:
    def __init__(self, BiGRU, name, x, y):
        torch.manual_seed(0)
        m = BiGRU(H, F, C, L, 50, 0.0, False, True, precision="bf16x3").cuda().train()
        m.add_loss_fn(nn.CrossEntropyLoss())
        if name == "adamw2_cosine":
            decay = [p for n, p in m.named_parameters() if "bias" not in n]
            no_decay = [p for n, p in m.named_parameters() if "bias" in n]
            opt = torch.optim.AdamW([{"params": decay, "weight_decay": 0.01}, {"params": no_decay, "weight_decay": 0.0}],
                                    lr=1e-3)
        else:
            opt = torch.optim.Adam(m.parameters(), lr=1e-3)
        m.add_optimizer(opt)
        self.sched = None if name == "adam_const" else torch.optim.lr_scheduler.CosineAnnealingLR(opt, T_max=10_000)
        self.m, self.x, self.y, self.fused, self.captures = m, x, y, m.can_fuse_step(), 0
        capture = m._capture

        def counted(*a, **k):
            self.captures += 1
            return capture(*a, **k)
        m._capture = counted

    def step(self):
        if self.fused:
            self.m.train_step(self.x, self.y)
        else:
            self.m._generic_step(self.x, self.y)
        if self.sched is not None:
            self.sched.step()


def window(case, n):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n):
        case.step()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pkg-root", required=True, help="checkout whose financial_market_data_analysis_b200 is measured")
    ap.add_argument("--label", default=None)
    ap.add_argument("--out", default="bench_fused_optim_out")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=7)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fused_optim needs a CUDA device")
    root = os.path.abspath(args.pkg_root)
    sys.path.insert(0, root)
    from financial_market_data_analysis_b200 import BiGRU
    import financial_market_data_analysis_b200 as pkg
    assert os.path.dirname(os.path.dirname(os.path.abspath(pkg.__file__))) == root, pkg.__file__
    g = torch.Generator().manual_seed(1)
    x = torch.randn(B, T, F, generator=g).cuda()
    y = torch.randint(0, C, (B,), generator=g).cuda()
    cases, peak = {}, {}
    for name in CASES:                                   # memory pass: what each case adds at its peak
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        cases[name] = Case(BiGRU, name, x, y)
        window(cases[name], 5)
        peak[name] = (torch.cuda.max_memory_allocated() - base) / 2 ** 30
    samples = {name: [] for name in CASES}
    for r in range(args.repeats):
        for name in CASES[r % len(CASES):] + CASES[:r % len(CASES)]:
            samples[name].append(window(cases[name], args.steps))
    out = {"label": args.label or root, "card": card(), "config": dict(B=B, T=T, F=F, H=H, L=L, C=C, precision="bf16x3"),
           "steps_per_window": args.steps, "repeats": args.repeats, "cases": {}}
    for name in CASES:
        s = samples[name]
        out["cases"][name] = {"path": "train_step" if cases[name].fused else "_generic_step",
                              "ms_per_step": {"median": statistics.median(s), "min": min(s), "max": max(s)},
                              "graph_captures": cases[name].captures, "graphs_held": len(cases[name].m._graphs),
                              "peak_added_gb": round(peak[name], 3)}
    os.makedirs(args.out, exist_ok=True)
    tag = "".join(ch if ch.isalnum() else "_" for ch in (args.label or "run"))
    with open(os.path.join(args.out, f"bench_fused_optim_{tag}.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
