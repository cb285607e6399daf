"""Eval-mode batch scoring: ``forward`` under ``torch.no_grad()`` (the training forward: full stash + scratch) against
``BiGRU.infer`` (bigru_infer: the inference workspace only) at BASELINE configs[1] (B512 T128 F64 H256 L2, bidirectional) in
bf16x3 and bf16, configs[4] (T1024 F128 H512 L2) in bf16 at B256, and configs[4] at the largest batch ``infer`` fits.

Per shape and path: ms per batch and sequences/s from CUDA events over windows of at least --window seconds, the two paths
alternating, --repeats windows each (median, min, max reported); the peak of torch.cuda.max_memory_allocated over the first
call of that path alone on the device; and whether the two paths' logits are bitwise equal.  The card's name, power limit and
maximum SM clock are read in the same run.  A path whose workspaces do not fit on the card is reported as such.

    python tools/bench_infer.py [--out DIR] [--window 0.5] [--repeats 5]      (writes DIR/bench_infer.json)"""
import argparse
import gc
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from financial_market_data_analysis_b200 import BiGRU, _lib   # noqa: E402
from financial_market_data_analysis_b200.biGRU_model import _PRECISIONS   # noqa: E402

CONFIGS = {1: dict(T=128, F=64, H=256, L=2, C=3), 4: dict(T=1024, F=128, H=512, L=2, C=3)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    line = q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else ""
    name, power, clock = ([s.strip() for s in line.split(",")] + ["", "", ""])[:3]
    return {"name": name or torch.cuda.get_device_name(), "power_limit": power or "unknown", "max_sm_clock": clock or "unknown"}


def plan_bytes(B, cfg, prec):
    """(stash + scratch of the training forward, inference workspace) of one plan, from the C ABI (no device memory)."""
    lib, C = _lib.load(), _lib.C
    h = C.c_void_p()
    _lib.check(lib.bigru_plan_create(B, cfg["T"], cfg["F"], cfg["H"], cfg["L"], cfg["C"], 1, _PRECISIONS[prec], C.byref(h)),
               "bigru_plan_create")
    try:
        a, b, c = C.c_size_t(), C.c_size_t(), C.c_size_t()
        _lib.check(lib.bigru_workspace_bytes(h, C.byref(a), C.byref(b)), "bigru_workspace_bytes")
        _lib.check(lib.bigru_infer_workspace_bytes(h, C.byref(c)), "bigru_infer_workspace_bytes")
        return a.value + b.value, c.value
    finally:
        lib.bigru_plan_destroy(h)


def largest_infer_batch(cfg, prec, tile=32):
    """The largest whole-tile batch whose inference workspace, input and logits fit in 90 % of the free device memory."""
    free = 0.9 * torch.cuda.mem_get_info()[0]
    row = 4 * cfg["T"] * cfg["F"] + 4 * cfg["C"]
    B = tile
    while True:
        nxt = B * 2
        if plan_bytes(nxt, cfg, prec)[1] + nxt * row > free:
            break
        B = nxt
    step = B // 2
    while step >= tile:                                  # bisect between B and 2B in whole tiles
        if plan_bytes(B + step, cfg, prec)[1] + (B + step) * row <= free:
            B += step
        step //= 2
    return B


def model(cfg, prec):
    torch.manual_seed(0)
    m = BiGRU(cfg["H"], cfg["F"], cfg["C"], cfg["L"], 50, 0.2, True, True, precision=prec).cuda()
    m.eval()
    return m


def first_call_peak(cfg, prec, x, path):
    """torch.cuda.max_memory_allocated over building the model and its first call, alone on the device."""
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    m = model(cfg, prec)
    out = path(m, x)
    torch.cuda.synchronize()
    return m, out, torch.cuda.max_memory_allocated()


def time_window(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / n


def forward_path(m, x):
    with torch.no_grad():
        return m(x)


def infer_path(m, x):
    return m.infer(x)


def run_shape(label, cfg, prec, B, window, repeats):
    print(f"[{label}] {prec} B{B}", file=sys.stderr, flush=True)
    trainfwd_bytes, infer_bytes = plan_bytes(B, cfg, prec)
    x = torch.randn(B, cfg["T"], cfg["F"], device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    free = torch.cuda.mem_get_info()[0]
    fits_forward = trainfwd_bytes + x.numel() * 4 < 0.9 * free
    res = {"label": label, "precision": prec, "B": B, **cfg, "bidirectional": True,
           "plan_bytes": {"forward_stash_plus_scratch": trainfwd_bytes, "infer_workspace": infer_bytes}}
    paths = {"infer": infer_path}
    if fits_forward:
        paths["forward_no_grad"] = forward_path
    else:
        res["forward_no_grad"] = {"skipped": f"stash + scratch ({trainfwd_bytes / 1e9:.1f} GB) do not fit on the card"}
    models, outs = {}, {}
    for name, fn in paths.items():
        m, out, peak = first_call_peak(cfg, prec, x, fn)
        outs[name] = out
        res[name] = {"max_memory_allocated_bytes": peak}
        del m                                             # measured alone: rebuilt for timing below
    if "forward_no_grad" in outs:
        res["bitwise_equal"] = bool(torch.equal(outs["infer"], outs["forward_no_grad"]))
    del outs
    gc.collect()
    torch.cuda.empty_cache()
    for name in paths:
        models[name] = model(cfg, prec)
    # warm-up, then calls per window from the warm-up's time
    per = {}
    for name, fn in paths.items():
        m = models[name]
        time_window(lambda: fn(m, x), 2)
        per[name] = max(1, int(window * 1e3 / time_window(lambda: fn(m, x), 2)) + 1)
    samples = {name: [] for name in paths}
    order = list(paths)
    for r in range(repeats):
        for name in (order if r % 2 == 0 else order[::-1]):
            m, fn = models[name], paths[name]
            samples[name].append(time_window(lambda: fn(m, x), per[name]))
    for name, s in samples.items():
        s = sorted(s)
        med = s[len(s) // 2]
        res[name].update({"ms_per_batch_median": med, "ms_per_batch_min": s[0], "ms_per_batch_max": s[-1],
                          "calls_per_window": per[name], "windows": len(s), "sequences_per_s": B / med * 1e3})
    del models, x
    gc.collect()
    torch.cuda.empty_cache()
    print(json.dumps(res), file=sys.stderr, flush=True)
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--out", default="bench_infer_out")
    ap.add_argument("--window", type=float, default=0.5, help="seconds of work per timed window")
    ap.add_argument("--repeats", type=int, default=5, help="timed windows per path and shape")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_infer needs a CUDA device (an H100); there is nothing to measure without one")
    info = {"card": card(), "torch": torch.__version__, "window_s": a.window, "repeats": a.repeats, "results": []}
    c1, c4 = CONFIGS[1], CONFIGS[4]
    info["results"].append(run_shape("configs[1]", c1, "bf16x3", 512, a.window, a.repeats))
    info["results"].append(run_shape("configs[1]", c1, "bf16", 512, a.window, a.repeats))
    info["results"].append(run_shape("configs[4]", c4, "bf16", 256, a.window, a.repeats))
    info["results"].append(run_shape("configs[4] largest infer batch", c4, "bf16", largest_infer_batch(c4, "bf16"),
                                     a.window, a.repeats))
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "bench_infer.json"), "w") as f:
        json.dump(info, f, indent=1)
    print(json.dumps(info))


if __name__ == "__main__":
    main()
