"""The tensor-core paths (BIGRU_PREC_BF16, BIGRU_PREC_BF16X3) against the oracle's rounding model of each.

oracle/bigru_ref.c with prec = bf16 / bf16x3 rounds the operands of every matrix product where the CUDA path rounds them and
keeps everything else in fp64.  What the kernels compute beyond that rounding is fp32 arithmetic, so kernel and model must
agree to within fp32 noise - one to two orders of magnitude below each path's own distance from the exact answer.  A
kernel that drops a cross term, rounds an operand the wrong way or reads a wrong time step lands far outside that noise
even where it stays well inside the path's own error (which is all the exact-answer tests in test_gpu_parity.py can see).

The C ABI is driven directly, with plans of whole 16-row batch tiles (nothing is padded), no dropout and a fixed random
dlogits.  Every layer's output at every time step, hn per layer and direction, every parameter gradient by name, dx and
dh0 are compared, each on its own.  The oracle's backward routes the max-pool gradient the way the kernel did
(bigru_stash_argmax_offset).
Run on an H100:  python -m pytest tests/test_gpu_rounding_model.py -m gpu -q
(BIGRU_ROUNDING_REPORT=path.json appends every measured distance to that file.)"""
import ctypes as C
import functools
import json
import os

import numpy as np
import pytest
import torch

import oracle_c

NSM = 132                  # SMs of an H100 SXM: what wg_splits (tc_hopper.cuh) aims its split-K at


def cdiv(a, b):
    return -(-a // b)


def wg_splits(tiles, kblocks):
    """Restates wg_splits of tc_hopper.cuh: split-K count of a weight-gradient GEMM with `tiles` output tiles."""
    s = min(cdiv(4 * NSM, tiles), kblocks // 8)
    if s <= 1:
        return 1
    return cdiv(kblocks, cdiv(kblocks, s))


def dw_gemms(s):
    """(splits, units) of every dW_ih and dW_hh launch of a shape: M = 3H, N = I_l or H, K = B*T, one batch per direction."""
    kb = cdiv(s["B"] * s["T"], 64)
    out = []
    for l in range(s["L"]):
        for n in (s["F"] if l == 0 else s["D"] * s["H"], s["H"]):
            tiles = cdiv(3 * s["H"], 128) * cdiv(n, 128) * s["D"]
            sp = wg_splits(tiles, kb)
            out.append((sp, tiles * sp))
    return out


# the regimes where these kernels go wrong, and how a shape proves it is in one
REGIMES = {
    "cluster2": lambda s: s["H"] == 128, "cluster4": lambda s: s["H"] == 256, "cluster8": lambda s: s["H"] == 512,
    "one_tile": lambda s: s["B"] == 16, "many_tiles": lambda s: s["B"] // 16 >= 2,
    "T1": lambda s: s["T"] == 1, "T2": lambda s: s["T"] == 2, "T_odd": lambda s: s["T"] % 2 == 1 and s["T"] > 1,
    "T_long": lambda s: s["T"] >= 300,
    "F_lt8": lambda s: s["F"] < 8, "F_ragged8": lambda s: s["F"] % 8 != 0, "F64": lambda s: s["F"] == 64,
    "F65": lambda s: s["F"] == 65, "F_wide_ragged": lambda s: s["F"] > 128 and s["F"] % 64 != 0 and cdiv(s["F"], 128) >= 2,
    "D1": lambda s: s["D"] == 1, "D2": lambda s: s["D"] == 2, "L3": lambda s: s["L"] == 3,
    "h0": lambda s: s["h0"],
    # split-K on every weight-gradient GEMM, and more units than SMs: CTAs run several units, the producer runs ahead
    "splitk_persistent": lambda s: all(sp > 1 and units > NSM for sp, units in dw_gemms(s)),
}

SHAPES = {
    "h128_b16_t1_f5": dict(B=16, T=1, F=5, H=128, L=1, C=3, D=2, h0=False, precs=("bf16",),
                           regimes=("cluster2", "one_tile", "T1", "F_lt8", "D2")),
    "h128_t2_f64_h0": dict(B=32, T=2, F=64, H=128, L=2, C=3, D=2, h0=True, precs=("bf16x3",),
                           regimes=("cluster2", "many_tiles", "T2", "F64", "h0", "D2")),
    "h256_l3_t7_f65": dict(B=64, T=7, F=65, H=256, L=3, C=4, D=2, h0=False, precs=("bf16", "bf16x3"),
                           regimes=("cluster4", "many_tiles", "T_odd", "F65", "F_ragged8", "L3")),
    "h128_t300_d1": dict(B=32, T=300, F=13, H=128, L=1, C=2, D=1, h0=False, precs=("bf16", "bf16x3"),
                         regimes=("cluster2", "T_long", "F_ragged8", "D1")),
    "h512_f200": dict(B=32, T=9, F=200, H=512, L=2, C=3, D=1, h0=False, precs=("bf16",),
                      regimes=("cluster8", "many_tiles", "F_wide_ragged", "T_odd", "D1")),
    "h256_f200_h0": dict(B=32, T=5, F=200, H=256, L=1, C=2, D=2, h0=True, precs=("bf16x3",),
                         regimes=("cluster4", "F_wide_ragged", "h0", "T_odd")),
    "h256_splitk": dict(B=32, T=128, F=136, H=256, L=2, C=3, D=2, h0=False, precs=("bf16", "bf16x3"),
                        regimes=("cluster4", "many_tiles", "splitk_persistent")),
}

# Kernel-vs-model tolerances (rel-L2, max-abs over max |model|) per tensor class: about 4x the worst value measured on an
# H100 80GB HBM3 (SXM, 700 W power limit) over the shapes above; the measurements are in tests/ROUNDING_MODEL.md.
# Classes of the free-running comparison: y, every layer, direction and time step; hn per layer and direction; logits;
# w, the w_ih, w_hh and lin_w gradients; b, the bias gradients; dx; dh0 per layer and direction.  Classes of the one-step
# comparison (_stepwise, the model restarted from the kernel's state): y_step, logits_step, w_step (the lin_w gradient).
# Why the two differ: once an activation differs from the model by d, its bf16 rounding lands on the other side of a
# rounding boundary for a fraction ~d / ulp of its elements, each off by a whole ulp, which amplifies fp32 noise to about
# sqrt(d * ulp) per rounded operand: a few 1e-4 at bf16 after one layer or a few hundred steps, a few 1e-6 at bf16x3.  The
# one-step comparison cannot compound flips and separates the bf16 kernels from their model by three orders of magnitude.
# At bf16x3 both stay near 1e-6 to 1e-5, the size of the model's own error: the tensor cores' fp32 accumulation is biased
# low (measured -1.4e-6 relative after a K = 512 projection), which no operand rounding model reproduces.
TOL = {
    "bf16": {"y_step": (1.8e-6, 3.6e-6), "logits_step": (8e-5, 3.6e-4), "w_step": (1e-4, 8.6e-4),
             "logits": (2.5e-3, 4e-3), "y": (1.2e-3, 2.8e-3), "hn": (1e-3, 1.6e-3),
             "w": (5e-3, 7e-3), "b": (1.5e-3, 1.5e-3), "dx": (5.5e-3, 8e-3), "dh0": (1e-3, 1e-3)},
    "bf16x3": {"y_step": (6.8e-6, 1e-5), "logits_step": (1.3e-5, 1.7e-5), "w_step": (1.3e-6, 7.8e-6),
               "logits": (2.8e-5, 3.7e-5), "y": (1.7e-5, 1.8e-5), "hn": (1.4e-5, 1.7e-5),
               "w": (3.8e-5, 4.7e-5), "b": (2.7e-5, 3e-5), "dx": (4.5e-5, 4.5e-5), "dh0": (1e-5, 1e-5)},
}
CODE = {"bf16": 1, "bf16x3": 2}


def test_shapes_are_in_the_regimes_they_claim():
    covered = set()
    for name, s in SHAPES.items():
        for r in s["regimes"]:
            assert REGIMES[r](s), (name, r)
        covered |= set(s["regimes"])
        assert s["B"] % 16 == 0 and ("bf16x3" not in s["precs"] or (s["B"] % 32 == 0 and s["H"] <= 256))
        assert not (s["h0"] and "bf16" in s["precs"])          # BIGRU_PREC_BF16 has no initial state
    assert covered == set(REGIMES), set(REGIMES) - covered
    assert set(SHAPES["h256_splitk"]["precs"]) == {"bf16", "bf16x3"}


def _pkg():
    import financial_market_data_analysis_b200 as pkg
    return pkg


def _inputs(s):
    B, T, F, H, L, C_, D = (s[k] for k in "BTFHLCD")
    rng = np.random.default_rng([B, T, F, H, L, D])
    k = 1 / np.sqrt(H)                                          # nn.GRU / nn.Linear initialisation scale
    flat = rng.uniform(-k, k, oracle_c.lib().bigru_ref_param_count(F, H, L, C_, D)).astype(np.float32)
    x = rng.standard_normal((B, T, F)).astype(np.float32)
    h0 = (0.5 * rng.standard_normal((L * D, B, H))).astype(np.float32) if s["h0"] else None
    dl = rng.standard_normal((B, C_)).astype(np.float32)
    return flat, x, h0, dl


def _param_names(plan, s):
    """name -> (offset, size) of every parameter block, from bigru_param_offset."""
    lib = _pkg()._lib.load()
    out = {}
    off, rows, cols = C.c_int64(), C.c_int64(), C.c_int64()
    for l in range(s["L"] + 1):
        for d in range(s["D"] if l < s["L"] else 1):
            for which, nm in enumerate(("w_ih", "w_hh", "b_ih", "b_hh")):
                if l == s["L"] and which in (1, 3):
                    continue
                assert lib.bigru_param_offset(plan, l, d, which, C.byref(off), C.byref(rows), C.byref(cols)) == 0
                name = ("lin_w" if which == 0 else "lin_b") if l == s["L"] else f"l{l}d{d}.{nm}"
                out[name] = (off.value, rows.value * cols.value)
    return out


def _kernel(s, prec, flat, x, h0, dl):
    pkg = _pkg()
    lib, L_ = pkg._lib.load(), pkg._lib
    B, T, F, H, L, C_, D = (s[k] for k in "BTFHLCD")
    plan = C.c_void_p()
    L_.check(lib.bigru_plan_create(B, T, F, H, L, C_, int(D == 2), CODE[prec], C.byref(plan)), "plan_create")
    try:
        sb, cb = C.c_size_t(), C.c_size_t()
        L_.check(lib.bigru_workspace_bytes(plan, C.byref(sb), C.byref(cb)), "workspace_bytes")
        dev = torch.device("cuda")
        stash = torch.zeros(sb.value // 4, dtype=torch.float32, device=dev)
        scratch = torch.zeros(cb.value // 4, dtype=torch.float32, device=dev)
        p, xd = torch.from_numpy(flat).to(dev), torch.from_numpy(x).to(dev)
        h0d = None if h0 is None else torch.from_numpy(h0).to(dev)
        logits = torch.zeros(B, C_, device=dev)
        hn = torch.zeros(L * D, B, H, device=dev)
        st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        ptr = L_.ptr
        L_.check(lib.bigru_forward(plan, ptr(p), ptr(xd), ptr(h0d), 0.0, 0, 0, 0, ptr(stash), ptr(scratch), ptr(logits), ptr(hn), st),
                 "forward")
        off = C.c_size_t()
        ys = []
        for l in range(L):
            L_.check(lib.bigru_stash_output_offset(plan, l, C.byref(off)), "stash_output_offset")
            ys.append(stash[off.value // 4: off.value // 4 + B * T * D * H].view(B, T, D * H).cpu().numpy().astype(np.float64))
        L_.check(lib.bigru_stash_argmax_offset(plan, C.byref(off)), "stash_argmax_offset")
        arg = stash.view(torch.int32)[off.value // 4: off.value // 4 + B * H].view(B, H).cpu().numpy().astype(np.int64)
        grads = torch.zeros(flat.size, device=dev)
        dx = torch.zeros(B, T, F, device=dev)
        dh0 = torch.zeros(L * D, B, H, device=dev) if h0 is not None else None
        dld = torch.from_numpy(dl).to(dev)                      # alive until the synchronize below: the backward reads it
        L_.check(lib.bigru_backward(plan, ptr(p), ptr(xd), ptr(h0d), 0.0, 0, 0, 0, ptr(stash), ptr(scratch),
                                    ptr(dld), ptr(grads), ptr(dx), ptr(dh0), st), "backward")
        torch.cuda.synchronize()
        names = _param_names(plan, s)
    finally:
        lib.bigru_plan_destroy(plan)
    f64 = lambda t: None if t is None else t.cpu().numpy().astype(np.float64)   # noqa: E731
    return dict(logits=f64(logits), hn=f64(hn), ys=ys, arg=arg, grads=f64(grads), dx=f64(dx), dh0=f64(dh0)), names


@functools.lru_cache(maxsize=None)
def _oracle_forward(name, prec):
    s = SHAPES[name]
    flat, x, h0, _ = _inputs(s)
    logits, hn, stash = oracle_c.forward(flat, x, s["H"], s["L"], s["C"], s["D"], h0, keep=True, prec=oracle_c.PRECISION[prec])
    return logits, hn, stash


def _oracle(name, prec, arg):
    """The oracle at `prec` (exact / bf16 / bf16x3), its backward routed through the max-pool choice `arg`."""
    s = SHAPES[name]
    flat, x, h0, dl = _inputs(s)
    B, T, H, L, C_, D = (s[k] for k in "BTHLCD")
    logits, hn, stash = _oracle_forward(name, prec)
    own_arg = oracle_c.routing(stash, B, H)
    stash = stash.copy()
    oracle_c.set_routing(stash, arg)
    grads, dx, dh0 = oracle_c.backward(flat, x, stash, dl, H, L, C_, D, prec=oracle_c.PRECISION[prec])
    return dict(logits=logits.astype(np.float64), hn=hn.astype(np.float64), ys=[y.copy() for y in oracle_c.layer_outputs(stash, B, T, H, L, D)],
                arg=own_arg, grads=grads.astype(np.float64), dx=dx.astype(np.float64),
                dh0=dh0.astype(np.float64) if h0 is not None else None)


def _bf16(v32):
    """Round float32 to the nearest bf16 (ties to even), returned as float32."""
    u = np.ascontiguousarray(v32, np.float32).view(np.uint32)
    u = (u + np.uint32(0x7FFF) + ((u >> np.uint32(16)) & np.uint32(1))) & np.uint32(0xFFFF0000)
    return u.view(np.float32)


def _mm(a, b, prec):
    """a[M,K] b[N,K]^T in float64 with both operands rounded as the kernels store them (fp32, then bf16 or a bf16 pair):
    ah bf + al bh = ah bh + ah bl + al bh, the rule of oracle/bigru_ref.c."""
    if prec == "exact":
        return a @ b.T
    def split(v):
        v32 = v.astype(np.float32)
        hi = _bf16(v32)
        lo = _bf16(v32 - hi) if prec == "bf16x3" else np.zeros_like(hi)
        return hi.astype(np.float64) + lo, hi.astype(np.float64), lo.astype(np.float64)
    _, ah, al = split(a)
    bf, bh, _ = split(b)
    return ah @ bf.T + al @ bh.T


def _stepwise(s, prec, flat, x, h0, dl, got, names):
    """The rounding model run one step at a time from the kernel's own state: every step of every layer starts from the
    kernel's h_{t-1} (its Y, or h0) and the kernel's layer input (x, or the previous layer's Y), the head from the kernel's
    top-layer Y.  Rounding flips cannot compound, so what is left of the kernel's distance is the fp32 arithmetic of one
    step.  Returns (name, class) -> array like _tensors: Y per layer, direction and step, the logits and the lin_w gradient."""
    B, T, H, L, C_, D = (s[k] for k in "BTHLCD")
    out = {}
    sig = lambda v: 1 / (1 + np.exp(-v))                        # noqa: E731
    inp = x.astype(np.float64)
    for l in range(L):
        Y = got["ys"][l]
        I = inp.shape[2]
        for d in range(D):
            o = names[f"l{l}d{d}.w_ih"][0]
            w_ih = flat[o:o + 3 * H * I].reshape(3 * H, I).astype(np.float64); o += 3 * H * I
            w_hh = flat[o:o + 3 * H * H].reshape(3 * H, H).astype(np.float64); o += 3 * H * H
            b_ih, b_hh = flat[o:o + 3 * H].astype(np.float64), flat[o + 3 * H:o + 6 * H].astype(np.float64)
            y = Y[:, :, d * H:(d + 1) * H]
            start = np.zeros((B, H)) if h0 is None else h0[l * D + d].astype(np.float64)
            if d == 0:
                hp = np.concatenate([start[:, None], y[:, :-1]], 1)
            else:
                hp = np.concatenate([y[:, 1:], start[:, None]], 1)
            gi = (_mm(inp.reshape(B * T, I), w_ih, prec) + b_ih).reshape(B, T, 3 * H)
            gh = (_mm(hp.reshape(B * T, H), w_hh, prec) + b_hh).reshape(B, T, 3 * H)
            r = sig(gi[..., :H] + gh[..., :H])
            z = sig(gi[..., H:2 * H] + gh[..., H:2 * H])
            n = np.tanh(gi[..., 2 * H:] + r * gh[..., 2 * H:])
            h = (1 - z) * n + z * hp
            for t in range(T):
                out[(f"step:y[l{l}d{d},t{t}]", "y_step")] = h[:, t]
        inp = Y
    top = got["ys"][-1]
    pooled = top[..., :H] + top[..., H:] if D == 2 else top
    last = top[:, T - 1, :H] + (top[:, 0, H:] if D == 2 else 0)
    cat = np.concatenate([last, pooled.max(1), pooled.sum(1) / T], 1)
    o = names["lin_w"][0]
    lin_w = flat[o:o + C_ * 3 * H].reshape(C_, 3 * H).astype(np.float64)
    lin_b = flat[names["lin_b"][0]:names["lin_b"][0] + C_].astype(np.float64)
    out[("step:logits", "logits_step")] = _mm(cat, lin_w, prec) + lin_b
    out[("step:grad:lin_w", "w_step")] = _mm(dl.astype(np.float64).T, cat.T, prec).ravel()
    return out


@pytest.mark.parametrize("prec", ["bf16", "bf16x3"])
def test_stepwise_model_reproduces_the_oracle(prec):
    """Fed the oracle's own state instead of the kernel's, the one-step model is the oracle's rounding model again."""
    name = "h128_t2_f64_h0"
    s = dict(SHAPES[name], T=5, L=2)
    flat, x, h0, dl = _inputs(s)
    B, T, H, L, C_, D = (s[k] for k in "BTHLCD")
    logits, _, stash = oracle_c.forward(flat, x, H, L, C_, D, h0, keep=True, prec=oracle_c.PRECISION[prec])
    grads = oracle_c.backward(flat, x, stash, dl, H, L, C_, D, prec=oracle_c.PRECISION[prec])[0]
    own = dict(ys=[y.copy() for y in oracle_c.layer_outputs(stash, B, T, H, L, D)], logits=logits.astype(np.float64),
               grads=grads.astype(np.float64))
    names = {}
    o = 0
    for l in range(L):
        for d in range(D):
            for nm, n in (("w_ih", 3 * H * (s["F"] if l == 0 else D * H)), ("w_hh", 3 * H * H), ("b_ih", 3 * H), ("b_hh", 3 * H)):
                names[f"l{l}d{d}.{nm}"] = (o, n)
                o += n
    names["lin_w"], names["lin_b"] = (o, C_ * 3 * H), (o + C_ * 3 * H, C_)
    want, got = _kernel_steps(own, s, names), _stepwise(s, prec, flat, x, h0, dl, own, names)
    for key, v in want.items():
        tol = 1e-12 if key[1] == "y_step" else 2e-7             # logits and gradients come back from the oracle as float32
        assert np.abs(got[key] - v).max() <= tol * np.abs(v).max(), key


def _kernel_steps(got, s, names):
    """The kernel's side of _stepwise."""
    H = s["H"]
    out = {}
    for l, y in enumerate(got["ys"]):
        for d in range(s["D"]):
            for t in range(s["T"]):
                out[(f"step:y[l{l}d{d},t{t}]", "y_step")] = y[:, t, d * H:(d + 1) * H]
    out[("step:logits", "logits_step")] = got["logits"]
    o, k = names["lin_w"]
    out[("step:grad:lin_w", "w_step")] = got["grads"][o:o + k]
    return out


def _tensors(r, s, names):
    """(name, class) -> array of every compared tensor; y per layer and time step, hn and dh0 per layer and direction."""
    out = {("logits", "logits"): r["logits"], ("dx", "dx"): r["dx"]}
    H, T = s["H"], s["T"]
    for l, y in enumerate(r["ys"]):
        for d in range(s["D"]):
            for t in range(T):
                out[(f"y[l{l}d{d},t{t}]", "y")] = y[:, t, d * H:(d + 1) * H]
    for i in range(s["L"] * s["D"]):
        out[(f"hn[l{i // s['D']}d{i % s['D']}]", "hn")] = r["hn"][i]
        if r["dh0"] is not None:
            out[(f"dh0[l{i // s['D']}d{i % s['D']}]", "dh0")] = r["dh0"][i]
    for n, (o, k) in names.items():
        out[(f"grad:{n}", "b" if n.split(".")[-1] in ("b_ih", "b_hh", "lin_b") else "w")] = r["grads"][o:o + k]
    return out


def _dist(a, b):
    """(rel-L2, max-abs / max |b|); a reference of zeros admits only zeros."""
    nb, mb = np.linalg.norm(b), np.abs(b).max()
    d = a - b
    if mb == 0:
        return (0.0, 0.0) if not d.any() else (np.inf, np.inf)
    return float(np.linalg.norm(d) / nb), float(np.abs(d).max() / mb)


CASES = [(n, p) for n, s in SHAPES.items() for p in s["precs"]]


@pytest.mark.gpu
@pytest.mark.parametrize("name,prec", CASES, ids=[f"{n}-{p}" for n, p in CASES])
def test_kernel_matches_its_rounding_model(name, prec):
    pkg = _pkg()
    if pkg._lib.load().bigru_device_check(0) != 0:
        pytest.fail("no H100: " + pkg._lib.load().bigru_last_error().decode())
    s = SHAPES[name]
    B, H, D = s["B"], s["H"], s["D"]
    flat, x, h0, dl = _inputs(s)
    got, names = _kernel(s, prec, flat, x, h0, dl)

    # max-pool routing: where the kernel picked another time step than the model, the two must tie to within the kernel's
    # own deviation from the model (if |s_k - s_m| <= e everywhere, the kernel's choice is at most 2e below the model's max)
    model = _oracle(name, prec, got["arg"])
    pool = lambda ys: ys[-1][..., :H] + ys[-1][..., H:] if D == 2 else ys[-1]   # noqa: E731
    sk, sm = pool(got["ys"]), pool(model["ys"])
    flips = got["arg"] != model["arg"]
    if flips.any():
        bi, ji = np.nonzero(flips)
        gap = sm[bi, model["arg"][bi, ji], ji] - sm[bi, got["arg"][bi, ji], ji]
        assert gap.max() <= 2 * np.abs(sk - sm).max(), (int(flips.sum()), float(gap.max()))
    exact = _oracle(name, "exact", got["arg"])

    tk, tm, te = _tensors(got, s, names), _tensors(model, s, names), _tensors(exact, s, names)
    # the same model one step at a time from the kernel's state, and the exact arithmetic from that state
    tk.update(_kernel_steps(got, s, names))
    tm.update(_stepwise(s, prec, flat, x, h0, dl, got, names))
    te.update(_stepwise(s, "exact", flat, x, h0, dl, got, names))
    rows, bad = [], []
    for key in tk:
        tname, cls = key
        km, me, ke = _dist(tk[key], tm[key]), _dist(tm[key], te[key]), _dist(tk[key], te[key])
        rows.append(dict(shape=name, prec=prec, tensor=tname, cls=cls, km_l2=km[0], km_max=km[1], me_l2=me[0], me_max=me[1],
                         ke_l2=ke[0], ke_max=ke[1]))
        tol = TOL[prec][cls]
        if km[0] > tol[0] or km[1] > tol[1]:
            bad.append(("kernel vs model", tname, km, tol))
        # the kernel is no less accurate than its own rounding model.  Once the bound above holds this cannot fail
        # (ke <= km + me <= tol + me): it records the intent, and the report keeps ke next to me
        if ke[0] > 1.25 * me[0] + tol[0] or ke[1] > 1.25 * me[1] + tol[1]:
            bad.append(("kernel vs exact", tname, ke, me))
    out = os.environ.get("BIGRU_ROUNDING_REPORT")
    if out:
        with open(out, "a") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")
    worst = {}
    for r in rows:
        w = worst.setdefault(r["cls"], [0.0, 0.0, np.inf])
        w[0], w[1], w[2] = max(w[0], r["km_l2"]), max(w[1], r["km_max"]), min(w[2], r["me_l2"] if r["me_l2"] > 0 else np.inf)
    print(f"\n{name} {prec} flips={int(flips.sum())} " +
          " ".join(f"{c}: km_l2 {w[0]:.1e} km_max {w[1]:.1e} me_l2(min) {w[2]:.1e}" for c, w in worst.items()))
    assert not bad, bad[:10]
