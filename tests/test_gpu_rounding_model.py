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
import functools
import json
import os

import numpy as np
import pytest

import oracle_c
from gru_driver import abi_names, dist as _dist, kernel, kernel_steps as _kernel_steps, stepwise as _stepwise, tensors as _tensors

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
    # bidirectional H = 512 (8-CTA clusters, both directions: bf16's largest backward shared-memory footprint), and an odd
    # number of 16-row batch tiles
    "cluster8_d2": lambda s: s["H"] == 512 and s["D"] == 2, "odd_tiles": lambda s: (s["B"] // 16) % 2 == 1 and s["B"] > 16,
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
    "h512_d2": dict(B=32, T=6, F=40, H=512, L=2, C=3, D=2, h0=False, precs=("bf16",),
                    regimes=("cluster8", "cluster8_d2", "many_tiles", "D2")),
    "h256_b48": dict(B=48, T=5, F=20, H=256, L=1, C=3, D=2, h0=False, precs=("bf16",),
                     regimes=("cluster4", "odd_tiles", "many_tiles", "D2", "T_odd")),
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
    names = abi_names(s)
    want, got = _kernel_steps(own, s, names), _stepwise(s, prec, flat, x, h0, dl, own, names)
    for key, v in want.items():
        tol = 1e-12 if key[1] == "y_step" else 2e-7             # logits and gradients come back from the oracle as float32
        assert np.abs(got[key] - v).max() <= tol * np.abs(v).max(), key


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
    got, names = kernel(s, prec, flat, x, h0, dl)

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
