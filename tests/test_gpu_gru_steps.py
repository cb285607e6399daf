"""The head-less plan (the nn.GRU drop-in, bigru_gru_*) one step and one GEMM at a time, from the kernels' own operands,
seeded from per-layer, per-direction h_n gradients.

test_gpu_tc_steps.py, test_gpu_scan_tiles.py and test_gpu_rd_steps.py check the scans only on plans with the pooling
head, where the only nonzero carry is the top layer's, the head's d(last), the same in both directions.  A head-less
plan starts every layer's carry from the caller's dhn slice, row by row and direction by direction, and its top layer
reads its output and upstream gradient from the caller's y and dy.  test_gpu_gru.py compares that path only free-running,
at parity bounds that a bf16-sized error passes.  Here gru_driver recomputes, with head=False:
  y_step, g_step   the forward, one step from the kernel's h_{t-1} (the top layer's from the caller's y);
  dg_step          layer 0's dgi and dgh per direction and step, from a carry seeded with dhn[0*D + d];
  dh0_step         dh_{-1} of layer 0;
  gemm_step        layer 0's backward GEMMs (tensor-core precisions);
and bit for bit: the Y, input (x, never dropped on a head-less plan), dgi and dgh planes, the recurrent-dropout masks and
masked states.  Exact checks need no tolerance: h_n is the output at each direction's last valid step; a seed in one
(layer, direction, row) reaches no layer above, not the layer's other direction and no other row of dx; a row's bits do
not depend on its tile; a head-less plan has the head plan's scan geometry.

configs[1] runs at full size (B512 T128 F64 H256 L2 D2) with its forward steps sampled by batch tile.
Run on an H100:  python -m pytest tests/test_gpu_gru_steps.py -m gpu -q
(BIGRU_GRU_STEPS_REPORT=path.jsonl appends every measured distance to that file.)  Measurements and mutations:
tests/ROUNDING_MODEL.md, section "The head-less plan, one step at a time"."""
import ctypes as C
import json
import os
import resource

import numpy as np
import pytest
import torch

from gru_driver import (CODE, abi_names, backward_steps, dist, dropout_mask, gemm_steps, kernel, kernel_gemm_steps,
                        kernel_steps, plane_checks, stepwise)
from test_gpu_rd_steps import _lengths, _ops
from test_gpu_scan_tiles import _assert_bitwise, _per_row
from test_recurrent_dropout_cpu import rd_masks

SEED = 20261019
NB = 16                    # rows of a batch tile (SCAN_NB)


def _geometry(prec, B, H, D, scan, rd_p=0.0, head=False):
    """(R, n_split) of bigru_scan_geometry for a plan of this batch (head=False: a head-less plan); scan 0 forward, 1
    backward."""
    import financial_market_data_analysis_b200 as pkg
    lib = pkg._lib.load()
    plan = C.c_void_p()
    if head:
        rc = lib.bigru_plan_create_rd(B, 2, 16, H, 1, 3, int(D == 2), CODE[prec], rd_p, C.byref(plan))
    else:
        rc = lib.bigru_gru_plan_create_rd(B, 2, 16, H, 1, int(D == 2), CODE[prec], rd_p, C.byref(plan))
    pkg._lib.check(rc, "plan_create")
    try:
        R, n2 = C.c_int(), C.c_int()
        pkg._lib.check(lib.bigru_scan_geometry(plan, scan, C.byref(R), C.byref(n2)), "scan_geometry")
        return R.value, n2.value
    finally:
        lib.bigru_plan_destroy(plan)


def _batch(H, D, kind, prec, rd_p):
    """A batch (a multiple of 32) whose head-less forward scan has two-tile and one-tile clusters ("mixed") or only
    two-tile clusters ("two"), or whose backward scan splits the tiles of its last round into 8-row clusters ("split")."""
    R = _geometry(prec, 32, H, D, int(kind == "split"), rd_p)[0]
    n = {"mixed": (R // (2 * D) + 1) * 2 * D, "two": 2 * R // (2 * D) * (2 * D), "split": (2 * R // (2 * D) + 1) * 2 * D}[kind]
    return NB * n // D


def _tile_rows(prec, B, H, D, rd_p):
    """Per direction, the rows in 32-row forward tiles and in 8-row backward clusters at batch B (the head-less plan's
    geometry)."""
    ntd = B // NB
    n2 = _geometry(prec, B, H, D, 0, rd_p)[1]
    L8 = _geometry(prec, B, H, D, 1, rd_p)[1]
    fwd32 = [np.arange(2 * NB * (n2 // D)) for _ in range(D)]
    bwd8 = [[] for _ in range(D)]
    for q in range(D * ntd - L8, D * ntd):
        bwd8[q // ntd].extend(range((q % ntd) * NB, (q % ntd + 1) * NB))
    return fwd32, [np.asarray(r, int) for r in bwd8]


# the regimes where the head-less scans go wrong, and how a shape proves it is in one.  Regimes marked "device" are proved
# from the head-less plan's scan geometry in test_shapes_are_in_the_regimes_they_claim.
REGIMES = {
    # scan: cluster size x direction count; H = 512 is bf16 only
    "cluster2_d1": lambda s: s["H"] == 128 and s["D"] == 1, "cluster2_d2": lambda s: s["H"] == 128 and s["D"] == 2,
    "cluster4_d1": lambda s: s["H"] == 256 and s["D"] == 1, "cluster4_d2": lambda s: s["H"] == 256 and s["D"] == 2,
    "cluster8_d1": lambda s: s["H"] == 512 and s["D"] == 1, "cluster8_d2": lambda s: s["H"] == 512 and s["D"] == 2,
    # layer 0 is the top layer: it reads the caller's y and dy, and its carry starts from dhn's slice 0
    "layer0_is_top": lambda s: s["L"] == 1 and s["dy"],
    # layer 0 below the top: a nonzero dhn slice seeds a layer that is not the top
    "layer0_below_top": lambda s: s["L"] >= 2 and s["dhn"],
    # tile kinds of the head-less scans (device): 32-row and 16-row forward clusters mixed, 32-row only, 8-row backward
    # clusters in the last round, each with dhn seeds
    "fwd_mixed_tiles": "device", "fwd_two_tile_only": "device", "bwd_split_8row": "device",
    # lengths: the forward direction's seed passes through padded steps to t = len - 1, also in 8-row clusters (device)
    "lengths_dhn": lambda s: s["lens"] and s["dhn"], "padded_8row_dhn": "device",
    # recurrent dropout with a seed; p = 0.9 scales kept units by 10
    "rd_dhn": lambda s: s["rd"] > 0 and s["dhn"], "rd_p0.9": lambda s: s["rd"] == 0.9 and s["dhn"],
    # an initial state and its gradient
    "h0_bf16x3": lambda s: s["h0"] and s["dhn"] and "bf16x3" in s["precs"],
    "h0_fp32": lambda s: s["h0"] and s["dhn"] and "fp32" in s["precs"],
    # inter-layer dropout: layers above 0 own their input planes, x is never dropped
    "dropout_x_kept": lambda s: s["drop"] > 0 and s["L"] >= 2,
    # gradient sources: no dhn; dy = 0 with only dhn (an encoder that uses h_n alone)
    "dhn_none": lambda s: not s["dhn"] and s["dy"], "dy_zero_dhn_only": lambda s: not s["dy"] and s["dhn"],
    # scan length
    "T1": lambda s: s["T"] == 1 and s["D"] == 2, "T_long": lambda s: s["T"] >= 300,
    "configs1_full": lambda s: (s["B"], s["T"], s["F"], s["H"], s["L"], s["D"]) == (512, 128, 64, 256, 2, 2) and s["dhn"],
    # the fp32 path: gates kernels seeded per direction, with ragged reverse rows
    "fp32_d2_lens_dhn": lambda s: "fp32" in s["precs"] and s["D"] == 2 and s["lens"] and s["dhn"],
}


def _shape(B, T, F, H, L, D, precs, regimes, rd=0.0, h0=False, lens=False, drop=0.0, dy=True, dhn=True, **kw):
    return dict(B=B, T=T, F=F, H=H, L=L, C=0, D=D, h0=h0, precs=precs, rd=rd, lens=lens, drop=drop, dy=dy, dhn=dhn,
                regimes=regimes, **kw)


SHAPES = {
    "h128_l1_d1": _shape(32, 7, 13, 128, 1, 1, ("bf16x3", "bf16"), ("cluster2_d1", "layer0_is_top")),
    "h128_t1_d2": _shape(32, 1, 5, 128, 1, 2, ("bf16",), ("cluster2_d2", "T1", "layer0_is_top")),
    "h128_t301_d2": _shape(32, 301, 13, 128, 1, 2, ("bf16",), ("cluster2_d2", "T_long", "dhn_none"), dhn=False),
    "h128_drop_dy0": _shape(32, 6, 16, 128, 2, 2, ("bf16x3",), ("cluster2_d2", "dropout_x_kept", "dy_zero_dhn_only",
                                                                  "layer0_below_top"), drop=0.3, dy=False),
    "h256_l2_d2_h0": _shape(32, 5, 20, 256, 2, 2, ("bf16x3",), ("cluster4_d2", "layer0_below_top", "h0_bf16x3"), h0=True),
    "h256_l3_d1_rd": _shape(64, 6, 16, 256, 3, 1, ("bf16",), ("cluster4_d1", "layer0_below_top", "rd_dhn", "rd_p0.9"),
                            rd=0.9),
    "h512_d1": _shape(32, 5, 40, 512, 1, 1, ("bf16",), ("cluster8_d1", "layer0_is_top")),
    "h512_l2_d2_lens": _shape(32, 9, 24, 512, 2, 2, ("bf16",), ("cluster8_d2", "layer0_below_top", "lengths_dhn"),
                              lens=True),
    "mixed_l1": _shape("mixed", 5, 16, 128, 1, 2, ("bf16x3",), ("cluster2_d2", "fwd_mixed_tiles", "layer0_is_top")),
    "two_h0_rd": _shape("two", 4, 16, 128, 2, 2, ("bf16x3",), ("fwd_two_tile_only", "h0_bf16x3", "rd_dhn",
                                                               "layer0_below_top"), h0=True, rd=0.3),
    "split_lens": _shape("split", 4, 16, 128, 1, 2, ("bf16x3", "bf16"), ("bwd_split_8row", "lengths_dhn", "padded_8row_dhn",
                                                                        "layer0_is_top"), lens=True),
    "split_rd_l2": _shape("split", 3, 16, 128, 2, 2, ("bf16",), ("bwd_split_8row", "rd_dhn", "layer0_below_top"), rd=0.3),
    "configs1": _shape(512, 128, 64, 256, 2, 2, ("bf16x3", "bf16"), ("configs1_full", "cluster4_d2", "layer0_below_top"),
                       sample_tiles=(0, 1, -1)),
    "fp32_lens": _shape(24, 7, 13, 40, 2, 2, ("fp32",), ("fp32_d2_lens_dhn", "lengths_dhn", "layer0_below_top"), lens=True),
    "fp32_l1_h0_rd": _shape(16, 6, 13, 48, 1, 2, ("fp32",), ("h0_fp32", "rd_dhn", "layer0_is_top"), h0=True, rd=0.3),
}

# Kernel-vs-model tolerances (rel-L2, max-abs over max |model|) per class: about 4x the worst value measured on an H100
# 80GB HBM3 (SXM, 700 W power limit) over the shapes above; the measurements are in tests/ROUNDING_MODEL.md.
TOL = {
    "bf16": {"y_step": (3.5e-6, 6.8e-6), "g_step": (6e-7, 2.5e-6), "dg_step": (1e-6, 1.6e-6), "dh0_step": (9.2e-7, 1.4e-6),
             "gemm_step": (1.3e-5, 1.4e-5)},
    "bf16x3": {"y_step": (6.8e-6, 8.8e-6), "g_step": (2.2e-6, 8.8e-6), "dg_step": (5.2e-7, 1.2e-6), "dh0_step": (7.6e-7, 1.1e-6),
               "gemm_step": (4e-5, 4.4e-5)},
    "fp32": {"y_step": (4.4e-7, 9.2e-7), "g_step": (2.2e-7, 7.6e-7), "dg_step": (3.6e-7, 8e-7), "dh0_step": (3.6e-7, 4e-7)},
}


def _need_h100():
    import financial_market_data_analysis_b200 as pkg
    if pkg._lib.load().bigru_device_check(0) != 0:
        pytest.fail("no H100: " + pkg._lib.load().bigru_last_error().decode())


def _resolve(s, prec):
    """The shape with its batch read off the head-less plan's geometry where it names a tile kind."""
    if isinstance(s["B"], str):
        return dict(s, B=_batch(s["H"], s["D"], s["B"], prec, s["rd"]))
    return dict(s)


def _holds(r, s, prec):
    """Whether shape s (resolved at prec) is in regime r; "device" regimes from the scans' geometry at s's batch."""
    rule = REGIMES[r]
    if rule != "device":
        return rule(s)
    if prec == "fp32" or not s["dhn"]:
        return False
    B, T, H, D = s["B"], s["T"], s["H"], s["D"]
    n = D * B // NB
    n2 = _geometry(prec, B, H, D, 0, s["rd"])[1]
    L8 = _geometry(prec, B, H, D, 1, s["rd"])[1]
    _, bwd8 = _tile_rows(prec, B, H, D, s["rd"])
    padded = (_lengths(B, T) if s["lens"] else np.full(B, T)) < T
    return {"fwd_mixed_tiles": 0 < n2 < n - n2, "fwd_two_tile_only": n2 > 0 and 2 * n2 == n, "bwd_split_8row": L8 > 0,
            "padded_8row_dhn": any(len(bwd8[d]) and padded[bwd8[d]].any() for d in range(D))}[r]


@pytest.mark.gpu
def test_shapes_are_in_the_regimes_they_claim():
    _need_h100()
    covered = set()
    for name, s0 in SHAPES.items():
        resolved = {prec: _resolve(s0, prec) for prec in s0["precs"]}
        for prec, s in resolved.items():
            assert s["B"] % 16 == 0 or prec == "fp32"
            assert "bf16x3" != prec or (s["B"] % 32 == 0 and s["H"] <= 256)
            assert not (s["h0"] and (prec == "bf16" or s["lens"]))   # the library refuses both
        for r in s0["regimes"]:
            assert any(_holds(r, s, prec) for prec, s in resolved.items()), (name, r)
        covered |= set(s0["regimes"])
    assert covered == set(REGIMES), set(REGIMES) - covered


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ("bf16x3", "bf16"))
@pytest.mark.parametrize("H", (128, 256, 512))
@pytest.mark.parametrize("D", (1, 2))
def test_headless_plans_have_the_head_plans_geometry(prec, H, D):
    """The tile-kind batches above are read off the head-less plan; the head is no part of the scans, so every geometry
    must equal that of the plan with a head, with and without recurrent dropout."""
    _need_h100()
    if H == 512 and prec == "bf16x3":
        pytest.skip("hidden 512 runs at bf16 only")
    Bs = {32, 512, 1024} | {_batch(H, D, k, prec, 0.0) for k in ("mixed", "two", "split")}
    for scan in (0, 1):
        for rd in (0.0, 0.3):
            for B in sorted(Bs):
                assert _geometry(prec, B, H, D, scan, rd) == _geometry(prec, B, H, D, scan, rd, head=True), (scan, rd, B)


def _inputs(s):
    B, T, F, H, L, D = (s[k] for k in "BTFHLD")
    rng = np.random.default_rng([B, T, F, H, L, D, 8])
    k = 1 / np.sqrt(H)                                          # nn.GRU initialisation scale
    flat = rng.uniform(-k, k, abi_names(s)["lin_w"][0]).astype(np.float32)
    x = rng.standard_normal((B, T, F)).astype(np.float32)
    h0 = (0.5 * rng.standard_normal((L * D, B, H))).astype(np.float32) if s["h0"] else None
    dy = rng.standard_normal((B, T, D * H)).astype(np.float32) if s["dy"] else None
    dhn = rng.standard_normal((L * D, B, H)).astype(np.float32) if s["dhn"] else None
    return flat, x, h0, dy, dhn


def _assert_hn_is_last_valid_output(got, s, lens):
    """hn[l, 0, b] == Y_l[b, len_b - 1, :H] and hn[l, 1, b] == Y_l[b, 0, H:], bitwise."""
    B, T, H, L, D = (s[k] for k in "BTHLD")
    n_b = np.full(B, T) if lens is None else np.asarray(lens)
    for l in range(L):
        y = got["ys"][l]
        assert np.array_equal(got["hn"][l * D], y[np.arange(B), n_b - 1, :H]), l
        if D == 2:
            assert np.array_equal(got["hn"][l * D + 1], y[:, 0, H:]), l


CASES = [(n, p) for n, s in SHAPES.items() for p in s["precs"]]


@pytest.mark.gpu
@pytest.mark.parametrize("name,prec", CASES, ids=[f"{n}-{p}" for n, p in CASES])
def test_kernel_steps_match_their_models(name, prec):
    _need_h100()
    s = _resolve(SHAPES[name], prec)
    B, T, F, H, L, D = (s[k] for k in "BTFHLD")
    flat, x, h0, dy, dhn = _inputs(s)
    lens = _lengths(B, T) if s["lens"] else None
    got, names = kernel(s, prec, flat, x, h0, None, p=s["drop"], seed=SEED, regions=True, rd_p=s["rd"], lens=lens,
                        head=False, dy=dy, dhn=dhn)
    assert got["logits"] is None and got["arg"] is None
    _assert_hn_is_last_valid_output(got, s, lens)
    ws = got["ws"]
    masks = rd_masks(SEED, s["rd"], L, D, B, H) if s["rd"] > 0 else None
    drops = None
    if s["drop"] > 0:                                           # between layers only: x is never dropped
        drops = [None] + [dropout_mask(SEED, l, B, T, D * H, s["drop"]) for l in range(1, L)]
    bad_planes = {k: v for k, v in plane_checks(got, s, prec, x, masks, lens, drop=s["drop"] > 0).items() if v}

    rows_out, bad = [], []

    def compare(key, k, m, e):
        tname, cls = key
        km, me, ke = dist(k, m), dist(m, e), dist(k, e)
        rows_out.append(dict(shape=name, prec=prec, B=B, tensor=tname, cls=cls, km_l2=km[0], km_max=km[1], me_l2=me[0],
                             me_max=me[1], ke_l2=ke[0], ke_max=ke[1]))
        tol = TOL[prec][cls]
        if not (km[0] <= tol[0] and km[1] <= tol[1]):
            bad.append((tname, km, tol))

    # forward: one step from the kernel's state (the top layer's from the caller's y), with the gate stash
    rows = None
    if "sample_tiles" in s:
        rows = np.concatenate([np.arange(NB) + NB * (t % (B // NB)) for t in s["sample_tiles"]])
    tk = kernel_steps(got, s, names, rows, gates=True, head=False)
    tm = stepwise(s, prec, flat, x, h0, None, got, names, rows, gates=True, masks=masks, lens=lens, drops=drops, head=False)
    te = stepwise(s, "exact", flat, x, h0, None, got, names, rows, gates=True, masks=masks, lens=lens, drops=drops, head=False)
    for key in tk:
        compare(key, tk[key], tm[key], te[key])
    del tk, tm, te
    # backward recurrence of layer 0 from the seeded carry, one step at a time from the kernel's operands
    m0 = None if masks is None else masks[0]
    bprec = "exact" if prec == "fp32" else prec
    kw = dict(masks=m0, lens=lens, head=False, dy=dy, dhn=dhn)
    for a, b in zip(backward_steps(s, bprec, flat, h0, ws, got["ys"], names, **kw),
                    backward_steps(s, "exact", flat, h0, ws, got["ys"], names, **kw)):
        kind, d, t = a[:3]
        if kind == "dg":
            compare((f"bstep:dgi[d{d},t{t}]", "dg_step"), ws["DGI"][d][:, t].astype(np.float64), a[3], b[3])
            compare((f"bstep:dgh[d{d},t{t}]", "dg_step"), ws["DGH"][d][:, t].astype(np.float64), a[4], b[4])
        else:
            i = 4 if prec == "fp32" and m0 is not None else 3
            compare((f"bstep:dh0[d{d}]", "dh0_step"), ws["DHC"][d].astype(np.float64), a[i], b[i])
    # the backward GEMMs of layer 0, from the kernel's operand planes (tensor-core precisions)
    if prec != "fp32":
        gk = kernel_gemm_steps(got, s, names, head=False)
        gm = gemm_steps(s, prec, flat, None, h0, _ops(got, s, x, masks, False), names, None, masks=m0, lens=lens, head=False)
        ge = gemm_steps(s, "exact", flat, None, h0, _ops(got, s, x, masks, True), names, None, masks=m0, lens=lens, head=False)
        for key in gk:
            compare(key, gk[key], gm[key], ge[key])

    peak_gb = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 2 ** 20
    out = os.environ.get("BIGRU_GRU_STEPS_REPORT")
    if out:
        with open(out, "a") as f:
            for r in rows_out:
                f.write(json.dumps(r) + "\n")
            f.write(json.dumps(dict(shape=name, prec=prec, B=B, peak_host_gb=peak_gb, planes_bad=bad_planes)) + "\n")
    worst = {}
    for r in rows_out:
        w = worst.setdefault(r["cls"], [0.0, 0.0, np.inf])
        w[0], w[1], w[2] = max(w[0], r["km_l2"]), max(w[1], r["km_max"]), min(w[2], r["me_l2"] if r["me_l2"] > 0 else np.inf)
    print(f"\n{name} {prec} B{B} peak host {peak_gb:.1f} GB " +
          " ".join(f"{c}: km_l2 {w[0]:.1e} km_max {w[1]:.1e} me_l2(min) {w[2]:.1e}" for c, w in worst.items()))
    assert not bad_planes, bad_planes
    assert not bad, sorted(bad, key=lambda b: -b[1][0])[:10]


# ---- exact checks ---------------------------------------------------------------------------------------------------------
def _flat(s, seed):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal(abi_names(s)["lin_w"][0]) * 0.08).astype(np.float32)


def _support_case(prec):
    """(shape, seeded row per direction): a batch whose backward splits tiles into 8-row clusters, the seeded row in the
    second half of such a cluster where the direction has them (the split tiles are the highest cluster ids, so at D = 2
    they may all be the reverse direction's; a direction without them is seeded in the same row)."""
    if prec == "fp32":
        return dict(B=24, T=4, F=13, H=40, L=2, C=0, D=2, h0=False), [21, 21]
    H, D = 128, 2
    B = _batch(H, D, "split", prec, 0.0)
    _, bwd8 = _tile_rows(prec, B, H, D, 0.0)
    split = [r for r in bwd8 if len(r)]
    assert split
    return dict(B=B, T=4, F=16, H=H, L=2, C=0, D=D, h0=False), [int((r if len(r) else split[0])[9]) for r in bwd8]


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ("bf16x3", "bf16", "fp32"))
def test_support_of_one_seed(prec):
    """dy = 0 and dhn nonzero only in slice (l, d), row b: every gradient of the layers above l, of layer l's other
    direction and of dx outside row b is exactly 0, and layer l's direction d is not.  A seed read from the wrong layer,
    direction or row fails this at any precision."""
    _need_h100()
    s, rows = _support_case(prec)
    B, T, F, H, L, D = (s[k] for k in "BTFHLD")
    rng = np.random.default_rng(13)
    flat = _flat(s, 12)
    x = rng.standard_normal((B, T, F)).astype(np.float32)
    lens = _lengths(B, T)
    names = abi_names(s)
    for l in range(L):
        for d in range(D):
            b = rows[d]
            dhn = np.zeros((L * D, B, H), np.float32)
            dhn[l * D + d, b] = rng.standard_normal(H).astype(np.float32)
            got, _ = kernel(s, prec, flat, x, None, None, lens=lens, head=False, dhn=dhn)
            g = got["grads"]
            blk = lambda ll, dd: np.concatenate([g[names[f"l{ll}d{dd}.{nm}"][0]:sum(names[f"l{ll}d{dd}.{nm}"])]   # noqa: E731
                                                 for nm in ("w_ih", "w_hh", "b_ih", "b_hh")])
            what = f"{prec} seed (l{l}, d{d}, b{b})"
            assert np.abs(blk(l, d)).max() > 0, what
            for ll in range(l + 1, L):
                for dd in range(D):
                    assert not blk(ll, dd).any(), f"{what}: layer {ll} direction {dd}"
            assert not blk(l, 1 - d).any(), f"{what}: other direction"
            assert not np.delete(got["dx"], b, 0).any(), f"{what}: dx rows other than {b}"
            assert np.abs(got["dx"][b]).max() > 0, what


def _rows(out, n):
    """Every per-row tensor of a head-less kernel() result with regions, for the first n rows: _per_row's, with dx in the
    place of the logits a head-less plan does not have."""
    r = _per_row(dict(out, logits=out["dx"]), np.arange(n))
    r["dx"] = r.pop("logits")
    if "RDS" in out["ws"]:
        for l, p in enumerate(out["ws"]["RDS"]):
            r[f"rds{l}"] = [None if a is None else a[:n] for a in p]
    return r


@pytest.mark.gpu
@pytest.mark.parametrize("kind,prec,rd", [("mixed", "bf16x3", 0.0), ("two", "bf16x3", 0.0), ("split", "bf16x3", 0.0),
                                          ("split", "bf16", 0.3)])
def test_rows_do_not_depend_on_the_tile(kind, prec, rd):
    """With a dhn seed in every row: the rows of 32-row forward tiles ("mixed", "two": the first 64 rows against a batch
    of 64) and of 8-row backward clusters ("split": against a larger batch whose backward splits nothing) must give the
    same bits where they sit in 16-row tiles."""
    _need_h100()
    H, D, T, L = 128, 2, 3, 2
    B = _batch(H, D, kind, prec, rd)
    fwd32, bwd8 = _tile_rows(prec, B, H, D, rd)
    if kind == "split":
        rows = np.unique(np.concatenate(bwd8))
        Bo = B + 32
        while _geometry(prec, Bo, H, D, 1, rd)[1]:
            Bo += 32
    else:
        rows = np.unique(np.concatenate(fwd32))
        Bo = 64
        assert _geometry(prec, Bo, H, D, 0, rd)[1] == 0 and _geometry(prec, Bo, H, D, 1, rd)[1] == 0
    assert (rows < min(B, Bo)).any()                # some compared rows sit in the tiles of interest at B only
    Bmax = max(B, Bo)
    s = dict(B=Bmax, T=T, F=16, H=H, L=L, C=0, D=D, h0=False)
    rng = np.random.default_rng(17)
    flat = _flat(s, 16)
    x = rng.standard_normal((Bmax, T, s["F"])).astype(np.float32)
    dy = rng.standard_normal((Bmax, T, D * H)).astype(np.float32)
    dhn = rng.standard_normal((L * D, Bmax, H)).astype(np.float32)
    lens = _lengths(Bmax, T)
    res = []
    for b in (B, Bo):
        out, _ = kernel(dict(s, B=b), prec, flat, np.ascontiguousarray(x[:b]), None, None, seed=SEED, regions=True, rd_p=rd,
                        lens=lens[:b], head=False, dy=np.ascontiguousarray(dy[:b]), dhn=np.ascontiguousarray(dhn[:, :b]))
        res.append(_rows(out, min(B, Bo)))
    _assert_bitwise(res[0], res[1], f"{kind} B{B} against B{Bo}")


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ("bf16x3", "fp32"))
def test_gru_module_hn_and_seed_support(prec):
    """Through ``GRU`` at H = 32 and B = 19, which the module pads in hidden and batch: h_n is the output at each
    direction's last valid step, bitwise, and a dhn seed in one (layer, direction, row) reaches only what it may."""
    from financial_market_data_analysis_b200 import GRU
    _need_h100()
    B, T, F, H, L, D = 19, 6, 13, 32, 2, 2
    torch.manual_seed(0)
    mine = GRU(F, H, L, batch_first=True, bidirectional=True, precision=prec).cuda()
    g = torch.Generator().manual_seed(9)
    x = torch.randn(B, T, F, generator=g).cuda()
    lens = torch.from_numpy(_lengths(B, T))
    y, hn = mine(x, lengths=lens)
    yc, hc = y.detach().cpu(), hn.detach().cpu()
    assert torch.equal(hc[(L - 1) * D], yc[torch.arange(B), lens - 1, :H])
    assert torch.equal(hc[(L - 1) * D + 1], yc[:, 0, H:])
    params = dict(mine.named_parameters())
    for l, d, b in ((0, 0, 18), (0, 1, 17), (1, 0, 1), (1, 1, 18)):
        mine.zero_grad(set_to_none=True)
        xg = x.clone().requires_grad_()
        y, hn = mine(xg, lengths=lens)
        dhn = torch.zeros_like(hn)
        dhn[l * D + d, b] = torch.randn(H, generator=g).cuda()
        torch.autograd.backward((y, hn), (torch.zeros_like(y), dhn))
        sfx = lambda ll, dd: f"_l{ll}" + ("_reverse" if dd else "")                # noqa: E731
        grads = lambda ll, dd: [params[n + sfx(ll, dd)].grad for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]  # noqa: E731
        what = f"{prec} seed (l{l}, d{d}, b{b})"
        assert any(bool(q.abs().max() > 0) for q in grads(l, d)), what
        for ll in range(l + 1, L):
            for dd in range(D):
                assert all(not bool(q.any()) for q in grads(ll, dd)), f"{what}: layer {ll} direction {dd}"
        assert all(not bool(q.any()) for q in grads(l, 1 - d)), f"{what}: other direction"
        gx = xg.grad.cpu()
        assert not torch.cat([gx[:b], gx[b + 1:]]).any() and bool(gx[b].abs().max() > 0), what
