"""Recurrent dropout and per-sequence lengths one step and one GEMM at a time, from the kernels' own operands, in every
tile geometry of the scans.

test_gpu_recurrent_dropout.py and test_gpu_lengths.py compare these paths only free-running, at parity bounds that a
bf16-sized operand error passes (tests/ROUNDING_MODEL.md, "Mutations of the backward"), and only at batches too small for
the scans' 32-row forward tiles or 8-row backward clusters.  Here, as in test_gpu_tc_steps.py, gru_driver recomputes from
the bits the kernels read (DESIGN.md §4.8 for the masks, §4.5 for the lengths):
  y_step, g_step, logits_step, w_step   the forward, one step from the kernel's h_{t-1}, through m * h_{t-1};
  dg_step    layer 0's dgi and dgh per direction and step: the gate math on m * h_{t-1}, the carry m (dh z + P) leaving a
             valid step and passed on unmasked by a padded one, dgi = dgh = 0 at padded steps;
  dh0_step   dh_{-1} of layer 0: masked by the scans, unmasked in the fp32 path's carry (mul_kernel masks it into dh0);
  gemm_step  layer 0's backward GEMMs: dW_hh from the masked-state planes R shifted by one row and m * h0, the rest as in
             the sibling file, the head's dY with the lengths' mean and padding;
and bit for bit: the masks in the stash against their host restatement, R = split_bf16(fp32(m * Y)) (the float32 product
at fp32), the Y planes to_planes_kernel writes for the next layer, the input, dgi and dgh planes (zero at padded steps).
The tile-kind shapes take their batch from the recurrent-dropout scans' geometry on the device (bigru_scan_geometry of a
plan with recurrent_p > 0), and a row's bits must not depend on its tile: rows of 32-row forward tiles and of 8-row backward
clusters are compared with the same rows in a prefix or an extended batch, where they sit in 16-row tiles.

configs[1] runs at full size (B512 T128 F64 H256 L2 D2) with its forward steps sampled by batch tile.
Run on an H100:  python -m pytest tests/test_gpu_rd_steps.py -m gpu -q
(BIGRU_RD_STEPS_REPORT=path.jsonl appends every measured distance to that file.)  Measurements and mutations:
tests/ROUNDING_MODEL.md, section "Recurrent dropout and lengths, one step at a time"."""
import ctypes as C
import json
import os
import resource

import numpy as np
import pytest

import oracle_c
from gru_driver import (CODE, abi_names, backward_steps, dist, dropout_mask, gemm_steps, kernel, kernel_gemm_steps,
                        kernel_steps, plane_checks, stepwise)
from test_gpu_scan_tiles import _assert_bitwise, _per_row
from test_gpu_tc_steps import _first_rows_zero
from test_recurrent_dropout_cpu import rd_masks

SEED = 20261018
NB = 16                    # rows of a batch tile (SCAN_NB)


def _geometry(prec, B, H, D, scan, rd_p):
    """(R, n_split) of bigru_scan_geometry for a plan of this batch with recurrent dropout rd_p; scan 0 forward, 1 backward."""
    import financial_market_data_analysis_b200 as pkg
    lib = pkg._lib.load()
    plan = C.c_void_p()
    pkg._lib.check(lib.bigru_plan_create_rd(B, 2, 16, H, 1, 3, int(D == 2), CODE[prec], rd_p, C.byref(plan)), "plan_create")
    try:
        R, n2 = C.c_int(), C.c_int()
        pkg._lib.check(lib.bigru_scan_geometry(plan, scan, C.byref(R), C.byref(n2)), "scan_geometry")
        return R.value, n2.value
    finally:
        lib.bigru_plan_destroy(plan)


def _batch(H, D, kind, prec, rd_p):
    """A batch (a multiple of 32) whose recurrent-dropout forward scan has two-tile and one-tile clusters ("mixed") or only
    two-tile clusters ("two"), or whose backward scan splits the tiles of its last round into 8-row clusters ("split")."""
    R = _geometry(prec, 32, H, D, int(kind == "split"), rd_p)[0]
    n = {"mixed": (R // (2 * D) + 1) * 2 * D, "two": 2 * R // (2 * D) * (2 * D), "split": (2 * R // (2 * D) + 1) * 2 * D}[kind]
    return NB * n // D


def _tile_rows(prec, B, H, D, rd_p):
    """Per direction, the rows in 32-row forward tiles and in 8-row backward clusters at batch B (the scans' geometry)."""
    ntd = B // NB
    n2 = _geometry(prec, B, H, D, 0, rd_p)[1]
    L8 = _geometry(prec, B, H, D, 1, rd_p)[1]
    fwd32 = [np.arange(2 * NB * (n2 // D)) for _ in range(D)]
    bwd8 = [[] for _ in range(D)]
    for q in range(D * ntd - L8, D * ntd):
        bwd8[q // ntd].extend(range((q % ntd) * NB, (q % ntd + 1) * NB))
    return fwd32, [np.asarray(r, int) for r in bwd8]


def _lengths(B, T):
    """Ragged lengths in [1, T]: len = 1 and len = T in the first and in the last 16-row tile."""
    rng = np.random.default_rng([B, T, 5])
    n = rng.integers(1, T + 1, B)
    n[0], n[1], n[-2], n[-1] = T, 1, 1, T
    return n


# the regimes where the masked and ragged scans go wrong, and how a shape proves it is in one.  Regimes marked "device"
# are proved from the scans' geometry in test_shapes_are_in_the_regimes_they_claim.
REGIMES = {
    # scan: cluster size x direction count, recurrent dropout on; H = 512 is bf16 only
    "cluster2_d1": lambda s: s["H"] == 128 and s["D"] == 1 and s["rd"] > 0,
    "cluster2_d2": lambda s: s["H"] == 128 and s["D"] == 2 and s["rd"] > 0,
    "cluster4_d1": lambda s: s["H"] == 256 and s["D"] == 1 and s["rd"] > 0,
    "cluster4_d2": lambda s: s["H"] == 256 and s["D"] == 2 and s["rd"] > 0,
    "cluster8_d1": lambda s: s["H"] == 512 and s["D"] == 1 and s["rd"] > 0,
    "cluster8_d2": lambda s: s["H"] == 512 and s["D"] == 2 and s["rd"] > 0,
    # scan length
    "T1_both_dirs": lambda s: s["T"] == 1 and s["D"] == 2 and s["rd"] > 0,
    "T2_both_dirs": lambda s: s["T"] == 2 and s["D"] == 2 and s["rd"] > 0,
    "T_long": lambda s: s["T"] >= 300 and s["rd"] > 0,
    # tile kinds of the recurrent-dropout scans (device): 32-row and 16-row forward clusters mixed, 32-row only, 8-row
    # backward clusters in the last round
    "fwd_mixed_tiles": "device", "fwd_two_tile_only": "device", "bwd_split_8row": "device",
    "configs1_full": lambda s: (s["B"], s["T"], s["F"], s["H"], s["L"], s["D"]) == (512, 128, 64, 256, 2, 2) and s["rd"] > 0,
    # lengths: with and without recurrent dropout; len = 1 and len = T rows in one 16-row tile; padded rows in 32-row,
    # 16-row and 8-row tiles (device)
    "lengths_rd": lambda s: s["lens"] and s["rd"] > 0, "lengths_plain": lambda s: s["lens"] and s["rd"] == 0,
    "len1_lenT_one_tile": lambda s: s["lens"] and s["T"] > 1,
    "padded_32row": "device", "padded_16row": "device", "padded_8row": "device",
    # an initial state: the masked h0 of the w0 term and the masked dh_{-1}
    "h0_bf16x3_rd": lambda s: s["h0"] and s["rd"] > 0 and "bf16x3" in s["precs"],
    "h0_fp32_rd": lambda s: s["h0"] and s["rd"] > 0 and "fp32" in s["precs"],
    # mask offsets of layers >= 2; input and inter-layer dropout with recurrent dropout (every layer owns its input planes)
    "L3": lambda s: s["L"] >= 3 and s["rd"] > 0,
    "dropout_own_planes": lambda s: s["drop"] > 0 and s["rd"] > 0 and s["L"] >= 2,
    # p: 1/(1-p) inexact; p = 0.9 scales kept units by 10
    "p0.05": lambda s: s["rd"] == 0.05, "p0.3": lambda s: s["rd"] == 0.3, "p0.9": lambda s: s["rd"] == 0.9,
    # the fp32 path: gates kernels with masks, with lengths (ragged reverse rows) and with h0
    "fp32_rd_lengths": lambda s: "fp32" in s["precs"] and s["rd"] > 0 and s["lens"] and s["D"] == 2,
}


def _shape(B, T, F, H, L, D, precs, regimes, rd=0.3, h0=False, lens=False, drop=0.0, C=3, **kw):
    return dict(B=B, T=T, F=F, H=H, L=L, C=C, D=D, h0=h0, precs=precs, rd=rd, lens=lens, drop=drop, regimes=regimes, **kw)


SHAPES = {
    "h128_t1_d2": _shape(32, 1, 5, 128, 1, 2, ("bf16",), ("cluster2_d2", "T1_both_dirs", "p0.3")),
    "h128_t2_h0": _shape(32, 2, 24, 128, 2, 2, ("bf16x3",), ("cluster2_d2", "T2_both_dirs", "h0_bf16x3_rd", "p0.05"),
                         rd=0.05, h0=True),
    # p = 0.9 only with a few steps: z * 10 h_{t-1} grows the state geometrically, and over 301 steps to inf
    "h128_t301_d1": _shape(32, 301, 13, 128, 1, 1, ("bf16", "bf16x3"), ("cluster2_d1", "T_long", "p0.3")),
    "h256_l3_d1": _shape(64, 6, 16, 256, 3, 1, ("bf16",), ("cluster4_d1", "L3", "p0.9"), rd=0.9),
    "h256_drop_d2": _shape(32, 7, 20, 256, 2, 2, ("bf16x3",), ("cluster4_d2", "dropout_own_planes", "p0.3"), drop=0.2),
    "h512_d1": _shape(32, 5, 40, 512, 1, 1, ("bf16",), ("cluster8_d1", "p0.3")),
    "h512_d2_lens": _shape(32, 9, 24, 512, 2, 2, ("bf16",), ("cluster8_d2", "lengths_rd", "len1_lenT_one_tile", "p0.3",
                                                            "padded_16row"), lens=True),
    "h128_lens_plain": _shape(64, 6, 16, 128, 2, 2, ("bf16x3", "bf16"), ("lengths_plain", "len1_lenT_one_tile",
                                                                        "padded_16row"), rd=0.0, lens=True),
    "mixed_lens": _shape("mixed", 5, 16, 128, 2, 2, ("bf16x3",), ("cluster2_d2", "fwd_mixed_tiles", "lengths_rd",
                                                                  "len1_lenT_one_tile", "padded_32row", "padded_16row"), lens=True),
    "two_h0": _shape("two", 4, 16, 128, 1, 2, ("bf16x3",), ("cluster2_d2", "fwd_two_tile_only", "h0_bf16x3_rd"), h0=True),
    "split_lens": _shape("split", 4, 16, 128, 2, 2, ("bf16x3", "bf16"), ("cluster2_d2", "bwd_split_8row", "lengths_rd",
                                                                        "padded_8row", "padded_16row"), lens=True),
    "split_lens_plain": _shape("split", 3, 16, 128, 1, 2, ("bf16",), ("bwd_split_8row", "lengths_plain", "padded_8row"),
                               rd=0.0, lens=True),
    "configs1": _shape(512, 128, 64, 256, 2, 2, ("bf16x3", "bf16"), ("configs1_full", "cluster4_d2", "p0.3"),
                       sample_tiles=(0, 1, -1)),
    "fp32_lens": _shape(24, 7, 13, 40, 2, 2, ("fp32",), ("fp32_rd_lengths", "lengths_rd", "len1_lenT_one_tile", "p0.3"),
                        lens=True),
    "fp32_h0_l3": _shape(16, 6, 13, 48, 3, 2, ("fp32",), ("h0_fp32_rd", "L3", "p0.9"), rd=0.9, h0=True),
}

# Kernel-vs-model tolerances (rel-L2, max-abs over max |model|) per class: about 4x the worst value measured on an H100
# 80GB HBM3 (SXM, 700 W power limit) over the shapes above; the measurements are in tests/ROUNDING_MODEL.md.
# fp32 w_step measured 0 (the float32 model forms the lin_w gradient as the kernel does); its bound is 1e-7.
TOL = {
    "bf16": {"y_step": (4e-6, 5.6e-6), "g_step": (1.6e-6, 3.4e-6), "logits_step": (7.2e-5, 1.8e-4), "w_step": (2.4e-5, 2.8e-4),
             "dg_step": (8e-7, 2e-6), "dh0_step": (4.8e-7, 1.1e-6), "gemm_step": (9.6e-6, 1.5e-5)},
    "bf16x3": {"y_step": (7.2e-6, 1e-5), "g_step": (4e-6, 7.6e-6), "logits_step": (1.4e-5, 1.4e-5), "w_step": (1.4e-5, 1.7e-5),
               "dg_step": (1.2e-6, 2.2e-6), "dh0_step": (8.8e-7, 1.2e-6), "gemm_step": (1.8e-5, 1.7e-5)},
    "fp32": {"y_step": (4.4e-7, 1e-6), "g_step": (2.2e-7, 7.6e-7), "logits_step": (1.1e-6, 1.9e-6), "w_step": (1e-7, 1e-7),
             "dg_step": (2e-6, 2.2e-6), "dh0_step": (5.6e-7, 7.2e-7)},
}


def _need_h100():
    import financial_market_data_analysis_b200 as pkg
    if pkg._lib.load().bigru_device_check(0) != 0:
        pytest.fail("no H100: " + pkg._lib.load().bigru_last_error().decode())


def _resolve(s, prec):
    """The shape with its batch read off the device geometry where it names a tile kind."""
    if isinstance(s["B"], str):
        return dict(s, B=_batch(s["H"], s["D"], s["B"], prec, s["rd"]))
    return dict(s)


def _holds(r, s, prec):
    """Whether shape s (resolved at prec) is in regime r; "device" regimes from the scans' geometry at s's batch."""
    rule = REGIMES[r]
    B, T, H, D = s["B"], s["T"], s["H"], s["D"]
    lens = _lengths(B, T) if s["lens"] else np.full(B, T)
    if r == "len1_lenT_one_tile":
        return rule(s) and lens[0] == T and lens[1] == 1
    if rule != "device":
        return rule(s)
    if prec == "fp32":
        return False
    n = D * B // NB
    n2 = _geometry(prec, B, H, D, 0, s["rd"])[1]
    L8 = _geometry(prec, B, H, D, 1, s["rd"])[1]
    fwd32, bwd8 = _tile_rows(prec, B, H, D, s["rd"])
    padded = lens < T
    one16 = [np.setdiff1d(np.arange(B), np.concatenate([fwd32[d], bwd8[d]])) for d in range(D)]
    return {"fwd_mixed_tiles": 0 < n2 < n - n2, "fwd_two_tile_only": n2 > 0 and 2 * n2 == n, "bwd_split_8row": L8 > 0,
            "padded_32row": all(len(fwd32[d]) and padded[fwd32[d]].any() for d in range(D)),
            "padded_8row": any(len(bwd8[d]) and padded[bwd8[d]].any() for d in range(D)),
            "padded_16row": all(padded[one16[d]].any() for d in range(D))}[r]


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
        # a shape is in a regime when one of its precisions puts it there
        for r in s0["regimes"]:
            assert any(_holds(r, s, prec) for prec, s in resolved.items()), (name, r)
        covered |= set(s0["regimes"])
    assert covered == set(REGIMES), set(REGIMES) - covered


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ("bf16x3", "bf16"))
@pytest.mark.parametrize("H", (128, 256, 512))
@pytest.mark.parametrize("D", (1, 2))
def test_recurrent_dropout_scans_have_the_plain_residency(prec, H, D):
    """DESIGN.md §4.8: the masks add no shared memory, so the recurrent-dropout scans' residency R, and with it every
    geometry, equals the plain scans'."""
    _need_h100()
    if H == 512 and prec == "bf16x3":
        pytest.skip("hidden 512 runs at bf16 only")
    for scan in (0, 1):
        for B in (32, 512, 1024):
            assert _geometry(prec, B, H, D, scan, 0.3) == _geometry(prec, B, H, D, scan, 0.0), (scan, B)


def _inputs(s):
    B, T, F, H, L, C_, D = (s[k] for k in "BTFHLCD")
    rng = np.random.default_rng([B, T, F, H, L, D, 7])
    k = 1 / np.sqrt(H)                                          # nn.GRU / nn.Linear initialisation scale
    flat = rng.uniform(-k, k, oracle_c.lib().bigru_ref_param_count(F, H, L, C_, D)).astype(np.float32)
    x = rng.standard_normal((B, T, F)).astype(np.float32)
    h0 = (0.5 * rng.standard_normal((L * D, B, H))).astype(np.float32) if s["h0"] else None
    dl = rng.standard_normal((B, C_)).astype(np.float32)
    return flat, x, h0, dl


def _ops(got, s, x, masks, exact):
    """gemm_steps' operands from the kernel's workspace: its planes, or (exact) the fp32 values they were split from."""
    ws, T, F, H, D = got["ws"], s["T"], s["F"], s["H"], s["D"]
    if not exact:
        ops = dict(DGIP=ws["DGIP"], DGHP=ws["DGHP"], XP=ws["XP"], YP=ws["YP"][0], DGI=ws["DGI"], DGH=ws["DGH"],
                   DCAT=ws["DCAT"])
        if masks is not None:
            ops["RDS"] = ws["RDS"][0]
        return ops
    xp = np.zeros(ws["XP"][0].shape, np.float32)
    xp[..., :F] = x
    ops = dict(DGIP=(ws["DGI"], None), DGHP=(_first_rows_zero(ws["DGH"], T), None), XP=(xp, None),
               YP=(got["ys"][0], None), DGI=ws["DGI"], DGH=ws["DGH"], DCAT=ws["DCAT"])
    if masks is not None:
        y = got["ys"][0].astype(np.float32)
        ops["RDS"] = (np.concatenate([masks[0][d][:, None, :] * y[..., d * H:(d + 1) * H] for d in range(D)], 2), None)
    return ops


CASES = [(n, p) for n, s in SHAPES.items() for p in s["precs"]]


@pytest.mark.gpu
@pytest.mark.parametrize("name,prec", CASES, ids=[f"{n}-{p}" for n, p in CASES])
def test_kernel_steps_match_their_models(name, prec):
    _need_h100()
    s = _resolve(SHAPES[name], prec)
    B, T, F, H, L, D = (s[k] for k in "BTFHLD")
    flat, x, h0, dl = _inputs(s)
    lens = _lengths(B, T) if s["lens"] else None
    got, names = kernel(s, prec, flat, x, h0, dl, p=s["drop"], seed=SEED, regions=True, rd_p=s["rd"], lens=lens)
    ws = got["ws"]
    masks = rd_masks(SEED, s["rd"], L, D, B, H) if s["rd"] > 0 else None
    drops = None
    xd = x
    if s["drop"] > 0:
        drops = [dropout_mask(SEED, 0, B, T, F, s["drop"])] + [dropout_mask(SEED, l, B, T, D * H, s["drop"]) for l in range(1, L)]
        xd = x * drops[0] + np.float32(0)                     # dropout_kernel writes +0 where it drops
    bad_planes = {k: v for k, v in plane_checks(got, s, prec, xd, masks, lens, drop=s["drop"] > 0).items() if v}

    rows_out, bad = [], []

    def compare(key, k, m, e):
        tname, cls = key
        km, me, ke = dist(k, m), dist(m, e), dist(k, e)
        rows_out.append(dict(shape=name, prec=prec, B=B, tensor=tname, cls=cls, km_l2=km[0], km_max=km[1], me_l2=me[0],
                             me_max=me[1], ke_l2=ke[0], ke_max=ke[1]))
        tol = TOL[prec][cls]
        if not (km[0] <= tol[0] and km[1] <= tol[1]):
            bad.append((tname, km, tol))

    # forward: one step from the kernel's state, with the gate stash
    rows = None
    if "sample_tiles" in s:
        rows = np.concatenate([np.arange(NB) + NB * (t % (B // NB)) for t in s["sample_tiles"]])
    tk = kernel_steps(got, s, names, rows, gates=True)
    tm = stepwise(s, prec, flat, x, h0, dl, got, names, rows, gates=True, masks=masks, lens=lens, drops=drops)
    te = stepwise(s, "exact", flat, x, h0, dl, got, names, rows, gates=True, masks=masks, lens=lens, drops=drops)
    for key in tk:
        compare(key, tk[key], tm[key], te[key])
    del tk, tm, te
    # backward recurrence of layer 0, one step at a time from the kernel's operands.  fp32: the float64 model is the
    # kernel's model (its products are fp32 GEMMs), and the fp32 carry is masked into dh0 after the scan
    m0 = None if masks is None else masks[0]
    bprec = "exact" if prec == "fp32" else prec
    for a, b in zip(backward_steps(s, bprec, flat, h0, ws, got["ys"], names, masks=m0, lens=lens),
                    backward_steps(s, "exact", flat, h0, ws, got["ys"], names, masks=m0, lens=lens)):
        kind, d, t = a[:3]
        if kind == "dg":
            compare((f"bstep:dgi[d{d},t{t}]", "dg_step"), ws["DGI"][d][:, t].astype(np.float64), a[3], b[3])
            compare((f"bstep:dgh[d{d},t{t}]", "dg_step"), ws["DGH"][d][:, t].astype(np.float64), a[4], b[4])
        else:
            i = 4 if prec == "fp32" and m0 is not None else 3
            compare((f"bstep:dh0[d{d}]", "dh0_step"), ws["DHC"][d].astype(np.float64), a[i], b[i])
    # the backward GEMMs of layer 0 and the head, from the kernel's operand planes (tensor-core precisions)
    if prec != "fp32":
        gk = kernel_gemm_steps(got, s, names)
        gm = gemm_steps(s, prec, flat, dl, h0, _ops(got, s, xd, masks, False), names, got["arg"], masks=m0, lens=lens)
        ge = gemm_steps(s, "exact", flat, dl, h0, _ops(got, s, xd, masks, True), names, got["arg"], masks=m0, lens=lens)
        if drops is not None:                                   # dropout_kernel applies the mask to dx after the GEMM
            gm[("gemm:dx", "gemm_step")] = gm[("gemm:dx", "gemm_step")] * drops[0]
            ge[("gemm:dx", "gemm_step")] = ge[("gemm:dx", "gemm_step")] * drops[0]
        for key in gk:
            compare(key, gk[key], gm[key], ge[key])

    peak_gb = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 2 ** 20
    out = os.environ.get("BIGRU_RD_STEPS_REPORT")
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


def _rows(out):
    """Every per-row tensor of a kernel() result with recurrent dropout, in batch order."""
    r = _per_row(out, np.arange(out["logits"].shape[0]))
    for l, p in enumerate(out["ws"]["RDS"]):
        r[f"rds{l}"] = list(p)
    return r


def _prefix(r, n):
    """The first n batch rows of every tensor of _rows (batch-leading: logits, Y, Y planes, R; else the batch is axis 1)."""
    out = {}
    for k, v in r.items():
        lead = k == "logits" or k.startswith(("y", "rds"))
        cut = lambda a: None if a is None else (a[:n] if lead else a[:, :n])   # noqa: E731
        out[k] = [cut(a) for a in v] if isinstance(v, list) else cut(v)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("kind,prec", [("mixed", "bf16x3"), ("two", "bf16x3"), ("split", "bf16x3"), ("split", "bf16")])
def test_rows_do_not_depend_on_the_tile(kind, prec):
    """Masks are keyed by batch row, so the batch is not reversed here (as in test_gpu_scan_tiles.py): the same rows, seed
    and lengths at a second batch size, where they sit in 16-row tiles, must give the same bits.  "mixed" and "two" compare
    the first 64 rows (32-row forward tiles) with a batch of 64; "split" compares the rows of the 8-row backward clusters
    with a larger batch whose backward splits nothing."""
    _need_h100()
    H, D, T, L, rd = 128, 2, 3, 2, 0.3
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
    s = dict(B=Bmax, T=T, F=16, H=H, L=L, C=3, D=D, h0=False)
    rng = np.random.default_rng(11)
    n = sum(v[1] for v in abi_names(s).values())
    flat = (rng.standard_normal(n) * 0.08).astype(np.float32)
    x = rng.standard_normal((Bmax, T, s["F"])).astype(np.float32)
    dl = rng.standard_normal((Bmax, s["C"])).astype(np.float32)
    lens = _lengths(Bmax, T)
    res = []
    for b in (B, Bo):
        out, _ = kernel(dict(s, B=b), prec, flat, np.ascontiguousarray(x[:b]), None, np.ascontiguousarray(dl[:b]),
                        seed=SEED, regions=True, rd_p=rd, lens=lens[:b])
        res.append(_prefix(_rows(out), min(B, Bo)))
    _assert_bitwise(res[0], res[1], f"{kind} B{B} against B{Bo}")
