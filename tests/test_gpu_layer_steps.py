"""The tensor-core backward of every layer above 0 (BIGRU_PREC_BF16, BIGRU_PREC_BF16X3) one step and one GEMM at a time,
from the kernels' own operands.

The backward runs layers L-1 .. 0 through one dgi / dgh / planes / dh_{-1} region of the scratch, so after a whole
backward only layer 0's intermediates are left: test_gpu_tc_steps.py, test_gpu_rd_steps.py and test_gpu_gru_steps.py stop
there.  bigru_plan_set_backward_stop(plan, s) ends the backward after layer s, and the scratch then holds layer s's
intermediates and the upstream gradients of layers s-1 and s.  For each shape, precision and stop s >= 1, gru_driver
recomputes in float64, from exactly the bits the kernels read:
  dg_step    dgi and dgh of layer s per direction and step (backward_steps at layer s: its dY, its gates, its h_{t-1} or
             h0[s*D + d], W_hh of layer s, the carry seeded from the head's `last` share on the top layer, from dhn[s*D + d]
             on a head-less plan, else from zero; recurrent-dropout masks of layer s, lengths);
  dh0_step   dh_{-1} of layer s (the scratch's dhc);
  gemm_step  layer s's backward GEMMs (gemm_steps at layer s): dW_ih from the dgi planes and the Y planes of layer s-1, or
             the layer's own input planes when its input was dropped; dW_hh from the Y planes (or the masked-state planes)
             of layer s with its h0 term; the bias column sums; the dX GEMM into dy[l{s-1}], times the dropout factor of
             stream s when the input was dropped; the head's dcat and, where it survives, the top layer's dY.
The planes (Y, the layer's own input planes = split_bf16(fp32(Y[s-1] * factor)), dgi, dgh) must equal split_bf16 of
their sources bit for bit, and with h0 the scratch's dh_{-1} must equal the caller's dh0 slice of layer s.  Without a
tolerance: the stop leaves the gradients of layers >= s bitwise those of a whole backward and those below exactly 0, dx
and the lower dh0 slices as the caller filled them; stop 0 is bitwise the plain backward, and resetting the stop to 0
restores it.  The forward is not compared: test_gpu_tc_steps.py checks every layer's forward one step at a time.

configs[1] runs at full size (B512 T128 F64 H256 L2 D2) at stop 1: its layer 1 is the head-seeded top layer, its dW_ih the
largest GEMM of the backward (M = 768, N = 512, K = 65 536), and at bf16x3 its backward scan splits the last round into
8-row clusters.  The whole file took 66 s on an H100 80GB HBM3 (SXM, 700 W power limit), with a peak host memory of
10.7 GB (configs[1]).
Run on an H100:  python -m pytest tests/test_gpu_layer_steps.py -m gpu -q
(BIGRU_LAYER_STEPS_REPORT=path.jsonl appends every measured distance to that file.)  Measurements and mutations:
tests/ROUNDING_MODEL.md, section "Upper layers one step and one GEMM at a time"."""
import ctypes as C
import json
import os
import resource

import numpy as np
import pytest
import torch

import test_gpu_gru_steps
import test_gpu_rd_steps
import test_gpu_tc_steps
from gru_driver import (CODE, WS, abi_names, backward_steps, dist, dropout_mask, dropped, gemm_steps, kernel,
                        kernel_gemm_steps, param_names, plane_checks, region)
from test_gpu_scan_tiles import _bwd_rule, _geometry
from test_gpu_tc_steps import NSM, _first_rows_zero, cdiv, wg_splits
from test_recurrent_dropout_cpu import rd_masks

SEED = 20261019


def dwih_gemms(s):
    """(splits, units, short last split) of an upper layer's dW_ih launch: M = 3H, N = D*H, K = B*T, 128 x 128 tiles, one
    batch per direction (dw0_gemms of test_gpu_tc_steps.py with the input width D*H)."""
    kb = cdiv(s["B"] * s["T"], 64)
    tiles = cdiv(3 * s["H"], 128) * cdiv(s["D"] * s["H"], 128) * s["D"]
    sp = wg_splits(tiles, kb)
    return sp, tiles * sp, sp > 1 and kb % cdiv(kb, sp) != 0


# the regimes where an upper layer's backward goes wrong, and how a shape proves it is in one.  "device": proved from
# the backward scan's geometry on the device in test_device_regimes_hold
REGIMES = {
    # where the stop is, and with it which ping-pong buffer the layer reads (L-1-s even: dYa) and writes
    "L2_stop1": lambda s: s["L"] == 2 and 1 in s["stops"],
    "L3_stop1": lambda s: s["L"] == 3 and 1 in s["stops"], "L3_stop2": lambda s: s["L"] == 3 and 2 in s["stops"],
    # the carry: the head's `last` share into the top layer at L >= 2, zero into a middle layer
    "head_seeded_top": lambda s: s["head"] and s["L"] - 1 in s["stops"],
    "zero_carry_middle": lambda s: s["head"] and any(0 < st < s["L"] - 1 for st in s["stops"]),
    # scan: cluster size x direction count; H = 512 is bf16 only
    "cluster2_d1": lambda s: s["H"] == 128 and s["D"] == 1, "cluster2_d2": lambda s: s["H"] == 128 and s["D"] == 2,
    "cluster4_d1": lambda s: s["H"] == 256 and s["D"] == 1, "cluster4_d2": lambda s: s["H"] == 256 and s["D"] == 2,
    "cluster8_d1": lambda s: s["H"] == 512 and s["D"] == 1, "cluster8_d2": lambda s: s["H"] == 512 and s["D"] == 2,
    # an initial state at bf16x3 on an upper layer: its h0 slice, dh0 slice and w0 term
    "h0_bf16x3_upper": lambda s: s["h0"] and "bf16x3" in s["precs"],
    # an upper layer's dW_ih (N = D*H): one split, a short last split, more units than SMs
    "dwih_one_split": lambda s: dwih_gemms(s)[0] == 1,
    "dwih_short_last_split": lambda s: dwih_gemms(s)[2],
    "dwih_units_gt_sms": lambda s: dwih_gemms(s)[1] > NSM,
    # the backward scan of an upper layer with 8-row split clusters in its last round
    "bwd_split_8row_upper": "device",
    # dropout between layers (the layer owns its input planes, dX is dropped in place with mask stream s)
    "drop_head_bf16": lambda s: s["head"] and s["drop"] > 0 and "bf16" in s["precs"],
    "drop_head_bf16x3": lambda s: s["head"] and s["drop"] > 0 and "bf16x3" in s["precs"],
    "drop_headless_bf16": lambda s: not s["head"] and s["drop"] > 0 and "bf16" in s["precs"],
    "drop_headless_bf16x3": lambda s: not s["head"] and s["drop"] > 0 and "bf16x3" in s["precs"],
    # recurrent dropout (masks and masked state of layer s) and lengths at an upper layer
    "rd_upper": lambda s: s["rd"] > 0, "lengths_upper": lambda s: s["lens"],
    # recurrent dropout with h0: the masked initial state S.H0M of layer s in the w0 term
    "rd_h0_upper": lambda s: s["rd"] > 0 and s["h0"],
    # head-less plans: the top layer on the caller's y / dy, a lower layer seeded from dhn[s*D + d]
    "headless_top": lambda s: not s["head"] and s["L"] - 1 in s["stops"],
    "headless_lower_dhn": lambda s: not s["head"] and s["dhn"] and any(st < s["L"] - 1 for st in s["stops"]),
    "configs1_full": lambda s: (s["B"], s["T"], s["F"], s["H"], s["L"], s["D"]) == (512, 128, 64, 256, 2, 2) and s["head"],
}


def _shape(B, T, F, H, L, D, precs, stops, regimes, head=True, h0=False, drop=0.0, rd=0.0, lens=False, C=3):
    return dict(B=B, T=T, F=F, H=H, L=L, C=C, D=D, precs=precs, stops=stops, regimes=regimes, head=head, h0=h0, drop=drop,
                rd=rd, lens=lens, dy=not head, dhn=not head)


SHAPES = {
    "h128_l2_d2": _shape(32, 9, 24, 128, 2, 2, ("bf16", "bf16x3"), (1,),
                         ("L2_stop1", "head_seeded_top", "cluster2_d2", "dwih_one_split")),
    "h128_l3_d1_h0": _shape(32, 7, 13, 128, 3, 1, ("bf16x3",), (1, 2),
                            ("L3_stop1", "L3_stop2", "head_seeded_top", "zero_carry_middle", "cluster2_d1",
                             "h0_bf16x3_upper", "dwih_one_split"), h0=True),
    "h256_l2_d1": _shape(48, 6, 20, 256, 2, 1, ("bf16",), (1,), ("L2_stop1", "cluster4_d1")),
    "h512_l2_d1": _shape(32, 5, 16, 512, 2, 1, ("bf16",), (1,), ("L2_stop1", "cluster8_d1")),
    "h512_l3_d2": _shape(32, 4, 16, 512, 3, 2, ("bf16",), (1, 2), ("L3_stop1", "L3_stop2", "cluster8_d2", "zero_carry_middle")),
    "drop_l3_d2": _shape(32, 6, 16, 128, 3, 2, ("bf16x3", "bf16"), (1, 2),
                         ("L3_stop1", "L3_stop2", "drop_head_bf16", "drop_head_bf16x3", "cluster2_d2"), drop=0.3),
    "rd_lens_l2": _shape(32, 7, 16, 256, 2, 2, ("bf16x3",), (1,), ("rd_upper", "lengths_upper", "cluster4_d2"),
                         rd=0.3, lens=True),
    "rd_h0_l2": _shape(32, 5, 16, 128, 2, 2, ("bf16x3",), (1,), ("rd_upper", "rd_h0_upper", "h0_bf16x3_upper"),
                       rd=0.3, h0=True),
    "gru_drop_l2": _shape(32, 5, 16, 128, 2, 2, ("bf16", "bf16x3"), (1,),
                          ("headless_top", "drop_headless_bf16", "drop_headless_bf16x3"), head=False, drop=0.3),
    "gru_rd_lens_l3": _shape(32, 6, 16, 256, 3, 1, ("bf16x3",), (1,), ("headless_lower_dhn", "rd_upper", "lengths_upper"),
                             head=False, rd=0.3, lens=True),
    "configs1": _shape(512, 128, 64, 256, 2, 2, ("bf16x3", "bf16"), (1,),
                       ("configs1_full", "head_seeded_top", "cluster4_d2", "bwd_split_8row_upper", "dwih_short_last_split",
                        "dwih_units_gt_sms")),
}


def test_shapes_are_in_the_regimes_they_claim():
    covered = set()
    for name, s in SHAPES.items():
        for r in s["regimes"]:
            if REGIMES[r] != "device":
                assert REGIMES[r](s), (name, r)
        covered |= set(s["regimes"])
        assert all(1 <= st < s["L"] for st in s["stops"]), name
        assert s["B"] % 16 == 0 and ("bf16x3" not in s["precs"] or (s["B"] % 32 == 0 and s["H"] <= 256))
        assert s["H"] != 512 or s["B"] % 32 == 0
        assert not (s["h0"] and ("bf16" in s["precs"] or s["lens"]))   # the library refuses both
    assert covered == set(REGIMES), set(REGIMES) - covered
    assert set(SHAPES["configs1"]["precs"]) == {"bf16", "bf16x3"}
    # configs[1]'s layer-1 dW_ih: 11 splits of 94 k-blocks (the last one 84), 48 tiles -> 528 units
    assert dwih_gemms(SHAPES["configs1"]) == (11, 528, True)


@pytest.mark.gpu
def test_device_regimes_hold():
    _need_h100()
    for name, s in SHAPES.items():
        if "bwd_split_8row_upper" in s["regimes"]:
            R, n8 = _geometry("bf16x3" if "bf16x3" in s["precs"] else "bf16", s["B"], s["H"], s["D"], 1)
            assert n8 > 0 and n8 == _bwd_rule(R, s["D"] * s["B"] // 16), (name, R, n8)


# ---- the stop's refusals and the regions it moves ------------------------------------------------------------------------
STOP_CASES = [(prec, L, D, head) for prec, in (("fp32",), ("bf16",), ("bf16x3",)) for L in (1, 2, 3, 4) for D in (1, 2)
              for head in (True, False)]


@pytest.mark.parametrize("case", STOP_CASES, ids=[f"{c[0]}-L{c[1]}-D{c[2]}-{'head' if c[3] else 'gru'}" for c in STOP_CASES])
def test_backward_stop_moves_the_regions(case):
    """bigru_plan_set_backward_stop refuses a null plan and stops outside [0, L); at stop s the backward's intermediates
    (DGI, DGH, their planes, DHC) are valid for layer s alone, DY for {0, 1} at stop 0 and {s-1, s} above (below L, and
    never a head-less plan's top layer), and no offset moves."""
    import financial_market_data_analysis_b200 as pkg
    lib = pkg._lib.load()
    prec, L, D, head = case
    B, T, F, H = (32, 3, 13, 128) if prec != "fp32" else (8, 3, 13, 24)
    plan = C.c_void_p()
    if head:
        pkg._lib.check(lib.bigru_plan_create(B, T, F, H, L, 3, int(D == 2), CODE[prec], C.byref(plan)), "plan_create")
    else:
        pkg._lib.check(lib.bigru_gru_plan_create(B, T, F, H, L, int(D == 2), CODE[prec], C.byref(plan)), "gru_plan_create")
    try:
        assert lib.bigru_plan_set_backward_stop(None, 0) == pkg._lib.ERR_ARG
        for bad in (-1, L, L + 1):
            assert lib.bigru_plan_set_backward_stop(plan, bad) == pkg._lib.ERR_ARG, bad
        sc_layout = test_gpu_tc_steps._layout(B, T, F, H, L, 3, D, prec)[1]
        ref = None
        for stop in list(range(L)) + [0]:
            assert lib.bigru_plan_set_backward_stop(plan, stop) == 0
            keep = [0, 1] if stop == 0 else [stop - 1, stop]
            got = {}
            for which in WS:
                for layer in range(-1, L + 2):
                    rc, sc, off, lo, pitch = region(plan, which, layer)
                    if which in ("GATES", "Y_PLANES", "IN_PLANES"):
                        ok = 0 <= layer < L
                    elif which == "DCAT":
                        ok = head and layer == L
                    elif which == "DY":
                        ok = layer in keep and layer < L and (head or layer < L - 1)
                    else:
                        ok = layer == stop
                    if not ok:
                        assert rc == pkg._lib.ERR_ARG, (stop, which, layer, rc)
                    elif which.endswith("PLANES") and prec == "fp32":
                        assert rc == pkg._lib.ERR_UNSUPPORTED, (stop, which, layer)
                    elif which == "DY":         # the ping-pong buffer of the layer's parity
                        assert rc == 0 and (sc, pitch) == (1, D * H), (stop, layer)
                        assert off == 4 * sc_layout["dYa" if (L - 1 - layer) % 2 == 0 else "dYb"], (stop, layer)
                    else:
                        assert rc == 0, (stop, which, layer, lib.bigru_last_error())
                        # the stop's own regions are keyed without their layer: their offsets are every layer's
                        per_layer = which in ("GATES", "Y_PLANES", "IN_PLANES", "DCAT")
                        got[(which, layer if per_layer else None)] = (sc, off, lo, pitch)
            ref = got if ref is None else ref
            assert got == ref, stop
    finally:
        lib.bigru_plan_destroy(plan)


# ---- the kernels of layer s against their step models on the GPU ----------------------------------------------------------
def _need_h100():
    import financial_market_data_analysis_b200 as pkg
    if pkg._lib.load().bigru_device_check(0) != 0:
        pytest.fail("no H100: " + pkg._lib.load().bigru_last_error().decode())


def _inputs(s):
    B, T, F, H, L, C_, D = (s[k] for k in "BTFHLCD")
    rng = np.random.default_rng([B, T, F, H, L, D, 9])
    k = 1 / np.sqrt(H)                                          # nn.GRU / nn.Linear initialisation scale
    names = abi_names(s)
    flat = rng.uniform(-k, k, names["lin_b"][0] + C_ if s["head"] else names["lin_w"][0]).astype(np.float32)
    x = rng.standard_normal((B, T, F)).astype(np.float32)
    h0 = (0.5 * rng.standard_normal((L * D, B, H))).astype(np.float32) if s["h0"] else None
    dl = rng.standard_normal((B, C_)).astype(np.float32) if s["head"] else None
    dy = rng.standard_normal((B, T, D * H)).astype(np.float32) if s["dy"] else None
    dhn = rng.standard_normal((L * D, B, H)).astype(np.float32) if s["dhn"] else None
    return flat, x, h0, dl, dy, dhn


def _tol(s, prec):
    """TOL of the sibling file of each feature the shape has (test_gpu_tc_steps.py's alone for a plain shape), the widest
    bound per class where it has several."""
    tabs = [test_gpu_tc_steps.TOL[prec]]
    if s["rd"] > 0 or s["lens"]:
        tabs.append(test_gpu_rd_steps.TOL[prec])
    if not s["head"]:
        tabs.append(test_gpu_gru_steps.TOL[prec])
    return {c: tuple(max(t[c][i] for t in tabs) for i in (0, 1)) for c in ("dg_step", "dh0_step", "gemm_step")}


def _ops(got, s, l, xin, masks, exact, own):
    """gemm_steps' operands of layer l from the kernel's workspace: its planes, or (exact) the fp32 values they were split
    from.  xin: the layer's input as float32 (Y[l-1], dropped when the layer owns its planes)."""
    ws, T, H, D = got["ws"], s["T"], s["H"], s["D"]
    if not exact:
        ops = dict(DGIP=ws["DGIP"], DGHP=ws["DGHP"], XP=ws["XP"] if own else ws["YP"][l - 1], YP=ws["YP"][l],
                   DGI=ws["DGI"], DGH=ws["DGH"], DCAT=ws["DCAT"])
        if masks is not None:
            ops["RDS"] = ws["RDS"][l]
        return ops
    ops = dict(DGIP=(ws["DGI"], None), DGHP=(_first_rows_zero(ws["DGH"], T), None), XP=(xin, None),
               YP=(got["ys"][l], None), DGI=ws["DGI"], DGH=ws["DGH"], DCAT=ws["DCAT"])
    if masks is not None:
        y = got["ys"][l].astype(np.float32)
        ops["RDS"] = (np.concatenate([masks[l][d][:, None, :] * y[..., d * H:(d + 1) * H] for d in range(D)], 2), None)
    return ops


CASES = [(n, p, st) for n, s in SHAPES.items() for p in s["precs"] for st in s["stops"]]


@pytest.mark.gpu
@pytest.mark.parametrize("name,prec,stop", CASES, ids=[f"{n}-{p}-stop{st}" for n, p, st in CASES])
def test_layer_steps_match_their_models(name, prec, stop):
    _need_h100()
    s = SHAPES[name]
    B, T, F, H, L, D = (s[k] for k in "BTFHLD")
    head, l = s["head"], stop
    flat, x, h0, dl, dy, dhn = _inputs(s)
    lens = test_gpu_rd_steps._lengths(B, T) if s["lens"] else None
    got, names = kernel(s, prec, flat, x, h0, dl, p=s["drop"], seed=SEED, regions=True, rd_p=s["rd"], lens=lens, head=head,
                        dy=dy, dhn=dhn, layer=l)
    ws = got["ws"]
    masks = rd_masks(SEED, s["rd"], L, D, B, H) if s["rd"] > 0 else None
    own = s["drop"] > 0                                         # layers above 0 own their input planes under dropout
    factor = dropout_mask(SEED, l, B, T, D * H, s["drop"]) if own else None
    xin = dropped(got["ys"][l - 1], factor) if own else got["ys"][l - 1].astype(np.float32)
    bad_planes = {k: v for k, v in plane_checks(got, s, prec, xin if own else None, masks, lens, drop=own, layer=l).items()
                  if v}
    # the stop: layers below s have zero gradients, dx and their dh0 slices stay as kernel() filled them (zeros)
    below = [v for k, v in names.items() if k[1].isdigit() and int(k[1:k.index("d")]) < l]
    assert all(not got["grads"][o:o + n].any() for o, n in below)
    assert not got["dx"].any()
    assert got["dh0"] is None or not got["dh0"][:l * D].any()

    tol = _tol(s, prec)
    rows_out, bad = [], []

    def compare(key, k, m, e):
        tname, cls = key
        km, me, ke = dist(k, m), dist(m, e), dist(k, e)
        rows_out.append(dict(shape=name, prec=prec, stop=l, tensor=tname, cls=cls, km_l2=km[0], km_max=km[1], me_l2=me[0],
                             me_max=me[1], ke_l2=ke[0], ke_max=ke[1]))
        if not (km[0] <= tol[cls][0] and km[1] <= tol[cls][1]):
            bad.append((tname, km, tol[cls]))

    ml = None if masks is None else masks[l]
    kw = dict(masks=ml, lens=lens, head=head, dy=dy, dhn=dhn, layer=l)
    for a, b in zip(backward_steps(s, prec, flat, h0, ws, got["ys"], names, **kw),
                    backward_steps(s, "exact", flat, h0, ws, got["ys"], names, **kw)):
        kind, d, t = a[:3]
        if kind == "dg":
            compare((f"bstep:l{l}:dgi[d{d},t{t}]", "dg_step"), ws["DGI"][d][:, t].astype(np.float64), a[3], b[3])
            compare((f"bstep:l{l}:dgh[d{d},t{t}]", "dg_step"), ws["DGH"][d][:, t].astype(np.float64), a[4], b[4])
        else:
            compare((f"bstep:l{l}:dh0[d{d}]", "dh0_step"), ws["DHC"][d].astype(np.float64), a[3], b[3])
    gk = kernel_gemm_steps(got, s, names, head=head, layer=l)
    kw = dict(masks=ml, lens=lens, head=head, layer=l, drop=factor)
    gm = gemm_steps(s, prec, flat, dl, h0, _ops(got, s, l, xin, masks, False, own), names, got["arg"], **kw)
    ge = gemm_steps(s, "exact", flat, dl, h0, _ops(got, s, l, xin, masks, True, own), names, got["arg"], **kw)
    assert gk.keys() == gm.keys()
    for key in gk:
        compare(key, gk[key], gm[key], ge[key])

    peak_gb = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 2 ** 20
    out = os.environ.get("BIGRU_LAYER_STEPS_REPORT")
    if out:
        with open(out, "a") as f:
            for r in rows_out:
                f.write(json.dumps(r) + "\n")
            f.write(json.dumps(dict(shape=name, prec=prec, stop=l, peak_host_gb=peak_gb, planes_bad=bad_planes)) + "\n")
    worst = {}
    for r in rows_out:
        w = worst.setdefault(r["cls"], [0.0, 0.0, np.inf])
        w[0], w[1], w[2] = max(w[0], r["km_l2"]), max(w[1], r["km_max"]), min(w[2], r["me_l2"] if r["me_l2"] > 0 else np.inf)
    print(f"\n{name} {prec} stop {l} peak host {peak_gb:.1f} GB " +
          " ".join(f"{c}: km_l2 {w[0]:.1e} km_max {w[1]:.1e} me_l2(min) {w[2]:.1e}" for c, w in worst.items()))
    assert not bad_planes, bad_planes
    assert not bad, sorted(bad, key=lambda b: -b[1][0])[:10]


# ---- the stop against the whole backward, bit for bit -------------------------------------------------------------------
EXACT_CASES = [("bf16x3", True, True), ("bf16", True, False), ("bf16x3", False, True), ("fp32", True, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("prec,head,h0", EXACT_CASES, ids=[f"{p}-{'head' if hd else 'gru'}{'-h0' if h else ''}"
                                                            for p, hd, h in EXACT_CASES])
def test_stop_is_the_whole_backward_cut_short(prec, head, h0):
    """One forward, then backward calls on the same plan: never stopped, stop 0 set explicitly, each stop s of L = 3 (with
    dx and dh0 filled with a sentinel), and stop 0 again.  Stop 0 and the reset are bitwise the plain backward; at stop s
    the gradients of layers >= s (and the head's) are bitwise the plain backward's, those below exactly 0, dx and the dh0
    slices below s keep the sentinel and the slices from s up are the plain backward's."""
    _need_h100()
    import financial_market_data_analysis_b200 as pkg
    lib, L_ = pkg._lib.load(), pkg._lib
    B, T, F, H, L, D = (32, 6, 16, 128, 3, 2) if prec != "fp32" else (8, 6, 13, 40, 3, 2)
    s = dict(B=B, T=T, F=F, H=H, L=L, C=3, D=D, head=head)
    rng = np.random.default_rng([B, T, F, H, L, D, int(head), 4])
    names0 = abi_names(s)
    n = names0["lin_b"][0] + 3 if head else names0["lin_w"][0]
    dev = torch.device("cuda")
    flat = torch.from_numpy(rng.uniform(-0.09, 0.09, n).astype(np.float32)).to(dev)
    x = torch.from_numpy(rng.standard_normal((B, T, F)).astype(np.float32)).to(dev)
    h0d = torch.from_numpy((0.5 * rng.standard_normal((L * D, B, H))).astype(np.float32)).to(dev) if h0 else None
    plan = C.c_void_p()
    if head:
        L_.check(lib.bigru_plan_create(B, T, F, H, L, 3, int(D == 2), CODE[prec], C.byref(plan)), "plan_create")
    else:
        L_.check(lib.bigru_gru_plan_create(B, T, F, H, L, int(D == 2), CODE[prec], C.byref(plan)), "gru_plan_create")
    try:
        sb, cb = C.c_size_t(), C.c_size_t()
        L_.check(lib.bigru_workspace_bytes(plan, C.byref(sb), C.byref(cb)), "workspace_bytes")
        stash = torch.zeros(sb.value // 4, device=dev)
        scratch = torch.zeros(cb.value // 4, device=dev)
        st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        ptr, p, seed = L_.ptr, 0.2, 99                         # training with dropout: every dropout backward runs
        dl = torch.from_numpy(rng.standard_normal((B, 3)).astype(np.float32)).to(dev) if head else None
        y = None if head else torch.zeros(B, T, D * H, device=dev)
        dy = None if head else torch.from_numpy(rng.standard_normal((B, T, D * H)).astype(np.float32)).to(dev)
        dhn = None if head else torch.from_numpy(rng.standard_normal((L * D, B, H)).astype(np.float32)).to(dev)
        logits = torch.zeros(B, 3, device=dev) if head else None
        if head:
            L_.check(lib.bigru_forward(plan, ptr(flat), ptr(x), ptr(h0d), p, 0, 1, seed, ptr(stash), ptr(scratch),
                                       ptr(logits), None, st), "forward")
        else:
            L_.check(lib.bigru_gru_forward(plan, ptr(flat), ptr(x), ptr(h0d), p, 1, seed, ptr(stash), ptr(scratch), ptr(y),
                                           None, None, st), "gru_forward")
        sentinel = 7.25

        def backward():
            grads = torch.full((n,), sentinel, device=dev)
            dx = torch.full((B, T, F), sentinel, device=dev)
            dh0 = torch.full((L * D, B, H), sentinel, device=dev) if h0 else None
            if head:
                L_.check(lib.bigru_backward(plan, ptr(flat), ptr(x), ptr(h0d), p, 0, 1, seed, ptr(stash), ptr(scratch),
                                            ptr(dl), ptr(grads), ptr(dx), ptr(dh0), st), "backward")
            else:
                L_.check(lib.bigru_gru_backward(plan, ptr(flat), ptr(x), ptr(h0d), p, 1, seed, ptr(stash), ptr(scratch),
                                                ptr(y), ptr(dy), ptr(dhn), ptr(grads), ptr(dx), ptr(dh0), None, st),
                         "gru_backward")
            torch.cuda.synchronize()
            return [None if t is None else t.cpu().numpy() for t in (grads, dx, dh0)]

        def same(a, b, what):
            for i, (u, v) in enumerate(zip(a, b)):
                assert (u is None) == (v is None), what
                if u is not None:
                    assert np.array_equal(u.view(np.uint32), v.view(np.uint32)), (what, i)

        plain = backward()
        assert not (plain[1] == sentinel).any() and (plain[2] is None or not (plain[2] == sentinel).any())
        L_.check(lib.bigru_plan_set_backward_stop(plan, 0), "set_backward_stop")
        same(backward(), plain, "stop 0")
        names = param_names(plan, s, head)
        for stop in range(1, L):
            L_.check(lib.bigru_plan_set_backward_stop(plan, stop), "set_backward_stop")
            grads, dx, dh0 = backward()
            for name, (o, k) in names.items():
                layer = int(name[1:name.index("d")]) if name[1].isdigit() else L
                if layer >= stop:
                    assert np.array_equal(grads[o:o + k].view(np.uint32), plain[0][o:o + k].view(np.uint32)), (stop, name)
                else:
                    assert np.array_equal(grads[o:o + k].view(np.uint32), np.zeros(k, np.uint32)), (stop, name)
            assert (dx == sentinel).all(), stop
            if h0:
                assert (dh0[:stop * D] == sentinel).all(), stop
                assert np.array_equal(dh0[stop * D:].view(np.uint32), plain[2][stop * D:].view(np.uint32)), stop
        L_.check(lib.bigru_plan_set_backward_stop(plan, 0), "set_backward_stop")
        same(backward(), plain, "stop reset to 0")
    finally:
        lib.bigru_plan_destroy(plan)
