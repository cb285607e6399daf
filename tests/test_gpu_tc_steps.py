"""The tensor-core backward (BIGRU_PREC_BF16, BIGRU_PREC_BF16X3) one step and one GEMM at a time, from the kernels' own
operands.

test_gpu_rounding_model.py compares the backward only free-running: the oracle's whole backward against the kernel's.
Rounding flips compound there, so its bf16 gradient bounds sit at the bf16 model's own distance from exact (about 2e-3).
Here bigru_workspace_region hands over what the backward kernels read and wrote (the gate stash G, the upstream gradient
dY, the fp32 dgi / dgh of layer 0 and their bf16 planes, the Y and input planes, dh_{-1}, the head's dcat), and
gru_driver recomputes in float64, from exactly those bits:
  g_step    G per layer, direction and step: stepwise, from the kernel's h_{t-1} and layer input;
  dg_step   dgi and dgh of layer 0 per direction and step: backward_steps, whose recurrent product takes the kernel's dgh;
  dh0_step  dh_{-1} of layer 0 per direction (the scratch's dhc; at bf16 the ABI refuses d_dh0, this is the only view);
  gemm_step every backward GEMM of layer 0 and of the head from the kernel's operand planes (gemm_steps): dW_ih, dW_hh
            with its h0 term, the bias column sums, dx, dcat and the top layer's dY;
plus y_step, logits_step and w_step of the forward, as in the sibling file.  The planes themselves must equal split_bf16
of their fp32 sources bit for bit.  The scratch keeps only the last layer the backward ran (each layer reuses it), so
this file checks layer 0; test_gpu_layer_steps.py stops the backward at each upper layer (bigru_plan_set_backward_stop)
and checks that layer's steps and GEMMs the same way.

configs[1] runs at full size (B512 T128 F64 H256 L2 D2) without the free-running oracle: its forward steps are sampled by
batch tile (the first, second and last 16-row tile, every step; configs[4]'s T = 1024 shape the first tile), its backward
steps and GEMMs are compared in full.
Run on an H100:  python -m pytest tests/test_gpu_tc_steps.py -m gpu -q
(BIGRU_TC_STEPS_REPORT=path.jsonl appends every measured distance to that file.)  Measurements and mutations:
tests/ROUNDING_MODEL.md, section "One step and one GEMM at a time"."""
import ctypes as C
import json
import os
import resource

import numpy as np
import pytest

import oracle_c
from gru_driver import (CODE, PLANE_REGIONS, WS, abi_names, backward_steps, dist, gemm_steps, head_dcat, head_dy, kernel,
                        kernel_gemm_steps, kernel_steps, plane_checks, region, split, stepwise)

NSM = 132                  # SMs of an H100 SXM: what wg_splits (tc_hopper.cuh) aims its split-K at


def cdiv(a, b):
    return -(-a // b)


def wg_splits(tiles, kblocks):
    """Restates wg_splits of tc_hopper.cuh: split-K count of a weight-gradient GEMM with `tiles` output tiles."""
    s = min(cdiv(4 * NSM, tiles), kblocks // 8)
    if s <= 1:
        return 1
    return cdiv(kblocks, cdiv(kblocks, s))


def wg_staged(splits, beta, base_bytes, ldc, zc, N):
    """Restates the epilogue decision of wg_gemm (tc_hopper.cuh): whether a job's output goes out through shared memory and
    bulk tensor stores (1) or element by element (0).  base_bytes, ldc, zc (elements) describe the kernel's output: C with
    its batch stride (M * ldc at batch 1), or with splits > 1 the partials [splits][batch][M][N] (ldc = N, zc = M * N).
    Rows must be whole 16-byte chunks (N % 4 == 0): a bulk tensor store clips columns only to 16 bytes."""
    return int((splits > 1 or not beta) and base_bytes % 16 == 0 and ldc % 4 == 0 and zc % 4 == 0 and N % 4 == 0)


def dw0_gemms(s):
    """(splits, units, short last split) of layer 0's dW_ih and dW_hh launches: M = 3H, N = F or H, K = B*T, 128 x 128
    tiles, one batch per direction."""
    kb = cdiv(s["B"] * s["T"], 64)
    out = []
    for n in (s["F"], s["H"]):
        tiles = cdiv(3 * s["H"], 128) * cdiv(n, 128) * s["D"]
        sp = wg_splits(tiles, kb)
        out.append((sp, tiles * sp, sp > 1 and kb % cdiv(kb, sp) != 0))
    return out


def scan_ctas(s):
    """CTAs of one scan launch: grid (CS = H/64, B/16 batch tiles, D), clusters of CS, one CTA per SM."""
    return s["H"] // 64 * (s["B"] // 16) * s["D"]


# the regimes where the backward kernels go wrong, and how a shape proves it is in one
REGIMES = {
    # scan: cluster size x direction count; bidirectional H = 512 (8-CTA clusters, 226 KB of shared memory) is bf16 only
    "cluster2_d1": lambda s: s["H"] == 128 and s["D"] == 1, "cluster2_d2": lambda s: s["H"] == 128 and s["D"] == 2,
    "cluster4_d1": lambda s: s["H"] == 256 and s["D"] == 1, "cluster4_d2": lambda s: s["H"] == 256 and s["D"] == 2,
    "cluster8_d1": lambda s: s["H"] == 512 and s["D"] == 1, "cluster8_d2": lambda s: s["H"] == 512 and s["D"] == 2,
    # scan length: one and two steps in both directions, long sequences, configs[4]'s T = 1024 at H = 512
    "T1_both_dirs": lambda s: s["T"] == 1 and s["D"] == 2, "T2_both_dirs": lambda s: s["T"] == 2 and s["D"] == 2,
    "T_long": lambda s: s["T"] >= 300, "T1024_h512": lambda s: s["T"] == 1024 and s["H"] == 512,
    # an initial state at bf16x3: dh0 and the w0 term of dW_hh
    "h0_bf16x3": lambda s: s["h0"] and "bf16x3" in s["precs"],
    # batch tiles: an odd count of 16-row tiles at bf16; at bf16x3 an odd count of 32-row tiles (half a 64-row tile);
    # more scan CTAs than one wave of the 132 SMs holds
    "odd_tiles_bf16": lambda s: (s["B"] // 16) % 2 == 1 and s["B"] > 16 and "bf16" in s["precs"],
    "odd_32_tiles_bf16x3": lambda s: (s["B"] // 32) % 2 == 1 and s["B"] > 32 and "bf16x3" in s["precs"],
    "two_waves": lambda s: scan_ctas(s) > NSM,
    # GEMMs: K = B*T ragged against the 64-deep k-block; F ragged against the 8-element plane pitch and the 64-wide box
    "K_ragged64": lambda s: (s["B"] * s["T"]) % 64 != 0,
    "F_ragged8": lambda s: s["F"] % 8 != 0, "F_ragged64": lambda s: s["F"] % 8 == 0 and s["F"] % 64 != 0,
    # layer 0's dW GEMMs: one split, a short last split, more units than SMs
    "dw_one_split": lambda s: any(sp == 1 for sp, _, _ in dw0_gemms(s)),
    "dw_short_last_split": lambda s: any(short for _, _, short in dw0_gemms(s)),
    "dw_units_gt_sms": lambda s: any(u > NSM for _, u, _ in dw0_gemms(s)),
    # dX: one K loop over one direction, or kcat over both
    "dx_d1": lambda s: s["D"] == 1, "dx_kcat_d2": lambda s: s["D"] == 2,
    "configs1_full": lambda s: (s["B"], s["T"], s["F"], s["H"], s["L"], s["D"]) == (512, 128, 64, 256, 2, 2),
}

SHAPES = {
    "h128_t1_f5": dict(B=16, T=1, F=5, H=128, L=1, C=3, D=2, h0=False, precs=("bf16",),
                       regimes=("cluster2_d2", "T1_both_dirs", "F_ragged8", "K_ragged64", "dw_one_split", "dx_kcat_d2")),
    "h128_t2_h0": dict(B=32, T=2, F=24, H=128, L=2, C=3, D=2, h0=True, precs=("bf16x3",),
                       regimes=("cluster2_d2", "T2_both_dirs", "h0_bf16x3", "F_ragged64", "dw_one_split")),
    "h128_t301_d1": dict(B=32, T=301, F=13, H=128, L=1, C=2, D=1, h0=False, precs=("bf16", "bf16x3"),
                         regimes=("cluster2_d1", "T_long", "K_ragged64", "F_ragged8", "dx_d1", "dw_short_last_split")),
    "h256_b48_d1": dict(B=48, T=9, F=64, H=256, L=2, C=3, D=1, h0=False, precs=("bf16",),
                        regimes=("cluster4_d1", "odd_tiles_bf16", "K_ragged64", "dx_d1")),
    "h256_b96_h0": dict(B=96, T=7, F=136, H=256, L=1, C=4, D=2, h0=True, precs=("bf16x3",),
                        regimes=("cluster4_d2", "odd_32_tiles_bf16x3", "h0_bf16x3", "F_ragged64", "K_ragged64")),
    "h512_d1": dict(B=32, T=5, F=40, H=512, L=1, C=2, D=1, h0=False, precs=("bf16",),
                    regimes=("cluster8_d1", "F_ragged64", "K_ragged64", "dx_d1")),
    "h512_d2": dict(B=32, T=9, F=200, H=512, L=2, C=3, D=2, h0=False, precs=("bf16",),
                    regimes=("cluster8_d2", "F_ragged64", "K_ragged64", "dx_kcat_d2")),
    "h512_t1024_d2": dict(B=32, T=1024, F=128, H=512, L=1, C=3, D=2, h0=False, precs=("bf16",), sample_tiles=(0,),
                          regimes=("cluster8_d2", "T_long", "T1024_h512", "dw_units_gt_sms",
                                   "dw_short_last_split")),
    "configs1": dict(B=512, T=128, F=64, H=256, L=2, C=3, D=2, h0=False, precs=("bf16x3", "bf16"), sample_tiles=(0, 1, -1),
                     regimes=("configs1_full", "cluster4_d2", "two_waves", "dw_units_gt_sms", "dx_kcat_d2")),
}

# Kernel-vs-model tolerances (rel-L2, max-abs over max |model|) per class: about 4x the worst value measured on an H100
# 80GB HBM3 (SXM, 700 W power limit) over the shapes above; the measurements are in tests/ROUNDING_MODEL.md.
TOL = {
    "bf16": {"y_step": (3.8e-6, 4.8e-6), "g_step": (9e-7, 4.8e-6), "logits_step": (1e-5, 1e-4), "w_step": (1.2e-5, 1.4e-4),
             "dg_step": (7.2e-7, 1.5e-6), "dh0_step": (4.4e-7, 8e-7), "gemm_step": (2.8e-5, 3.2e-5)},
    "bf16x3": {"y_step": (6.8e-6, 9.6e-6), "g_step": (1.4e-6, 8e-6), "logits_step": (1.1e-5, 1.3e-5), "w_step": (5.6e-6, 9.2e-6),
               "dg_step": (6.8e-7, 9.6e-7), "dh0_step": (6.4e-7, 6.4e-7), "gemm_step": (4e-5, 4e-5)},
}


def test_shapes_are_in_the_regimes_they_claim():
    covered = set()
    for name, s in SHAPES.items():
        for r in s["regimes"]:
            assert REGIMES[r](s), (name, r)
        covered |= set(s["regimes"])
        assert s["B"] % 16 == 0 and ("bf16x3" not in s["precs"] or (s["B"] % 32 == 0 and s["H"] <= 256))
        assert s["H"] != 512 or s["B"] % 32 == 0
        assert not (s["h0"] and "bf16" in s["precs"])          # BIGRU_PREC_BF16 has no initial state
    assert covered == set(REGIMES), set(REGIMES) - covered
    assert set(SHAPES["configs1"]["precs"]) == {"bf16", "bf16x3"}
    # configs[1]'s dW GEMMs of layer 0: 43 splits of dW_ih (44 asked, no empty split), 22 of dW_hh
    assert [sp for sp, _, _ in dw0_gemms(SHAPES["configs1"])] == [43, 22]


# ---- bigru_workspace_region against a restatement of stash_layout / scratch_layout (api.cu) ----------------------------
def _rup(v, m):
    return -(-v // m) * m


def _layout(B, T, F, H, L, C_, D, prec):
    """stash_layout / scratch_layout of api.cu up to the planes of dgi and dgh (float offsets)."""
    BT, tc = B * T, prec != "fp32"
    I = lambda l: F if l == 0 else D * H                                             # noqa: E731
    pitch = lambda l: _rup(I(l), 8)                                                  # noqa: E731
    planes = lambda n: _rup((2 if prec == "bf16x3" else 1) * n, 128) // 2 if tc else 0   # noqa: E731
    st, o = {}, 0
    for l in range(L):
        st[("Y", l)] = o; o += BT * D * H
        st[("G", l)] = o; o += D * BT * 4 * H
        o += BT * I(l)
        o = _rup(o, 64)
        st[("YP", l)] = o; o += planes(BT * D * H)
        st[("XP", l)] = o; o += planes(BT * pitch(l))
    sc, o = {}, 0
    wide = max(D * H, F)
    o += D * BT * 3 * H + D * B * 3 * H                                              # gi, gh
    sc["dgi"] = o; o += D * BT * 3 * H
    sc["dgh"] = o; o += D * BT * 3 * H
    sc["dYa"] = o; o += BT * wide
    sc["dYb"] = o; o += BT * wide
    sc["dhc"] = o; o += D * B * H
    sc["dcat"] = o; o += B * 3 * H
    o += 64 * max(3 * H, C_)                                                          # colsum partials
    o = _rup(o, 64)
    sc["dgiP"] = o; o += planes(D * BT * 3 * H)
    sc["dghP"] = o
    return st, sc, pitch


LAYOUT_CASES = [(B, T, F, H, L, D, prec) for prec, B, H in (("fp32", 8, 24), ("bf16", 16, 128), ("bf16", 32, 512), ("bf16x3", 32, 256))
                for T, F in ((3, 13), (5, 64)) for L in (1, 2, 3) for D in (1, 2)]


@pytest.mark.parametrize("case", LAYOUT_CASES, ids=[f"B{c[0]}T{c[1]}F{c[2]}H{c[3]}L{c[4]}D{c[5]}-{c[6]}" for c in LAYOUT_CASES])
def test_workspace_regions_match_the_layout(case):
    import financial_market_data_analysis_b200 as pkg
    lib = pkg._lib.load()
    B, T, F, H, L, D, prec = case
    C_ = 3
    plan = C.c_void_p()
    pkg._lib.check(lib.bigru_plan_create(B, T, F, H, L, C_, int(D == 2), CODE[prec], C.byref(plan)), "plan_create")
    try:
        sb, cb = C.c_size_t(), C.c_size_t()
        pkg._lib.check(lib.bigru_workspace_bytes(plan, C.byref(sb), C.byref(cb)), "workspace_bytes")
        st, sc, pitch = _layout(B, T, F, H, L, C_, D, prec)
        BT, H3, DH, x3 = B * T, 3 * H, D * H, prec == "bf16x3"
        # which -> [(layer, buffer, float offset, pitch, elements of one plane or of the fp32 region, bytes per element)]
        want = {"GATES": [(l, 0, st[("G", l)], 4 * H, D * BT * 4 * H, 4) for l in range(L)],
                "Y_PLANES": [(l, 0, st[("YP", l)], DH, BT * DH, 2) for l in range(L)],
                "IN_PLANES": [(l, 0, st[("XP", l)], pitch(l), BT * pitch(l), 2) for l in range(L)],
                "DGI": [(0, 1, sc["dgi"], H3, D * BT * H3, 4)], "DGH": [(0, 1, sc["dgh"], H3, D * BT * H3, 4)],
                "DGI_PLANES": [(0, 1, sc["dgiP"], H3, D * BT * H3, 2)], "DGH_PLANES": [(0, 1, sc["dghP"], H3, D * BT * H3, 2)],
                "DY": [(l, 1, sc["dYa" if (L - 1 - l) % 2 == 0 else "dYb"], DH, BT * DH, 4) for l in range(min(L, 2))],
                "DHC": [(0, 1, sc["dhc"], H, D * B * H, 4)], "DCAT": [(L, 1, sc["dcat"], H3, B * H3, 4)]}
        assert set(want) == set(WS)
        spans = {0: [], 1: []}
        for which, regs in want.items():
            is_plane = which in PLANE_REGIONS
            for layer, buf, off, pt, n, es in regs:
                rc, in_sc, b, lo, p = region(plan, which, layer)
                if is_plane and prec == "fp32":
                    assert rc == pkg._lib.ERR_UNSUPPORTED, (which, layer)
                    continue
                assert rc == 0, (which, layer, lib.bigru_last_error())
                assert (in_sc, b, p) == (buf, 4 * off, pt), (which, layer)
                end = b + n * es
                if is_plane:
                    assert b % 16 == 0, (which, layer)
                    if x3:
                        assert lo == end and lo % 16 == 0, (which, layer)
                        end = lo + n * es
                    else:
                        assert lo == 2 ** 64 - 1, (which, layer)
                else:
                    assert lo == 2 ** 64 - 1, (which, layer)
                assert end <= (sb.value, cb.value)[buf], (which, layer)
                spans[buf].append((b, end, which, layer))
        # no two regions alias (the DY of layers 0 and 1 are the two ping-pong buffers)
        for regs in spans.values():
            regs.sort()
            for a, b in zip(regs, regs[1:]):
                assert a[1] <= b[0], (a, b)
        # refusals: unknown region, a layer the region does not have, null outputs
        for which, layer in ((-1, 0), (len(WS), 0)):
            assert lib.bigru_workspace_region(plan, which, layer, C.byref(C.c_int()), C.byref(C.c_size_t()),
                                              C.byref(C.c_size_t()), C.byref(C.c_int64())) == pkg._lib.ERR_ARG
        for which, layer in (("GATES", L), ("GATES", -1), ("Y_PLANES", L), ("DGI", 1), ("DGH_PLANES", 1), ("DHC", 1),
                             ("DY", 2), ("DY", L), ("DCAT", 0), ("DCAT", L + 1)):
            if which in PLANE_REGIONS and prec == "fp32":
                continue
            assert region(plan, which, layer)[0] == pkg._lib.ERR_ARG, (which, layer)
        assert lib.bigru_workspace_region(plan, 0, 0, None, None, None, None) == pkg._lib.ERR_ARG
    finally:
        lib.bigru_plan_destroy(plan)


# ---- the step models, fed their own operands, are the oracle's rounding model again -------------------------------------
def _inputs(s):
    B, T, F, H, L, C_, D = (s[k] for k in "BTFHLCD")
    rng = np.random.default_rng([B, T, F, H, L, D])
    k = 1 / np.sqrt(H)                                          # nn.GRU / nn.Linear initialisation scale
    flat = rng.uniform(-k, k, oracle_c.lib().bigru_ref_param_count(F, H, L, C_, D)).astype(np.float32)
    x = rng.standard_normal((B, T, F)).astype(np.float32)
    h0 = (0.5 * rng.standard_normal((L * D, B, H))).astype(np.float32) if s["h0"] else None
    dl = rng.standard_normal((B, C_)).astype(np.float32)
    return flat, x, h0, dl


def _first_rows_zero(a, T):
    a = a.copy()
    a[0, :, 0] = 0
    if a.shape[0] == 2:
        a[1, :, T - 1] = 0
    return a


def _pair(p, f=lambda a: a):
    return f(p[0]), (None if p[1] is None else f(p[1]))


@pytest.mark.parametrize("prec", ["exact", "bf16", "bf16x3"])
@pytest.mark.parametrize("D", [1, 2])
def test_step_models_reproduce_the_oracle(prec, D):
    """backward_steps and gemm_steps run free-running (each step's recurrent product takes the model's own dgh, each GEMM
    the split of the model's own dgi / dgh) from the oracle's forward stash and routing: that is oracle/bigru_ref.c's
    backward at `prec`, so dW_ih, dW_hh, the biases, dx and dh0 of layer 0 must be the oracle's to within the float32 it
    returns.  This is what makes the GPU comparisons mean "kernel against its rounding model"."""
    s = dict(B=3, T=5, F=13, H=8, L=1, C=3, D=D, h0=True)
    flat, x, h0, dl = _inputs(s)
    B, T, F, H, L, C_ = (s[k] for k in "BTFHLC")
    P = oracle_c.PRECISION[prec]
    _, _, stash = oracle_c.forward(flat, x, H, L, C_, D, h0, keep=True, prec=P)
    grads, dx, dh0 = oracle_c.backward(flat, x, stash, dl, H, L, C_, D, prec=P)
    ys = [y.copy() for y in oracle_c.layer_outputs(stash, B, T, H, L, D)]
    BT, o = B * T, B * T * D * H
    gates = []
    for d in range(D):
        r, z, n, hn = (stash[o + i * BT * H: o + (i + 1) * BT * H].reshape(B, T, H) for i in range(4))
        gates.append(np.concatenate([r, z, n, hn], 2))
        o += 5 * BT * H
    arg = oracle_c.routing(stash, B, H)
    names = abi_names(s)
    dcat = head_dcat(s, prec, flat, dl, names)
    ws = dict(G=[np.stack(gates)], DY=[head_dy(s, dcat, arg)], DCAT=dcat)
    dgi, dgh, dh0m = np.zeros((D, B, T, 3 * H)), np.zeros((D, B, T, 3 * H)), np.zeros((D, B, H))
    for kind, d, t, a, b in backward_steps(s, prec, flat, h0, ws, ys, names, own=True):
        if kind == "dg":
            dgi[d][:, t], dgh[d][:, t] = a, b
        else:
            dh0m[d] = a
    xp = np.zeros((B, T, _rup(F, 8)))
    xp[..., :F] = x
    ops = dict(DGIP=split(dgi, prec), DGHP=_pair(split(dgh, prec), lambda a: _first_rows_zero(a, T)),
               XP=split(xp, prec), YP=split(ys[0], prec), DGI=dgi, DGH=dgh, DCAT=dcat)
    model = gemm_steps(s, prec, flat, dl, h0, ops, names, arg)
    want = {}
    for d in range(D):
        for nm in ("w_ih", "w_hh", "b_ih", "b_hh"):
            off, k = names[f"l0d{d}.{nm}"]
            want[f"gemm:grad:l0d{d}.{nm}"] = grads[off:off + k]
    want["gemm:dx"] = dx
    assert set(want) <= {k for k, _ in model}
    for key, v in want.items():
        got = model[(key, "gemm_step")]
        assert np.abs(got - v).max() <= 2e-7 * np.abs(v).max(), (key, np.abs(got - v).max(), np.abs(v).max())
    assert np.abs(dh0m - dh0[:D]).max() <= 2e-7 * np.abs(dh0).max()


# ---- the kernels against their step models on the GPU ----------------------------------------------------------------
def _ops(got, s, x, exact):
    """gemm_steps' operands from the kernel's workspace: its planes, or (exact) the fp32 values they were split from."""
    ws, B, T, F = got["ws"], s["B"], s["T"], s["F"]
    if not exact:
        return dict(DGIP=ws["DGIP"], DGHP=ws["DGHP"], XP=ws["XP"], YP=ws["YP"][0], DGI=ws["DGI"], DGH=ws["DGH"],
                    DCAT=ws["DCAT"])
    xp = np.zeros(ws["XP"][0].shape, np.float32)
    xp[..., :F] = x
    return dict(DGIP=(ws["DGI"], None), DGHP=(_first_rows_zero(ws["DGH"], T), None), XP=(xp, None),
                YP=(got["ys"][0], None), DGI=ws["DGI"], DGH=ws["DGH"], DCAT=ws["DCAT"])


CASES = [(n, p) for n, s in SHAPES.items() for p in s["precs"]]


@pytest.mark.gpu
@pytest.mark.parametrize("name,prec", CASES, ids=[f"{n}-{p}" for n, p in CASES])
def test_kernel_steps_match_their_models(name, prec):
    import financial_market_data_analysis_b200 as pkg
    if pkg._lib.load().bigru_device_check(0) != 0:
        pytest.fail("no H100: " + pkg._lib.load().bigru_last_error().decode())
    s = SHAPES[name]
    B, T, H = s["B"], s["T"], s["H"]
    flat, x, h0, dl = _inputs(s)
    got, names = kernel(s, prec, flat, x, h0, dl, regions=True)
    ws = got["ws"]
    bad_planes = {k: v for k, v in plane_checks(got, s, prec, x).items() if v}

    rows_out, bad = [], []

    def compare(key, k, m, e):
        tname, cls = key
        km, me, ke = dist(k, m), dist(m, e), dist(k, e)
        rows_out.append(dict(shape=name, prec=prec, tensor=tname, cls=cls, km_l2=km[0], km_max=km[1], me_l2=me[0],
                             me_max=me[1], ke_l2=ke[0], ke_max=ke[1]))
        tol = TOL[prec][cls]
        if not (km[0] <= tol[0] and km[1] <= tol[1]):
            bad.append((tname, km, tol))

    # forward: one step from the kernel's state, with the gate stash
    rows = None
    if "sample_tiles" in s:
        rows = np.concatenate([np.arange(16) + 16 * (t % (B // 16)) for t in s["sample_tiles"]])
        assert len(np.unique(rows)) == len(rows)
    tk = kernel_steps(got, s, names, rows, gates=True)
    tm = stepwise(s, prec, flat, x, h0, dl, got, names, rows, gates=True)
    te = stepwise(s, "exact", flat, x, h0, dl, got, names, rows, gates=True)
    for key in tk:
        compare(key, tk[key], tm[key], te[key])
    del tk, tm, te
    # backward recurrence of layer 0, one step at a time from the kernel's operands
    for a, b in zip(backward_steps(s, prec, flat, h0, ws, got["ys"], names),
                    backward_steps(s, "exact", flat, h0, ws, got["ys"], names)):
        kind, d, t = a[:3]
        if kind == "dg":
            compare((f"bstep:dgi[d{d},t{t}]", "dg_step"), ws["DGI"][d][:, t].astype(np.float64), a[3], b[3])
            compare((f"bstep:dgh[d{d},t{t}]", "dg_step"), ws["DGH"][d][:, t].astype(np.float64), a[4], b[4])
        else:
            compare((f"bstep:dh0[d{d}]", "dh0_step"), ws["DHC"][d].astype(np.float64), a[3], b[3])
    # the backward GEMMs of layer 0 and the head, from the kernel's operand planes
    gk = kernel_gemm_steps(got, s, names)
    gm = gemm_steps(s, prec, flat, dl, h0, _ops(got, s, x, False), names, got["arg"])
    ge = gemm_steps(s, "exact", flat, dl, h0, _ops(got, s, x, True), names, got["arg"])
    for key in gk:
        compare(key, gk[key], gm[key], ge[key])

    peak_gb = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 2 ** 20
    out = os.environ.get("BIGRU_TC_STEPS_REPORT")
    if out:
        with open(out, "a") as f:
            for r in rows_out:
                f.write(json.dumps(r) + "\n")
            f.write(json.dumps(dict(shape=name, prec=prec, peak_host_gb=peak_gb, planes_bad=bad_planes)) + "\n")
    worst = {}
    for r in rows_out:
        w = worst.setdefault(r["cls"], [0.0, 0.0, np.inf])
        w[0], w[1], w[2] = max(w[0], r["km_l2"]), max(w[1], r["km_max"]), min(w[2], r["me_l2"] if r["me_l2"] > 0 else np.inf)
    print(f"\n{name} {prec} peak host {peak_gb:.1f} GB " +
          " ".join(f"{c}: km_l2 {w[0]:.1e} km_max {w[1]:.1e} me_l2(min) {w[2]:.1e}" for c, w in worst.items()))
    assert not bad_planes, bad_planes
    assert not bad, sorted(bad, key=lambda b: -b[1][0])[:10]
