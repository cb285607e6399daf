"""Recurrent dropout without a GPU: the constructor and ``*_rd`` creator refusals, p = 0 plans equal to the plain creators'
plans, the stash of plans with p > 0 against a restatement of its layout, the two new workspace regions, and the host
restatement of the mask (DESIGN.md §4.8)."""
import ctypes as C
import sys
import os

import numpy as np
import pytest
import torch

from financial_market_data_analysis_b200 import GRU, BiGRU, _lib

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from gru_driver import bigru_uniform  # noqa: E402

PREC = {"fp32": _lib.PREC_FP32, "bf16": _lib.PREC_BF16, "bf16x3": _lib.PREC_BF16X3}
RD_STREAM = 65536                          # BIGRU_RD_STREAM of include/bigru_b200.h
WS_RD_MASK, WS_RD_STATE = 10, 11           # BIGRU_WS_RD_MASK, BIGRU_WS_RD_STATE


def _rup(a, m):
    return (a + m - 1) // m * m


def _plan(B, T, F, H, L, D, prec, p=None, C_=0):
    """A plan from the plain creator (p None) or its _rd twin."""
    lib = _lib.load()
    h = C.c_void_p()
    if C_:
        rc = (lib.bigru_plan_create(B, T, F, H, L, C_, int(D == 2), PREC[prec], C.byref(h)) if p is None
              else lib.bigru_plan_create_rd(B, T, F, H, L, C_, int(D == 2), PREC[prec], p, C.byref(h)))
    else:
        rc = (lib.bigru_gru_plan_create(B, T, F, H, L, int(D == 2), PREC[prec], C.byref(h)) if p is None
              else lib.bigru_gru_plan_create_rd(B, T, F, H, L, int(D == 2), PREC[prec], p, C.byref(h)))
    assert rc == 0, lib.bigru_last_error()
    return h


def _sizes(h):
    lib = _lib.load()
    a, b, c = C.c_size_t(), C.c_size_t(), C.c_size_t()
    assert lib.bigru_workspace_bytes(h, C.byref(a), C.byref(b)) == 0
    assert lib.bigru_infer_workspace_bytes(h, C.byref(c)) == 0
    return a.value, b.value, c.value


def _region(h, which, layer):
    lib = _lib.load()
    sc, off, lo, pitch = C.c_int(), C.c_size_t(), C.c_size_t(), C.c_int64()
    rc = lib.bigru_workspace_region(h, which, layer, C.byref(sc), C.byref(off), C.byref(lo), C.byref(pitch))
    return rc, sc.value, off.value, lo.value, pitch.value


def _stash_layout(B, T, F, H, L, D, prec, head, rd):
    """The stash restated in words: per layer Y [BT][DH] (not the top layer's without a head), G [D][BT][4H], the dropped
    input [BT][I]; from a 64-word boundary the planes of Y and of the layer input, then (p > 0) the masked state R [BT][DH]
    (planes at the tensor-core precisions, fp32 at fp32).  Then cat [B][3H] and arg [B][H] with a head, and (p > 0) the
    masks [L][D][B][H] and the masked initial state [L*D][B][H].  Returns (R offsets, mask offset, total)."""
    BT, DH, tc = B * T, D * H, prec != "fp32"
    n = 2 if prec == "bf16x3" else 1

    def planes(elems):
        return _rup(n * elems, 128) // 2 if tc else 0

    w, R = 0, []
    for l in range(L):
        I = F if l == 0 else DH
        w += (BT * DH if head or l < L - 1 else 0) + D * BT * 4 * H + BT * I
        w = _rup(w, 64) + planes(BT * DH) + planes(BT * _rup(I, 8))
        R.append(w)
        if rd:
            w += planes(BT * DH) if tc else BT * DH
    w += B * 4 * H if head else 0
    M = w
    if rd:
        w += 2 * L * D * B * H
    return R, M, w


SHAPES = [(32, 5, 13, 128, 1, 1, "bf16x3"), (64, 7, 16, 256, 2, 2, "bf16x3"), (32, 4, 9, 128, 3, 2, "bf16"),
          (32, 4, 9, 512, 2, 2, "bf16"), (37, 6, 13, 32, 3, 2, "fp32"), (5, 3, 7, 300, 2, 1, "fp32")]


@pytest.mark.parametrize("head", [False, True])
@pytest.mark.parametrize("B,T,F,H,L,D,prec", SHAPES)
def test_p0_plans_equal_the_plain_creators(B, T, F, H, L, D, prec, head):
    a = _plan(B, T, F, H, L, D, prec, None, 3 if head else 0)
    b = _plan(B, T, F, H, L, D, prec, 0.0, 3 if head else 0)
    try:
        assert _sizes(a) == _sizes(b)
        for which in (WS_RD_MASK, WS_RD_STATE):            # no recurrent-dropout regions on a plan without it
            assert _region(b, which, 0)[0] == _lib.ERR_ARG
    finally:
        _lib.load().bigru_plan_destroy(a)
        _lib.load().bigru_plan_destroy(b)


@pytest.mark.parametrize("head", [False, True])
@pytest.mark.parametrize("B,T,F,H,L,D,prec", SHAPES)
def test_rd_stash_layout_and_regions(B, T, F, H, L, D, prec, head):
    lib = _lib.load()
    plain = _plan(B, T, F, H, L, D, prec, None, 3 if head else 0)
    h = _plan(B, T, F, H, L, D, prec, 0.25, 3 if head else 0)
    try:
        R, M, total = _stash_layout(B, T, F, H, L, D, prec, head, True)
        st, sc, inf = _sizes(h)
        assert st == 4 * total
        assert (sc, inf) == _sizes(plain)[1:]               # only the stash grows
        assert _sizes(plain)[0] == 4 * _stash_layout(B, T, F, H, L, D, prec, head, False)[2]
        tc = prec != "fp32"
        for l in range(L):
            rc, ins, off, lo, pitch = _region(h, WS_RD_MASK, l)
            assert (rc, ins, off, lo, pitch) == (0, 0, 4 * (M + l * D * B * H), 2 ** 64 - 1, H)
            rc, ins, off, lo, pitch = _region(h, WS_RD_STATE, l)
            assert (rc, ins, off, pitch) == (0, 0, 4 * R[l], D * H)
            assert lo == (off + 2 * B * T * D * H if prec == "bf16x3" else 2 ** 64 - 1)
            assert off + (2 if tc else 4) * B * T * D * H * (2 if prec == "bf16x3" else 1) <= st
        for which, layer in ((WS_RD_MASK, L), (WS_RD_MASK, -1), (WS_RD_STATE, L), (12, 0)):
            assert _region(h, which, layer)[0] == _lib.ERR_ARG
    finally:
        lib.bigru_plan_destroy(plain)
        lib.bigru_plan_destroy(h)


def test_configs1_stash_estimate():
    """configs[1] at bf16x3: two layers of masked planes (about 134 MB each) on top of the plain plan's stash."""
    plain, rd = _plan(512, 128, 64, 256, 2, 2, "bf16x3", None, 3), _plan(512, 128, 64, 256, 2, 2, "bf16x3", 0.25, 3)
    try:
        grow = _sizes(rd)[0] - _sizes(plain)[0]
        assert grow == 2 * 4 * 512 * 128 * 512 + 2 * 4 * 2 * 2 * 512 * 256
        assert round(_sizes(plain)[0] / 1e6) == 1915 and round(_sizes(rd)[0] / 1e6) == 2187
    finally:
        _lib.load().bigru_plan_destroy(plain)
        _lib.load().bigru_plan_destroy(rd)


@pytest.mark.parametrize("p", [-0.1, 1.0, 1.5, float("nan"), float("inf")])
def test_rd_creators_refuse_p_outside_0_1(p):
    lib = _lib.load()
    h = C.c_void_p()
    assert lib.bigru_plan_create_rd(32, 4, 8, 128, 1, 3, 1, PREC["bf16x3"], p, C.byref(h)) == _lib.ERR_ARG
    assert lib.bigru_gru_plan_create_rd(32, 4, 8, 128, 1, 1, PREC["bf16x3"], p, C.byref(h)) == _lib.ERR_ARG
    # the head-less rule of the plain creators holds for the _rd twin too
    assert lib.bigru_plan_create_rd(32, 4, 8, 128, 1, 0, 1, PREC["bf16x3"], 0.25, C.byref(h)) == _lib.ERR_ARG


@pytest.mark.parametrize("p", [-0.1, 1.0, 2.0, float("nan")])
def test_constructors_refuse_p_outside_0_1(p):
    with pytest.raises(ValueError, match="recurrent_dropout"):
        BiGRU(32, 8, 3, recurrent_dropout=p)
    with pytest.raises(ValueError, match="recurrent_dropout"):
        GRU(8, 32, recurrent_dropout=p)


def test_keyword_is_not_a_parameter():
    torch.manual_seed(0)
    a = BiGRU(32, 8, 3, 2, precision="fp32")
    torch.manual_seed(0)
    b = BiGRU(32, 8, 3, 2, precision="fp32", recurrent_dropout=0.3)
    assert list(a.state_dict()) == list(b.state_dict())
    assert all(torch.equal(a.state_dict()[k], b.state_dict()[k]) for k in a.state_dict())
    assert b.recurrent_dropout == 0.3 and "recurrent_dropout=0.3" in repr(b) and "recurrent_dropout" not in repr(a)
    g = GRU(8, 32, 2, recurrent_dropout=0.5)
    assert "recurrent_dropout=0.5" in repr(g) and "recurrent_dropout" not in repr(GRU(8, 32))
    assert g.state_dict().keys() == GRU(8, 32, 2).state_dict().keys()


def rd_masks(seed, p, L, D, B, H):
    """The masks rd_mask_kernel writes, restated: m[l][d][b][j] = 0 where bigru_uniform(seed, BIGRU_RD_STREAM + l,
    (b*D + d)*H + j) < p, else 1/(1-p) rounded to float32."""
    p32 = np.float32(p)
    scale = np.float32(1) / (np.float32(1) - p32)
    d, b, j = np.meshgrid(np.arange(D), np.arange(B), np.arange(H), indexing="ij")
    key = (b * D + d) * H + j
    return np.stack([np.where(bigru_uniform(seed, RD_STREAM + l, key).astype(np.float32) < p32, np.float32(0), scale)
                     for l in range(L)]).astype(np.float32)


def test_mask_restatement_is_batch_major_and_per_layer():
    m = rd_masks(1234, 0.25, 2, 2, 40, 32)
    assert m.shape == (2, 2, 40, 32)
    # a row's masks do not depend on how many rows follow it
    assert np.array_equal(rd_masks(1234, 0.25, 2, 2, 7, 32), m[:, :, :7])
    assert not np.array_equal(m[0], m[1])                  # one stream per layer
    assert set(np.unique(m)) == {np.float32(0), np.float32(1) / np.float32(0.75)}
    # the streams never meet the input / inter-layer dropout streams l < 16
    u_drop = bigru_uniform(1234, 0, np.arange(64))
    u_rd = bigru_uniform(1234, RD_STREAM, np.arange(64))
    assert not np.array_equal(u_drop, u_rd)


@pytest.mark.parametrize("p", [0.1, 0.25, 0.5])
def test_mask_statistics(p):
    """The zeroed fraction lies within 5 binomial standard deviations of p."""
    m = rd_masks(99, p, 2, 2, 512, 256)
    n = m.size
    frac = float((m == 0).mean())
    assert abs(frac - p) < 5 * np.sqrt(p * (1 - p) / n), (frac, p)
