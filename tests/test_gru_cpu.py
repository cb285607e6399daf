"""The head-less plan and ``GRU`` without a GPU: exports, nn.GRU's parameter order and count, workspace sizes against a
restatement of their layouts, refusals, and nn.GRU's initialisation and state_dict."""
import ctypes as C

import pytest
import torch
import torch.nn as nn

import financial_market_data_analysis_b200 as pkg
from financial_market_data_analysis_b200 import GRU, BiGRU, _lib

PREC = {"fp32": _lib.PREC_FP32, "bf16": _lib.PREC_BF16, "bf16x3": _lib.PREC_BF16X3}


def _rup(a, m):
    return (a + m - 1) // m * m


def _plan(B, T, F, H, L, D, prec, C_=0):
    lib = _lib.load()
    h = C.c_void_p()
    rc = (lib.bigru_gru_plan_create(B, T, F, H, L, int(D == 2), PREC[prec], C.byref(h)) if C_ == 0
          else lib.bigru_plan_create(B, T, F, H, L, C_, int(D == 2), PREC[prec], C.byref(h)))
    assert rc == 0, lib.bigru_last_error()
    return h


def _sizes(h):
    lib = _lib.load()
    a, b, c = C.c_size_t(), C.c_size_t(), C.c_size_t()
    assert lib.bigru_workspace_bytes(h, C.byref(a), C.byref(b)) == 0
    assert lib.bigru_infer_workspace_bytes(h, C.byref(c)) == 0
    return a.value, b.value, c.value


def test_exports():
    assert pkg.GRU is GRU and "GRU" in pkg.__all__
    lib = _lib.load()
    for name in ("bigru_gru_plan_create", "bigru_gru_forward", "bigru_gru_infer", "bigru_gru_backward"):
        assert hasattr(lib, name)
    assert lib.bigru_version() >= 209


@pytest.mark.parametrize("F,H,L,D", [(13, 32, 1, 1), (64, 256, 2, 2), (5, 128, 3, 2), (7, 300, 2, 1)])
def test_param_count_and_order_follow_nn_gru(F, H, L, D):
    lib = _lib.load()
    h = _plan(4, 3, F, H, L, D, "fp32")
    ref = nn.GRU(F, H, L, bidirectional=D == 2)
    assert lib.bigru_param_count(h) == sum(p.numel() for p in ref.parameters())
    off, rows, cols = C.c_int64(), C.c_int64(), C.c_int64()
    expect = 0
    for (name, p) in ref.named_parameters():
        kind, _, lay = name.rpartition("_l")
        layer, d = int(lay.split("_")[0]), int(lay.endswith("_reverse"))
        which = ("weight_ih", "weight_hh", "bias_ih", "bias_hh").index(kind)
        assert lib.bigru_param_offset(h, layer, d, which, C.byref(off), C.byref(rows), C.byref(cols)) == 0
        assert off.value == expect and rows.value * cols.value == p.numel()
        expect += p.numel()
    for which in (0, 2):
        assert lib.bigru_param_offset(h, L, 0, which, C.byref(off), C.byref(rows), C.byref(cols)) == _lib.ERR_ARG
    lib.bigru_plan_destroy(h)


def _infer_words(B, T, F, H, L, D, prec):
    """bigru_infer_workspace_bytes of a head-less plan restated: gi [D][BT][3H], gh [D][B][3H] (fp32 only), the fp32 Y
    buffers of the layers below the top at fp32 (ping-pong, at most two), then from a 64-word boundary the bf16 planes:
    the layer-0 input [BT][rup(F, 8)], the Y planes of min(L - 1, 2) lower layers and the packed W_ih image."""
    BT, DH, tc = B * T, D * H, prec != "fp32"
    n = 2 if prec == "bf16x3" else 1

    def planes(elems):
        return _rup(n * elems, 128) // 2 if tc else 0

    def pack(R, K, batch):
        return n * batch * _rup(R, 128) * _rup(K, 64)

    w = D * BT * 3 * H + (0 if tc else D * B * 3 * H)
    w += 0 if tc else BT * DH * min(L - 1, 2)
    w = _rup(w, 64)
    w += planes(BT * _rup(F, 8)) + planes(BT * DH) * min(L - 1, 2)
    if tc:
        w += planes(max(pack(3 * H, I, D) for I in [F] + [DH] * (L - 1)))
    return 4 * w


def _stash_words(B, T, F, H, L, D, prec, head=False):
    """bigru_workspace_bytes' stash restated: per layer Y [BT][DH] (not the top layer's without a head), G [D][BT][4H], the
    dropped input [BT][I], then from a 64-word boundary the planes of Y and of the layer input; cat and arg with a head."""
    BT, DH, tc = B * T, D * H, prec != "fp32"
    n = 2 if prec == "bf16x3" else 1

    def planes(elems):
        return _rup(n * elems, 128) // 2 if tc else 0

    w = 0
    for l in range(L):
        I = F if l == 0 else DH
        w += (BT * DH if head or l < L - 1 else 0) + D * BT * 4 * H + BT * I
        w = _rup(w, 64) + planes(BT * DH) + planes(BT * _rup(I, 8))
    return 4 * (w + (B * 4 * H if head else 0))


def _cdiv(a, b):
    return -(-a // b)


def _wg_splits(tiles, kblocks):
    """wg_splits (tc_hopper.cuh) restated: split-K count of a weight-gradient GEMM."""
    s = min(_cdiv(4 * 132, tiles), kblocks // 8)
    return 1 if s <= 1 else _cdiv(kblocks, _cdiv(kblocks, s))


def _scratch_words(B, T, F, H, L, D, prec, C_=0):
    """bigru_workspace_bytes' scratch restated: gi, dgi, dgh [D][BT][3H], gh [D][B][3H], dYa and dYb [BT][max(DH, F)], dhc
    [D][B][H], dcat [B][3H] (with a head only), the column-sum partials [64][max(3H, C)]; from a 64-word boundary the planes of
    dgi and dgh; then, at the tensor-core precisions, the packed operands (W_ih, W_ih^T of every layer, the head's three GEMMs
    with a head, the w0 GEMM always) and the split-K partials of dW_ih / dW_hh."""
    BT, DH, H3, tc = B * T, D * H, 3 * H, prec != "fp32"
    n = 2 if prec == "bf16x3" else 1

    def planes(elems):
        return _rup(n * elems, 128) // 2 if tc else 0

    def pack(R, K, batch):                 # tc_pack_elems: hi (and lo) images, rows to 128, K to 64
        return n * batch * _rup(R, 128) * _rup(K, 64)

    def gemm_ws(M, N, K):
        return pack(M, K, 1) + pack(N, K, 1)

    def part(N):
        s = _wg_splits(_cdiv(H3, 128) * _cdiv(N, 128) * D, _cdiv(BT, 64))
        return s * D * H3 * N if s > 1 else 0

    w = 3 * D * BT * H3 + D * B * H3 + 2 * BT * max(DH, F) + D * B * H + (B * H3 if C_ else 0) + 64 * max(H3, C_)
    w = _rup(w, 64) + 2 * planes(D * BT * H3)
    if tc:
        ins = [F] + [DH] * (L - 1)
        need = max([pack(H3, I, D) for I in ins] + [pack(I, H3, D) for I in ins] + [gemm_ws(H3, H, B)]
                   + ([gemm_ws(B, C_, H3), gemm_ws(B, H3, C_), gemm_ws(C_, H3, B)] if C_ else []))
        w += planes(need) + max(max(part(I), part(H)) for I in ins)
    return 4 * w


@pytest.mark.parametrize("prec,B,T,F,H,L,D", [("fp32", 3, 5, 13, 32, 1, 1), ("fp32", 4, 6, 7, 40, 2, 2),
                                              ("fp32", 2, 3, 5, 16, 3, 2), ("bf16x3", 32, 8, 13, 128, 1, 2),
                                              ("bf16x3", 64, 4, 64, 256, 2, 2), ("bf16", 16, 5, 9, 128, 3, 1),
                                              ("bf16", 32, 3, 16, 512, 2, 2), ("bf16x3", 64, 64, 64, 256, 2, 2),
                                              ("fp32", 64, 64, 400, 32, 2, 1), ("bf16", 32, 2, 700, 128, 1, 1)])
def test_workspace_layouts(prec, B, T, F, H, L, D):
    """The head-less stash is the head plan's without the top layer's fp32 Y, cat and arg, its scratch without dcat and the
    head's operands; stash and scratch of both kinds of plan, and the head-less inference workspace, match the restatements
    above."""
    hg, hb = _plan(B, T, F, H, L, D, prec), _plan(B, T, F, H, L, D, prec, C_=3)
    (sg, wg, ig), (sb, wb, ib) = _sizes(hg), _sizes(hb)
    assert sg == _stash_words(B, T, F, H, L, D, prec)
    assert sb == _stash_words(B, T, F, H, L, D, prec, head=True)
    assert wg == _scratch_words(B, T, F, H, L, D, prec)
    assert wb == _scratch_words(B, T, F, H, L, D, prec, C_=3)
    assert ig == _infer_words(B, T, F, H, L, D, prec)
    lib = _lib.load()
    for h in (hg, hb):
        lib.bigru_plan_destroy(h)


def test_refusals():
    lib = _lib.load()
    h = C.c_void_p()
    assert lib.bigru_plan_create(32, 4, 8, 128, 1, 0, 1, _lib.PREC_BF16X3, C.byref(h)) == _lib.ERR_ARG      # C = 0: gru plan
    assert lib.bigru_gru_plan_create(0, 4, 8, 128, 1, 1, _lib.PREC_FP32, C.byref(h)) == _lib.ERR_ARG
    assert lib.bigru_gru_plan_create(32, 4, 8, 128, 1, 1, 7, C.byref(h)) == _lib.ERR_ARG
    assert lib.bigru_gru_plan_create(33, 4, 8, 128, 1, 1, _lib.PREC_BF16X3, C.byref(h)) == _lib.ERR_UNSUPPORTED
    g, b = _plan(32, 4, 8, 128, 2, 2, "bf16x3"), _plan(32, 4, 8, 128, 2, 2, "bf16x3", C_=3)
    dev = C.c_void_p(256)                                # stands for a device pointer; every call below returns before using it
    # head entry points refuse the head-less plan, and the other way round
    assert lib.bigru_forward_lengths(g, dev, dev, None, 0.0, 0, 0, 0, dev, dev, dev, None, None, None) == _lib.ERR_ARG
    assert b"bigru_gru_" in lib.bigru_last_error()
    assert lib.bigru_infer_lengths(g, dev, dev, None, dev, dev, None, None) == _lib.ERR_ARG
    assert lib.bigru_backward_lengths(g, dev, dev, None, 0.0, 0, 0, 0, dev, dev, dev, dev, None, None, None, None) == _lib.ERR_ARG
    assert lib.bigru_gru_forward(b, dev, dev, None, 0.0, 0, 0, dev, dev, dev, None, None, None) == _lib.ERR_ARG
    assert lib.bigru_gru_infer(b, dev, dev, None, dev, dev, None, None, None) == _lib.ERR_ARG
    assert lib.bigru_gru_backward(b, dev, dev, None, 0.0, 0, 0, dev, dev, dev, dev, None, dev, None, None, None, None) == _lib.ERR_ARG
    # null d_y / d_dy, dropout out of range
    assert lib.bigru_gru_forward(g, dev, dev, None, 0.0, 0, 0, dev, dev, None, None, None, None) == _lib.ERR_ARG
    assert lib.bigru_gru_forward(g, dev, dev, None, 1.0, 1, 0, dev, dev, dev, None, None, None) == _lib.ERR_ARG
    assert lib.bigru_gru_backward(g, dev, dev, None, 0.0, 0, 0, dev, dev, dev, None, None, dev, None, None, None, None) == _lib.ERR_ARG
    # regions that do not exist without a head
    off = C.c_size_t()
    assert lib.bigru_stash_output_offset(g, 1, C.byref(off)) == _lib.ERR_ARG
    assert lib.bigru_stash_output_offset(g, 0, C.byref(off)) == 0
    assert lib.bigru_stash_argmax_offset(g, C.byref(off)) == _lib.ERR_ARG
    ins, lo, pitch = C.c_int(), C.c_size_t(), C.c_int64()
    assert lib.bigru_workspace_region(g, 9, 2, C.byref(ins), C.byref(off), C.byref(lo), C.byref(pitch)) == _lib.ERR_ARG   # DCAT
    assert lib.bigru_workspace_region(b, 9, 2, C.byref(ins), C.byref(off), C.byref(lo), C.byref(pitch)) == 0
    for h in (g, b):
        lib.bigru_plan_destroy(h)


@pytest.mark.parametrize("kw", [dict(), dict(num_layers=3, bidirectional=True), dict(num_layers=2, batch_first=True, dropout=0.3)])
def test_init_and_state_dict_match_nn_gru(kw):
    torch.manual_seed(0)
    ref = nn.GRU(13, 24, **kw)
    torch.manual_seed(0)
    mine = GRU(13, 24, **kw)
    sd_ref, sd = ref.state_dict(), mine.state_dict()
    assert list(sd_ref) == list(sd)
    assert all(torch.equal(sd_ref[k], sd[k]) for k in sd)
    assert [n for n, _ in ref.named_parameters()] == [n for n, _ in mine.named_parameters()]
    for a in ("input_size", "hidden_size", "num_layers", "bias", "batch_first", "dropout", "bidirectional", "proj_size", "mode"):
        assert getattr(ref, a) == getattr(mine, a), a
    # load_state_dict round trip, into the flat vector
    torch.manual_seed(1)
    other = nn.GRU(13, 24, **kw)
    mine.load_state_dict(other.state_dict())
    assert mine._is_flat() and all(torch.equal(other.state_dict()[k], v) for k, v in mine.state_dict().items())
    ref.load_state_dict(mine.state_dict())
    assert all(torch.equal(ref.state_dict()[k], v) for k, v in mine.state_dict().items())
    flat = mine.flat_parameters()
    mine.weight_hh_l0.data = mine.weight_hh_l0.data.clone()        # breaks the flat layout
    assert not mine._is_flat()
    mine.flatten_parameters()
    assert mine._is_flat() and mine.flat_parameters() is not flat


def test_constructor_refusals_and_cpu():
    with pytest.raises(ValueError):
        GRU(4, 8, bias=False)
    with pytest.raises(ValueError):
        GRU(4, 8, proj_size=2)
    with pytest.raises(ValueError):
        GRU(4, 8, dtype=torch.float64)
    with pytest.raises(ValueError):
        GRU(4, 8, precision="fp16")
    with pytest.raises(RuntimeError, match="no CPU path"):
        GRU(4, 8)(torch.zeros(3, 2, 4))


def test_bigru_gru_is_a_gru_on_the_prefix():
    torch.manual_seed(0)
    ref = BiGRU(16, 5, 3, 2, 50, 0.1, True, True)
    assert isinstance(ref.gru, GRU) and ref.gru.batch_first and ref.gru.dropout == 0.1
    assert BiGRU(16, 5, 3, 1, 50, 0.1, True, True).gru.dropout == 0
    flat, g = ref.flat_parameters(), ref.gru.flat_parameters()
    assert g.data_ptr() == flat.data_ptr() and g.numel() == flat.numel() - ref.linear.weight.numel() - ref.linear.bias.numel()
    assert ref.gru._is_flat() and ref._is_flat()
    # the parameter objects are the BiGRU's and nn.GRU's initialisation is kept
    torch.manual_seed(0)
    nng = (nn.Dropout(0.1), nn.Dropout2d(0.1), nn.GRU(5, 16, 2, batch_first=True, dropout=0.1, bidirectional=True))[2]
    assert all(torch.equal(a, b) for a, b in zip(nng.state_dict().values(), ref.gru.state_dict().values()))
    assert {id(p) for p in ref.gru.parameters()} <= {id(p) for p in ref.parameters()}
