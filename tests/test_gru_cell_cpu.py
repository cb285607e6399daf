"""``GRUCell`` without a GPU: the export, nn.GRUCell's parameters, initialisation and state_dict, the refusals, the
workspace sizes against a restatement of their layout, and argument checks that come before any launch."""
import ctypes as C

import pytest
import torch
import torch.nn as nn

import financial_market_data_analysis_b200 as pkg
from financial_market_data_analysis_b200 import GRU, GRUCell, _lib

PREC = {"fp32": _lib.PREC_FP32, "bf16": _lib.PREC_BF16, "bf16x3": _lib.PREC_BF16X3}


def test_export():
    assert pkg.GRUCell is GRUCell and "GRUCell" in pkg.__all__
    lib = _lib.load()
    for name in ("bigru_cell_workspace_bytes", "bigru_cell_forward", "bigru_cell_backward"):
        assert hasattr(lib, name)
    assert lib.bigru_version() >= 210


@pytest.mark.parametrize("I,H", [(1, 1), (13, 100), (64, 256)])
def test_parameters_follow_nn_grucell(I, H):
    torch.manual_seed(7)
    mine = GRUCell(I, H)
    torch.manual_seed(7)
    ref = nn.GRUCell(I, H)
    assert [n for n, _ in mine.named_parameters()] == [n for n, _ in ref.named_parameters()]
    for (n, p), (_, q) in zip(mine.named_parameters(), ref.named_parameters()):
        assert p.shape == q.shape and torch.equal(p, q), n
    # the flat vector is a GRU(I, H, 1)'s: the same order and count
    gru = GRU(I, H, 1)
    assert mine.flat_parameters().numel() == gru.flat_parameters().numel()
    assert mine.flat_parameters().numel() == sum(p.numel() for p in ref.parameters())


def test_state_dict_round_trips():
    torch.manual_seed(1)
    ref = nn.GRUCell(13, 32)
    mine = GRUCell(13, 32)
    mine.load_state_dict(ref.state_dict())
    assert all(torch.equal(a, b) for a, b in zip(mine.parameters(), ref.parameters()))
    assert mine._is_flat()                                   # still views of one flat vector
    back = nn.GRUCell(13, 32)
    back.load_state_dict(mine.state_dict())
    assert all(torch.equal(a, b) for a, b in zip(back.parameters(), ref.parameters()))


def test_refusals():
    with pytest.raises(ValueError):
        GRUCell(4, 8, bias=False)
    with pytest.raises(ValueError):
        GRUCell(4, 8, dtype=torch.float64)
    with pytest.raises(ValueError):
        GRUCell(4, 8, precision="fp16")
    with pytest.raises(RuntimeError, match="no CPU path"):
        GRUCell(4, 8)(torch.randn(2, 4))
    with pytest.raises(ValueError):
        GRUCell(4, 8)(torch.randn(2, 3, 4))


@pytest.mark.parametrize("H,want", [(8, "bf16x3"), (256, "bf16x3"), (257, "fp32"), (1024, "fp32")])
def test_auto_precision_is_grus(H, want, monkeypatch):
    monkeypatch.delenv("BIGRU_B200_PRECISION", raising=False)
    cell = GRUCell(3, H)
    assert cell._precision_code() == PREC[want]
    assert GRU(3, H)._pad.precision == want


@pytest.mark.parametrize("prec", ["fp32", "bf16x3", "bf16"])
@pytest.mark.parametrize("B,I,H", [(1, 1, 1), (3, 13, 100), (512, 64, 256), (17, 200, 1024)])
def test_workspace_sizes(prec, B, I, H):
    lib = _lib.load()
    st, sc = C.c_size_t(), C.c_size_t()
    assert lib.bigru_cell_workspace_bytes(B, I, H, PREC[prec], C.byref(st), C.byref(sc)) == 0
    assert st.value == 4 * B * 4 * H                          # G [B][4H] fp32: r, z, n, W_hn h + b_hn
    assert sc.value == 4 * 2 * B * 3 * H                      # dgi, dgh [B][3H] fp32


def test_entry_points_refuse_bad_arguments_before_launching():
    lib = _lib.load()
    st, sc = C.c_size_t(), C.c_size_t()
    p = C.c_void_p(16)                                        # never dereferenced: every call below fails its checks first
    assert lib.bigru_cell_workspace_bytes(1, 1, 1, 0, None, C.byref(sc)) == _lib.ERR_ARG
    assert lib.bigru_cell_workspace_bytes(1, 1, 1, 0, C.byref(st), None) == _lib.ERR_ARG
    for B, I, H, prec in ((0, 1, 1, 0), (1, 0, 1, 0), (1, 1, 0, 0), (-1, 1, 1, 0), (1, 1, 1, 3), (1, 1, 1, -1)):
        assert lib.bigru_cell_workspace_bytes(B, I, H, prec, C.byref(st), C.byref(sc)) == _lib.ERR_ARG
        assert lib.bigru_cell_forward(B, I, H, prec, p, p, p, p, p, None) == _lib.ERR_ARG
        assert lib.bigru_cell_backward(B, I, H, prec, p, p, p, p, p, p, p, p, p, None) == _lib.ERR_ARG
    assert lib.bigru_cell_workspace_bytes(32769, 1, 1, 0, C.byref(st), C.byref(sc)) == _lib.ERR_UNSUPPORTED
    assert lib.bigru_cell_workspace_bytes(1, 65537, 1, 0, C.byref(st), C.byref(sc)) == _lib.ERR_UNSUPPORTED
    fwd = [p, p, p, p, p]                                     # params, x, h, hout, stash
    for i in (0, 1, 3):                                       # h and stash may be null
        args = list(fwd)
        args[i] = None
        assert lib.bigru_cell_forward(2, 3, 4, 0, *args, None) == _lib.ERR_ARG
    bwd = [p] * 9                                             # params, x, h, stash, dhout, grads, dx, dh, scratch
    for i in (0, 1, 3, 4, 5, 8):                              # h, dx and dh may be null
        args = list(bwd)
        args[i] = None
        assert lib.bigru_cell_backward(2, 3, 4, 0, *args, None) == _lib.ERR_ARG
    assert b"null" in lib.bigru_last_error()
