"""The step models of gru_driver with recurrent-dropout masks and per-sequence lengths, without a GPU.

test_gpu_rd_steps.py compares the kernels with gru_driver's stepwise / backward_steps / gemm_steps fed the kernels' own
operands.  Here the same models run free-running (each step's recurrent product takes the model's own dgh, each GEMM the
model's own dgi / dgh) from a float64 forward, so they must be torch float64 autograd through the masked-cell loop of
test_gpu_recurrent_dropout.py: layer 0's dW_ih, dW_hh, biases, dx and dh0.  With masks of ones and full lengths they
must be bitwise the models without masks and lengths, which test_step_models_reproduce_the_oracle ties to
oracle/bigru_ref.c."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from gru_driver import abi_names, backward_steps, gemm_steps, head_dcat, head_dy, stepwise  # noqa: E402
from test_gpu_recurrent_dropout import _head, _oracle  # noqa: E402

P = 0.3                                     # 1 / (1 - p) is inexact in float32


def _case(D, lengths, h0):
    s = dict(B=6, T=5, F=7, H=8, L=1, C=3, D=D, h0=h0)
    B, T, F, H, C_ = (s[k] for k in "BTFHC")
    rng = np.random.default_rng([D, int(lengths), int(h0)])
    names = abi_names(s)
    n = names["lin_b"][0] + C_
    flat = rng.uniform(-0.4, 0.4, n).astype(np.float32)
    x = rng.standard_normal((B, T, F)).astype(np.float32)
    h0v = (0.5 * rng.standard_normal((D, B, H))).astype(np.float32) if h0 else None
    dl = rng.standard_normal((B, C_)).astype(np.float32)
    m = np.where(rng.uniform(size=(D, B, H)) < P, np.float32(0), np.float32(1) / (np.float32(1) - np.float32(P)))
    m = m.astype(np.float32)
    assert (m == 0).any() and (m != 0).any()
    lens = np.array([1, T, 3, T, 2, 4]) if lengths else None
    return s, names, flat, x, h0v, dl, m, lens


def _blk(flat, names, name, shape):
    o = names[name][0]
    return torch.from_numpy(flat[o:o + int(np.prod(shape))].astype(np.float64).reshape(shape)).requires_grad_()


def _models(s, names, flat, x, h0, dl, ys, m, lens, prec="exact"):
    """Free-running models from the layer outputs ys: gates (stepwise), the backward recurrence, the GEMMs."""
    B, T, F, H, D = (s[k] for k in "BTFHD")
    masks = None if m is None else [m]
    got = dict(ys=ys)
    steps = stepwise(s, prec, flat, x, h0, dl, got, names, gates=True, masks=masks, lens=lens)
    G = np.stack([np.stack([steps[(f"step:g[l0d{d},t{t}]", "g_step")] for t in range(T)], 1) for d in range(D)])
    top = ys[0]
    pooled = top[..., :H] + top[..., H:] if D == 2 else top
    ok = np.ones((B, T), bool) if lens is None else np.arange(T)[None, :] < lens[:, None]
    arg = np.where(ok[..., None], pooled, -np.inf).argmax(1)
    dcat = head_dcat(s, prec, flat, dl, names)
    ws = dict(G=[G], DY=[head_dy(s, dcat, arg, lens)], DCAT=dcat)
    dgi, dgh = np.zeros((D, B, T, 3 * H)), np.zeros((D, B, T, 3 * H))
    dh0, dh0_raw = np.zeros((D, B, H)), [None] * D
    for kind, d, t, a, b in backward_steps(s, prec, flat, h0, ws, ys, names, own=True, masks=m, lens=lens):
        if kind == "dg":
            dgi[d][:, t], dgh[d][:, t] = a, b
        else:
            dh0[d], dh0_raw[d] = a, b
    ghp = dgh.copy()
    ghp[0, :, 0] = 0
    if D == 2:
        ghp[1, :, T - 1] = 0
    xp = np.zeros((B, T, -(-F // 8) * 8))
    xp[..., :F] = x
    ops = dict(DGIP=(dgi, None), DGHP=(ghp, None), XP=(xp, None), YP=(ys[0], None), DGI=dgi, DGH=dgh, DCAT=dcat)
    if m is not None:
        ops["RDS"] = (np.concatenate([m[d][:, None, :].astype(np.float64) * ys[0][..., d * H:(d + 1) * H]
                                      for d in range(D)], 2), None)
    gm = gemm_steps(s, prec, flat, dl, h0, ops, names, arg, masks=m, lens=lens)
    return steps, gm, dgi, dgh, dh0, dh0_raw


@pytest.mark.parametrize("D", [1, 2])
@pytest.mark.parametrize("lengths,h0", [(True, False), (False, True)], ids=["ragged_lengths", "h0"])
def test_masked_step_models_are_autograd_of_the_masked_cell_loop(D, lengths, h0):
    """Lengths and h0 are tested apart: the library refuses them together."""
    s, names, flat, x, h0v, dl, m, lens = _case(D, lengths, h0)
    B, T, F, H, C_ = (s[k] for k in "BTFHC")
    W = [[[_blk(flat, names, f"l0d{d}.{nm}", shp) for nm, shp in
           (("w_ih", (3 * H, F)), ("w_hh", (3 * H, H)), ("b_ih", (3 * H,)), ("b_hh", (3 * H,)))] for d in range(D)]]
    lw, lb = _blk(flat, names, "lin_w", (C_, 3 * H)), _blk(flat, names, "lin_b", (C_,))
    xr = torch.from_numpy(x.astype(np.float64)).requires_grad_()
    h0r = None if h0v is None else torch.from_numpy(h0v.astype(np.float64)).requires_grad_()
    lt = torch.from_numpy(lens if lens is not None else np.full(B, T))
    y, _ = _oracle(W, xr, h0r, lt, [[torch.from_numpy(m[d]).double() for d in range(D)]], [None], H, 1, D)
    ref = _head(y, lt, lw, lb, H, D)
    ref.backward(torch.from_numpy(dl.astype(np.float64)))
    ys = [y.detach().numpy()]
    steps, gm, _, _, dh0, _ = _models(s, names, flat, x, h0v, dl, ys, m, lens)
    # the gate model's outputs are the loop's outputs
    for d in range(D):
        for t in range(T):
            got = steps[(f"step:y[l0d{d},t{t}]", "y_step")]
            assert np.abs(got - ys[0][:, t, d * H:(d + 1) * H]).max() <= 1e-12, (d, t)
    assert np.abs(steps[("step:logits", "logits_step")] - ref.detach().numpy()).max() <= 1e-12
    want = {}
    for d in range(D):
        for i, nm in enumerate(("w_ih", "w_hh", "b_ih", "b_hh")):
            want[f"gemm:grad:l0d{d}.{nm}"] = W[0][d][i].grad.numpy().ravel()
    want["gemm:dx"] = xr.grad.numpy()
    for key, v in want.items():
        err = np.abs(gm[(key, "gemm_step")] - v).max()
        assert err <= 1e-10 * np.abs(v).max(), (key, err)
    if h0:
        assert np.abs(dh0 - h0r.grad.numpy()).max() <= 1e-10 * np.abs(h0r.grad.numpy()).max()


@pytest.mark.parametrize("prec", ["exact", "bf16", "bf16x3"])
@pytest.mark.parametrize("D", [1, 2])
def test_masks_of_ones_and_full_lengths_change_no_bit(prec, D):
    s, names, flat, x, h0v, dl, m, _ = _case(D, False, True)
    T = s["T"]
    rng = np.random.default_rng(3)
    ys = [rng.uniform(-0.9, 0.9, (s["B"], T, D * s["H"])).astype(np.float32).astype(np.float64)]  # values of a float32 Y
    plain = _models(s, names, flat, x, h0v, dl, ys, None, None, prec)
    ones = _models(s, names, flat, x, h0v, dl, ys, np.ones_like(m), np.full(s["B"], T), prec)
    for a, b in zip(plain[:2], ones[:2]):
        assert a.keys() == b.keys()
        for k in a:
            assert np.array_equal(a[k], b[k]), k
    for a, b in zip(plain[2:5], ones[2:5]):
        assert np.array_equal(a, b)
    assert plain[5] == [None] * D and all(np.array_equal(r, c) for r, c in zip(ones[5], ones[4]))
