"""The step models of gru_driver on a head-less plan (the nn.GRU drop-in), without a GPU.

test_gpu_gru_steps.py compares the kernels of bigru_gru_forward / bigru_gru_backward with gru_driver's stepwise /
backward_steps / gemm_steps with head=False, fed the kernels' own operands.  Here the same models run free-running (each
step's recurrent product takes the model's own dgh, each GEMM the model's own dgi / dgh) from a float64 forward, seeded
as the library seeds a head-less plan: layer 0's carry from the caller's dhn slice of its direction, its upstream
gradient from the caller's dy when it is the top layer, else from the layer above.  They must be torch float64 autograd
through nn.GRU (packed for lengths), or through the masked-cell loop of test_gpu_recurrent_dropout.py under recurrent
dropout, with backward((y, h_n), (dy, dhn)): layer 0's dW_ih, dW_hh, biases, dx and dh0."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn as nn
from torch.nn.utils.rnn import pack_padded_sequence, pad_packed_sequence

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from gru_driver import abi_names, backward_steps, gemm_steps, stepwise  # noqa: E402
from test_gpu_recurrent_dropout import _oracle  # noqa: E402

P = 0.3                                     # 1 / (1 - p) is inexact in float32
NM = ("w_ih", "w_hh", "b_ih", "b_hh")


def _case(L, D, lengths, h0, masked):
    s = dict(B=6, T=5, F=7, H=8, L=L, C=3, D=D, h0=h0)
    B, T, F, H = (s[k] for k in "BTFH")
    rng = np.random.default_rng([L, D, int(lengths), int(h0), int(masked)])
    names = abi_names(s)
    flat = rng.uniform(-0.4, 0.4, names["lin_w"][0]).astype(np.float32)      # the recurrent prefix: a GRU's vector
    x = rng.standard_normal((B, T, F)).astype(np.float32)
    h0v = (0.5 * rng.standard_normal((L * D, B, H))).astype(np.float32) if h0 else None
    dy = rng.standard_normal((B, T, D * H)).astype(np.float32)
    dhn = rng.standard_normal((L * D, B, H)).astype(np.float32)              # a different seed per layer and direction
    m = None
    if masked:
        m = np.where(rng.uniform(size=(L, D, B, H)) < P, np.float32(0), np.float32(1) / (np.float32(1) - np.float32(P)))
        m = m.astype(np.float32)
        assert (m == 0).any() and (m != 0).any()
    lens = np.array([1, T, 3, T, 2, 4]) if lengths else None
    return s, names, flat, x, h0v, dy, dhn, m, lens


def _reference(s, names, flat, x, h0, dy, dhn, m, lens):
    """float64 autograd, one layer at a time so that layer 0's output keeps its gradient: nn.GRU (packed with lengths)
    without masks, the masked-cell loop with them.  Returns (ys, per-layer parameter gradients, dx, dh0, dY of layer 0)."""
    B, T, F, H, L, D = (s[k] for k in "BTFHLD")
    W = [[[torch.from_numpy(flat[names[f"l{l}d{d}.{nm}"][0]:sum(names[f"l{l}d{d}.{nm}"])].astype(np.float64))
           for nm in NM] for d in range(D)] for l in range(L)]
    for l in range(L):
        for d in range(D):
            I = F if l == 0 else D * H
            W[l][d] = [w.reshape(3 * H, I if i == 0 else H) if i < 2 else w for i, w in enumerate(W[l][d])]
            W[l][d] = [w.clone().requires_grad_() for w in W[l][d]]
    xr = torch.from_numpy(x.astype(np.float64)).requires_grad_()
    h0r = None if h0 is None else torch.from_numpy(h0.astype(np.float64)).requires_grad_()
    lt = torch.from_numpy(lens if lens is not None else np.full(B, T))
    inp, ys, hns = xr, [], []
    for l in range(L):
        hl = None if h0r is None else h0r[l * D:(l + 1) * D]
        if m is None:
            gru = nn.GRU(inp.shape[2], H, 1, batch_first=True, bidirectional=D == 2).double()
            for d in range(D):
                sfx = "_l0" + ("_reverse" if d else "")
                W[l][d] = [nn.Parameter(w.detach()) for w in W[l][d]]    # the module's leaves: their .grad is the reference
                for nm, w in zip(("weight_ih", "weight_hh", "bias_ih", "bias_hh"), W[l][d]):
                    setattr(gru, nm + sfx, w)
            if lens is None:
                y, hn = gru(inp, hl)
            else:
                pk, hn = gru(pack_padded_sequence(inp, lt, batch_first=True, enforce_sorted=False), hl)
                y, _ = pad_packed_sequence(pk, batch_first=True, total_length=T)
        else:
            rdm = [[torch.from_numpy(m[l][d]).double() for d in range(D)]]
            y, hn = _oracle(W[l:l + 1], inp, hl, lt, rdm, [None], H, 1, D)
        y.retain_grad()
        ys.append(y)
        hns.append(hn)
        inp = y
    torch.autograd.backward((ys[-1], torch.cat(hns)), (torch.from_numpy(dy.astype(np.float64)),
                                                        torch.from_numpy(dhn.astype(np.float64))))
    grads = {f"gemm:grad:l0d{d}.{nm}": W[0][d][i].grad.numpy().ravel() for d in range(D) for i, nm in enumerate(NM)}
    grads["gemm:dx"] = xr.grad.numpy()
    dY0 = ys[0].grad.numpy() if L > 1 else None
    return ([y.detach().numpy() for y in ys], grads, None if h0r is None else h0r.grad.numpy()[:D], dY0,
            torch.cat(hns).detach().numpy())


def _models(s, names, flat, x, h0, dy, dhn, ys, dY0, m, lens, prec="exact"):
    """Free-running head-less models from the layer outputs ys: gates (stepwise), layer 0's backward recurrence seeded
    from dhn[0*D + d], the GEMMs."""
    B, T, F, H, L, D = (s[k] for k in "BTFHLD")
    masks = None if m is None else list(m)
    m0 = None if m is None else m[0]
    got = dict(ys=ys)
    steps = stepwise(s, prec, flat, x, h0, None, got, names, gates=True, masks=masks, lens=lens, head=False)
    G = np.stack([np.stack([steps[(f"step:g[l0d{d},t{t}]", "g_step")] for t in range(T)], 1) for d in range(D)])
    ws = dict(G=[G], DY=[dY0] + [None] * (min(L, 2) - 1))
    dgi, dgh = np.zeros((D, B, T, 3 * H)), np.zeros((D, B, T, 3 * H))
    dh0 = np.zeros((D, B, H))
    for kind, d, t, a, b in backward_steps(s, prec, flat, None if h0 is None else h0[:D], ws, ys, names, own=True,
                                           masks=m0, lens=lens, head=False, dy=dy, dhn=dhn):
        if kind == "dg":
            dgi[d][:, t], dgh[d][:, t] = a, b
        else:
            dh0[d] = a
    ghp = dgh.copy()
    ghp[0, :, 0] = 0
    if D == 2:
        ghp[1, :, T - 1] = 0
    xp = np.zeros((B, T, -(-F // 8) * 8))
    xp[..., :F] = x
    ops = dict(DGIP=(dgi, None), DGHP=(ghp, None), XP=(xp, None), YP=(ys[0], None), DGI=dgi, DGH=dgh)
    if m is not None:
        ops["RDS"] = (np.concatenate([m0[d][:, None, :].astype(np.float64) * ys[0][..., d * H:(d + 1) * H]
                                      for d in range(D)], 2), None)
    gm = gemm_steps(s, prec, flat, None, None if h0 is None else h0[:D], ops, names, None, masks=m0, lens=lens, head=False)
    return steps, gm, dh0


@pytest.mark.parametrize("masked", [False, True], ids=["nn_gru", "recurrent_dropout"])
@pytest.mark.parametrize("L", [1, 2])
@pytest.mark.parametrize("D", [1, 2])
@pytest.mark.parametrize("lengths,h0", [(True, False), (False, True)], ids=["ragged_lengths", "h0"])
def test_headless_step_models_are_autograd_of_nn_gru(masked, L, D, lengths, h0):
    """L = 1: layer 0 is the top layer and takes the caller's dy; L = 2: it takes dhn's slice 0 under the layer above.
    Lengths and h0 are tested apart: the library refuses them together."""
    s, names, flat, x, h0v, dy, dhn, m, lens = _case(L, D, lengths, h0, masked)
    T, H = s["T"], s["H"]
    ys, want, dh0_ref, dY0, hn = _reference(s, names, flat, x, h0v, dy, dhn, m, lens)
    steps, gm, dh0 = _models(s, names, flat, x, h0v, dy, dhn, ys, dY0, m, lens)
    assert ("step:logits", "logits_step") not in steps and ("gemm:dcat", "gemm_step") not in gm
    # the gate model's outputs are the reference's outputs, at every layer
    for l in range(L):
        for d in range(D):
            for t in range(T):
                got = steps[(f"step:y[l{l}d{d},t{t}]", "y_step")]
                assert np.abs(got - ys[l][:, t, d * H:(d + 1) * H]).max() <= 1e-12, (l, d, t)
    # h_n is the output at each direction's last valid step (the exact test of test_gpu_gru_steps.py)
    n_b = lens if lens is not None else np.full(s["B"], T)
    for l in range(L):
        assert np.array_equal(hn[l * D], ys[l][np.arange(s["B"]), n_b - 1, :H])
        if D == 2:
            assert np.array_equal(hn[l * D + 1], ys[l][:, 0, H:])
    for key, v in want.items():
        err = np.abs(gm[(key, "gemm_step")] - v).max()
        assert err <= 1e-10 * np.abs(v).max(), (key, err)
    if h0:
        assert np.abs(dh0 - dh0_ref).max() <= 1e-10 * np.abs(dh0_ref).max()


def test_headless_seed_is_per_direction_and_layer():
    """The seed the model reads is dhn[0*D + d]: swapping the directions' slices, or putting layer 1's slice in layer 0's
    place, changes layer 0's gradients (so the comparison above would see either error)."""
    s, names, flat, x, h0v, dy, dhn, m, lens = _case(2, 2, True, False, False)
    ys, want, _, dY0, _ = _reference(s, names, flat, x, h0v, dy, dhn, m, lens)
    base = _models(s, names, flat, x, h0v, dy, dhn, ys, dY0, m, lens)[1]
    for wrong in (dhn[[1, 0, 2, 3]], dhn[[2, 3, 0, 1]]):
        other = _models(s, names, flat, x, h0v, dy, wrong, ys, dY0, m, lens)[1]
        k = ("gemm:grad:l0d0.w_hh", "gemm_step")
        assert np.abs(other[k] - base[k]).max() > 1e-3 * np.abs(base[k]).max()
