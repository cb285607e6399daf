"""Recurrent dropout on the GPU (DESIGN.md §4.8): the masks read back from the stash against their host restatement, parity
of BiGRU and GRU with a float64 loop of ``h_t = GRUCell(x_t, m * h_{t-1})`` built from those masks, eval / infer / p = 0
against models without the keyword, and reproducibility."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn as nn

from financial_market_data_analysis_b200 import GRU, BiGRU, _lib

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from gru_driver import dropout_mask  # noqa: E402
from test_recurrent_dropout_cpu import WS_RD_MASK, rd_masks  # noqa: E402

pytestmark = pytest.mark.gpu
TOL = {"fp32": (1e-4, 1e-3), "bf16x3": (1e-4, 1e-3), "bf16": (3e-2, 6e-2)}    # logits / outputs rel-max, gradients rel-L2


def _rel_max(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def _rel_l2(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _cell(x, h, wih, whh, bih, bhh):
    gi, gh = x @ wih.T + bih, h @ whh.T + bhh
    H = h.shape[-1]
    r = torch.sigmoid(gi[:, :H] + gh[:, :H])
    z = torch.sigmoid(gi[:, H:2 * H] + gh[:, H:2 * H])
    n = torch.tanh(gi[:, 2 * H:] + r * gh[:, 2 * H:])
    return (1 - z) * n + z * h


def _oracle(W, x, h0, lens, rdm, drops, H, L, D):
    """float64 GRU stack: per layer the input times drops[l] (None: not dropped), then per direction a loop of
    GRUCell(x_t, m * h_{t-1}) over the valid steps (a padded step keeps h and outputs 0).  Returns (y [B][T][D*H], h_n)."""
    B, T, _ = x.shape
    inp, hns = x, []
    for l in range(L):
        if drops[l] is not None:
            inp = inp * drops[l]
        outs = []
        for d in range(D):
            w = W[l][d]
            h = h0[l * D + d] if h0 is not None else x.new_zeros(B, H)
            m = rdm[l][d]
            ys = [None] * T
            for t in (range(T) if d == 0 else reversed(range(T))):
                valid = (lens > t)[:, None]
                h = torch.where(valid, _cell(inp[:, t], m * h, *w), h)
                ys[t] = torch.where(valid, h, torch.zeros_like(h))
            outs.append(torch.stack(ys, 1))
            hns.append(h)
        inp = torch.cat(outs, -1)
    return inp, torch.stack(hns)


def _head(y, lens, lw, lb, H, D):
    s = y[..., :H] + (y[..., H:] if D == 2 else 0)
    B, T = s.shape[:2]
    idx = torch.arange(B)
    last = y[idx, lens - 1, :H] + (y[:, 0, H:] if D == 2 else 0)
    valid = (torch.arange(T)[None, :] < lens[:, None])[..., None]
    mx = torch.where(valid, s, torch.full_like(s, -float("inf"))).max(1).values
    mean = (s * valid).sum(1) / lens[:, None].double()
    return torch.cat([last, mx, mean], 1) @ lw.T + lb


def _weights(gru, L, D):
    return [[[getattr(gru, f"{n}_l{l}{'_reverse' if d else ''}").detach().double().cpu().requires_grad_()
              for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")] for d in range(D)] for l in range(L)]


def _masks(model, seed, L, D, B, H, p):
    Hp = model._pad.hidden
    return [[torch.from_numpy(m[:, :H].copy()).double() for m in layer] for layer in rd_masks(seed, p, L, D, B, Hp)]


def _input_drop(seed, l, B, T, width, cols, p, spatial):
    """dropout_kernel's factor for layer l's input [B][T][width] (the plan's columns) at the real columns `cols`."""
    m = dropout_mask(seed, l, B, T, width, p, spatial)
    return torch.from_numpy(m[..., cols].copy()).double()


def _plan_cols(H, Hp, D):
    return np.concatenate([d * Hp + np.arange(H) for d in range(D)])


CASES = {
    # prec, B, T, F, H, L, D, lengths, h0, drop, spatial
    "bf16x3_l1_d1": ("bf16x3", 32, 9, 13, 128, 1, 1, False, False, 0.0, False),
    "bf16x3_l2_d2_ragged_h32": ("bf16x3", 37, 8, 13, 32, 2, 2, False, False, 0.0, False),
    "bf16x3_l3_h0": ("bf16x3", 32, 6, 16, 128, 3, 2, False, True, 0.0, False),
    "bf16x3_l2_lengths_drop_spatial": ("bf16x3", 48, 9, 13, 256, 2, 2, True, False, 0.2, True),
    "bf16x3_l2_drop": ("bf16x3", 32, 7, 16, 128, 2, 2, False, False, 0.3, False),
    "bf16_l2_lengths": ("bf16", 37, 8, 13, 128, 2, 2, True, False, 0.2, False),
    "bf16_h512": ("bf16", 32, 5, 13, 512, 1, 2, False, False, 0.0, False),
    "fp32_l3_ragged_h32": ("fp32", 37, 7, 13, 32, 3, 2, False, False, 0.0, False),
    "fp32_h0_d1": ("fp32", 16, 6, 13, 48, 2, 1, False, True, 0.0, False),
    "fp32_lengths_drop": ("fp32", 21, 8, 13, 40, 2, 2, True, False, 0.3, True),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_bigru_parity_with_masked_cell_loop(name):
    prec, B, T, F, H, L, D, use_len, use_h0, pdrop, spatial = CASES[name]
    p = 0.25
    torch.manual_seed(0)
    model = BiGRU(H, F, 3, L, 50, pdrop, spatial, D == 2, precision=prec, recurrent_dropout=p).cuda().train()
    g = torch.Generator().manual_seed(7)
    x = torch.randn(B, T, F, generator=g, dtype=torch.float64)
    lens = torch.randint(1, T + 1, (B,), generator=g) if use_len else torch.full((B,), T)
    lens[0] = T
    h0 = 0.5 * torch.randn(L * D, B, H, generator=g, dtype=torch.float64) if use_h0 else None
    xm = x.float().cuda().requires_grad_()
    h0m = h0.float().cuda().requires_grad_() if use_h0 else None
    logits = model(xm, h0m, lengths=lens if use_len else None)
    seed = model._last_seed
    assert seed != 0
    # the oracle's masks: recurrent (host restatement), input and inter-layer dropout (dropout_kernel's)
    rdm = _masks(model, seed, L, D, B, H, p)
    Hp = model._pad.hidden
    drops = [None] * L
    if pdrop > 0:
        drops[0] = _input_drop(seed, 0, B, T, F, np.arange(F), pdrop, spatial)
        for l in range(1, L):
            drops[l] = _input_drop(seed, l, B, T, D * Hp, _plan_cols(H, Hp, D), pdrop, False)
    W = _weights(model.gru, L, D)
    lw = model.linear.weight.detach().double().cpu().requires_grad_()
    lb = model.linear.bias.detach().double().cpu().requires_grad_()
    xr = x.clone().requires_grad_()
    h0r = h0.clone().requires_grad_() if use_h0 else None
    y, hn = _oracle(W, xr, h0r, lens, rdm, drops, H, L, D)
    ref = _head(y, lens, lw, lb, H, D)
    tl, tg = TOL[prec]
    assert _rel_max(logits, ref) <= tl, name
    assert _rel_max(model._last_hidden, hn) <= tl, name
    dl = torch.randn(ref.shape, generator=g, dtype=torch.float64)
    ref.backward(dl)
    logits.backward(dl.float().cuda())
    ref_grads = [q.grad for l in range(L) for d in range(D) for q in W[l][d]] + [lw.grad, lb.grad]
    for (n, a), b in zip(model.named_parameters(), ref_grads):
        assert _rel_l2(a.grad, b) <= tg, (name, n, _rel_l2(a.grad, b))
    assert _rel_l2(xm.grad, xr.grad) <= tg, name
    if use_h0:
        assert _rel_l2(h0m.grad, h0r.grad) <= tg, name


@pytest.mark.parametrize("prec,H,L,D,use_h0", [("bf16x3", 128, 2, 2, True), ("bf16", 256, 2, 1, False), ("fp32", 40, 2, 2, True)])
def test_gru_parity_with_dhn(prec, H, L, D, use_h0):
    B, T, F, p = 37, 6, 13, 0.3
    torch.manual_seed(1)
    mine = GRU(F, H, L, batch_first=True, dropout=0.2, bidirectional=D == 2, precision=prec, recurrent_dropout=p).cuda().train()
    g = torch.Generator().manual_seed(3)
    x = torch.randn(B, T, F, generator=g, dtype=torch.float64)
    h0 = 0.5 * torch.randn(L * D, B, H, generator=g, dtype=torch.float64) if use_h0 else None
    xm = x.float().cuda().requires_grad_()
    h0m = h0.float().cuda().requires_grad_() if use_h0 else None
    ym, hnm = mine(xm, h0m)
    seed = mine._last_seed
    rdm = _masks(mine, seed, L, D, B, H, p)
    Hp = mine._pad.hidden
    drops = [None] + [_input_drop(seed, l, B, T, D * Hp, _plan_cols(H, Hp, D), 0.2, False) for l in range(1, L)]
    W = _weights(mine, L, D)
    xr = x.clone().requires_grad_()
    h0r = h0.clone().requires_grad_() if use_h0 else None
    yr, hnr = _oracle(W, xr, h0r, torch.full((B,), T), rdm, drops, H, L, D)
    tl, tg = TOL[prec]
    assert _rel_max(ym, yr) <= tl and _rel_max(hnm, hnr) <= tl
    dy, dhn = torch.randn(yr.shape, generator=g, dtype=torch.float64), torch.randn(hnr.shape, generator=g, dtype=torch.float64)
    torch.autograd.backward((yr, hnr), (dy, dhn))
    torch.autograd.backward((ym, hnm), (dy.float().cuda(), dhn.float().cuda()))
    ref_grads = [q.grad for l in range(L) for d in range(D) for q in W[l][d]]
    for a, b in zip(mine.parameters(), ref_grads):
        assert _rel_l2(a.grad, b) <= tg
    assert _rel_l2(xm.grad, xr.grad) <= tg
    if use_h0:
        assert _rel_l2(h0m.grad, h0r.grad) <= tg
    # without grad mode, training mode still masks (the training forward runs with a seed of its own)
    with torch.no_grad():
        yn, _ = mine(x.float().cuda(), None if h0 is None else h0.float().cuda())
        rdm = _masks(mine, mine._last_seed, L, D, B, H, p)
        drops = [None] + [_input_drop(mine._last_seed, l, B, T, D * Hp, _plan_cols(H, Hp, D), 0.2, False) for l in range(1, L)]
        yr2, _ = _oracle(W, x, h0, torch.full((B,), T), rdm, drops, H, L, D)
    assert _rel_max(yn, yr2) <= tl


@pytest.mark.parametrize("prec", ["fp32", "bf16x3", "bf16"])
def test_mask_read_back_equals_restatement(prec):
    B, T, F, H, L, D, p = 32, 4, 8, 128, 2, 2, 0.4
    model = BiGRU(H, F, 3, L, 50, 0.0, False, True, precision=prec, recurrent_dropout=p).cuda().train()
    x = torch.randn(B, T, F, device="cuda")
    model(x)
    torch.cuda.synchronize()
    plan, stash, _ = model._last_forward
    lib = _lib.load()
    ref = rd_masks(model._last_seed, p, L, D, B, H)
    for l in range(L):
        sc, off, lo, pitch = C.c_int(), C.c_size_t(), C.c_size_t(), C.c_int64()
        assert lib.bigru_workspace_region(plan.handle, WS_RD_MASK, l, C.byref(sc), C.byref(off), C.byref(lo), C.byref(pitch)) == 0
        got = stash[off.value:off.value + 4 * D * B * H].view(torch.float32).view(D, B, H).cpu().numpy()
        assert np.array_equal(got.view(np.uint32), ref[l].view(np.uint32)), l


@pytest.mark.parametrize("prec", ["fp32", "bf16x3", "bf16"])
def test_eval_infer_and_p0_equal_model_without_keyword(prec):
    B, T, F, H, L, C_ = 40, 6, 13, 128, 2, 3
    torch.manual_seed(0)
    plain = BiGRU(H, F, C_, L, 50, 0.2, True, True, precision=prec).cuda()
    torch.manual_seed(0)
    rd = BiGRU(H, F, C_, L, 50, 0.2, True, True, precision=prec, recurrent_dropout=0.3).cuda()
    x = torch.randn(B, T, F, device="cuda")
    plain.eval(); rd.eval()
    with torch.no_grad():
        assert torch.equal(plain(x), rd(x))
    assert torch.equal(plain.infer(x), rd.infer(x))
    gp, gr = GRU(F, H, L, batch_first=True, precision=prec), GRU(F, H, L, batch_first=True, precision=prec, recurrent_dropout=0.3)
    gr.load_state_dict(gp.state_dict())
    gp.cuda().eval(); gr.cuda().eval()
    with torch.no_grad():
        a, b = gp(x), gr(x)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    # p = 0 with graphs on: three train steps are bitwise those of a model built without the keyword
    torch.manual_seed(0)
    m0 = BiGRU(H, F, C_, L, 50, 0.0, False, True, precision=prec).cuda().train()
    torch.manual_seed(0)
    m1 = BiGRU(H, F, C_, L, 50, 0.0, False, True, precision=prec, recurrent_dropout=0.0).cuda().train()
    tgt = torch.randint(0, C_, (B,), device="cuda")
    outs = []
    for m in (m0, m1):
        m.use_cuda_graph = True
        m.add_loss_fn(nn.CrossEntropyLoss())
        m.add_optimizer(torch.optim.Adam(m.parameters(), lr=1e-3))
        outs.append([m.train_step(x, tgt) for _ in range(3)])
    for (l0, g0), (l1, g1) in zip(*outs):
        assert torch.equal(l0, l1) and torch.equal(g0, g1)
    assert torch.equal(m0.flat_parameters(), m1.flat_parameters())
    assert len(m0._graphs) == 1 and len(m1._graphs) == 1


def test_assigning_the_attribute_takes_effect():
    B, T, F, H = 32, 5, 8, 128
    torch.manual_seed(0)
    m = BiGRU(H, F, 3, 1, 50, 0.0, False, True, precision="bf16x3").cuda().train()
    x = torch.randn(B, T, F, device="cuda")
    with torch.no_grad():
        a = m(x)
        m.recurrent_dropout = 0.5
        torch.manual_seed(3)
        b = m(x)
        seed = m._last_seed
        m.eval()
        c = m(x)
    assert seed != 0 and not torch.equal(a, b) and torch.equal(a, c)


def _train(seed_model, B, p=0.25, x=None, tgt=None):
    torch.manual_seed(seed_model)
    m = BiGRU(256, 64, 3, 2, 50, 0.2, True, True, precision="bf16x3", recurrent_dropout=p).cuda().train()
    m.add_loss_fn(nn.CrossEntropyLoss())
    m.add_optimizer(torch.optim.Adam(m.parameters(), lr=1e-3))
    torch.manual_seed(11)
    res = [m.train_step(x, tgt) for _ in range(3)]
    return m, res


def test_reproducible_train_steps_and_row_independence():
    B, T, F = 512, 128, 64
    g = torch.Generator().manual_seed(2)
    x = torch.randn(B, T, F, generator=g).cuda()
    tgt = torch.randint(0, 3, (B,), generator=g).cuda()
    m1, r1 = _train(0, B, x=x, tgt=tgt)
    m2, r2 = _train(0, B, x=x, tgt=tgt)
    for (l1, g1), (l2, g2) in zip(r1, r2):
        assert torch.equal(l1, l2) and torch.equal(g1, g2)
    assert torch.equal(m1.flat_parameters(), m2.flat_parameters())
    assert not m1._graphs                                   # masks are drawn: no graph capture
    # a row's outputs do not depend on the rows after it: the first 64 rows inside a batch of 64 and of 512, same seed
    torch.manual_seed(0)
    m = BiGRU(256, 64, 3, 2, 50, 0.0, False, True, precision="bf16x3", recurrent_dropout=0.25).cuda().train()
    with torch.no_grad():
        torch.manual_seed(5)
        small = m(x[:64])
        torch.manual_seed(5)
        big = m(x)
    assert torch.equal(small, big[:64])
