"""``GRU`` (bigru_gru_*) on the H100: parity with torch.nn.GRU in float64, lengths and PackedSequence, bit identity with
the recurrence inside BiGRU, nn.GRU's dropout placement, reproducibility, a custom head on ``BiGRU.gru`` and the refusals."""
import ctypes as C

import pytest
import torch
import torch.nn as nn
from torch.nn.utils.rnn import pack_padded_sequence, pad_packed_sequence

from financial_market_data_analysis_b200 import GRU, BiGRU, _lib
from gru_driver import dropout_mask

pytestmark = pytest.mark.gpu

TOL = {"fp32": (1e-4, 1e-3), "bf16x3": (1e-4, 1e-3), "bf16": (3e-2, 6e-2)}


def _prec(p, H):
    return ("bf16x3" if H <= 256 else "fp32") if p == "auto" else p


def _rel_max(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def _rel_l2(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _pair(F, H, L, D, prec, batch_first=True, seed=0):
    torch.manual_seed(seed)
    mine = GRU(F, H, L, batch_first=batch_first, bidirectional=D == 2, precision=prec).cuda()
    ref = nn.GRU(F, H, L, batch_first=batch_first, bidirectional=D == 2).double()
    ref.load_state_dict({k: v.double().cpu() for k, v in mine.state_dict().items()})
    return mine, ref


def _check_grads(mine, ref, tol, what):
    for (n, p), (_, q) in zip(mine.named_parameters(), ref.named_parameters()):
        assert _rel_l2(p.grad, q.grad) <= tol, (what, n, _rel_l2(p.grad, q.grad))


# (precision, H, L, D, B (None: unbatched), F, T, hx, batch_first)
CASES = [
    ("fp32", 32, 1, 1, 1, 13, 1, True, True),
    ("fp32", 128, 2, 2, 19, 64, 8, False, False),
    ("fp32", 512, 2, 1, 1, 13, 4, True, True),
    ("bf16x3", 32, 2, 2, 19, 13, 7, True, False),
    ("bf16x3", 128, 3, 2, 64, 64, 9, False, True),
    ("bf16x3", 256, 2, 1, 19, 64, 5, True, True),
    ("bf16x3", 128, 2, 2, None, 13, 6, True, True),
    ("bf16", 128, 2, 2, 19, 13, 7, False, True),
    ("bf16", 256, 3, 1, 1, 64, 1, False, False),
    ("bf16", 512, 1, 2, 64, 64, 5, False, True),
    ("auto", 32, 1, 2, 64, 13, 3, True, False),
    ("auto", 300, 2, 2, 19, 13, 6, True, True),
]


@pytest.mark.parametrize("prec,H,L,D,B,F,T,hx,bf", CASES)
def test_parity_with_nn_gru(prec, H, L, D, B, F, T, hx, bf):
    mine, ref = _pair(F, H, L, D, prec, batch_first=bf)
    g = torch.Generator().manual_seed(1)
    shape = (T, F) if B is None else ((B, T, F) if bf else (T, B, F))
    x = torch.randn(*shape, generator=g, dtype=torch.float64)
    hshape = (L * D, H) if B is None else (L * D, B, H)
    h0 = 0.5 * torch.randn(*hshape, generator=g, dtype=torch.float64) if hx else None
    xr, xm = x.clone().requires_grad_(), x.float().cuda().requires_grad_()
    hr = h0.clone().requires_grad_() if hx else None
    hm = h0.float().cuda().requires_grad_() if hx else None
    yr, hnr = ref(xr, hr)
    ym, hnm = mine(xm, hm)
    assert ym.shape == yr.shape and hnm.shape == hnr.shape
    to, tg = TOL[_prec(prec, H)]
    assert _rel_max(ym, yr) <= to and _rel_max(hnm, hnr) <= to, (_rel_max(ym, yr), _rel_max(hnm, hnr))
    dy, dhn = torch.randn(yr.shape, generator=g, dtype=torch.float64), torch.randn(hnr.shape, generator=g, dtype=torch.float64)
    torch.autograd.backward((yr, hnr), (dy, dhn))
    torch.autograd.backward((ym, hnm), (dy.float().cuda(), dhn.float().cuda()))
    assert _rel_l2(xm.grad, xr.grad) <= tg
    if hx:
        assert _rel_l2(hm.grad, hr.grad) <= tg
    _check_grads(mine, ref, tg, prec)
    with torch.no_grad():                                    # the inference path gives the training path's bits
        yi, hni = mine(xm, hm)
    assert torch.equal(yi, ym.detach()) and torch.equal(hni, hnm.detach())


def test_parity_configs1_bf16x3():
    B, T, F, H, L = 512, 128, 64, 256, 2
    mine, ref = _pair(F, H, L, 2, "bf16x3")
    g = torch.Generator().manual_seed(2)
    x = torch.randn(B, T, F, generator=g, dtype=torch.float64)
    xr, xm = x.clone().requires_grad_(), x.float().cuda().requires_grad_()
    yr, hnr = ref(xr)
    ym, hnm = mine(xm)
    assert _rel_max(ym, yr) <= 1e-4 and _rel_max(hnm, hnr) <= 1e-4
    dy, dhn = torch.randn(yr.shape, generator=g, dtype=torch.float64), torch.randn(hnr.shape, generator=g, dtype=torch.float64)
    torch.autograd.backward((yr, hnr), (dy, dhn))
    torch.autograd.backward((ym, hnm), (dy.float().cuda(), dhn.float().cuda()))
    assert _rel_l2(xm.grad, xr.grad) <= 1e-3
    _check_grads(mine, ref, 1e-3, "configs[1]")


@pytest.mark.parametrize("prec,H,D,B", [("fp32", 40, 2, 7), ("bf16x3", 128, 2, 19), ("bf16x3", 32, 1, 32), ("bf16", 128, 2, 16)])
def test_lengths_and_packed_sequence(prec, H, D, B):
    T, F, L = 9, 13, 2
    mine, ref = _pair(F, H, L, D, prec)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(B, T, F, generator=g, dtype=torch.float64)
    lens = torch.randint(1, T + 1, (B,), generator=g)
    lens[0], lens[-1] = 1, T
    to, tg = TOL[prec]
    xr = x.clone().requires_grad_()
    pr, hnr = ref(pack_padded_sequence(xr, lens, batch_first=True, enforce_sorted=False))
    yr, _ = pad_packed_sequence(pr, batch_first=True, total_length=T)
    dy = torch.randn(B, T, D * H, generator=g, dtype=torch.float64)
    dhn = torch.randn(L * D, B, H, generator=g, dtype=torch.float64)
    torch.autograd.backward((yr, hnr), (dy, dhn))
    ref_grads = [p.grad.clone() for p in ref.parameters()]
    # lengths=: output 0 at padded steps, h_n after each direction's last valid step
    xm = x.float().cuda().requires_grad_()
    ym, hnm = mine(xm, lengths=lens)
    pad = torch.arange(T)[None, :] >= lens[:, None]
    assert torch.all(ym.detach().cpu()[pad] == 0)
    assert _rel_max(ym, yr) <= to and _rel_max(hnm, hnr) <= to
    torch.autograd.backward((ym, hnm), (dy.float().cuda(), dhn.float().cuda()))
    assert _rel_l2(xm.grad, xr.grad) <= tg and torch.all(xm.grad.cpu()[pad] == 0)
    _check_grads(mine, ref, tg, "lengths")
    # a PackedSequence in, the same packing out
    mine.zero_grad()
    xp = x.float().cuda().requires_grad_()
    packed = pack_padded_sequence(xp, lens, batch_first=True, enforce_sorted=False)
    pm, hnp = mine(packed)
    assert torch.equal(pm.batch_sizes, packed.batch_sizes) and torch.equal(pm.sorted_indices, packed.sorted_indices)
    yp, lp = pad_packed_sequence(pm, batch_first=True, total_length=T)
    assert torch.equal(lp, lens) and torch.equal(yp, ym.detach()) and torch.equal(hnp, hnm.detach())
    torch.autograd.backward((yp, hnp), (dy.float().cuda(), dhn.float().cuda()))
    assert torch.equal(xp.grad, xm.grad)
    for p, q in zip(mine.parameters(), ref_grads):
        assert _rel_l2(p.grad, q) <= tg


def _region(plan, which, layer, nfloats, buf):
    ins, off, lo, pitch = C.c_int(), C.c_size_t(), C.c_size_t(), C.c_int64()
    _lib.check(_lib.load().bigru_workspace_region(plan.handle, which, layer, C.byref(ins), C.byref(off), C.byref(lo), C.byref(pitch)),
               "bigru_workspace_region")
    return buf[off.value:off.value + 4 * nfloats].view(torch.float32)


@pytest.mark.parametrize("prec", ["fp32", "bf16x3", "bf16"])
@pytest.mark.parametrize("L,D", [(1, 1), (1, 2), (2, 1), (2, 2)])
@pytest.mark.parametrize("ragged", [False, True])
def test_bitwise_identity_with_bigru(prec, L, D, ragged):
    B, T, F, H, Cn = 32, 6, 13, 128, 3
    torch.manual_seed(0)
    model = BiGRU(H, F, Cn, L, 50, 0.0, False, D == 2, precision=prec).cuda().train()
    g = torch.Generator().manual_seed(4)
    x = torch.randn(B, T, F, generator=g).cuda()
    lens = torch.randint(1, T + 1, (B,), generator=g) if ragged else None
    xb = x.clone().requires_grad_()
    logits = model(xb, lengths=lens)
    plan, stash, _ = model._last_forward
    off = C.c_size_t()
    _lib.check(_lib.load().bigru_stash_output_offset(plan.handle, L - 1, C.byref(off)), "bigru_stash_output_offset")
    y_bigru = stash[off.value:off.value + 4 * B * T * D * H].view(torch.float32).view(B, T, D * H).clone()
    hn_bigru = model._last_hidden.clone()
    logits.backward(torch.randn(B, Cn, generator=g).cuda())
    dY = _region(plan, 7, L - 1, B * T * D * H, plan.scratch).view(B, T, D * H).clone()       # BIGRU_WS_DY
    dcat = _region(plan, 9, L, B * 3 * H, plan.scratch).view(B, 3 * H).clone()                # BIGRU_WS_DCAT
    n_gru = model.gru_param_count()
    g_bigru = [p.grad.clone() for p in model.gru.parameters()]
    dx_bigru = xb.grad.clone()
    model.zero_grad()
    xg = x.clone().requires_grad_()
    y, hn = model.gru(xg, lengths=lens)
    assert torch.equal(y, y_bigru) and torch.equal(hn, hn_bigru)
    dhn = torch.zeros(L * D, B, H, device="cuda")
    dhn[(L - 1) * D:] = dcat[:, :H]
    torch.autograd.backward((y, hn), (dY, dhn))
    for a, b in zip(model.gru.parameters(), g_bigru):
        assert torch.equal(a.grad, b)
    assert torch.equal(xg.grad, dx_bigru)
    assert sum(p.numel() for p in model.gru.parameters()) == n_gru
    with torch.no_grad():
        yi, hni = model.gru(x, lengths=lens)
    assert torch.equal(yi, y_bigru) and torch.equal(hni, hn_bigru)


@pytest.mark.parametrize("prec", ["fp32", "bf16x3"])
def test_dropout_between_layers_only(prec):
    B, T, F, H, L, D, p = 32, 5, 13, 128, 2, 2, 0.3
    torch.manual_seed(0)
    mine = GRU(F, H, L, batch_first=True, dropout=p, bidirectional=True, precision=prec).cuda().train()
    g = torch.Generator().manual_seed(5)
    x = torch.randn(B, T, F, generator=g, dtype=torch.float64)
    xm = x.float().cuda().requires_grad_()
    ym, hnm = mine(xm)
    mask = torch.from_numpy(dropout_mask(mine._last_seed, 1, B, T, D * H, p)).double()
    # float64 reference: one nn.GRU per layer, the kernel's own mask on layer 1's input
    layers = []
    for l in range(L):
        m = nn.GRU(F if l == 0 else D * H, H, 1, batch_first=True, bidirectional=True).double()
        m.load_state_dict({k.replace(f"_l{l}", "_l0"): v.double().cpu() for k, v in mine.state_dict().items() if f"_l{l}" in k})
        layers.append(m)
    xr = x.clone().requires_grad_()
    y0, h0 = layers[0](xr)
    yr, h1 = layers[1](y0 * mask)
    hnr = torch.cat([h0, h1])
    assert _rel_max(ym, yr) <= 1e-4 and _rel_max(hnm, hnr) <= 1e-4
    dy, dhn = torch.randn(yr.shape, generator=g, dtype=torch.float64), torch.randn(hnr.shape, generator=g, dtype=torch.float64)
    torch.autograd.backward((yr, hnr), (dy, dhn))
    torch.autograd.backward((ym, hnm), (dy.float().cuda(), dhn.float().cuda()))
    assert _rel_l2(xm.grad, xr.grad) <= 1e-3
    ref_grads = [q.grad for l in range(L) for q in layers[l].parameters()]
    for a, b in zip(mine.parameters(), ref_grads):
        assert _rel_l2(a.grad, b) <= 1e-3
    # without grad mode, training mode drops as nn.GRU does: the training forward runs, with masks of its own seed
    with torch.no_grad():
        yn, hnn = mine(x.float().cuda())
    mask = torch.from_numpy(dropout_mask(mine._last_seed, 1, B, T, D * H, p)).double()
    with torch.no_grad():
        y0, h0 = layers[0](x)
        yr, h1 = layers[1](y0 * mask)
    assert _rel_max(yn, yr) <= 1e-4 and _rel_max(hnn, torch.cat([h0, h1])) <= 1e-4
    # one layer: nothing is dropped, x included
    one = GRU(F, H, 1, batch_first=True, dropout=0.5, bidirectional=True, precision=prec).cuda().train()
    xa = x.float().cuda()
    ya, ha = one(xa.clone().requires_grad_())
    one.dropout = 0.0
    yb, hb = one(xa.clone().requires_grad_())
    assert torch.equal(ya, yb) and torch.equal(ha, hb)


def test_reproducible_and_inference_workspace_only():
    B, T, F, H, L = 512, 128, 64, 256, 2
    torch.manual_seed(0)
    mine = GRU(F, H, L, batch_first=True, bidirectional=True, precision="bf16x3").cuda()
    g = torch.Generator().manual_seed(6)
    x = torch.randn(B, T, F, generator=g).cuda()
    dy, dhn = torch.randn(B, T, 2 * H, generator=g).cuda(), torch.randn(2 * L, B, H, generator=g).cuda()
    runs = []
    for _ in range(2):
        mine.zero_grad()
        xg = x.clone().requires_grad_()
        y, hn = mine(xg)
        torch.autograd.backward((y, hn), (dy, dhn))
        runs.append([y.detach().clone(), hn.detach().clone(), xg.grad] + [p.grad.clone() for p in mine.parameters()])
    assert all(torch.equal(a, b) for a, b in zip(*runs))
    fresh = GRU(F, H, L, batch_first=True, bidirectional=True, precision="bf16x3").cuda()
    with torch.no_grad():
        fresh(x)
    (plan,) = fresh._plans.values()
    assert plan._infer_ws is not None and plan._scratch is None and not plan._free_stash


class _HeadOnGRU(BiGRU):
    """The reference's head (biGRU_model.py:101-137) in torch ops on ``self.gru``."""

    def forward(self, input_seq, hidden=None):
        self.batch_size, self.input_length = input_seq.size(0), input_seq.size(1)
        gru_out, hidden = self.gru(input_seq, hidden)
        hidden = hidden.view(self.n_layers, self.n_directions, self.batch_size, self.hidden_size)
        last_hidden = torch.sum(hidden[-1], dim=0)
        if self.bidirectional:
            gru_out = gru_out[:, :, :self.hidden_size] + gru_out[:, :, self.hidden_size:]
        max_pool = torch.nn.functional.adaptive_max_pool1d(gru_out.permute(0, 2, 1), (1,)).view(self.batch_size, -1)
        avg_pool = torch.sum(gru_out, dim=1) / self.input_length
        return self.linear(torch.cat([last_hidden, max_pool, avg_pool], dim=1))


@pytest.mark.parametrize("prec", ["fp32", "bf16x3"])
def test_custom_head_matches_bigru(prec):
    B, T, F, H, L, Cn = 19, 7, 13, 128, 2, 3
    torch.manual_seed(0)
    base = BiGRU(H, F, Cn, L, 50, 0.0, False, True, precision=prec).cuda()
    torch.manual_seed(0)
    custom = _HeadOnGRU(H, F, Cn, L, 50, 0.0, False, True, precision=prec).cuda()
    g = torch.Generator().manual_seed(7)
    x = torch.randn(B, T, F, generator=g).cuda()
    dl = torch.randn(B, Cn, generator=g).cuda()
    la, lb = base(x), custom(x)
    assert _rel_max(lb, la) <= 1e-4
    la.backward(dl)
    lb.backward(dl)
    for (n, p), q in zip(base.named_parameters(), custom.parameters()):
        assert _rel_l2(q.grad, p.grad) <= 1e-3, n


@pytest.mark.parametrize("B,H", [(32, 128), (19, 32)])
def test_forward_without_backward_frees_on_refcount(B, H):
    """Outputs dropped without a backward free the training stash at once, without the garbage collector: the autograd
    node keeps no reference cycle through the output (unpadded plans return the kernels' own y)."""
    import gc
    import weakref
    mine = GRU(13, H, 2, batch_first=True, bidirectional=True, precision="bf16x3").cuda()
    x = torch.randn(B, 5, 13, device="cuda")
    gc.collect()
    gc.disable()
    try:
        y, hn = mine(x)                                   # parameters require grad: the autograd path
        node = hn.grad_fn
        stash, out = weakref.ref(node.stash), weakref.ref(y)
        del y, hn, node
        assert stash() is None and out() is None
    finally:
        gc.enable()


def test_refusals():
    mine = GRU(13, 128, 2, batch_first=True, precision="bf16x3").cuda()
    x = torch.randn(4, 5, 13, device="cuda")
    with pytest.raises(ValueError, match="dropout = 1"):
        GRU(13, 128, 2, batch_first=True, dropout=1.0, precision="bf16x3").cuda().train()(x)
    GRU(13, 128, 1, batch_first=True, dropout=1.0, precision="bf16x3").cuda().train()(x)      # one layer: nothing to drop
    with pytest.raises(RuntimeError):
        mine(x, torch.zeros(2, 3, 128, device="cuda"))                  # wrong batch
    with pytest.raises(RuntimeError):
        mine(x, torch.zeros(2, 4, 64, device="cuda"))                   # wrong hidden
    with pytest.raises(ValueError):
        mine(x, torch.zeros(2, 4, 128, device="cuda"), lengths=[5, 4, 3, 2])
    with pytest.raises(ValueError):
        mine(x, lengths=[5, 4, 3, 6])
    with pytest.raises(ValueError):
        GRU(13, 128, 2, batch_first=True, precision="bf16").cuda()(x, torch.zeros(2, 4, 128, device="cuda"))
    with pytest.raises(RuntimeError):
        mine(torch.randn(4, 5, 12, device="cuda"))
    with pytest.raises(ValueError):
        mine(torch.randn(5, device="cuda"))
