"""Per-sequence lengths (``lengths=`` of BiGRU.forward / infer / train_step; bigru_*_lengths of the C ABI).

1. Every length equal to T is bitwise the call without lengths: logits, every gradient, dx, h_n, infer and three train
   steps, graphed and plain.
2. Padded inputs do not leak: large finite values at padded steps instead of zeros change no bit of the logits, the
   gradients, h_n or the max-pool routing, and dx is exactly 0 there.
3. Against the float64 oracle (oracle/lengths_oracle.py, torch's pack_padded_sequence) at the parity tolerances, under the
   kernel's own max-pool routing.
4. infer(lengths=...) is bitwise the eval-mode forward with the same lengths, also sliced by max_batch.
5. The Y planes and the dgi / dgh planes (bigru_workspace_region) are zero at padded steps.
6. Bad lengths raise ValueError; lengths with an initial state are refused by the library too.
7. Dropout with lengths, by mask injection.

At "fp32" the weight-gradient SGEMM adds split-K partials with atomics once B*T >= 1024 (DESIGN.md §4.3), so the bitwise
gradient checks run below that; the tensor-core precisions are bitwise at every shape."""
import ctypes as C

import numpy as np
import pytest
import torch

from gru_driver import dropout_mask, region
from oracle.lengths_oracle import LengthsOracle

PRECS = ("fp32", "bf16x3", "bf16")
TOL = {"fp32": (1e-4, 1e-3), "bf16x3": (1e-4, 1e-3), "bf16": (3e-2, 6e-2)}      # logits (rel max), gradients (rel L2)


def _pkg():
    import financial_market_data_analysis_b200 as pkg
    return pkg


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-30)


def rel_l2(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30)


def _model(prec, H, F, C_, L, D, p=0.0, spatial=False, seed=0):
    torch.manual_seed(seed)
    return _pkg().BiGRU(H, F, C_, L, 50, p, spatial, D == 2, precision=prec).cuda()


def _lengths(B, T, g, lo=1):
    """Random lengths in [lo, T] with T and lo both present."""
    n = torch.randint(lo, T + 1, (B,), generator=g)
    n[0], n[-1] = T, lo
    return n


def _run(m, x, dl, lengths=None):
    """Forward + backward through autograd: logits, flat gradient (C-ABI order), dx, h_n, max-pool routing."""
    for p in m.parameters():
        p.grad = None
    xg = x.clone().requires_grad_(True)
    y = m(xg, lengths=lengths)
    hn, arg = m._last_hidden.clone(), m.pooled_argmax()
    y.backward(dl)
    grads = torch.cat([p.grad.reshape(-1) for p in m._ordered_params()])
    torch.cuda.synchronize()
    return dict(logits=y.detach(), grads=grads, dx=xg.grad, hn=hn, arg=arg)


# ---------------------------------------------------------------------------------------------------------------- 1
@pytest.mark.gpu
@pytest.mark.parametrize("prec", PRECS)
def test_full_lengths_bitwise_equal_no_lengths(prec):
    B, T, F, H, L, C_, D = 40, 12, 13, 33, 2, 3, 2          # B*T < 1024: one split at fp32; ragged batch, padded units
    m = _model(prec, H, F, C_, L, D)
    g = torch.Generator().manual_seed(1)
    x, dl = torch.randn(B, T, F, generator=g).cuda(), torch.randn(B, C_, generator=g).cuda()
    want = _run(m, x, dl)
    forms = ([T] * B, torch.full((B,), T, dtype=torch.int64), torch.full((B,), T, dtype=torch.int32).cuda())
    for lens in forms:
        got = _run(m, x, dl, lens)
        for k in want:
            assert torch.equal(got[k], want[k]), (prec, k, type(lens))
    m.eval()
    with torch.no_grad():
        assert torch.equal(m.infer(x, lengths=[T] * B), m.infer(x))
        assert torch.equal(m.infer(x, lengths=[T] * B, max_batch=16), m.infer(x))


@pytest.mark.gpu
@pytest.mark.parametrize("graph", [True, False])
@pytest.mark.parametrize("prec", PRECS)
def test_full_lengths_train_steps_bitwise(prec, graph):
    import torch.nn as nn
    B, T, F, H, L, C_, D = 40, 12, 13, 33, 2, 3, 2
    ms = []
    for _ in range(2):
        m = _model(prec, H, F, C_, L, D)
        m.use_cuda_graph = graph
        m.add_loss_fn(nn.CrossEntropyLoss())
        m.add_optimizer(torch.optim.Adam(m.parameters(), lr=1e-3))
        m.train()
        ms.append(m)
    g = torch.Generator().manual_seed(2)
    for step in range(3):
        x, tgt = torch.randn(B, T, F, generator=g).cuda(), torch.randint(0, C_, (B,), generator=g).cuda()
        l0, y0 = ms[0].train_step(x, tgt)
        l1, y1 = ms[1].train_step(x, tgt, lengths=torch.full((B,), T))
        assert torch.equal(l0, l1) and torch.equal(y0, y1), (prec, graph, step)
        assert torch.equal(ms[0].flat_parameters(), ms[1].flat_parameters()), (prec, graph, step)
    if graph:
        assert len(ms[1]._graphs) == 1 and next(iter(ms[1]._graphs))[-1] is True


@pytest.mark.gpu
@pytest.mark.parametrize("prec", PRECS)
def test_train_step_graph_reads_new_lengths(prec):
    """A replayed graph reads the lengths of each call from its static buffer: graphed and plain steps agree bitwise."""
    import torch.nn as nn
    B, T, F, H, L, C_, D = 32, 10, 16, 128, 1, 3, 2
    ms = []
    for graph in (True, False):
        m = _model(prec, H, F, C_, L, D)
        m.use_cuda_graph = graph
        m.add_loss_fn(nn.CrossEntropyLoss())
        m.add_optimizer(torch.optim.Adam(m.parameters(), lr=1e-3))
        m.train()
        ms.append(m)
    g = torch.Generator().manual_seed(5)
    for step in range(3):
        x, tgt = torch.randn(B, T, F, generator=g).cuda(), torch.randint(0, C_, (B,), generator=g).cuda()
        lens = _lengths(B, T, g)
        (l0, y0), (l1, y1) = (m.train_step(x, tgt, lengths=lens) for m in ms)
        assert torch.equal(l0, l1) and torch.equal(y0, y1), (prec, step)
        assert torch.equal(ms[0].flat_parameters(), ms[1].flat_parameters()), (prec, step)
    assert len(ms[0]._graphs) == 1


# ---------------------------------------------------------------------------------------------------------------- 2
@pytest.mark.gpu
@pytest.mark.parametrize("prec", PRECS)
def test_padding_does_not_leak(prec):
    B, T, F, H, L, C_, D = 40, 12, 13, 33, 2, 3, 2
    m = _model(prec, H, F, C_, L, D)
    g = torch.Generator().manual_seed(3)
    lens = _lengths(B, T, g)
    x, dl = torch.randn(B, T, F, generator=g), torch.randn(B, C_, generator=g).cuda()
    pad = torch.arange(T)[None, :] >= lens[:, None]
    x0 = x.masked_fill(pad[..., None], 0.0)
    x1 = torch.where(pad[..., None], 1e4 * torch.randn(B, T, F, generator=g), x)
    a, b = _run(m, x0.cuda(), dl, lens), _run(m, x1.cuda(), dl, lens.cuda())
    for k in ("logits", "grads", "hn", "arg"):
        assert torch.equal(a[k], b[k]), (prec, k)
    padc = pad.cuda()
    for r in (a, b):
        assert (r["dx"][padc] == 0).all(), prec
    assert torch.equal(a["dx"], b["dx"]), prec


# ---------------------------------------------------------------------------------------------------------------- 3
ORACLE_CASES = {                     # B, T, F, H, L, D, lengths: "mixed" (a 16-row tile of length 1, then 1..T) or lo
    "mixed_l2": (48, 10, 16, 128, 2, 2, "mixed"),
    "ragged_f13_h33_l1": (37, 9, 13, 33, 1, 2, 1),
    "l3_d1": (32, 8, 16, 128, 3, 1, 1),
    "h512": (32, 6, 16, 512, 1, 2, 1),
    "configs1": (512, 128, 64, 256, 2, 2, 64),
}


def _oracle_lengths(B, T, kind, g):
    if kind == "mixed":
        lens = _lengths(B, T, g)
        lens[:16] = 1
        lens[16], lens[17] = T, 1
        return lens
    return _lengths(B, T, g, lo=kind)


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(ORACLE_CASES))
@pytest.mark.parametrize("prec", PRECS)
def test_lengths_against_oracle(prec, case):
    B, T, F, H, L, D, kind = ORACLE_CASES[case]
    if H == 512 and prec != "bf16":
        pytest.skip("hidden 512 runs at bf16 only (DESIGN.md §7)")
    C_ = 3
    m = _model(prec, H, F, C_, L, D)
    g = torch.Generator().manual_seed(4)
    lens = _oracle_lengths(B, T, kind, g)
    x, dl = torch.randn(B, T, F, generator=g), torch.randn(B, C_, generator=g)
    got = _run(m, x.cuda(), dl.cuda(), lens)
    orc = LengthsOracle(m.state_dict(), H, F, L, D == 2)
    xr = x.double().requires_grad_(True)
    want, hn, _ = orc(xr, lens, idx=got["arg"].cpu())
    want.backward(dl.double())
    tl, tg = TOL[prec]
    assert rel(got["logits"].cpu(), want.detach()) < tl, (prec, case)
    assert rel_l2(got["grads"].cpu(), orc.flat_grads()) < tg, (prec, case)
    assert rel_l2(got["dx"].cpu(), xr.grad) < tg, (prec, case)
    assert rel_l2(got["hn"].cpu(), hn.detach()) < tg, (prec, case)
    pad = (torch.arange(T)[None, :] >= lens[:, None]).cuda()
    assert (got["dx"][pad] == 0).all()
    assert (got["arg"].cpu() < lens[:, None].to(got["arg"].dtype)).all()      # the max-pool never picks a padded step


# ---------------------------------------------------------------------------------------------------------------- 4
@pytest.mark.gpu
@pytest.mark.parametrize("prec", PRECS)
def test_infer_lengths_bitwise_equal_eval_forward(prec):
    B, T, F, H, L, C_, D = 37, 9, 13, 128, 2, 3, 2
    m = _model(prec, H, F, C_, L, D)
    g = torch.Generator().manual_seed(6)
    lens = _lengths(B, T, g)
    x = torch.randn(B, T, F, generator=g).cuda()
    m.eval()
    with torch.no_grad():
        want = m(x, lengths=lens)
        assert torch.equal(m.infer(x, lengths=lens), want), prec
        assert torch.equal(m.infer(x, lengths=lens.cuda(), max_batch=16), want), prec
        assert not torch.equal(m.infer(x), want)


# ---------------------------------------------------------------------------------------------------------------- 5
@pytest.mark.gpu
@pytest.mark.parametrize("prec", ("bf16x3", "bf16"))
def test_planes_zero_at_padded_steps(prec):
    B, T, F, H, L, C_, D = 32, 10, 16, 128, 2, 3, 2
    m = _model(prec, H, F, C_, L, D)
    g = torch.Generator().manual_seed(7)
    lens = _lengths(B, T, g)
    x, dl = torch.randn(B, T, F, generator=g).cuda(), torch.randn(B, C_, generator=g).cuda()
    _run(m, x, dl, lens)
    plan, stash, _ = m._last_forward
    assert plan.B == B
    bufs = (stash, plan.scratch)
    pad = torch.arange(T)[None, :] >= lens[:, None]                      # [B, T]

    def planes(which, layer, shape):
        rc, sc, off, lo, _ = region(plan.handle, which, layer)
        assert rc == 0
        n, v = int(np.prod(shape)), bufs[sc].view(torch.int16)
        out = [v[off // 2: off // 2 + n].view(*shape).cpu()]
        if prec == "bf16x3":
            out.append(v[lo // 2: lo // 2 + n].view(*shape).cpu())
        return out

    for l in range(L):
        for p in planes("Y_PLANES", l, (B, T, D * H)):
            assert (p[pad] == 0).all(), (prec, l)
            assert (p[~pad] != 0).any()
    for which in ("DGI_PLANES", "DGH_PLANES"):
        for p in planes(which, 0, (D, B, T, 3 * H)):
            for d in range(D):
                assert (p[d][pad] == 0).all(), (prec, which, d)
                assert (p[d][~pad] != 0).any()


# ---------------------------------------------------------------------------------------------------------------- 6
@pytest.mark.gpu
def test_bad_lengths_raise():
    import torch.nn as nn
    B, T, F, H, L, C_, D = 8, 6, 5, 16, 2, 3, 2
    m = _model("fp32", H, F, C_, L, D)
    m.add_loss_fn(nn.CrossEntropyLoss())
    m.add_optimizer(torch.optim.Adam(m.parameters(), lr=1e-3))
    x, tgt = torch.randn(B, T, F).cuda(), torch.randint(0, C_, (B,)).cuda()
    h0 = torch.zeros(L * D, B, H).cuda()
    bad = ([0] + [T] * (B - 1), [T + 1] + [T] * (B - 1), [T] * (B - 1), torch.full((B, 1), T), [float(T)] * B)
    for lens in bad:
        with pytest.raises(ValueError):
            m(x, lengths=lens)
        with pytest.raises(ValueError):
            m.infer(x, lengths=lens)
        with pytest.raises(ValueError):
            m.train_step(x, tgt, lengths=lens)
    with pytest.raises(ValueError):
        m(x, h0, lengths=[T] * B)
    with pytest.raises(ValueError):
        m.infer(x, h0, lengths=[T] * B)
    with pytest.raises(ValueError):
        m.train_step(x, tgt, h0, lengths=[T] * B)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ("fp32", "bf16x3"))
def test_library_refuses_lengths_with_initial_state(prec):
    pkg = _pkg()
    lib, L_ = pkg._lib.load(), pkg._lib
    B, T, F, H, L, C_ = 32, 4, 8, 128, 1, 3
    plan = C.c_void_p()
    L_.check(lib.bigru_plan_create(B, T, F, H, L, C_, 1, {"fp32": 0, "bf16x3": 2}[prec], C.byref(plan)), "plan_create")
    try:
        buf = torch.zeros(1 << 16, device="cuda")
        lens = torch.full((B,), T, dtype=torch.int32, device="cuda")
        p, st = L_.ptr, C.c_void_p(torch.cuda.current_stream().cuda_stream)
        assert lib.bigru_forward_lengths(plan, p(buf), p(buf), p(buf), 0.0, 0, 0, 0, p(buf), p(buf), p(buf), None, p(lens),
                                         st) == L_.ERR_UNSUPPORTED
        assert lib.bigru_infer_lengths(plan, p(buf), p(buf), p(buf), p(buf), p(buf), p(lens), st) == L_.ERR_UNSUPPORTED
        for h0, dh0 in ((p(buf), None), (None, p(buf))):
            assert lib.bigru_backward_lengths(plan, p(buf), p(buf), h0, 0.0, 0, 0, 0, p(buf), p(buf), p(buf), p(buf), None,
                                              dh0, p(lens), st) == L_.ERR_UNSUPPORTED
        torch.cuda.synchronize()
    finally:
        lib.bigru_plan_destroy(plan)


# ---------------------------------------------------------------------------------------------------------------- 7
@pytest.mark.gpu
@pytest.mark.parametrize("spatial", [False, True])
@pytest.mark.parametrize("prec", PRECS)
def test_dropout_mask_injection_with_lengths(prec, spatial):
    """The kernels' dropout masks are a pure function of (seed, element index): rebuilt on the host and applied to each
    layer's input in the oracle before packing, the logits, gradients and dx match at the parity tolerances."""
    p = 0.3
    B, T, F, H, L, C_, D = (8, 6, 10, 16, 2, 3, 2) if prec == "fp32" else (32, 6, 16, 128, 2, 3, 2)
    m = _model(prec, H, F, C_, L, D, p=p, spatial=spatial, seed=12)
    m.train()
    g = torch.Generator().manual_seed(8)
    lens = _lengths(B, T, g)
    x, dl = torch.randn(B, T, F, generator=g), torch.randn(B, C_, generator=g)
    got = _run(m, x.cuda(), dl.cuda(), lens)
    seed = m._last_seed
    masks = [torch.from_numpy(dropout_mask(seed, 0, B, T, F, p, spatial)).double(),
             torch.from_numpy(dropout_mask(seed, 1, B, T, D * H, p)).double()]
    orc = LengthsOracle(m.state_dict(), H, F, L, D == 2)
    xr = x.double().requires_grad_(True)
    want, _, _ = orc(xr, lens, masks=masks, idx=got["arg"].cpu())
    want.backward(dl.double())
    tl, tg = TOL[prec]
    assert rel(got["logits"].cpu(), want.detach()) < tl, (prec, spatial)
    assert rel_l2(got["grads"].cpu(), orc.flat_grads()) < 5 * tg, (prec, spatial)
    assert rel_l2(got["dx"].cpu(), xr.grad) < 5 * tg, (prec, spatial)
    pad = torch.arange(T)[None, :] >= lens[:, None]
    dx = got["dx"].cpu()
    assert (dx[pad] == 0).all()
