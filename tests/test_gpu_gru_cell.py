"""``GRUCell`` (bigru_cell_*) on the H100: parity with float64 nn.GRUCell, a 64-step loop, a rounding model that splits
operands into bf16 where the kernels do, bit properties, agreement with ``GRU`` unrolled, launch counts and memory."""
import ctypes as C

import pytest
import torch
import torch.nn as nn

from financial_market_data_analysis_b200 import GRU, GRUCell, _lib

pytestmark = pytest.mark.gpu

TOL = {"fp32": (1e-4, 1e-3), "bf16x3": (1e-4, 1e-3), "bf16": (3e-2, 6e-2)}     # those of tests/test_gpu_gru.py
PRECS = ["fp32", "bf16x3", "bf16"]


def _rel_max(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def _rel_l2(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _pair(I, H, prec, seed=0):
    torch.manual_seed(seed)
    mine = GRUCell(I, H, precision=prec).cuda()
    ref = nn.GRUCell(I, H).double()
    ref.load_state_dict({k: v.double().cpu() for k, v in mine.state_dict().items()})
    return mine, ref


# every B, I and H of the issue's grid appears, with and without hx; None: unbatched.  The kernels' CTAs take 8, 16 or 32
# batch rows (cell_nblk): B = 13 runs the 16-row instantiations, B = 45 one 32-row CTA and a ragged tail of 13 rows (and
# two 32-row chunks in the weight-gradient kernel)
SHAPES = [(1, 13, 1), (3, 64, 8), (17, 200, 100), (512, 1, 128), (1, 64, 256), (3, 200, 512), (17, 13, 1024),
          (512, 64, 256), (None, 13, 100), (13, 64, 256), (45, 200, 100)]


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("B,I,H", SHAPES)
@pytest.mark.parametrize("hx", [True, False])
def test_parity_with_nn_grucell(prec, B, I, H, hx):
    mine, ref = _pair(I, H, prec)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(*((I,) if B is None else (B, I)), generator=g, dtype=torch.float64)
    h = 0.5 * torch.randn(*((H,) if B is None else (B, H)), generator=g, dtype=torch.float64) if hx else None
    xr, xm = x.clone().requires_grad_(), x.float().cuda().requires_grad_()
    hr = h.clone().requires_grad_() if hx else None
    hm = h.float().cuda().requires_grad_() if hx else None
    yr, ym = ref(xr, hr), mine(xm, hm)
    assert ym.shape == yr.shape
    to, tg = TOL[prec]
    assert _rel_max(ym, yr) <= to, _rel_max(ym, yr)
    dy = torch.randn(yr.shape, generator=g, dtype=torch.float64)
    yr.backward(dy)
    ym.backward(dy.float().cuda())
    assert _rel_l2(xm.grad, xr.grad) <= tg, _rel_l2(xm.grad, xr.grad)
    if hx:
        assert _rel_l2(hm.grad, hr.grad) <= tg, _rel_l2(hm.grad, hr.grad)
    for (n, p), (_, q) in zip(mine.named_parameters(), ref.named_parameters()):
        assert _rel_l2(p.grad, q.grad) <= tg, (n, _rel_l2(p.grad, q.grad))


@pytest.mark.parametrize("prec", PRECS)
def test_loop_of_64_steps(prec):
    """h' fed back for 64 steps with a loss on every step: the gradients of the parameters accumulate across 64 backward
    calls and the state's gradient flows back through every step."""
    I, H, B, T = 13, 128, 5, 64
    mine, ref = _pair(I, H, prec)
    g = torch.Generator().manual_seed(2)
    xs = 0.5 * torch.randn(T, B, I, generator=g, dtype=torch.float64)
    w = torch.randn(T, B, H, generator=g, dtype=torch.float64)
    xr, xm = xs.clone().requires_grad_(), xs.float().cuda().requires_grad_()
    hr, hm = None, None
    lr, lm = 0.0, 0.0
    for t in range(T):
        hr, hm = ref(xr[t], hr), mine(xm[t], hm)
        lr = lr + (hr * w[t]).sum()
        lm = lm + (hm * w[t].float().cuda()).sum()
    lr.backward()
    lm.backward()
    to, tg = TOL[prec]
    assert _rel_max(hm, hr) <= to * 10, _rel_max(hm, hr)          # 64 steps of one precision's rounding
    assert _rel_l2(xm.grad, xr.grad) <= tg * 10, _rel_l2(xm.grad, xr.grad)
    for (n, p), (_, q) in zip(mine.named_parameters(), ref.named_parameters()):
        assert _rel_l2(p.grad, q.grad) <= tg * 10, (n, _rel_l2(p.grad, q.grad))


# ---- rounding model ---------------------------------------------------------------------------------------------------------
def _split(t, ns):
    """(hi, lo) of an fp32 tensor as the kernels split it (lo = 0 at bf16), in float64; ns = 0: unsplit (the fp32 cell's
    FFMA products read the fp32 values themselves)."""
    t = t.float()
    if ns == 0:
        return t.double(), torch.zeros_like(t, dtype=torch.float64)
    hi = t.bfloat16().float()
    lo = (t - hi).bfloat16().float() if ns == 3 else torch.zeros_like(t)
    return hi.double(), lo.double()


def _mm(a, b, ns):
    """a @ b.T with both operands split where the kernels split them: hi*lo + lo*hi + hi*hi (bf16x3) or hi*hi, in fp64."""
    ah, al = _split(a, ns)
    bh, bl = _split(b, ns)
    out = ah @ bh.T
    if ns == 3:
        out = out + ah @ bl.T + al @ bh.T
    return out


CODE = {"fp32": _lib.PREC_FP32, "bf16": _lib.PREC_BF16, "bf16x3": _lib.PREC_BF16X3}


def _stash(B, I, H, prec):
    st, sc = C.c_size_t(), C.c_size_t()
    assert _lib.load().bigru_cell_workspace_bytes(B, I, H, CODE[prec], C.byref(st), C.byref(sc)) == 0
    return st.value, sc.value


# Tolerances (relative max-norm): about 4x the worst error measured over these shapes on an H100 80GB HBM3 (700 W), where
# what is left is fp32 accumulation order and the kernels' fp32 gate math against fp64, as in tests/ROUNDING_MODEL.md.  A
# misplaced rounding (an operand not split, or split twice) costs 1e-3 at bf16 and about 1e-5 at bf16x3.
#   worst measured:  h 5.0e-7   G 7.7e-7   dg (dgi, dgh) 1.4e-7   dx 9.0e-7   dh 2.8e-7   dW 7.1e-7
RM_TOL = {"h": 2e-6, "G": 3e-6, "dg": 6e-7, "dx": 4e-6, "dh": 2e-6, "dW": 3e-6}
# The fp32 cell against the same model with unsplit operands: what is left is its fp32 FFMA accumulation order and gate
# math, the same size as the tensor-core cells' remainder.  About 4x the worst error measured over the shapes below on the
# same card (tests/ROUNDING_MODEL.md).
#   worst measured:  h 1.3e-7   G 2.8e-7   dg 1.4e-7   dx 8.9e-7   dh 2.7e-7   dW 7.6e-7
RM_TOL_FP32 = {"h": 5e-7, "G": 1.2e-6, "dg": 6e-7, "dx": 3.6e-6, "dh": 1.1e-6, "dW": 3e-6}


@pytest.mark.parametrize("prec", ["bf16x3", "bf16", "fp32"])
@pytest.mark.parametrize("B,I,H", [(1, 64, 256), (17, 13, 100), (512, 64, 256), (3, 200, 1024), (13, 64, 256),
                                   (45, 200, 100)])
def test_rounding_model(prec, B, I, H):
    ns = {"bf16x3": 3, "bf16": 1, "fp32": 0}[prec]
    code = CODE[prec]
    tol = RM_TOL_FP32 if prec == "fp32" else RM_TOL
    torch.manual_seed(3)
    cell = GRUCell(I, H, precision=prec).cuda()
    flat = cell.flat_parameters()
    x = torch.randn(B, I, device="cuda")
    h = 0.5 * torch.randn(B, H, device="cuda")
    dhout = torch.randn(B, H, device="cuda")
    stash_b, scratch_b = _stash(B, I, H, prec)
    stash = torch.empty(stash_b, dtype=torch.uint8, device="cuda")
    scratch = torch.empty(scratch_b, dtype=torch.uint8, device="cuda")
    hout = torch.empty(B, H, device="cuda")
    grads, dx, dh = torch.empty_like(flat), torch.empty_like(x), torch.empty_like(h)
    lib = _lib.load()
    P = _lib.ptr
    assert lib.bigru_cell_forward(B, I, H, code, P(flat), P(x), P(h), P(hout), P(stash), None) == 0
    assert lib.bigru_cell_backward(B, I, H, code, P(flat), P(x), P(h), P(stash), P(dhout), P(grads), P(dx), P(dh), P(scratch),
                                   None) == 0
    torch.cuda.synchronize()
    G = stash.view(torch.float32).view(B, 4, H).cpu()
    H3 = 3 * H
    wih, whh = flat[:H3 * I].view(H3, I).cpu(), flat[H3 * I:H3 * (I + H)].view(H3, H).cpu()
    bih, bhh = flat[H3 * (I + H):H3 * (I + H) + H3].cpu().double(), flat[H3 * (I + H) + H3:].cpu().double()
    xc, hc, dc = x.cpu(), h.cpu(), dhout.cpu()
    # forward: four products, bias, gate math in fp64
    gi, gh = _mm(xc, wih, ns), _mm(hc, whh, ns)
    r = torch.sigmoid(gi[:, :H] + gh[:, :H] + bih[:H] + bhh[:H])
    z = torch.sigmoid(gi[:, H:2 * H] + gh[:, H:2 * H] + bih[H:2 * H] + bhh[H:2 * H])
    ghn = gh[:, 2 * H:] + bhh[2 * H:]
    n = torch.tanh(gi[:, 2 * H:] + bih[2 * H:] + r * ghn)
    hm = (1 - z) * n + z * hc.double()
    err = {"h": _rel_max(hout, hm), "G": max(_rel_max(G[:, k], v) for k, v in enumerate((r, z, n, ghn)))}
    # backward from the kernel's own stash: the gate gradients in fp64 from G, against the fp32 dgi, dgh the kernel left in
    # its scratch; the products split those (as the kernels do: a flipped bf16 rounding of one element would show at bf16)
    rs, zs, ns_, hs = (G[:, k].double() for k in range(4))
    dan = dc.double() * (1 - zs) * (1 - ns_ * ns_)
    dar = dan * hs * rs * (1 - rs)
    daz = dc.double() * (hc.double() - ns_) * zs * (1 - zs)
    dgi, dgh = scratch.view(torch.float32).view(2, B, H3).cpu()
    err["dg"] = max(_rel_max(dgi, torch.cat([dar, daz, dan], 1)), _rel_max(dgh, torch.cat([dar, daz, dan * rs], 1)))
    dxm = _mm(dgi, wih.T.contiguous(), ns)
    dhm = dc.double() * zs + _mm(dgh, whh.T.contiguous(), ns)
    gm = torch.cat([(dgi.double().T @ xc.double()).reshape(-1), (dgh.double().T @ hc.double()).reshape(-1),
                    dgi.double().sum(0), dgh.double().sum(0)])
    err.update(dx=_rel_max(dx, dxm), dh=_rel_max(dh, dhm), dW=_rel_max(grads, gm))
    print(f"rounding model {prec} B={B} I={I} H={H}: " + " ".join(f"{k}={v:.2e}" for k, v in err.items()))
    for k, v in err.items():
        assert v <= tol[k], (k, v)


# ---- bit properties -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", PRECS)
def test_bits_independent_of_grad_mode_batch_and_position(prec):
    I, H, B = 64, 256, 512
    cell = GRUCell(I, H, precision=prec).cuda()
    g = torch.Generator(device="cuda").manual_seed(4)
    x = torch.randn(B, I, device="cuda", generator=g)
    h = 0.5 * torch.randn(B, H, device="cuda", generator=g)
    dy = torch.randn(B, H, device="cuda", generator=g)

    def run(xx, hh, yy):
        xx, hh = xx.clone().requires_grad_(), hh.clone().requires_grad_()
        out = cell(xx, hh)
        out.backward(yy)
        return out.detach(), xx.grad, hh.grad

    y, dx, dh = run(x, h, dy)
    with torch.no_grad():
        assert torch.equal(cell(x, h), y)                      # with and without grad mode (no stash)
    for b in (0, 1, 255, 511):
        y1, dx1, dh1 = run(x[b:b + 1], h[b:b + 1], dy[b:b + 1])
        assert torch.equal(y1, y[b:b + 1]) and torch.equal(dx1, dx[b:b + 1]) and torch.equal(dh1, dh[b:b + 1]), b
    yr, dxr, dhr = run(x.flip(0), h.flip(0), dy.flip(0))
    assert torch.equal(yr, y.flip(0)) and torch.equal(dxr, dx.flip(0)) and torch.equal(dhr, dh.flip(0))
    # other tile shapes: 8, 16 and 32 batch rows per CTA, and a 32-row CTA with a ragged 13-row tail
    for b in (3, 13, 17, 45):
        yb, dxb, dhb = run(x[:b], h[:b], dy[:b])
        assert torch.equal(yb, y[:b]) and torch.equal(dxb, dx[:b]) and torch.equal(dhb, dh[:b]), b


@pytest.mark.parametrize("prec", PRECS)
def test_parameter_gradients_reproducible(prec):
    cell = GRUCell(64, 256, precision=prec).cuda()
    x = torch.randn(512, 64, device="cuda")
    h = torch.randn(512, 256, device="cuda")
    grads = []
    for _ in range(2):
        cell.zero_grad(set_to_none=True)
        cell(x, h).square().sum().backward()
        grads.append([p.grad.clone() for p in cell.parameters()])
    assert all(torch.equal(a, b) for a, b in zip(*grads))


@pytest.mark.parametrize("prec", PRECS)
def test_unrolled_cell_matches_gru(prec):
    I, H, B, T = 13, 128, 9, 16
    torch.manual_seed(5)
    gru = GRU(I, H, 1, batch_first=True, precision=prec).cuda()
    cell = GRUCell(I, H, precision=prec).cuda()
    cell.load_state_dict({k[:-3]: v for k, v in gru.state_dict().items()})       # weight_ih_l0 -> weight_ih
    x = torch.randn(B, T, I, device="cuda")
    h0 = 0.5 * torch.randn(1, B, H, device="cuda") if prec != "bf16" else None     # GRU refuses hx at bf16
    with torch.no_grad():
        y, hn = gru(x, h0)
        hc = None if h0 is None else h0[0]
        outs = []
        for t in range(T):
            hc = cell(x[:, t], hc)
            outs.append(hc)
    to = TOL[prec][0]
    assert _rel_max(torch.stack(outs, 1), y) <= to and _rel_max(hc, hn[0]) <= to


# ---- launches and memory ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", PRECS)
def test_launch_counts(prec):
    """A forward is one launch; a backward three (gate gradients, dx / dh, weight gradients), two without dx and dh
    (DESIGN.md §4.7)."""
    lib = _lib.load()
    cell = GRUCell(64, 256, precision=prec).cuda()
    x = torch.randn(32, 64, device="cuda", requires_grad=True)
    h = torch.randn(32, 256, device="cuda")
    n0 = lib.bigru_launch_count()
    with torch.no_grad():
        cell(x, h)
    n1 = lib.bigru_launch_count()
    y = cell(x, h)
    n2 = lib.bigru_launch_count()
    y.sum().backward()
    n3 = lib.bigru_launch_count()
    y = cell(x.detach())
    n4 = lib.bigru_launch_count()
    y.sum().backward()
    n5 = lib.bigru_launch_count()
    assert (n1 - n0, n2 - n1, n3 - n2, n4 - n3, n5 - n4) == (1, 1, 3, 1, 2)


def test_memory_stash_freed_on_refcount_and_none_without_grad():
    import gc
    import weakref
    B, I, H = 64, 64, 256
    cell = GRUCell(I, H, precision="bf16x3").cuda()
    x = torch.randn(B, I, device="cuda")
    torch.cuda.synchronize()
    gc.collect()
    gc.disable()
    try:
        m0 = torch.cuda.memory_allocated()
        with torch.no_grad():
            y = cell(x)
        assert torch.cuda.memory_allocated() - m0 == B * H * 4          # h' only (a multiple of the allocator's 512 bytes)
        del y
        y = cell(x)                                                     # parameters require grad: the autograd path
        assert torch.cuda.memory_allocated() - m0 == B * H * 4 + B * 4 * H * 4
        out = weakref.ref(y)
        del y
        assert out() is None and torch.cuda.memory_allocated() == m0
    finally:
        gc.enable()


def test_refusals_and_shapes():
    cell = GRUCell(13, 32, precision="bf16").cuda()
    x = torch.randn(4, 13, device="cuda")
    assert cell(x, torch.zeros(4, 32, device="cuda")).shape == (4, 32)      # hx at bf16
    assert cell(torch.randn(13, device="cuda"), torch.zeros(32, device="cuda")).shape == (32,)
    with pytest.raises(ValueError):
        cell(torch.randn(2, 4, 13, device="cuda"))
    with pytest.raises(ValueError):
        cell(x, torch.zeros(1, 4, 32, device="cuda"))
    with pytest.raises(RuntimeError):
        cell(torch.randn(4, 12, device="cuda"))
    with pytest.raises(RuntimeError):
        cell(x, torch.zeros(3, 32, device="cuda"))
    with pytest.raises(RuntimeError):
        cell(x, torch.zeros(4, 31, device="cuda"))
    lib = _lib.load()
    buf = torch.zeros(16, device="cuda")
    assert lib.bigru_cell_forward(1, 1, 65537, _lib.PREC_FP32, _lib.ptr(buf), _lib.ptr(buf), None, _lib.ptr(buf), None,
                                  None) == _lib.ERR_UNSUPPORTED
