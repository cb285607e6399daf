"""Stash-free batched inference (bigru_infer, BiGRU.infer / infer_windows).

CPU: the inference workspace size against a restatement of its layout, and the null-argument checks.  GPU: the logits are
bitwise those of the eval-mode forward (the same launch sequence and kernels; only where the outputs go differs), slicing by
max_batch and the window path change nothing, the first call allocates the inference workspace and nothing of the training
forward's stash or scratch, and an inference call between training calls leaves them bitwise unchanged."""
import os

import numpy as np
import pytest
import torch
import torch.nn as nn


@pytest.fixture(scope="module")
def pkg():
    import financial_market_data_analysis_b200 as p
    from financial_market_data_analysis_b200 import build as b
    if not os.path.exists(p._lib.LIB_PATH):
        b.build()
    return p


PRECS = ("fp32", "bf16", "bf16x3")


def _rup(v, m):
    return (v + m - 1) // m * m


def infer_bytes(B, T, F, H, L, C, D, prec):
    """bigru_infer_workspace_bytes restated: fp32 words of gi [D][BT][3H], gh [D][B][3H] (fp32 only), the fp32 Y buffers
    [BT][DH] (the top layer's; at fp32 a second one for ping-pong from L = 2), cat [B][3H], arg [B][H], then from a 64-word
    boundary the bf16 planes (hi, and lo at bf16x3; each plane set rounded up to 128 bf16): the layer-0 input
    [BT][rup(F, 8)], the Y planes of min(L - 1, 2) lower layers, and the packed W_ih / head operand image."""
    BT, DH, tc = B * T, D * H, prec != "fp32"
    n = 2 if prec == "bf16x3" else 1

    def planes(elems):
        return _rup(n * elems, 128) // 2 if tc else 0

    def pack(R, K, batch):                 # zero-padded K-major image: rows to 128, K to 64
        return n * batch * _rup(R, 128) * _rup(K, 64)

    w = D * BT * 3 * H
    w += 0 if tc else D * B * 3 * H
    w += BT * DH * (2 if not tc and L > 1 else 1)
    w += B * 3 * H + B * H
    w = _rup(w, 64)
    w += planes(BT * _rup(F, 8))
    w += planes(BT * DH) * min(L - 1, 2)
    if tc:
        ins = [F] + [DH] * (L - 1)
        w += planes(max([pack(B, 3 * H, 1) + pack(C, 3 * H, 1)] + [pack(3 * H, I, D) for I in ins]))
    return 4 * w


SIZE_CASES = {                                     # B, T, F, H, L, C, D
    "configs1": (512, 128, 64, 256, 2, 3, 2),
    "configs4": (256, 1024, 128, 512, 2, 3, 2),
    "l1": (64, 8, 16, 128, 1, 3, 2),
    "l3": (64, 8, 16, 256, 3, 3, 2),
    "l4": (64, 8, 16, 128, 4, 5, 2),
    "d1": (32, 8, 16, 256, 2, 3, 1),
    "f13": (32, 8, 13, 128, 2, 3, 2),
}


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("case", sorted(SIZE_CASES))
def test_infer_workspace_bytes_match_layout(pkg, case, prec):
    lib, C = pkg._lib.load(), pkg._lib.C
    B, T, F, H, L, Cn, D = SIZE_CASES[case]
    code = {"fp32": pkg._lib.PREC_FP32, "bf16": pkg._lib.PREC_BF16, "bf16x3": pkg._lib.PREC_BF16X3}[prec]
    h = C.c_void_p()
    rc = lib.bigru_plan_create(B, T, F, H, L, Cn, int(D == 2), code, C.byref(h))
    if prec == "bf16x3" and H == 512:
        assert rc == pkg._lib.ERR_UNSUPPORTED                 # hi/lo weight planes of H = 512 exceed shared memory
        return
    assert rc == 0
    try:
        got, st, sc = C.c_size_t(), C.c_size_t(), C.c_size_t()
        assert lib.bigru_infer_workspace_bytes(h, C.byref(got)) == 0
        assert got.value == infer_bytes(B, T, F, H, L, Cn, D, prec)
        assert lib.bigru_workspace_bytes(h, C.byref(st), C.byref(sc)) == 0
        assert got.value < st.value + sc.value
        if case == "configs1" and prec == "bf16x3":
            assert got.value < (st.value + sc.value) / 5
            assert abs(got.value / 1e9 - 0.69) < 0.01
    finally:
        lib.bigru_plan_destroy(h)


def test_infer_null_arguments_refused_before_launch(pkg):
    """Refused with ERR_ARG before anything is launched, so this holds with or without a device."""
    lib, C = pkg._lib.load(), pkg._lib.C
    h = C.c_void_p()
    assert lib.bigru_plan_create(32, 4, 8, 128, 1, 3, 1, pkg._lib.PREC_BF16X3, C.byref(h)) == 0
    try:
        dev = C.c_void_p(256)                                   # stands for a device pointer; never dereferenced
        assert lib.bigru_infer(h, dev, None, None, dev, dev, None) == pkg._lib.ERR_ARG                 # d_x
        assert b"null argument" in lib.bigru_last_error()
        assert lib.bigru_infer(h, dev, dev, None, None, dev, None) == pkg._lib.ERR_ARG                 # d_workspace
        assert lib.bigru_infer(h, None, dev, None, dev, dev, None) == pkg._lib.ERR_ARG                 # d_params
        assert lib.bigru_infer(h, dev, dev, None, dev, None, None) == pkg._lib.ERR_ARG                 # d_logits
        assert lib.bigru_infer(None, dev, dev, None, dev, dev, None) == pkg._lib.ERR_ARG
        assert lib.bigru_infer_workspace_bytes(h, None) == pkg._lib.ERR_ARG
    finally:
        lib.bigru_plan_destroy(h)


# ---------------------------------------------------------------------------------------------------------------- GPU
def _model(pkg, prec, H, F, C, L, D, dropout=0.0, seed=0):
    torch.manual_seed(seed)
    return pkg.BiGRU(H, F, C, L, 50, dropout, True, D == 2, precision=prec).cuda()


def _eval_forward(m, x, h=None):
    was = m.training
    m.eval()
    with torch.no_grad():
        out = m(x, h)
    m.train(was)
    return out


IDENTITY_CASES = {                                 # precision, B, T, F, H, L, D, with hidden
    "bf16x3_h128": ("bf16x3", 64, 16, 16, 128, 2, 2, False),
    "bf16x3_h256_l3_f13_hidden": ("bf16x3", 32, 12, 13, 256, 3, 2, True),
    "bf16x3_h8_ragged_l1": ("bf16x3", 37, 10, 13, 8, 1, 2, False),
    "bf16x3_h32_d1_hidden": ("bf16x3", 37, 10, 16, 32, 2, 1, True),
    "bf16_h128_l1": ("bf16", 48, 16, 16, 128, 1, 2, False),
    "bf16_h256_l3_d1_f13_ragged": ("bf16", 37, 12, 13, 256, 3, 1, False),
    "bf16_h512": ("bf16", 64, 6, 16, 512, 2, 2, False),
    "bf16_h32": ("bf16", 20, 9, 16, 32, 2, 2, False),
    "fp32_h32_l3_f13_ragged_hidden": ("fp32", 37, 10, 13, 32, 3, 2, True),
    "fp32_h8_d1": ("fp32", 5, 7, 16, 8, 2, 1, False),
    "fp32_h64_l1_hidden": ("fp32", 16, 9, 13, 64, 1, 2, True),
    "fp32_h128": ("fp32", 32, 8, 16, 128, 2, 2, False),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(IDENTITY_CASES))
def test_infer_bitwise_equals_eval_forward(pkg, case):
    prec, B, T, F, H, L, D, with_h = IDENTITY_CASES[case]
    m = _model(pkg, prec, H, F, 3, L, D, dropout=0.3)
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(B, T, F, device="cuda", generator=g)
    h = 0.5 * torch.randn(L * D, B, H, device="cuda", generator=g) if with_h else None
    m.train()                                                   # infer runs eval semantics whatever the mode
    got = m.infer(x, h)
    assert m.training
    assert not got.requires_grad and got.shape == (B, 3)
    want = _eval_forward(m, x, h)
    assert torch.equal(got, want), (got - want).abs().max().item()


@pytest.mark.gpu
def test_infer_bitwise_equals_eval_forward_configs1(pkg):
    """BASELINE configs[1] at full size: B512 T128 F64 H256 L2, bidirectional, bf16x3."""
    m = _model(pkg, "bf16x3", 256, 64, 3, 2, 2, dropout=0.2)
    x = torch.randn(512, 128, 64, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
    m.eval()
    got = m.infer(x)
    assert torch.equal(got, _eval_forward(m, x))


@pytest.mark.gpu
@pytest.mark.parametrize("prec,H,k", [("bf16x3", 128, 16), ("bf16", 128, 20), ("fp32", 32, 10)])
def test_infer_slices_bitwise_equal_whole_batch(pkg, prec, H, k):
    B, T, F, L, D = 37, 9, 13, 2, 2
    m = _model(pkg, prec, H, F, 4, L, D)
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(B, T, F, device="cuda", generator=g)
    whole = m.infer(x)
    assert torch.equal(m.infer(x, max_batch=k), whole)
    assert torch.equal(m.infer(x, max_batch=10 * B), whole)
    if prec != "bf16":
        h = 0.5 * torch.randn(L * D, B, H, device="cuda", generator=g)
        assert torch.equal(m.infer(x, h, max_batch=k), m.infer(x, h))
    with pytest.raises(ValueError):
        m.infer(x, max_batch=0)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", PRECS)
def test_infer_windows_bitwise_equal_forward_windows(pkg, prec):
    F, T, C, N = 13, 12, 4, 200
    H = 32 if prec == "fp32" else 128
    rng = np.random.default_rng(4)
    x_rows = torch.from_numpy(rng.normal(size=(N, F)).astype(np.float32))
    y_rows = torch.from_numpy((rng.uniform(size=(N, C)) > 0.5).astype(np.float32))
    norm = (x_rows.min(0, keepdim=True).values, x_rows.max(0, keepdim=True).values)
    ds = pkg.MySQLBatchLoader.from_tensors(x_rows.cuda(), y_rows.cuda(), norm, window=T)
    m = _model(pkg, prec, H, F, C, 2, 2, dropout=0.2)
    m.eval()
    want = m.forward_windows(ds, 5, 70)
    assert torch.equal(m.infer_windows(ds, 5, 70), want)
    assert torch.equal(m.infer_windows(ds, 5, 70, max_batch=32), want)
    with pytest.raises(ValueError):
        m.infer_windows(ds, 170, 32)                            # past the chunk, as forward_windows


@pytest.mark.gpu
def test_first_infer_allocates_only_the_inference_workspace(pkg):
    """configs[1] bf16x3 on a fresh model: nothing is padded (H = 256, B = 512 whole tiles), so the first infer may add the
    plan's inference workspace and the logits; 4 MB of slack covers the caching allocator's rounding."""
    m = _model(pkg, "bf16x3", 256, 64, 3, 2, 2)
    x = torch.randn(512, 128, 64, device="cuda")
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    logits = m.infer(x)
    torch.cuda.synchronize()
    rise = torch.cuda.max_memory_allocated() - base
    (plan,) = m._plans.values()
    assert rise <= plan.infer_bytes + logits.numel() * 4 + (4 << 20), (rise, plan.infer_bytes)
    assert rise < plan.stash_bytes and rise < plan.scratch_bytes
    assert plan._scratch is None and not plan._free_stash


def _trained(pkg, use_graph, with_infer, x, tgt):
    m = _model(pkg, "bf16x3", 128, 16, 3, 2, 2)
    m.use_cuda_graph = use_graph
    m.add_loss_fn(nn.CrossEntropyLoss())
    m.add_optimizer(torch.optim.Adam(m.parameters(), lr=1e-2))
    m.train()
    m.train_step(x, tgt)
    if with_infer:
        m.infer(x)
        m.infer(x[:7], max_batch=5)
    loss, logits = m.train_step(x, tgt)
    m.train_step(x, tgt)                                        # a graph replay when graphs are on
    torch.cuda.synchronize()
    return loss.clone(), logits.clone(), m.flat_parameters().detach().clone()


@pytest.mark.gpu
@pytest.mark.parametrize("use_graph", [True, False])
def test_infer_between_train_steps_changes_nothing(pkg, use_graph):
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn(64, 16, 16, device="cuda", generator=g)
    tgt = torch.randint(0, 3, (64,), device="cuda", generator=g)
    a = _trained(pkg, use_graph, False, x, tgt)
    b = _trained(pkg, use_graph, True, x, tgt)
    for u, v in zip(a, b):
        assert torch.equal(u, v)


@pytest.mark.gpu
def test_infer_between_forward_and_backward_changes_nothing(pkg):
    g = torch.Generator(device="cuda").manual_seed(6)
    x = torch.randn(37, 12, 16, device="cuda", generator=g)
    runs = []
    for with_infer in (False, True):
        m = _model(pkg, "bf16x3", 128, 16, 3, 2, 2)
        m.train()
        out = m(x)
        arg = m.pooled_argmax()
        if with_infer:
            m.infer(x)
            m.infer(x, max_batch=16)
            assert m.training
            assert torch.equal(m.pooled_argmax(), arg)
        (out * torch.arange(1, 4, device="cuda")).sum().backward()
        runs.append((out.detach(), m.pooled_argmax(), torch.cat([p.grad.reshape(-1) for p in m.parameters()])))
    for u, v in zip(*runs):
        assert torch.equal(u, v)


@pytest.mark.gpu
def test_infer_errors(pkg):
    with pytest.raises(RuntimeError):
        pkg.BiGRU(8, 4, 2, 1).infer(torch.zeros(2, 3, 4))            # CPU model: no CPU path
    m = pkg.BiGRU(8, 4, 2, 1).cuda()
    with pytest.raises(ValueError):
        m.infer(torch.zeros(2, 3, 5, device="cuda"))                  # wrong feature count
    with pytest.raises(RuntimeError):
        m.infer(torch.zeros(2, 3, 4, device="cuda"), torch.zeros(1, 2, 8, device="cuda"))   # wrong hidden shape
    mb = _model(pkg, "bf16", 128, 4, 2, 1, 2)
    with pytest.raises(ValueError):
        mb.infer(torch.zeros(16, 3, 4, device="cuda"), torch.zeros(2, 16, 128, device="cuda"))   # no initial state at bf16
