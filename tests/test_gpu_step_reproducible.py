"""Bit-reproducibility of the tensor-core paths at the benchmark shape (BASELINE configs[1]: B512 T128 F64 H256 L2,
bidirectional).  Every cross-block sum of a step runs in a fixed order (split-K partials, bias column sums, loss, gradient
norm), so two identically seeded models fed the same inputs must agree bit for bit.
Run on an H100:  python -m pytest tests/test_gpu_step_reproducible.py -m gpu -q"""
import os
import sys

import pytest
import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import financial_market_data_analysis_b200 as pkg  # noqa: E402

pytestmark = pytest.mark.gpu

B, T, F, H, L, C = 512, 128, 64, 256, 2, 3


def _model(precision):
    torch.manual_seed(0)
    m = pkg.BiGRU(H, F, C, L, 50, 0.0, False, True, precision=precision).cuda()
    m.add_loss_fn(nn.CrossEntropyLoss())
    m.add_optimizer(torch.optim.Adam(m.parameters(), lr=1e-3))
    return m.train()


def _inputs():
    g = torch.Generator().manual_seed(1234)
    x = torch.randn(B, T, F, generator=g).cuda()
    y = torch.randint(0, C, (B,), generator=g).cuda()
    return x, y


def _same(a, b):
    return torch.equal(a.detach().cpu(), b.detach().cpu())


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
def test_train_steps_bit_identical(precision):
    x, y = _inputs()
    runs = []
    for _ in range(2):
        m = _model(precision)
        assert m.resolved_precision(B) == precision
        steps = [m.train_step(x, y) for _ in range(2)]
        torch.cuda.synchronize()
        runs.append(([(loss.clone(), logits.clone()) for loss, logits in steps], m.flat_parameters().clone()))
        del m
    for (l0, g0), (l1, g1) in zip(runs[0][0], runs[1][0]):
        assert _same(l0, l1), (float(l0), float(l1))
        assert _same(g0, g1)
    assert _same(runs[0][1], runs[1][1])


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
def test_forward_backward_bit_identical(precision):
    x, y = _inputs()
    outs = []
    for _ in range(2):
        m = _model(precision)
        logits = m(x)
        nn.functional.cross_entropy(logits, y).backward()
        grads = torch.cat([p.grad.reshape(-1) for p in m.parameters()])
        torch.cuda.synchronize()
        outs.append((logits.detach().clone(), grads.clone()))
        del m
    assert _same(outs[0][0], outs[1][0])
    assert _same(outs[0][1], outs[1][1])
