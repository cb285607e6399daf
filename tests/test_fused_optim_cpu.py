"""CPU checks of the fused step's optimizer and loss coverage: which losses and optimizers fuse, the per-tensor segment
table against the flat vector's views, the graph key without optimizer hyperparameters, and the fp64 references of
tests/fused_optim_ref.py against torch in float64."""
import numpy as np
import pytest
import torch
import torch.nn as nn

import fused_optim_ref as ref
from financial_market_data_analysis_b200 import BiGRU, _lib


def _model(H=8, F=5, C=3, L=2, **kw):
    return BiGRU(H, F, C, L, 50, 0.0, False, True, **kw)


def _decay_groups(m):
    """Two groups the usual way: weights with decay, biases without."""
    decay = [p for n, p in m.named_parameters() if "bias" not in n]
    no_decay = [p for n, p in m.named_parameters() if "bias" in n]
    return [{"params": decay, "weight_decay": 0.05}, {"params": no_decay, "weight_decay": 0.0}]


def test_which_losses_fuse():
    C = 3
    m = _model(C=C)
    m.add_optimizer(torch.optim.Adam(m.parameters()))
    w = torch.tensor([0.5, 1.0, 3.0])
    fuse = [(nn.CrossEntropyLoss(), _lib.LOSS_CE, 0.0), (nn.CrossEntropyLoss(weight=w), _lib.LOSS_CE_WEIGHTED, 0.0),
            (nn.BCEWithLogitsLoss(weight=w), _lib.LOSS_BCE, 0.0), (nn.MultiLabelSoftMarginLoss(), _lib.LOSS_MLSM, 0.0),
            (nn.MSELoss(), _lib.LOSS_MSE, 0.0), (nn.L1Loss(), _lib.LOSS_L1, 0.0),
            (nn.SmoothL1Loss(), _lib.LOSS_SMOOTH_L1, 1.0), (nn.SmoothL1Loss(beta=0.0), _lib.LOSS_SMOOTH_L1, 0.0),
            (nn.SmoothL1Loss(beta=0.25), _lib.LOSS_SMOOTH_L1, 0.25), (nn.HuberLoss(delta=2.5), _lib.LOSS_HUBER, 2.5)]
    for fn, kind, param in fuse:
        m.add_loss_fn(fn)
        spec = m._loss_spec()
        assert spec is not None and spec[0] == kind and spec[3] == param and m.can_fuse_step(), fn
    assert m._loss_spec()[0] == _lib.LOSS_HUBER
    m.add_loss_fn(nn.CrossEntropyLoss(weight=w))
    assert m._loss_spec()[1] is w
    refuse = [nn.CrossEntropyLoss(label_smoothing=0.1), nn.CrossEntropyLoss(weight=w, label_smoothing=0.1),
              nn.CrossEntropyLoss(reduction="sum"), nn.CrossEntropyLoss(weight=w, reduction="none"),
              nn.CrossEntropyLoss(weight=w, ignore_index=1), nn.CrossEntropyLoss(weight=torch.ones(C + 1)),
              nn.CrossEntropyLoss(weight=torch.ones(1, C)), nn.BCEWithLogitsLoss(weight=w.reshape(C, 1)),
              nn.BCEWithLogitsLoss(weight=torch.rand(4, C)), nn.MSELoss(reduction="sum"), nn.L1Loss(reduction="none"),
              nn.SmoothL1Loss(reduction="sum"), nn.HuberLoss(reduction="sum"), nn.NLLLoss(), nn.KLDivLoss()]
    for fn in refuse:
        m.add_loss_fn(fn)
        assert m._loss_spec() is None and not m.can_fuse_step(), fn


def test_which_optimizers_fuse():
    m = _model()
    m.add_loss_fn(nn.CrossEntropyLoss())
    ps = list(m.parameters())
    fuse = [torch.optim.Adam(ps), torch.optim.AdamW(ps), torch.optim.Adam(ps, weight_decay=0.1),
            torch.optim.AdamW(_decay_groups(m)), torch.optim.Adam(_decay_groups(m), lr=3e-4),
            torch.optim.AdamW([{"params": [p]} for p in ps], lr=1e-3)]
    for opt in fuse:
        m.add_optimizer(opt)
        assert m._adam_spec() is opt.param_groups and m.can_fuse_step(), opt
    other = nn.Parameter(torch.zeros(3))
    refuse = [torch.optim.SGD(ps, lr=0.1), torch.optim.Adam(ps, amsgrad=True), torch.optim.AdamW(ps, maximize=True),
              torch.optim.AdamW([{"params": ps[:3]}, {"params": ps[3:], "amsgrad": True}]), torch.optim.Adam(ps[1:]),
              torch.optim.Adam([{"params": ps}, {"params": [other]}]), torch.optim.RMSprop(ps), torch.optim.Adagrad(ps),
              torch.optim.AdamW([{"params": [p]} for p in ps] + [{"params": [nn.Parameter(torch.zeros(1))]}
                                                                 for _ in range(_lib.ADAM_MAX_GROUPS)])]
    for opt in refuse:
        m.add_optimizer(opt)
        assert m._adam_spec() is None and not m.can_fuse_step(), opt
    m.add_optimizer(None)
    assert not m.can_fuse_step()


@pytest.mark.parametrize("H,F,L,bidir,prec", [(8, 5, 2, True, "auto"), (33, 7, 3, True, "bf16x3"), (7, 3, 2, False, "bf16"),
                                              (300, 9, 2, True, "fp32"), (256, 64, 2, True, "bf16x3")])
def test_segment_table_matches_the_flat_views(H, F, L, bidir, prec):
    """One (offset, count, group) row per tensor of _ordered_params, in order, covering the flat vector exactly once,
    whether or not the plan pads hidden units (the update runs on the unpadded flat vector)."""
    m = BiGRU(H, F, 3, L, 50, 0.0, False, bidir, precision=prec)
    opt = torch.optim.AdamW(_decay_groups(m), lr=2e-3, betas=(0.8, 0.95), eps=1e-7)
    opt.param_groups[1]["lr"] = 5e-4
    m.add_optimizer(opt)
    hyper, segs = m._adam_tables(m._adam_spec())
    assert len(segs) == len(m._views) == len(m._ordered_params()) == 4 * L * (2 if bidir else 1) + 2
    off = 0
    for (o, n, k), (vo, vn, _), p in zip(segs, m._views, m._ordered_params()):
        assert (o, n) == (vo, vn) == (off, p.numel())
        is_bias = p.dim() == 1
        assert k == (1 if is_bias else 0)
        off += n
    assert off == m.flat_parameters().numel()
    assert hyper == ((2e-3, 0.8, 0.95, 1e-7, 0.05, 1.0), (5e-4, 0.8, 0.95, 1e-7, 0.0, 1.0))
    m.add_optimizer(torch.optim.Adam(m.parameters(), lr=1e-3, weight_decay=0.1))
    hyper, segs = m._adam_tables(m._adam_spec())
    assert hyper == ((1e-3, 0.9, 0.999, 1e-8, 0.1, 0.0),) and {k for _, _, k in segs} == {0}


def test_graph_key_holds_no_optimizer_hyperparameter():
    m = _model()
    w = torch.ones(3)
    opt = torch.optim.AdamW(_decay_groups(m), lr=1e-3)
    m.add_optimizer(opt)
    dev = torch.device("cpu")
    loss = (_lib.LOSS_CE_WEIGHTED, w, None, 1.0, 0.0)
    key = m._graph_key(32, 12, loss, len(opt.param_groups), dev, True)
    for g in opt.param_groups:
        g.update(lr=7e-2, betas=(0.5, 0.6), eps=1e-3, weight_decay=0.3)
    assert m._graph_key(32, 12, loss, len(opt.param_groups), dev, True) == key
    assert 1e-3 not in key and 7e-2 not in key and key[-1] is True
    assert m._graph_key(32, 12, loss, len(opt.param_groups), dev, False)[-1] is False
    m.clip = 5.0
    assert m._graph_key(32, 12, loss, len(opt.param_groups), dev, True) != key


# ---- the fp64 references against torch in float64 ------------------------------------------------------------------
def _torch_loss(fn, x, t):
    x = torch.from_numpy(x).requires_grad_(True)
    v = fn(x, torch.from_numpy(t))
    v.backward()
    return v.item(), x.grad.numpy()


@pytest.mark.parametrize("B,C", [(1, 1), (1, 3), (7, 1), (300, 4)])
def test_loss_references_match_torch_float64(B, C):
    rng = np.random.default_rng([B, C])
    x = rng.standard_normal((B, C)) * 3
    # regressions: targets at the kinks of each loss (x - y in {0, +-beta, +-delta}) and away from them
    y = x - rng.choice([0.0, 0.5, -0.5, 2.0, -2.0, 1.7], (B, C))
    for kind, fn, param in ((ref.MSE, nn.MSELoss(), 0.0), (ref.L1, nn.L1Loss(), 0.0),
                            (ref.SMOOTH_L1, nn.SmoothL1Loss(beta=0.5), 0.5), (ref.SMOOTH_L1, nn.SmoothL1Loss(beta=0.0), 0.0),
                            (ref.SMOOTH_L1, nn.SmoothL1Loss(beta=2.0), 2.0), (ref.HUBER, nn.HuberLoss(delta=0.5), 0.5),
                            (ref.HUBER, nn.HuberLoss(delta=2.0), 2.0)):
        tv, tg = _torch_loss(fn, x, y)
        rv, rg = ref.loss(kind, x, y, param=param, denom=B * C)
        assert rv == pytest.approx(tv, rel=1e-12, abs=1e-15), (kind, param)
        np.testing.assert_allclose(rg, tg, rtol=1e-12, atol=1e-15, err_msg=str((kind, param)))
    t = rng.integers(0, C, B)
    for w in (rng.uniform(0.5, 2.0, C), np.where(np.arange(C) % 2 == 0, 0.0, 1.5)):
        if w[t].sum() == 0:
            continue
        tv, tg = _torch_loss(nn.CrossEntropyLoss(weight=torch.from_numpy(w)), x, t)
        rv, rg = ref.loss(ref.CE_WEIGHTED, x, t, w)
        assert rv == pytest.approx(tv, rel=1e-12)
        np.testing.assert_allclose(rg, tg, rtol=1e-12, atol=1e-15)
    zero = np.zeros(C)
    tv, _ = _torch_loss(nn.CrossEntropyLoss(weight=torch.from_numpy(zero)), x, t)
    assert np.isnan(tv) and np.isnan(ref.loss(ref.CE_WEIGHTED, x, t, zero)[0])


@pytest.mark.parametrize("opt_cls", [torch.optim.Adam, torch.optim.AdamW])
@pytest.mark.parametrize("clip", [1e3, 0.05])
def test_grouped_update_reference_matches_torch_float64(opt_cls, clip):
    """Three steps of clip_grad_norm_ + Adam / AdamW over three groups (one without decay, two with their own lr and
    betas) in float64, against the reference fed the same gradients."""
    rng = np.random.default_rng(5)
    sizes = (40, 7, 13, 5)
    ps = [nn.Parameter(torch.from_numpy(rng.standard_normal(n))) for n in sizes]
    groups = [dict(params=[ps[0], ps[2]], lr=1e-2, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.1),
              dict(params=[ps[1]], lr=3e-3, betas=(0.8, 0.95), eps=1e-6, weight_decay=0.0),
              dict(params=[ps[3]], lr=5e-2, betas=(0.5, 0.9), eps=1e-7, weight_decay=0.3)]
    opt = opt_cls(groups, foreach=False)
    table = [(g["lr"], *g["betas"], g["eps"], g["weight_decay"], float(opt_cls is torch.optim.AdamW)) for g in groups]
    offs = np.cumsum((0,) + sizes)
    segs = [(int(offs[0]), sizes[0], 0), (int(offs[1]), sizes[1], 1), (int(offs[2]), sizes[2], 0), (int(offs[3]), sizes[3], 2)]
    n = int(offs[-1])
    p = np.concatenate([q.detach().numpy() for q in ps])
    m, v = np.zeros(n), np.zeros(n)
    for step in (1, 2, 3):
        g = rng.standard_normal(n)
        for q, o, k in zip(ps, offs, sizes):
            q.grad = torch.from_numpy(g[o:o + k].copy())
        nn.utils.clip_grad_norm_(ps, clip)
        opt.step()
        p, gq, m, v, norm = ref.clip_adam_groups(p, g, m, v, clip, table, segs, step)
        assert norm == pytest.approx(np.linalg.norm(g), rel=1e-14)
        for q, o, k in zip(ps, offs, sizes):
            st = opt.state[q]
            np.testing.assert_allclose(p[o:o + k], q.detach().numpy(), rtol=1e-13, atol=1e-15)
            np.testing.assert_allclose(gq[o:o + k], q.grad.numpy(), rtol=1e-14, atol=0)
            np.testing.assert_allclose(m[o:o + k], st["exp_avg"].numpy(), rtol=1e-13, atol=1e-16)
            np.testing.assert_allclose(v[o:o + k], st["exp_avg_sq"].numpy(), rtol=1e-13, atol=1e-18)
