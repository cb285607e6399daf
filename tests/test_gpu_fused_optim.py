"""The fused train step with AdamW, parameter groups, learning-rate schedules, weighted cross-entropy and regression
losses, on the GPU.

- bigru_loss_param against the fp64 references of fused_optim_ref.py: weighted CE (weights with zeros, all target weights
  zero), MSE, L1, SmoothL1 (beta 0 and > 0) and Huber, at B = 1, B below, at and above the kernel's 256 threads, C = 1,
  targets exactly at each loss's kinks, N(0,1) and +-1e4 logits; the old kinds through bigru_loss_param bitwise as
  bigru_loss.
- bigru_clip_adam_groups_dev against fused_optim_ref.clip_adam_groups element by element: one and several groups, weight
  decay 0 and > 0, decoupled and coupled, clipping inactive and binding, at the vector lengths on both sides of the
  sqnorm and update grid edges; bigru_clip_adam_step_dev bitwise equal to the grouped entry with one group.
- BiGRU.train_step with AdamW (two groups, biases without decay) and CrossEntropyLoss(weight=...) against the same model
  under _generic_step (torch's autograd loss, clip_grad_norm_ and AdamW), at fp32 and bf16x3.
- 20 steps under CosineAnnealingLR and OneCycleLR (which also cycles beta1): CUDA graph on and off bitwise equal, one
  captured graph.
- A checkpoint of an AdamW fused run resumes bit for bit, and the generic step continues from it.

Tolerances are scale-free (error over the magnitude of what the kernel adds up).  BIGRU_FUSED_OPTIM_REPORT=path.jsonl
appends every measured value to that file.

Run on an H100:  python -m pytest tests/test_gpu_fused_optim.py -m gpu -q"""
import copy
import json
import os
import warnings

import numpy as np
import pytest
import torch
import torch.nn as nn

import fused_optim_ref as ref

pytestmark = pytest.mark.gpu

# about 4x the worst value measured on an H100 80GB HBM3 (700 W power limit, 1980 MHz max SM clock):
#   loss 1.6e-7   dlogits 7.9e-8   g 1.9e-7   m 2.7e-7   v 4.4e-7   p 1.8e-6 (coupled weight decay, clipping binding)
#   end to end: parameters 1.1e-6, their change over five steps 7.3e-6
TOL = {"loss": 7e-7, "dlogits": 3.2e-7, "g": 8e-7, "m": 1.1e-6, "v": 1.8e-6, "p": 7.5e-6,
       "e2e_params": 5e-6, "e2e_change": 3e-5}


def _L():
    from financial_market_data_analysis_b200 import _lib
    return _lib


def _st():
    return torch.cuda.current_stream().cuda_stream


def _scaled(k, r, mag, slack=0.0):
    """max (|k - r| - slack) / mag; where mag is 0 the two must agree within slack.  NaN anywhere gives NaN."""
    k, r = np.asarray(k, np.float64), np.asarray(r, np.float64)
    d = np.maximum(np.abs(k - r) - slack, 0.0)
    mag = np.broadcast_to(np.asarray(mag, np.float64), d.shape)
    if np.isnan(d).any():
        return float("nan")
    z = mag == 0
    if (d[z] != 0).any():
        return float("inf")
    return float((d[~z] / mag[~z]).max()) if (~z).any() else 0.0


class _Checks:
    def __init__(self, test):
        self.test, self.rows, self.bad = test, [], []

    def __call__(self, cls, err, **ctx):
        self.rows.append(dict(test=self.test, cls=cls, err=err, **ctx))
        if not err <= TOL[cls]:
            self.bad.append((cls, err, TOL[cls], ctx))

    def done(self):
        out = os.environ.get("BIGRU_FUSED_OPTIM_REPORT")
        if out:
            with open(out, "a") as f:
                for r in self.rows:
                    f.write(json.dumps(r) + "\n")
        assert not self.bad, (len(self.bad), self.bad[:8])


# ---- losses ---------------------------------------------------------------------------------------------------------
LOSS_B = (1, 31, 256, 257, 1000)
LOSS_C = (1, 3, 33)
KINDS = {"ce_weighted": (ref.CE_WEIGHTED, 0.0), "mse": (ref.MSE, 0.0), "l1": (ref.L1, 0.0),
         "smooth_l1": (ref.SMOOTH_L1, 0.5), "smooth_l1_beta0": (ref.SMOOTH_L1, 0.0), "huber": (ref.HUBER, 0.25),
         "huber_wide": (ref.HUBER, 4.0)}


def _kernel_loss(kind, lg, tg, w, param, denom, old=False):
    L = _L()
    lib = L.load()
    dev = torch.device("cuda")
    lgd, tgd = torch.from_numpy(lg).to(dev), torch.from_numpy(tg).to(dev)
    wd = None if w is None else torch.from_numpy(w).to(dev)
    loss = torch.full((1,), 7.0, device=dev)
    dl = torch.full(lg.shape, 5.0, device=dev)
    if old:
        L.check(lib.bigru_loss(kind, L.ptr(lgd), L.ptr(tgd), L.ptr(wd), None, lg.shape[0], lg.shape[1], denom, L.ptr(loss),
                               L.ptr(dl), _st()), "bigru_loss")
    else:
        L.check(lib.bigru_loss_param(kind, L.ptr(lgd), L.ptr(tgd), L.ptr(wd), None, lg.shape[0], lg.shape[1], denom, param,
                                     L.ptr(loss), L.ptr(dl), _st()), "bigru_loss_param")
    return loss.item(), dl.cpu().numpy()


def _loss_inputs(name, fam, B, C_):
    rng = np.random.default_rng([B, C_, list(KINDS).index(name), fam == "1e4"])
    if fam == "1e4":
        lg = rng.choice([-1.0, 1.0], (B, C_)) * 1e4 * rng.uniform(0.5, 1.0, (B, C_))
    else:
        lg = rng.standard_normal((B, C_))
    kind, param = KINDS[name]
    if kind == ref.CE_WEIGHTED:
        w = rng.uniform(0.25, 3.0, C_).astype(np.float32)
        if C_ > 1:
            w[0] = 0.0                                          # a class of weight 0
        tg = rng.integers(0, C_, B).astype(np.int64)
        if C_ > 1:
            tg[-1] = C_ - 1                                     # the weight sum is never zero
            if B > 1:
                tg[0] = 0
        return lg.astype(np.float32), tg, w
    # logits and differences on a 1/64 grid so that x - y is exact in fp32: the kinks are hit exactly
    lg = np.round(lg * 64) / 64
    kinks = np.array([0.0, param, -param, 1.0, -1.0, 0.015625, 3.5], np.float64)
    diff = np.where(rng.random((B, C_)) < 0.5, rng.choice(kinks, (B, C_)), np.round(rng.standard_normal((B, C_)) * 64) / 64)
    return lg.astype(np.float32), (lg - diff).astype(np.float32), None


@pytest.mark.parametrize("B", LOSS_B)
@pytest.mark.parametrize("name", list(KINDS))
def test_loss_param_matches_fp64_reference(name, B):
    kind, param = KINDS[name]
    chk = _Checks(f"loss[{name}-{B}]")
    for C_ in LOSS_C:
        for fam in ("normal", "1e4"):
            lg, tg, w = _loss_inputs(name, fam, B, C_)
            for world in (1, 4):
                if kind == ref.CE_WEIGHTED:
                    denom = float(world)
                    ok = tg >= 0
                    wy = w.astype(np.float64)[tg]
                    row = 1.0 + np.abs(lg.astype(np.float64)).max(1, keepdims=True)
                    W = wy.sum()
                    lmag = (wy[:, None] * row).sum() / (W * denom)
                    dscale = np.broadcast_to(wy[:, None] * row / (W * denom), lg.shape)
                    assert ok.all()
                else:
                    denom = float(B * C_ * world)
                    x, y = lg.astype(np.float64), tg.astype(np.float64)
                    sc = np.abs(x) + np.abs(y)
                    lmag = (sc * sc / (param if kind == ref.SMOOTH_L1 and 0 < param < 1 else 1.0) + sc + 1.0 + param).sum() / denom
                    dscale = (2.0 * sc / (param if kind == ref.SMOOTH_L1 and param > 0 else 1.0) + 1.0 + param) / denom
                got, dl = _kernel_loss(kind, lg, tg, w, param, denom)
                want, dwant = ref.loss(kind, lg, tg, w, param, denom)
                ctx = dict(C=C_, fam=fam, world=world)
                chk("loss", abs(got - want) / lmag, **ctx)
                chk("dlogits", _scaled(dl, dwant, dscale), **ctx)
                if kind != ref.CE_WEIGHTED:                     # torch's gradient at the kinks, exactly (times fp32 1/denom)
                    d = lg.astype(np.float64) - tg.astype(np.float64)
                    at = (d == 0) | (np.abs(d) == param)
                    exact = (dwant[at] * denom).astype(np.float32) * np.float32(1.0 / denom)
                    if at.any() and (dl[at] != exact).any():
                        chk.bad.append(("kink gradient", name, ctx))
    chk.done()


def test_weighted_ce_with_every_target_weight_zero_is_nan():
    lg = np.random.default_rng(1).standard_normal((5, 3)).astype(np.float32)
    tg = np.array([0, 0, 2, 2, 0], np.int64)
    w = np.array([0.0, 1.0, 0.0], np.float32)
    loss, dl = _kernel_loss(ref.CE_WEIGHTED, lg, tg, w, 0.0, 1.0)
    assert np.isnan(loss) and np.isnan(dl).all()


@pytest.mark.parametrize("kind", [0, 1, 2])
def test_old_kinds_through_loss_param_are_bitwise_bigru_loss(kind):
    rng = np.random.default_rng(kind)
    B, C_ = 257, 5
    lg = (3 * rng.standard_normal((B, C_))).astype(np.float32)
    tg = rng.integers(0, C_, B).astype(np.int64) if kind == 0 else (rng.random((B, C_)) < 0.4).astype(np.float32)
    w = rng.uniform(0.5, 2, C_).astype(np.float32)
    a = _kernel_loss(kind, lg, tg, w, 0.0, float(B * C_), old=True)
    b = _kernel_loss(kind, lg, tg, w, 0.75, float(B * C_))
    assert np.float32(a[0]).tobytes() == np.float32(b[0]).tobytes() and a[1].tobytes() == b[1].tobytes()


# ---- the grouped update ---------------------------------------------------------------------------------------------
UPDATE_N = (1, 257, 8193, 135169, 270337, 300001)
GROUP_SETS = {
    "one_adam": [(1e-3, 0.9, 0.999, 1e-8, 0.0, 0.0)],
    "one_adamw": [(3e-3, 0.8, 0.95, 1e-6, 0.1, 1.0)],
    "one_adam_l2": [(2e-3, 0.9, 0.99, 1e-7, 0.05, 0.0)],
    "mixed": [(1e-3, 0.9, 0.999, 1e-8, 0.01, 1.0), (5e-4, 0.85, 0.99, 1e-7, 0.0, 1.0), (2e-2, 0.5, 0.9, 1e-6, 0.2, 0.0)],
}
CLIP = {"inactive": 4.0, "binding": 0.3}


def _segments(n, G, rng):
    """Ranges of random lengths tiling [0, n), groups cycling over G (so that every group appears, unless n is tiny)."""
    cuts = np.unique(np.concatenate([[0, n], rng.integers(1, n, min(n - 1, 9)) if n > 1 else []])).astype(np.int64)
    return [(int(a), int(b - a), k % G) for k, (a, b) in enumerate(zip(cuts[:-1], cuts[1:]))]


def _kernel_groups(p, g, m, v, clip, groups, segs, step, legacy=False):
    L = _L()
    lib = L.load()
    dev = torch.device("cuda")
    pd, gd, md, vd = (torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (p, g, m, v))
    sq = torch.full((1,), 123.0, device=dev)
    ws = torch.full((L.SQNORM_WS,), float("nan"), device=dev)
    dstep = torch.full((1,), step - 1, dtype=torch.int32, device=dev)
    n = p.size
    L.check(lib.bigru_adam_tick(L.ptr(dstep), L.ptr(sq), _st()), "bigru_adam_tick")
    L.check(lib.bigru_sqnorm(L.ptr(gd), n, L.ptr(sq), L.ptr(ws), _st()), "bigru_sqnorm")
    if legacy:
        lr, b1, b2, eps, _, _ = groups[0]
        L.check(lib.bigru_clip_adam_step_dev(L.ptr(pd), L.ptr(gd), L.ptr(md), L.ptr(vd), n, L.ptr(sq), clip, lr, b1, b2, eps,
                                             L.ptr(dstep), 1.0, _st()), "bigru_clip_adam_step_dev")
    else:
        hd = torch.tensor(groups, dtype=torch.float32, device=dev)
        sd = torch.tensor(segs, dtype=torch.int64, device=dev)
        L.check(lib.bigru_clip_adam_groups_dev(L.ptr(pd), L.ptr(gd), L.ptr(md), L.ptr(vd), n, L.ptr(sq), clip, L.ptr(hd),
                                               len(groups), L.ptr(sd), len(segs), L.ptr(dstep), 1.0, _st()),
                "bigru_clip_adam_groups_dev")
    return tuple(t.cpu().numpy() for t in (pd, gd, md, vd))


def _f32_groups(groups):
    return [tuple(float(np.float32(x)) for x in g) for g in groups]


@pytest.mark.parametrize("clip_kind", list(CLIP))
@pytest.mark.parametrize("gset", list(GROUP_SETS))
@pytest.mark.parametrize("n", UPDATE_N)
def test_grouped_update_matches_fp64_reference(n, gset, clip_kind):
    groups = _f32_groups(GROUP_SETS[gset])
    rng = np.random.default_rng([n, list(GROUP_SETS).index(gset), list(CLIP).index(clip_kind)])
    segs = _segments(n, len(groups), rng)
    chk = _Checks(f"groups[{n}-{gset}-{clip_kind}]")
    g = (1e-3 * rng.standard_normal(n)).astype(np.float32)
    g[np.arange(n) % 7 == 3] = 0.0
    clip = float(np.float32(CLIP[clip_kind] * np.linalg.norm(g.astype(np.float64))))
    p = (1e-2 * rng.standard_normal(n)).astype(np.float32)
    m = (1e-3 * rng.standard_normal(n)).astype(np.float32)
    v = ((1e-3 * rng.standard_normal(n)) ** 2).astype(np.float32)
    for step in (1, 10):
        got = _kernel_groups(p, g, m, v, clip, groups, segs, step)
        pr, gr, mr, vr, _ = ref.clip_adam_groups(p, g, m, v, clip, groups, segs, step)
        # per element: the group's hyperparameters, and magnitudes of what each quantity adds up
        b1, b2, lr, eps, wd, dec = (np.empty(n) for _ in range(6))
        for off, cnt, k in segs:
            lr[off:off + cnt], b1[off:off + cnt], b2[off:off + cnt], eps[off:off + cnt], wd[off:off + cnt], dec[off:off + cnt] = groups[k]
        ge = np.abs(gr) + np.where(dec == 0, wd * np.abs(p), 0.0)
        m_mag = b1 * np.abs(m) + (1 - b1) * ge
        v_mag = b2 * v + (1 - b2) * ge * ge + np.finfo(np.float32).tiny
        p_mag = lr / (1 - b1 ** step) * m_mag / (np.sqrt(vr / (1 - b2 ** step)) + eps)
        slack = 2 * np.spacing(np.abs(pr).astype(np.float32)).astype(np.float64)
        ctx = dict(step=step)
        chk("g", _scaled(got[1], gr, np.abs(gr)), **ctx)
        chk("m", _scaled(got[2], mr, m_mag), **ctx)
        chk("v", _scaled(got[3], vr, v_mag), **ctx)
        chk("p", _scaled(got[0], pr, p_mag, slack), **ctx)
    chk.done()


@pytest.mark.parametrize("n", (1, 257, 270337, 300001))
def test_clip_adam_step_dev_is_the_grouped_update_with_one_group(n):
    """Bit for bit: the legacy entry point, the grouped one with one segment, and the grouped one with the same
    hyperparameters split over several segments and identical groups."""
    rng = np.random.default_rng(n)
    g = (1e-3 * rng.standard_normal(n)).astype(np.float32)
    p = (1e-2 * rng.standard_normal(n)).astype(np.float32)
    m = (1e-3 * rng.standard_normal(n)).astype(np.float32)
    v = ((1e-3 * rng.standard_normal(n)) ** 2).astype(np.float32)
    one = _f32_groups([(2e-3, 0.85, 0.99, 1e-7, 0.0, 0.0)])
    for clip in (1e3, 0.3 * float(np.linalg.norm(g))):
        clip = float(np.float32(clip))
        for step in (1, 7):
            a = _kernel_groups(p, g, m, v, clip, one, None, step, legacy=True)
            b = _kernel_groups(p, g, m, v, clip, one, [(0, n, 0)], step)
            c = _kernel_groups(p, g, m, v, clip, one * 3, _segments(n, 3, rng), step)
            for x, y, z in zip(a, b, c):
                assert x.tobytes() == y.tobytes() == z.tobytes()


# ---- the fused step end to end --------------------------------------------------------------------------------------
def _decay_groups(m, **kw):
    decay = [p for n, p in m.named_parameters() if "bias" not in n]
    no_decay = [p for n, p in m.named_parameters() if "bias" in n]
    return [{"params": decay, "weight_decay": 0.05, **kw}, {"params": no_decay, "weight_decay": 0.0, **kw}]


def _model(prec, H=128, F=16, C=3, L=2, clip=1.0):
    from financial_market_data_analysis_b200 import BiGRU
    torch.manual_seed(7)
    return BiGRU(H, F, C, L, clip, 0.0, False, True, precision=prec).cuda().train()


def _batches(k, B=64, T=12, F=16, C=3, seed=3):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(B, T, F, generator=g).cuda(), torch.randint(0, C, (B,), generator=g).cuda()) for _ in range(k)]


@pytest.mark.parametrize("prec", ["fp32", "bf16x3"])
def test_fused_adamw_weighted_ce_matches_generic_step(prec):
    """Five steps: the fused step against autograd + torch's CrossEntropyLoss(weight=), clip_grad_norm_ (clip binding) and
    AdamW over two groups.  Both run the same forward / backward kernels; they differ in the loss, clip and update
    arithmetic (torch forms 1 - beta2 in double, the kernel in fp32): relative L2 of the parameters and of their change
    over the five steps."""
    w = torch.tensor([0.3, 1.0, 2.5], device="cuda")
    data = _batches(5)
    out = []
    for fused in (True, False):
        m = _model(prec)
        p0 = m.flat_parameters().clone()
        m.add_loss_fn(nn.CrossEntropyLoss(weight=w))
        m.add_optimizer(torch.optim.AdamW(_decay_groups(m), lr=3e-3))
        assert m.can_fuse_step()
        for x, y in data:
            m.train_step(x, y) if fused else m._generic_step(x, y)
        out.append((m.flat_parameters().clone() - p0, m.flat_parameters().clone()))
    chk = _Checks(f"e2e[{prec}]")
    rel = lambda a, b: float((a - b).norm() / b.norm())                     # noqa: E731
    chk("e2e_params", rel(out[0][1], out[1][1]))
    chk("e2e_change", rel(out[0][0], out[1][0]))
    chk.done()


@pytest.mark.parametrize("sched", ["cosine", "onecycle"])
def test_schedule_replays_one_graph_bitwise_as_plain_launches(sched):
    """20 steps under a scheduler stepped between train_step calls: CUDA graph on and off give bitwise equal
    parameters and moments, and the graph run captured one graph.  OneCycleLR also cycles beta1."""
    data = _batches(20, B=48)
    res = []
    for graph in (True, False):
        m = _model("bf16x3")
        m.use_cuda_graph = graph
        m.add_loss_fn(nn.CrossEntropyLoss(weight=torch.tensor([0.5, 1.0, 2.0], device="cuda")))
        opt = torch.optim.AdamW(_decay_groups(m), lr=2e-3)
        m.add_optimizer(opt)
        s = (torch.optim.lr_scheduler.CosineAnnealingLR(opt, T_max=20) if sched == "cosine" else
             torch.optim.lr_scheduler.OneCycleLR(opt, max_lr=1e-2, total_steps=20))
        lrs = []
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            for x, y in data:
                m.train_step(x, y)
                lrs.append(opt.param_groups[0]["lr"])
                s.step()
        # the fused step is the optimizer's step: the scheduler sees it as one
        assert not [w for w in caught if "lr_scheduler.step()" in str(w.message)]
        assert len(set(lrs)) > 10
        if graph:
            assert len(m._graphs) == 1
        else:
            assert not m._graphs
        res.append([t.clone() for t in (m.flat_parameters(), m._adam.m, m._adam.v)])
    for a, b in zip(*res):
        assert torch.equal(a, b)


def test_adamw_checkpoint_resumes_bitwise_and_the_generic_step_continues():
    data = _batches(6)
    w = torch.tensor([0.5, 1.0, 2.0], device="cuda")

    def fresh(state=None):
        m = _model("fp32", H=32)
        m.add_loss_fn(nn.CrossEntropyLoss(weight=w))                       # a submodule: its weight is in state_dict
        if state is not None:
            m.load_state_dict(state)
        m.add_optimizer(torch.optim.AdamW(_decay_groups(m), lr=5e-3))
        return m

    m1 = fresh()
    for x, y in data[:3]:
        m1.train_step(x, y)
    sd_opt = copy.deepcopy(m1.optimizer.state_dict())
    sd_model = {k: v.clone() for k, v in m1.state_dict().items()}
    assert all(int(float(v["step"])) == 3 for v in sd_opt["state"].values())
    for x, y in data[3:]:
        m1.train_step(x, y)
    m2 = fresh(sd_model)
    m2.optimizer.load_state_dict(sd_opt)
    for x, y in data[3:]:
        m2.train_step(x, y)
    assert torch.equal(m1.flat_parameters(), m2.flat_parameters())
    assert torch.equal(m1._adam.m, m2._adam.m) and torch.equal(m1._adam.v, m2._adam.v)
    # the generic step (torch's own AdamW) continues from the mirrored moments
    m3 = fresh(sd_model)
    m3.optimizer.load_state_dict(sd_opt)
    for x, y in data[3:]:
        m3._generic_step(x, y)
    assert all(int(float(v["step"])) == 6 for v in m3.optimizer.state_dict()["state"].values())
    rel = float((m3.flat_parameters() - m1.flat_parameters()).norm() / m1.flat_parameters().norm())
    assert rel < 1e-5, rel
