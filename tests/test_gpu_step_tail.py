"""The kernels after the backward pass of every train step, and the two behind the metrics and the live predictor, against
fp64 references at their edges.

- bigru_loss against bigru_ref_loss_ce / _bce / _mlsm (oracle/bigru_ref.c): CE, BCE with every weight / pos_weight form,
  MLSM; batches below, at and above one row per thread of the kernel's single 256-thread block; one to 33 classes;
  N(0,1), x30, +-88, +-1e4 logits and rows whose largest logit is far from the rest; the mean over the batch and over four
  times the batch (data parallelism at world size 4).  Targets outside [0, C) must poison the loss with NaN, never be read.
- bigru_adam_tick -> bigru_sqnorm -> bigru_clip_adam_step_dev against bigru_ref_clip_adam element by element, at vector
  lengths on both sides of each kernel's grid-stride boundary, with clipping inactive and binding, at steps 1 to 10^4.
- BiGRU.train_step for five steps with clipping binding on every step: each update against the oracle, from a snapshot of
  the state it started from.
- bigru_multilabel_counts against torch.sigmoid(logits) > 0.5 on the same device, across the fp32 logits where that
  differs from logits > 0.
- bigru_infer_window at D*H = 1024 threads, above 48 KB of shared memory, at L = 3, F > D*H and C above the thread count.

Every comparison is scale-free: an error over the magnitude of what the kernel adds up (see each test).  The tolerances
are about 4x the worst value measured on an H100 80GB HBM3 (700 W power limit); BIGRU_TAIL_REPORT=path.jsonl appends
every measured value to that file.

Worst values measured on an H100 80GB HBM3 (700 W power limit, 1980 MHz max SM clock):
    loss 8.5e-7 (BCE, B = 4096, C = 33, +-88 logits)   dlogits 2.4e-7   torch_loss 8.6e-7   torch_dlogits 2.4e-7
    norm 3.7e-8   g 2.3e-7   m 2.9e-7   v 5.8e-7   p 3.8e-7   (kernel test and five fused steps together)
    against torch.optim.Adam: g 0, m 3.7e-7, v 1.3e-5, p 1.9e-5 (fp32 betas, see that test)
    infer_logits 1.5e-6 (L = 3)   infer_probs 9.1e-8

Single mutations of kernels_f32.cuh, each run against the whole GPU suite but the rounding-model file (which calls none of
these kernels).  Tests of this file that fail, then tests elsewhere that fail:
    clip coefficient without min(1, .)      clip_adam[*-inactive] (6)
                                            test_golden_fused_train_step[c0, small_uni_bce], test_fused_step_matches_generic_step,
                                            test_fused_adam_state_lives_in_the_optimizer, test_zero_copy_windows_against_...[24]
    bias correction 2 formed from b1        clip_adam (18), clip_adam_torch, train_step_clip
                                            test_golden_fused_train_step (3), test_fused_step_matches_generic_step,
                                            test_fused_adam_state_lives_in_the_optimizer, test_training_trajectories_agree,
                                            test_zero_copy_windows_against_loader_and_model_oracles (2)
    sqnorm_kernel: one grid pass            clip_adam[135169, 270337, config1] (9), clip_adam_torch, train_step_clip
                                            none
    sqnorm_finish_kernel: ws[0..31] only    clip_adam[8193 and up] (12), clip_adam_torch, train_step_clip
                                            test_golden_fused_train_step[c0]
    loss: warp 0's partial only             loss[B >= 256] (44), ce_invalid[1000-33]
                                            test_auto_precision_and_batch_padding
    BCE: pos_weight on the negative term    loss[bce with pos_weight] (36)
                                            test_golden_fused_train_step[small_uni_bce]
    clip_adam reads step - 1                clip_adam (18), clip_adam_torch, train_step_clip
                                            14 tests of test_gpu_parity.py and test_gpu_step_reproducible.py

Run on an H100:  python -m pytest tests/test_gpu_step_tail.py -m gpu -q"""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

import oracle_c

pytestmark = pytest.mark.gpu

TOL = {
    "loss": 3.5e-6, "dlogits": 1e-6, "torch_loss": 3.5e-6, "torch_dlogits": 1e-6,
    "norm": 1.5e-7, "g": 1e-6, "m": 1.2e-6, "v": 2.4e-6, "p": 1.6e-6,
    "torch_g": 1e-6, "torch_m": 1.5e-6, "torch_v": 5.3e-5, "torch_p": 7.5e-5,
    "infer_logits": 6e-6, "infer_probs": 4e-7,
}

f32 = lambda v: float(np.float32(v))          # noqa: E731  - the C ABI takes these scalars as float


def _lib():
    from financial_market_data_analysis_b200 import _lib as L
    return L


def _st():
    return torch.cuda.current_stream().cuda_stream


def _scaled(k, r, mag, slack=0.0):
    """max (|k - r| - slack) / mag over the elements; where mag is 0 the two must agree to within slack.  NaN anywhere
    fails."""
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
    """Collects every measured error of a test: all are reported, the test fails at the end if any exceeds its bound."""

    def __init__(self, test):
        self.test, self.rows, self.bad = test, [], []

    def __call__(self, cls, err, **ctx):
        self.rows.append(dict(test=self.test, cls=cls, err=err, **ctx))
        if not err <= TOL[cls]:
            self.bad.append((cls, err, TOL[cls], ctx))

    def done(self):
        out = os.environ.get("BIGRU_TAIL_REPORT")
        if out:
            with open(out, "a") as f:
                for r in self.rows:
                    f.write(json.dumps(r) + "\n")
        assert not self.bad, (len(self.bad), self.bad[:8])


# ---- bigru_loss -----------------------------------------------------------------------------------------------------
LOSS_B = (1, 31, 256, 257, 1000, 4096)
LOSS_C = (1, 2, 3, 4, 33)
FAMILIES = ("normal", "x30", "pm88", "1e4", "far")
# BCE weight / pos_weight: none, one value per class, one value for all classes (the C ABI takes it expanded to [C])
WEIGHTS = ("none", "class", "single")
LOSS_KINDS = ["ce", "mlsm"] + [f"bce-w{w}-pw{p}" for w in WEIGHTS for p in WEIGHTS]


def _logits(rng, fam, B, C_):
    if fam == "normal":
        return rng.standard_normal((B, C_))
    if fam == "x30":
        return 30 * rng.standard_normal((B, C_))
    if fam == "pm88":                                           # rows mixing +-88 with 0: exp at the edge of fp32's range
        return rng.choice([-88.0, 0.0, 88.0], (B, C_))
    if fam == "1e4":
        return rng.choice([-1.0, 1.0], (B, C_)) * 1e4 * rng.uniform(0.5, 1.0, (B, C_))
    lg = rng.standard_normal((B, C_))                           # "far": one logit per row 60 above the rest
    lg[np.arange(B), rng.integers(0, C_, B)] += 60.0
    return lg


def _loss_inputs(kind, fam, B, C_):
    rng = np.random.default_rng([B, C_, FAMILIES.index(fam), LOSS_KINDS.index(kind)])
    lg = _logits(rng, fam, B, C_).astype(np.float32)
    w = pw = None
    if kind == "ce":
        tg = rng.integers(0, C_, B)
        if fam == "far":                                        # half the rows target the far logit, half another class
            top = lg.argmax(1)
            tg = np.where(np.arange(B) % 2 == 0, top, tg)
        return lg, tg.astype(np.int64), w, pw
    tg = (rng.random((B, C_)) < 0.5).astype(np.float32)
    soft = rng.random((B, C_)) < 0.1                            # soft labels too
    tg[soft] = rng.random(int(soft.sum()))
    if kind.startswith("bce"):
        wk, pk = kind[5:].split("-pw")
        form = {"none": lambda lo, hi: None, "class": lambda lo, hi: rng.uniform(lo, hi, C_).astype(np.float32),
                "single": lambda lo, hi: np.full(C_, rng.uniform(lo, hi), np.float32)}
        w, pw = form[wk](0.5, 2.0), form[pk](0.25, 4.0)
    return lg, tg, w, pw


def _kernel_loss(kind, lg, tg, w, pw, denom):
    """bigru_loss twice on the same d_loss (it must be overwritten, not accumulated; the second call without dlogits)."""
    L = _lib()
    lib = L.load()
    code = L.LOSS_CE if kind == "ce" else (L.LOSS_MLSM if kind == "mlsm" else L.LOSS_BCE)
    B, C_ = lg.shape
    dev = torch.device("cuda")
    lgd, tgd = torch.from_numpy(lg).to(dev), torch.from_numpy(tg).to(dev)
    wd = None if w is None else torch.from_numpy(w).to(dev)
    pwd = None if pw is None else torch.from_numpy(pw).to(dev)
    loss = torch.full((1,), 7.0, device=dev)
    dl = torch.full((B, C_), 5.0, device=dev)
    L.check(lib.bigru_loss(code, L.ptr(lgd), L.ptr(tgd), L.ptr(wd), L.ptr(pwd), B, C_, denom, L.ptr(loss), L.ptr(dl), _st()),
            "bigru_loss")
    first = loss.item()
    L.check(lib.bigru_loss(code, L.ptr(lgd), L.ptr(tgd), L.ptr(wd), L.ptr(pwd), B, C_, denom, L.ptr(loss), None, _st()),
            "bigru_loss")
    return first, loss.item(), dl.cpu().numpy()


def _oracle_loss(kind, lg, tg, w, pw, denom):
    if kind == "ce":
        return oracle_c.loss_ce(lg, tg, scale=1.0 / denom)
    if kind == "mlsm":
        return oracle_c.loss_mlsm(lg, tg, scale=1.0 / denom)
    return oracle_c.loss_bce(lg, tg, w, pw, scale=1.0 / denom)


def _loss_scales(kind, lg, tg, w, pw, denom):
    """(magnitude of the loss's summands, per-element scale of dlogits).  CE: the row's log-sum-exp is formed around its
    largest logit, so its rounding error, and that of every softmax entry, scales with 1 + max|logit| of the row.  BCE:
    the gradient w (1 - y - lw (1 - sigmoid)) has absolute error of order w max(1, lw) eps, lw = 1 + (pw - 1) y."""
    lg = lg.astype(np.float64)
    if kind == "ce":
        row = 1.0 + np.abs(lg).max(1, keepdims=True)
        return row.sum() / denom, np.broadcast_to(row / denom, lg.shape)
    C_ = lg.shape[1]
    wv = np.ones(C_) if w is None else w.astype(np.float64)
    pv = np.ones(C_) if pw is None else pw.astype(np.float64)
    amp = wv * np.maximum(1.0, 1.0 + (pv - 1.0) * tg)
    return (amp * (1.0 + np.abs(lg))).sum() / denom, amp / denom


def _torch_loss(kind, lg, tg, w, pw, single_w, single_pw):
    """torch's own fp32 loss and gradient on the same device (mean reduction): a second check of semantics."""
    dev = torch.device("cuda")
    x = torch.from_numpy(lg).to(dev).requires_grad_(True)
    t = torch.from_numpy(tg).to(dev)
    if kind == "ce":
        fn = nn.CrossEntropyLoss()
    elif kind == "mlsm":
        fn = nn.MultiLabelSoftMarginLoss()
    else:
        as_t = lambda a, single: None if a is None else torch.from_numpy(a[:1] if single else a).to(dev)   # noqa: E731
        fn = nn.BCEWithLogitsLoss(weight=as_t(w, single_w), pos_weight=as_t(pw, single_pw))
    v = fn(x, t)
    v.backward()
    return v.item(), x.grad.cpu().numpy()


@pytest.mark.parametrize("B", LOSS_B)
@pytest.mark.parametrize("kind", LOSS_KINDS)
def test_loss_matches_fp64_oracle(kind, B):
    chk = _Checks(f"loss[{kind}-{B}]")
    for C_ in LOSS_C:
        for fam in FAMILIES:
            lg, tg, w, pw = _loss_inputs(kind, fam, B, C_)
            base = float(B if kind == "ce" else B * C_)
            for world in (1, 4):
                denom = base * world
                first, second, dl = _kernel_loss(kind, lg, tg, w, pw, denom)
                ref, dref = _oracle_loss(kind, lg, tg, w, pw, denom)
                lmag, dscale = _loss_scales(kind, lg, tg, w, pw, denom)
                ctx = dict(C=C_, fam=fam, world=world)
                # overwritten, not accumulated: the second call on the same d_loss gives the same bits
                if not (first == second or (np.isnan(first) and np.isnan(second))):
                    chk.bad.append(("loss accumulated", first, second, ctx))
                chk("loss", abs(first - ref) / lmag, **ctx)
                chk("dlogits", _scaled(dl, dref, dscale), **ctx)
                if world == 1:
                    tv, tgrad = _torch_loss(kind, lg, tg, w, pw, "-wsingle" in kind, "-pwsingle" in kind)
                    chk("torch_loss", abs(first - tv) / lmag, **ctx)
                    chk("torch_dlogits", _scaled(dl, tgrad, dscale), **ctx)
    chk.done()


@pytest.mark.parametrize("B,C_", [(1, 1), (1, 3), (257, 1), (257, 3), (1000, 33)])
def test_ce_target_outside_the_classes_poisons_its_row_and_is_never_read(B, C_):
    """nn.CrossEntropyLoss's ignore_index (-100) and any other target outside [0, C) are not implemented: the row's loss
    and dlogits are NaN.  The logits sit inside 256 guard floats on each side holding a large finite value, so that even
    a kernel that read lg[target] would read memory this test owns; dlogits too, so that no write outside it passes."""
    G, GUARD = 256, 1e30
    L = _lib()
    lib = L.load()
    dev = torch.device("cuda")
    chk = _Checks(f"ce_invalid[{B}-{C_}]")
    rng = np.random.default_rng([B, C_])
    for bad_value in (-100, -1, C_, None):
        lg = rng.standard_normal((B, C_)).astype(np.float32)
        tg = rng.integers(0, C_, B).astype(np.int64)
        bad = np.zeros(B, bool)
        if bad_value is None:                                   # a mixture, first and last row included
            bad[[0, B - 1]] = True
            bad |= rng.random(B) < 0.1
            tg[bad] = rng.choice([-100, -1, C_], int(bad.sum()))
        else:
            bad[rng.integers(0, B)] = True
            bad[B - 1] = True
            tg[bad] = bad_value
        lbuf = torch.full((B * C_ + 2 * G,), GUARD, device=dev)
        lbuf[G:G + B * C_] = torch.from_numpy(lg.ravel()).to(dev)
        dbuf = torch.full((B * C_ + 2 * G,), 3 * GUARD, device=dev)
        tgd = torch.from_numpy(tg).to(dev)
        loss = torch.zeros(1, device=dev)
        L.check(lib.bigru_loss(L.LOSS_CE, C.c_void_p(lbuf.data_ptr() + 4 * G), L.ptr(tgd), None, None, B, C_, float(B),
                               L.ptr(loss), C.c_void_p(dbuf.data_ptr() + 4 * G), _st()), "bigru_loss")
        dl = dbuf[G:G + B * C_].view(B, C_).cpu().numpy()
        ctx = dict(bad_value=str(bad_value))
        assert np.isnan(loss.item()), (loss.item(), ctx)
        assert np.isnan(dl[bad]).all(), ctx
        assert (lbuf[:G] == GUARD).all() and (lbuf[G + B * C_:] == GUARD).all()
        assert (dbuf[:G] == 3 * GUARD).all() and (dbuf[G + B * C_:] == 3 * GUARD).all()
        ok = ~bad
        if ok.any():                                            # the other rows: as if the bad ones were absent
            _, dref = oracle_c.loss_ce(lg[ok], tg[ok], scale=1.0 / B)
            _, dscale = _loss_scales("ce", lg[ok], tg[ok], None, None, float(B))
            chk("dlogits", _scaled(dl[ok], dref, dscale), **ctx)
    chk.done()


# ---- clip_grad_norm_ + Adam -----------------------------------------------------------------------------------------
# BASELINE.json configs[1]: batch 512, seq_len 128, 64 features, hidden 256, 2 layers, 3 classes, bidirectional
CONFIG1 = (512, 128, 64, 256, 2, 3, 1)
# 1, one block and a bit, the 33rd sqnorm block (sqnorm_finish's lanes stride), the second grid pass of sqnorm_kernel
# (528 x 256 = 135168 elements), the second pass of clip_adam_dev_kernel (1056 x 256 = 270336), configs[1]'s parameters
UPDATE_N = (1, 257, 8193, 135169, 270337, "config1")
CLIP = {"inactive": 4.0, "half": 0.5, "milli": 1e-3}           # clip / ||g||: the coefficient min(1, clip / ||g||)
HYPER = (dict(lr=1e-3, b1=0.9, b2=0.999, eps=1e-8, gscale=1.0),       # torch.optim.Adam's defaults; what the mirror passes
         dict(lr=3e-3, b1=0.8, b2=0.95, eps=1e-6, gscale=0.25))       # a data-parallel scale, exact in fp32


def _config1_params():
    L = _lib()
    lib = L.load()
    h = C.c_void_p()
    B, T, F, H, L_, C_, D = CONFIG1
    L.check(lib.bigru_plan_create(B, T, F, H, L_, C_, D, L.PREC_FP32, C.byref(h)), "bigru_plan_create")
    try:
        return int(lib.bigru_param_count(h))
    finally:
        lib.bigru_plan_destroy(h)


def _grad(rng, n, kind):
    if kind == "span":                                          # |g| from 1e-20 to 1e3, the largest last
        g = np.logspace(3, -20, n)[::-1] * rng.choice([-1.0, 1.0], n)
    else:
        g = 1e-3 * rng.standard_normal(n)
    g[np.arange(n) % 7 == 3] = 0.0                              # some gradients exactly zero
    return g.astype(np.float32)


def _kernel_update(p, g, m, v, clip, hp, step, dstep0=None):
    """adam_tick -> sqnorm -> clip_adam_step_dev on device copies; returns p, g, m, v, sqnorm, the device step counter."""
    L = _lib()
    lib = L.load()
    dev = torch.device("cuda")
    pd, gd, md, vd = (torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (p, g, m, v))
    sq = torch.full((1,), 123.0, device=dev)                    # adam_tick clears it
    ws = torch.full((L.SQNORM_WS,), float("nan"), device=dev)
    dstep = torch.full((1,), step - 1 if dstep0 is None else dstep0, dtype=torch.int32, device=dev)
    n = p.size
    L.check(lib.bigru_adam_tick(L.ptr(dstep), L.ptr(sq), _st()), "bigru_adam_tick")
    L.check(lib.bigru_sqnorm(L.ptr(gd), n, L.ptr(sq), L.ptr(ws), _st()), "bigru_sqnorm")
    L.check(lib.bigru_clip_adam_step_dev(L.ptr(pd), L.ptr(gd), L.ptr(md), L.ptr(vd), n, L.ptr(sq), f32(clip), f32(hp["lr"]),
                                         f32(hp["b1"]), f32(hp["b2"]), f32(hp["eps"]), L.ptr(dstep), f32(hp["gscale"]), _st()),
            "bigru_clip_adam_step_dev")
    return (pd.cpu().numpy(), gd.cpu().numpy(), md.cpu().numpy(), vd.cpu().numpy(), float(sq.item()), int(dstep.item()))


def _oracle_update(p, g, m, v, clip, hp, step):
    """bigru_ref_clip_adam on copies, with the hyperparameters rounded to fp32 as the C ABI receives them."""
    p, g, m, v = (np.array(a, np.float32, copy=True) for a in (p, g, m, v))
    norm = oracle_c.clip_adam(p, g, m, v, f32(clip), f32(hp["lr"]), f32(hp["b1"]), f32(hp["b2"]), f32(hp["eps"]), step)
    return p, g, m, v, norm


def _update_errors(chk, prefix, before, got, ref, hp, step, **ctx):
    """Element-wise errors of (p, g, m, v) over the magnitude of what each update adds up: g relative; m over
    b1 |m| + (1 - b1) |g|; v over b2 v + (1 - b2) g^2 plus the smallest normal fp32 (below it v is subnormal and keeps
    fewer bits); p over the step formed from m's magnitude instead of m (m can cancel to far below the terms it is made
    of, and its absolute error is that of the terms), after one ulp of p: p - step rounds, and a step off by an ulp of
    its own can move that rounding by one ulp of p."""
    m0, v0 = (np.asarray(a, np.float64) for a in (before[2], before[3]))
    pr, gr, mr, vr = (np.asarray(a, np.float64) for a in ref[:4])
    lr, b1, b2, eps = (f32(hp[k]) for k in ("lr", "b1", "b2", "eps"))
    m_mag = b1 * np.abs(m0) + (1 - b1) * np.abs(gr)
    p_mag = lr / (1 - b1 ** step) * m_mag / (np.sqrt(vr / (1 - b2 ** step)) + eps)
    chk(prefix + "g", _scaled(got[1], gr, np.abs(gr)), step=step, **ctx)
    chk(prefix + "m", _scaled(got[2], mr, m_mag), step=step, **ctx)
    chk(prefix + "v", _scaled(got[3], vr, b2 * v0 + (1 - b2) * gr * gr + np.finfo(np.float32).tiny), step=step, **ctx)
    chk(prefix + "p", _scaled(got[0], pr, p_mag, np.spacing(np.abs(ref[0]).astype(np.float32))), step=step, **ctx)


@pytest.fixture(scope="module")
def config1_n():
    return _config1_params()


@pytest.mark.parametrize("clip_kind", list(CLIP))
@pytest.mark.parametrize("n_kind", UPDATE_N, ids=[str(n) for n in UPDATE_N])
def test_clip_adam_matches_fp64_oracle(n_kind, clip_kind, config1_n):
    n = config1_n if n_kind == "config1" else n_kind
    chk = _Checks(f"clip_adam[{n}-{clip_kind}]")
    rng = np.random.default_rng([n, list(CLIP).index(clip_kind)])
    for gkind in ("normal", "span"):
        g = _grad(rng, n, gkind)
        for hi, hp in enumerate(HYPER):
            gs = (g * np.float32(hp["gscale"])).astype(np.float32)  # exact: gscale is a power of two
            gnorm = float(np.linalg.norm(gs.astype(np.float64)))
            clip = CLIP[clip_kind] * gnorm
            p = (hp["lr"] * rng.standard_normal(n)).astype(np.float32)   # parameters the size of a step: every step resolves
            for state in ("zero", "prev"):
                if state == "zero":
                    m = np.zeros(n, np.float32); v = np.zeros(n, np.float32)
                else:
                    m = (1e-3 * rng.standard_normal(n)).astype(np.float32)
                    v = ((1e-3 * rng.standard_normal(n)) ** 2).astype(np.float32)
                for step in (1, 2, 10, 10_000):
                    ctx = dict(g=gkind, hyper=hi, state=state)
                    got = _kernel_update(p, g, m, v, clip, hp, step)
                    ref = _oracle_update(p, gs, m, v, clip, hp, step)
                    if got[5] != step:
                        chk.bad.append(("device step", got[5], step, ctx))
                    exact = float(np.linalg.norm(g.astype(np.float64)))
                    chk("norm", abs(np.sqrt(got[4]) - exact) / exact, step=step, **ctx)
                    _update_errors(chk, "", (p, g, m, v), got, ref, hp, step, **ctx)
    chk.done()


def test_clip_adam_matches_torch_adam_and_clip_grad_norm():
    """Two steps against torch.optim.Adam(foreach=False) and clip_grad_norm_ on the same device, clipping binding.  The C
    ABI takes the betas in fp32 and forms 1 - beta2 from that, torch forms it in double: at beta2 = 0.999 the two
    second moments differ by 1.3e-5 relative, which bounds this comparison from below."""
    n, hp = 270337, HYPER[0]
    rng = np.random.default_rng(7)
    chk = _Checks("clip_adam_torch")
    dev = torch.device("cuda")
    p0 = (0.1 * rng.standard_normal(n)).astype(np.float32)
    gs = [_grad(rng, n, "normal") for _ in range(2)]
    clip = 0.5 * float(np.linalg.norm(gs[0].astype(np.float64)))
    prm = nn.Parameter(torch.from_numpy(p0).to(dev))
    opt = torch.optim.Adam([prm], lr=hp["lr"], betas=(hp["b1"], hp["b2"]), eps=hp["eps"], foreach=False)
    p, m, v = p0, np.zeros(n, np.float32), np.zeros(n, np.float32)
    for step, g in enumerate(gs, 1):
        prm.grad = torch.from_numpy(g).to(dev)
        nn.utils.clip_grad_norm_([prm], clip)
        opt.step()
        got = _kernel_update(p, g, m, v, clip, hp, step)
        st = opt.state[prm]
        ref = (prm.detach().cpu().numpy(), prm.grad.cpu().numpy(), st["exp_avg"].cpu().numpy(), st["exp_avg_sq"].cpu().numpy())
        _update_errors(chk, "torch_", (p, g, m, v), got, ref, hp, step)
        p, m, v = got[0], got[2], got[3]
    chk.done()


def test_fused_train_step_with_clipping_follows_the_oracle_update_every_step():
    """BiGRU.train_step at fp32, plain launches, clip = 0.05 so that clipping binds on every step.  Each update is
    compared with bigru_ref_clip_adam fed a snapshot of the state it started from (the unclipped flat gradient, p, m, v),
    so the recurrence's own error does not compound into the comparison."""
    from financial_market_data_analysis_b200 import BiGRU
    B, T, F, H, L, C_ = 64, 12, 16, 128, 2, 3
    torch.manual_seed(11)
    m = BiGRU(H, F, C_, L, 0.05, 0.0, False, True, precision="fp32").cuda()
    m.use_cuda_graph = False
    m.add_loss_fn(nn.CrossEntropyLoss())
    hp = dict(lr=2e-3, b1=0.85, b2=0.99, eps=1e-7, gscale=1.0)
    m.add_optimizer(torch.optim.Adam(m.parameters(), lr=hp["lr"], betas=(hp["b1"], hp["b2"]), eps=hp["eps"]))
    m.train()
    snaps = []
    launch_update = m._launch_update

    def read(st):
        return (m._flat.cpu().numpy(), st.grad.cpu().numpy(), st.m.cpu().numpy(), st.v.cpu().numpy(),
                float(st.scal[1].item()), int(st.dstep.item()))

    def update(g, st, s):
        before = read(st)
        launch_update(g, st, s)
        snaps.append((before, read(st), st.step))

    m._launch_update = update
    g = torch.Generator().manual_seed(12)
    chk = _Checks("train_step_clip")
    assert m._flat.numel() > 270336                              # past the second grid pass of sqnorm and of the update
    for k in range(5):
        x, t = torch.randn(B, T, F, generator=g).cuda(), torch.randint(0, C_, (B,), generator=g).cuda()
        m.train_step(x, t)
        st = m._adam
        assert st.step == int(st.dstep.item()) == k + 1
        before, after, host_step = snaps[k]
        assert host_step == k and before[5] == k and after[5] == k + 1
        ref = _oracle_update(before[0], before[1], before[2], before[3], 0.05, hp, k + 1)
        assert ref[4] > 2 * 0.05, ref[4]                         # clipping binds
        chk("norm", abs(np.sqrt(after[4]) - ref[4]) / ref[4], step=k + 1)
        _update_errors(chk, "", before, after, ref, hp, k + 1)
    chk.done()


# ---- bigru_multilabel_counts ----------------------------------------------------------------------------------------
def _boundary_logits():
    """Every fp32 value in [8e-8, 1.3e-7]: where 1 + expf(-x) stops rounding to 2, so that torch's fp32 sigmoid of a
    positive logit stops being exactly 0.5 (about 9e-8 with a correctly rounded expf)."""
    lo, hi = np.float32(8e-8).view(np.uint32), np.float32(1.3e-7).view(np.uint32)
    return np.arange(lo, hi + 1, dtype=np.uint32).view(np.float32)


# signed zeros, NaN, infinities, and positive logits far below the boundary (fp32 sigmoid exactly 0.5)
SPECIAL = np.array([0.0, -0.0, 1e-8, -1e-8, 5e-8, 1e-20, 1e-45, -1e-45, np.nan, -np.nan, 2e-7, -1e-7, 1.0, -1.0, np.inf,
                    -np.inf], np.float32)


def _metric_reference(lg_dev, tg):
    pred = (torch.sigmoid(lg_dev) > 0.5).cpu().numpy()
    tru = tg > 0.5
    C_ = tg.shape[1]
    row = np.zeros(2 + 3 * C_, np.int64)
    row[0] = (pred == tru).all(1).sum()
    row[1] = (pred != tru).sum()
    row[2::3] = (pred & tru).sum(0)
    row[3::3] = (pred & ~tru).sum(0)
    row[4::3] = (~pred & tru).sum(0)
    return row, pred


@pytest.mark.parametrize("C_", (1, 4, 37))
@pytest.mark.parametrize("B", (1, 127, 128, 129, 100_000))
def test_multilabel_counts_match_torch_sigmoid_threshold(B, C_):
    L = _lib()
    lib = L.load()
    dev = torch.device("cuda")
    rng = np.random.default_rng([B, C_])
    edge = _boundary_logits()
    n = B * C_
    counts = torch.zeros(2 + 3 * C_, dtype=torch.int64, device=dev)
    want = np.zeros(2 + 3 * C_, np.int64)
    keep, todo = [], edge                                         # edge values not yet placed
    for call in range(2):                                        # the counters accumulate over calls
        if n >= 1_000_000:                                       # every boundary value, over the two calls
            part, todo = todo[:n - SPECIAL.size], todo[n - SPECIAL.size:]
            lg = np.concatenate([part, SPECIAL, rng.standard_normal(n - part.size - SPECIAL.size).astype(np.float32)])
            rng.shuffle(lg)
        else:
            pool = np.concatenate([rng.choice(edge, max(1, n // 2)), SPECIAL, rng.standard_normal(n).astype(np.float32)])
            lg = rng.permutation(pool)[:n]
            lg[rng.integers(0, n)] = 1e-8                        # at least one positive logit whose sigmoid is 0.5
        lg = lg.astype(np.float32).reshape(B, C_)
        tg = rng.choice(np.array([0.0, 1.0, 0.5, 0.7, 0.3], np.float32), (B, C_), p=[0.4, 0.4, 0.1, 0.05, 0.05])
        lgd, tgd = torch.from_numpy(lg).to(dev), torch.from_numpy(tg).to(dev)
        keep.append((lgd, tgd))
        row, pred = _metric_reference(lgd, tg)
        want += row
        assert ((lg > 0) != pred).any()                          # this batch separates the fp32 sigmoid from logit > 0
        L.check(lib.bigru_multilabel_counts(L.ptr(lgd), L.ptr(tgd), B, C_, L.ptr(counts), _st()), "bigru_multilabel_counts")
    assert todo.size == 0 or n < 1_000_000
    got = counts.cpu().numpy()
    assert (got == want).all(), (got[:8], want[:8])


# ---- bigru_infer_window ---------------------------------------------------------------------------------------------
INFER = {
    "dh1024": dict(B=2, T=6, F=16, H=512, L=1, C=3, D=2, norm=False),         # 1024 threads of 64 registers; 62 KB smem
    "dh1024_smem198k": dict(B=1, T=23, F=16, H=512, L=1, C=3, D=2, norm=True),  # next to the 200 KB the entry point allows
    "l3": dict(B=3, T=5, F=12, H=16, L=3, C=3, D=2, norm=True),
    "f_above_dh": dict(B=2, T=5, F=100, H=8, L=2, C=3, D=2, norm=True),
    "c_above_threads": dict(B=2, T=4, F=6, H=8, L=1, C=40, D=1, norm=False),
}


def _infer_smem(s):
    DH = s["D"] * s["H"]
    return 4 * (s["T"] * max(s["F"], DH) + s["T"] * DH + 2 * DH + 3 * s["H"])


def test_infer_cases_are_in_the_regimes_they_claim():
    threads = lambda s: max(32, -(-s["D"] * s["H"] // 32) * 32)   # noqa: E731  - bigru_infer_window's block size
    assert INFER["dh1024"]["D"] * INFER["dh1024"]["H"] == 1024 and _infer_smem(INFER["dh1024"]) > 48 * 1024
    assert 190 * 1024 < _infer_smem(INFER["dh1024_smem198k"]) <= 200 * 1024
    assert INFER["l3"]["L"] == 3
    assert INFER["f_above_dh"]["F"] > INFER["f_above_dh"]["D"] * INFER["f_above_dh"]["H"]
    assert INFER["c_above_threads"]["C"] > threads(INFER["c_above_threads"])


@pytest.mark.parametrize("name", list(INFER))
def test_infer_window_matches_fp64_oracle(name):
    s = INFER[name]
    B, T, F, H, L_, C_, D = (s[k] for k in "BTFHLCD")
    rng = np.random.default_rng(list(map(ord, name)))
    k = 1 / np.sqrt(H)
    flat = rng.uniform(-k, k, oracle_c.lib().bigru_ref_param_count(F, H, L_, C_, D)).astype(np.float32)
    if s["norm"]:
        mn = rng.uniform(-5, 0, F).astype(np.float32)
        mx = (mn + rng.uniform(0.5, 3, F)).astype(np.float32)
        raw = (mn + rng.uniform(0, 1, (B, T, F)) * (mx - mn)).astype(np.float32)
        x = ((raw.astype(np.float64) - mn) / (mx.astype(np.float64) - mn)).astype(np.float32)
    else:
        mn = mx = None
        raw = x = rng.standard_normal((B, T, F)).astype(np.float32)
    ref, _ = oracle_c.forward(flat, x, H, L_, C_, D)
    L = _lib()
    lib = L.load()
    dev = torch.device("cuda")
    to = lambda a: None if a is None else torch.from_numpy(a).to(dev)   # noqa: E731
    pd, xd, mnd, mxd = to(flat), to(raw), to(mn), to(mx)
    logits = torch.full((B, C_), float("nan"), device=dev)
    probs = torch.full((B, C_), float("nan"), device=dev)
    L.check(lib.bigru_infer_window(L.ptr(pd), L.ptr(xd), L.ptr(mnd), L.ptr(mxd), B, T, F, H, L_, C_, int(D == 2), L.ptr(logits),
                                   L.ptr(probs), _st()), "bigru_infer_window")
    chk = _Checks(f"infer[{name}]")
    ref64 = ref.astype(np.float64)
    chk("infer_logits", _scaled(logits.cpu().numpy(), ref64, max(np.abs(ref64).max(), 1e-3)))
    chk("infer_probs", _scaled(probs.cpu().numpy(), 1 / (1 + np.exp(-ref64)), 1.0))
    chk.done()
