"""fp64 references of the fused step's weighted cross-entropy, regression losses and grouped Adam / AdamW update
(bigru_loss_param, bigru_clip_adam_groups_dev in include/bigru_b200.h).  Plain numpy in float64, written from torch's
documented formulas; tests/test_fused_optim_cpu.py checks them against torch in float64."""
import numpy as np

CE_WEIGHTED, MSE, L1, SMOOTH_L1, HUBER = 3, 4, 5, 6, 7        # BIGRU_LOSS_* of include/bigru_b200.h


def loss(kind, logits, target, weight=None, param=0.0, denom=1.0):
    """(loss, dlogits) in float64.  CE_WEIGHTED: sum_b w[y_b] nll_b / (sum_b w[y_b] * denom); the regressions: the mean
    of the elementwise loss over denom elements, with torch's gradient at the kinks."""
    x = np.asarray(logits, np.float64)
    if kind == CE_WEIGHTED:
        y = np.asarray(target, np.int64)
        w = np.asarray(weight, np.float64)[y]
        m = x.max(1, keepdims=True)
        lse = m[:, 0] + np.log(np.exp(x - m).sum(1))
        nll = lse - x[np.arange(x.shape[0]), y]
        W = w.sum()
        with np.errstate(invalid="ignore", divide="ignore"):
            sm = np.exp(x - lse[:, None])
            sm[np.arange(x.shape[0]), y] -= 1.0
            return float((w * nll).sum() / (W * denom)), sm * (w / (W * denom))[:, None]
    d = x - np.asarray(target, np.float64)
    ad = np.abs(d)
    if kind == SMOOTH_L1 and param == 0.0:
        kind = L1
    if kind == MSE:
        val, gr = d * d, 2.0 * d
    elif kind == L1:
        val, gr = ad, np.sign(d)
    elif kind == SMOOTH_L1:
        val = np.where(ad < param, 0.5 * d * d / param, ad - 0.5 * param)
        gr = np.where(d < -param, -1.0, np.where(d > param, 1.0, d / param))
    elif kind == HUBER:
        val = np.where(ad < param, 0.5 * d * d, param * (ad - 0.5 * param))
        gr = np.where(d < -param, -param, np.where(d > param, param, d))
    else:
        raise ValueError(kind)
    return float(val.sum() / denom), gr / denom


def clip_adam_groups(p, g, m, v, clip, groups, segments, step, gscale=1.0):
    """clip_grad_norm_(clip) of g * gscale, then Adam / AdamW per segment with its group's (lr, beta1, beta2, eps,
    weight_decay, decoupled), on float64 copies.  Elements in no segment are left as they are.  Returns
    (p, g, m, v, norm)."""
    p, g, m, v = (np.array(a, np.float64, copy=True) for a in (p, g, m, v))
    gs = g * gscale
    norm = float(np.sqrt((gs * gs).sum()))
    coef = min(1.0, clip / (norm + 1e-6))
    for off, n, k in segments:
        lr, b1, b2, eps, wd, dec = (float(t) for t in groups[k])
        s = slice(off, off + n)
        g[s] = gs[s] * coef
        ge = g[s].copy()
        if wd != 0.0:
            if dec:
                p[s] *= 1.0 - lr * wd
            else:
                ge += wd * p[s]
        m[s] = b1 * m[s] + (1.0 - b1) * ge
        v[s] = b2 * v[s] + (1.0 - b2) * ge * ge
        p[s] -= lr / (1.0 - b1 ** step) * m[s] / (np.sqrt(v[s] / (1.0 - b2 ** step)) + eps)
    return p, g, m, v, norm
