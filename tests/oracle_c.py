"""ctypes binding of oracle/_build/libbigru_oracle.so (plain-C restatement).  Test infrastructure."""
import ctypes as C
import os
import subprocess

import numpy as np

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SO = os.path.join(_ROOT, "oracle", "_build", "libbigru_oracle.so")


def build():
    if not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(os.path.join(_ROOT, "oracle", "bigru_ref.c")):
        subprocess.check_call(["make", "-C", os.path.join(_ROOT, "oracle")], stdout=subprocess.DEVNULL)
    return _SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
        _lib.bigru_ref_param_count.restype = C.c_int64
        _lib.bigru_ref_stash_doubles.restype = C.c_int64
        assert _lib.bigru_ref_rounding_points() == len(ROUNDING_POINTS)
        for f in ("bigru_ref_loss_ce", "bigru_ref_loss_bce", "bigru_ref_loss_mlsm", "bigru_ref_clip_adam"):
            getattr(_lib, f).restype = C.c_double
    return _lib


def _p(a, t=C.c_float):
    return None if a is None else a.ctypes.data_as(C.POINTER(t))


# precision of the rounding model (oracle/bigru_ref.c): every product exact, or its operands rounded where the bf16 /
# bf16x3 tensor-core path rounds them
EXACT, BF16, BF16X3 = 0, 1, 2
PRECISION = {"exact": EXACT, "bf16": BF16, "bf16x3": BF16X3}
# rounding points of the model, in bit order of the `mask` argument (see the table in oracle/bigru_ref.c)
ROUNDING_POINTS = ("proj_x", "proj_w", "rec_h", "rec_w", "head_cat", "head_w", "hb_dl", "hb_w", "hb_cat", "br_dgh", "br_w",
                   "dwih_dgi", "dwih_x", "dwhh_dgh", "dwhh_y", "dwhh_h0", "dx_dgi", "dx_w", "rec_h0")
ALL_POINTS = (1 << len(ROUNDING_POINTS)) - 1


def without(*points):
    """Rounding mask with the named points left exact."""
    m = ALL_POINTS
    for p in points:
        m &= ~(1 << ROUNDING_POINTS.index(p))
    return m


PARAM_ORDER = ("weight_ih", "weight_hh", "bias_ih", "bias_hh")


def flatten_params(sd, L, D):
    """nn.GRU/nn.Linear-named dict -> flat float32 vector in the C-ABI order."""
    parts = []
    for l in range(L):
        for d in range(D):
            sfx = f"l{l}" + ("_reverse" if d else "")
            for n in PARAM_ORDER:
                parts.append(np.asarray(sd[f"gru.{n}_{sfx}"], np.float32).ravel())
    parts.append(np.asarray(sd["linear.weight"], np.float32).ravel())
    parts.append(np.asarray(sd["linear.bias"], np.float32).ravel())
    return np.ascontiguousarray(np.concatenate(parts))


def forward(flat, x, H, L, C_, D, h0=None, keep=False, prec=EXACT, mask=ALL_POINTS):
    """logits[B,C], hn[L*D,B,H] (and the stash for backward with keep).  prec / mask select the rounding model; the
    default is the exact restatement."""
    B, T, F = x.shape
    x = np.ascontiguousarray(x, np.float32)
    logits = np.zeros((B, C_), np.float32)
    hn = np.zeros((L * D, B, H), np.float32)
    n = lib().bigru_ref_stash_doubles(B, T, F, H, L, C_, D)
    stash = np.zeros(n, np.float64)
    h0c = None if h0 is None else np.ascontiguousarray(h0, np.float32)
    rc = lib().bigru_ref_forward_p(B, T, F, H, L, C_, D, prec, C.c_uint(mask), _p(flat), _p(x), _p(h0c), _p(logits), _p(hn),
                                   _p(stash, C.c_double))
    assert rc == 0
    return (logits, hn, stash) if keep else (logits, hn)


def backward(flat, x, stash, dlogits, H, L, C_, D, prec=EXACT, mask=ALL_POINTS):
    """grads (flat), dx, dh0 from a stash of forward(..., keep=True) run with the same prec and mask."""
    B, T, F = x.shape
    x = np.ascontiguousarray(x, np.float32)
    grads = np.zeros_like(flat)
    dx = np.zeros_like(x)
    dh0 = np.zeros((L * D, B, H), np.float32)
    dl = np.ascontiguousarray(dlogits, np.float32)
    rc = lib().bigru_ref_backward_p(B, T, F, H, L, C_, D, prec, C.c_uint(mask), _p(flat), _p(x), _p(stash, C.c_double), _p(dl),
                                    _p(grads), _p(dx), _p(dh0))
    assert rc == 0
    return grads, dx, dh0


def layer_outputs(stash, B, T, H, L, D):
    """Views of every layer's output Y[B,T,D*H] inside a forward stash."""
    BT, out, o = B * T, [], 0
    for _ in range(L):
        out.append(stash[o:o + BT * D * H].reshape(B, T, D * H))
        o += BT * D * H + D * 5 * BT * H
    return out


def set_routing(stash, arg):
    """Overwrite the stash's max-pool routing (argmax over T of the pooled top-layer output, int [B,H]) so that the
    backward routes the max-pool gradient as given."""
    arg = np.asarray(arg)
    stash[-arg.size:] = arg.ravel()


def routing(stash, B, H):
    return stash[-B * H:].reshape(B, H).astype(np.int64)


def loss_ce(logits, target, scale=None):
    B, C_ = logits.shape
    lg = np.ascontiguousarray(logits, np.float32)
    tg = np.ascontiguousarray(target, np.int64)
    d = np.zeros_like(lg)
    v = lib().bigru_ref_loss_ce(B, C_, _p(lg), _p(tg, C.c_int64), _p(d), C.c_double(scale or 1.0 / B))
    return v, d


def loss_bce(logits, target, weight=None, pos_weight=None, scale=None):
    B, C_ = logits.shape
    lg = np.ascontiguousarray(logits, np.float32)
    tg = np.ascontiguousarray(target, np.float32)
    w = None if weight is None else np.ascontiguousarray(weight, np.float32)
    pw = None if pos_weight is None else np.ascontiguousarray(pos_weight, np.float32)
    d = np.zeros_like(lg)
    v = lib().bigru_ref_loss_bce(B, C_, _p(lg), _p(tg), _p(w), _p(pw), _p(d), C.c_double(scale or 1.0 / (B * C_)))
    return v, d


def loss_mlsm(logits, target, scale=None):
    B, C_ = logits.shape
    lg = np.ascontiguousarray(logits, np.float32)
    tg = np.ascontiguousarray(target, np.float32)
    d = np.zeros_like(lg)
    v = lib().bigru_ref_loss_mlsm(B, C_, _p(lg), _p(tg), _p(d), C.c_double(scale or 1.0 / (B * C_)))
    return v, d


def clip_adam(params, grads, m, v, clip, lr, b1, b2, eps, step):
    """clip_grad_norm_ + one Adam step in fp64, on float32 arrays updated in place (grads become the clipped gradient).
    Returns the norm of the unclipped gradient."""
    return lib().bigru_ref_clip_adam(C.c_int64(params.size), _p(params), _p(grads), _p(m), _p(v), C.c_double(clip),
                                     C.c_double(lr), C.c_double(b1), C.c_double(b2), C.c_double(eps), step)


def window_gather_norm(src, xmin, xmax, start, B, T):
    F = src.shape[1]
    out = np.zeros((B, T, F), np.float32)
    lib().bigru_ref_window_gather_norm(_p(np.ascontiguousarray(src, np.float32)), _p(np.ascontiguousarray(xmin, np.float32)),
                                       _p(np.ascontiguousarray(xmax, np.float32)), C.c_int64(start), B, T, F, _p(out))
    return out
