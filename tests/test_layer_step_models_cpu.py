"""The step models of gru_driver at every layer, without a GPU.

test_gpu_layer_steps.py stops the backward at layer s (bigru_plan_set_backward_stop) and compares layer s's kernels with
backward_steps / gemm_steps at layer=s, fed the kernels' own operands.  Here the same models run free-running down the
whole stack (each step's recurrent product takes the model's own dgh, each GEMM the model's own dgi / dgh): the head's dY
(or the caller's dy) into layer L-1, each layer's modelled dX (times its dropout factor) into the layer below, each
layer's carry seeded from the head's `last` share, the caller's dhn or zero.  Run so, they must be
  oracle/bigru_ref.c's backward at exact, bf16 and bf16x3, for every layer's dW_ih, dW_hh and biases, dx and every dh0
  slice, to the float32 the oracle returns (as test_step_models_reproduce_the_oracle does for layer 0); and
  torch float64 autograd through the masked-cell loop of test_gpu_recurrent_dropout.py with dropout between layers,
  recurrent-dropout masks and lengths, on plans with a head and on head-less plans seeded from dhn.
So that a wrong layer index in any of the models (a layer's dY, carry seed, h0 slice, masks, input planes, dropout
factor or dX destination) fails here, and the GPU comparisons mean "kernel against its rounding model" at every layer."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import oracle_c  # noqa: E402
from gru_driver import (_dx_name, abi_names, backward_steps, dropout_mask, gemm_steps, head_dcat, head_dy,  # noqa: E402
                        split, stepwise)
from test_gpu_recurrent_dropout import _head, _oracle  # noqa: E402

NM = ("w_ih", "w_hh", "b_ih", "b_hh")
SEED = 77


def _first_rows_zero(a, T):
    a = a.copy()
    a[0, :, 0] = 0
    if a.shape[0] == 2:
        a[1, :, T - 1] = 0
    return a


def _layer_input(prec, x, ys, drops, l):
    """Layer l's input as its projection and dW_ih read it: x or Y[l-1], times the layer's dropout factor (a float32 product
    below "exact", as dropout_kernel forms it)."""
    v = x if l == 0 else ys[l - 1]
    if drops is None or drops[l] is None:
        return np.asarray(v, np.float64)
    if prec == "exact":
        return np.asarray(v, np.float64) * drops[l]
    return (np.asarray(v, np.float32) * drops[l]).astype(np.float64)


def _gates(s, flat, names, x, ys, h0, masks, lens, drops):
    """Every layer's gate stash G [D, B, T, 4H] in float64, from stepwise run on one layer at a time (its input exactly the
    float64 dropped input, which stepwise's own drops would round to float32)."""
    B, T, H, L, D = (s[k] for k in "BTHLD")
    out = []
    for l in range(L):
        inp = _layer_input("exact", x, ys, drops, l)
        one = dict(s, L=1, F=inp.shape[2])
        nm1 = {f"l0d{d}.{k}": names[f"l{l}d{d}.{k}"] for d in range(D) for k in NM}
        st = stepwise(one, "exact", flat, inp, None if h0 is None else h0[l * D:(l + 1) * D], None, dict(ys=[ys[l]]), nm1,
                      gates=True, masks=None if masks is None else [masks[l]], lens=lens, head=False)
        out.append(np.stack([np.stack([st[(f"step:g[l0d{d},t{t}]", "g_step")] for t in range(T)], 1) for d in range(D)]))
    return out


def chain(s, prec, flat, x, h0, names, G, ys, dl=None, arg=None, masks=None, lens=None, drops=None, head=True, dy=None,
          dhn=None):
    """The layer-l models free-running from layer L-1 down to 0.  Returns (gradient name -> array, dx, dh0 [L*D, B, H])."""
    B, T, H, L, D = (s[k] for k in "BTHLD")
    grads, dh0 = {}, np.zeros((L * D, B, H))
    dcat = head_dcat(s, prec, flat, dl, names) if head else None
    dY = head_dy(s, dcat, arg, lens) if head else None
    for l in reversed(range(L)):
        ws = dict(G=G, DY=[dY if i == l else None for i in range(L)], DCAT=dcat)
        m = None if masks is None else masks[l]
        dgi, dgh = np.zeros((D, B, T, 3 * H)), np.zeros((D, B, T, 3 * H))
        for kind, d, t, a, b in backward_steps(s, prec, flat, h0, ws, ys, names, own=True, masks=m, lens=lens, head=head,
                                               dy=dy, dhn=dhn, layer=l):
            if kind == "dg":
                dgi[d][:, t], dgh[d][:, t] = a, b
            else:
                dh0[l * D + d] = a
        inp = _layer_input(prec, x, ys, drops, l)
        xp = np.zeros(inp.shape[:2] + (-(-inp.shape[2] // 8) * 8,))
        xp[..., :inp.shape[2]] = inp
        ops = dict(DGIP=split(dgi, prec), DGHP=tuple(None if p is None else _first_rows_zero(p, T) for p in split(dgh, prec)),
                   XP=split(xp, prec), YP=split(ys[l], prec), DGI=dgi, DGH=dgh, DCAT=dcat)
        if m is not None:
            ops["RDS"] = split(np.concatenate([m[d][:, None, :].astype(np.float64) * ys[l][..., d * H:(d + 1) * H]
                                               for d in range(D)], 2), prec)
        gm = gemm_steps(s, prec, flat, dl, h0, ops, names, arg, masks=m, lens=lens, head=head, layer=l,
                        drop=None if drops is None else drops[l])
        for d in range(D):
            for nm in NM:
                grads[f"l{l}d{d}.{nm}"] = gm[(f"gemm:grad:l{l}d{d}.{nm}", "gemm_step")]
        dY = gm[(_dx_name(l), "gemm_step")]
    return grads, dY, dh0


# ---- against oracle/bigru_ref.c at every precision of its rounding model ----------------------------------------------
@pytest.mark.parametrize("h0", [False, True], ids=["no_h0", "h0"])
@pytest.mark.parametrize("prec", ["exact", "bf16", "bf16x3"])
@pytest.mark.parametrize("D", [1, 2])
@pytest.mark.parametrize("L", [2, 3])
def test_layer_models_reproduce_the_oracle(L, D, prec, h0):
    s = dict(B=3, T=5, F=13, H=8, L=L, C=3, D=D)
    B, T, F, H, C_ = (s[k] for k in "BTFHC")
    rng = np.random.default_rng([L, D, int(h0), 3])
    flat = rng.uniform(-0.5, 0.5, oracle_c.lib().bigru_ref_param_count(F, H, L, C_, D)).astype(np.float32)
    x = rng.standard_normal((B, T, F)).astype(np.float32)
    h0v = (0.5 * rng.standard_normal((L * D, B, H))).astype(np.float32) if h0 else None
    dl = rng.standard_normal((B, C_)).astype(np.float32)
    P = oracle_c.PRECISION[prec]
    _, _, stash = oracle_c.forward(flat, x, H, L, C_, D, h0v, keep=True, prec=P)
    want, dx, dh0 = oracle_c.backward(flat, x, stash, dl, H, L, C_, D, prec=P)
    ys = [y.copy() for y in oracle_c.layer_outputs(stash, B, T, H, L, D)]
    BT, o, G = B * T, 0, []
    for l in range(L):
        o += BT * D * H
        per = []
        for d in range(D):
            r, z, n, hn = (stash[o + i * BT * H: o + (i + 1) * BT * H].reshape(B, T, H) for i in range(4))
            per.append(np.concatenate([r, z, n, hn], 2))
            o += 5 * BT * H
        G.append(np.stack(per))
    names = abi_names(s)
    grads, mdx, mdh0 = chain(s, prec, flat, x, h0v, names, G, ys, dl=dl, arg=oracle_c.routing(stash, B, H))
    for name, v in grads.items():
        off, k = names[name]
        ref = want[off:off + k]
        assert np.abs(v - ref).max() <= 2e-7 * np.abs(ref).max(), (name, np.abs(v - ref).max(), np.abs(ref).max())
    assert np.abs(mdx - dx).max() <= 2e-7 * np.abs(dx).max()
    for i in range(L * D):
        assert np.abs(mdh0[i] - dh0[i]).max() <= 2e-7 * np.abs(dh0[i]).max(), i


# ---- against torch float64 autograd: dropout between layers, recurrent dropout, lengths, head-less seeds ----------------
# head, L, D, input / inter-layer dropout p, recurrent-dropout masks, lengths, h0
AUTOGRAD_CASES = {
    "head_drop_l2_lens": (True, 2, 2, 0.3, False, True, False),
    "head_drop_l3_d1": (True, 3, 1, 0.3, False, False, False),
    "head_rd_l3_h0": (True, 3, 2, 0.0, True, False, True),
    "head_rd_drop_l2_lens": (True, 2, 1, 0.2, True, True, False),
    "headless_drop_l3_lens": (False, 3, 2, 0.3, False, True, False),
    "headless_rd_l2_h0": (False, 2, 1, 0.0, True, False, True),
    "headless_rd_drop_l3_d1": (False, 3, 1, 0.3, True, False, False),
    "headless_l2_d2_h0": (False, 2, 2, 0.0, False, False, True),
}


def _torch_blocks(flat, names, s):
    H, L, D, F = (s[k] for k in "HLDF")
    W = []
    for l in range(L):
        I = F if l == 0 else D * H
        W.append([[torch.from_numpy(flat[names[f"l{l}d{d}.{nm}"][0]:sum(names[f"l{l}d{d}.{nm}"])].astype(np.float64)
                                    .reshape(shp)).requires_grad_()
                   for nm, shp in zip(NM, ((3 * H, I), (3 * H, H), (3 * H,), (3 * H,)))] for d in range(D)])
    return W


@pytest.mark.parametrize("case", list(AUTOGRAD_CASES))
def test_layer_models_are_autograd(case):
    head, L, D, p, masked, lengths, h0 = AUTOGRAD_CASES[case]
    s = dict(B=6, T=5, F=7, H=8, L=L, C=3, D=D, h0=h0)
    B, T, F, H, C_ = (s[k] for k in "BTFHC")
    rng = np.random.default_rng(list(map(int, (head, L, D, 10 * p, masked, lengths, h0))))
    names = abi_names(s)
    n = names["lin_b"][0] + C_ if head else names["lin_w"][0]
    flat = rng.uniform(-0.4, 0.4, n).astype(np.float32)
    x = rng.standard_normal((B, T, F)).astype(np.float32)
    h0v = (0.5 * rng.standard_normal((L * D, B, H))).astype(np.float32) if h0 else None
    lens = np.array([1, T, 3, T, 2, 4]) if lengths else None
    m = None
    if masked:
        m = np.where(rng.uniform(size=(L, D, B, H)) < 0.3, np.float32(0), np.float32(1) / np.float32(0.7)).astype(np.float32)
    drops = None
    if p > 0:
        # BiGRU drops every layer's input; a head-less plan (nn.GRU) only between layers
        drops = [dropout_mask(SEED, l, B, T, F if l == 0 else D * H, p) if (l > 0 or head) else None for l in range(L)]
        assert all((f == 0).any() for f in drops if f is not None)
    dl = rng.standard_normal((B, C_)).astype(np.float32) if head else None
    dy = None if head else rng.standard_normal((B, T, D * H)).astype(np.float32)
    dhn = None if head else rng.standard_normal((L * D, B, H)).astype(np.float32)

    W = _torch_blocks(flat, names, s)
    xr = torch.from_numpy(x.astype(np.float64)).requires_grad_()
    h0r = None if h0v is None else torch.from_numpy(h0v.astype(np.float64)).requires_grad_()
    lt = torch.from_numpy(lens if lens is not None else np.full(B, T))
    rdm = [[torch.from_numpy(m[l][d] if masked else np.ones((B, H), np.float32)).double() for d in range(D)] for l in range(L)]
    tdrops = [None if drops is None or drops[l] is None else torch.from_numpy(drops[l]).double() for l in range(L)]
    # one layer at a time, so that every layer's output is at hand for the models
    inp, ys_t, hns = xr, [], []
    for l in range(L):
        y, hn = _oracle(W[l:l + 1], inp, None if h0r is None else h0r[l * D:(l + 1) * D], lt, rdm[l:l + 1], tdrops[l:l + 1],
                        H, 1, D)
        ys_t.append(y)
        hns.append(hn)
        inp = y
    if head:
        lw = torch.from_numpy(flat[names["lin_w"][0]:sum(names["lin_w"])].astype(np.float64).reshape(C_, 3 * H))
        lb = torch.from_numpy(flat[names["lin_b"][0]:sum(names["lin_b"])].astype(np.float64))
        _head(ys_t[-1], lt, lw, lb, H, D).backward(torch.from_numpy(dl.astype(np.float64)))
    else:
        torch.autograd.backward((ys_t[-1], torch.cat(hns)), (torch.from_numpy(dy.astype(np.float64)),
                                                              torch.from_numpy(dhn.astype(np.float64))))
    ys = [y.detach().numpy() for y in ys_t]
    arg = None
    if head:
        top = ys[-1]
        pooled = top[..., :H] + top[..., H:] if D == 2 else top
        ok = np.ones((B, T), bool) if lens is None else np.arange(T)[None, :] < lens[:, None]
        arg = np.where(ok[..., None], pooled, -np.inf).argmax(1)
    G = _gates(s, flat, names, x, ys, h0v, m, lens, drops)
    grads, mdx, mdh0 = chain(s, "exact", flat, x, h0v, names, G, ys, dl=dl, arg=arg, masks=m, lens=lens, drops=drops,
                             head=head, dy=dy, dhn=dhn)
    for l in range(L):
        for d in range(D):
            for i, nm in enumerate(NM):
                ref = W[l][d][i].grad.numpy().ravel()
                err = np.abs(grads[f"l{l}d{d}.{nm}"] - ref).max()
                assert err <= 1e-10 * np.abs(ref).max(), (f"l{l}d{d}.{nm}", err)
    assert np.abs(mdx - xr.grad.numpy()).max() <= 1e-10 * np.abs(xr.grad.numpy()).max()
    if h0:
        ref = h0r.grad.numpy()
        for i in range(L * D):
            assert np.abs(mdh0[i] - ref[i]).max() <= 1e-10 * np.abs(ref[i]).max(), i


def test_layer_models_see_a_wrong_layer_index():
    """The chain reads the h0 slice and the masks of the layer it models: giving layer 1 layer 0's h0 or layer 0's masks
    changes layer 1's gradients far beyond the autograd test's bound (so a model that made one of these slips fails it)."""
    head, L, D = True, 2, 2
    s = dict(B=6, T=5, F=7, H=8, L=L, C=3, D=D, h0=True)
    B, T, F, H, C_ = (s[k] for k in "BTFHC")
    rng = np.random.default_rng(5)
    names = abi_names(s)
    flat = rng.uniform(-0.4, 0.4, names["lin_b"][0] + C_).astype(np.float32)
    x = rng.standard_normal((B, T, F)).astype(np.float32)
    h0v = (0.5 * rng.standard_normal((L * D, B, H))).astype(np.float32)
    m = np.where(rng.uniform(size=(L, D, B, H)) < 0.3, np.float32(0), np.float32(1) / np.float32(0.7)).astype(np.float32)
    ys = [rng.uniform(-0.9, 0.9, (B, T, D * H)) for _ in range(L)]
    dl = rng.standard_normal((B, C_)).astype(np.float32)
    arg = rng.integers(0, T, (B, H))
    G = _gates(s, flat, names, x, ys, h0v, m, None, None)
    base = chain(s, "exact", flat, x, h0v, names, G, ys, dl=dl, arg=arg, masks=m)[0]["l1d0.w_hh"]
    wrong_h0 = h0v.copy()
    wrong_h0[D:] = h0v[:D]
    wrong_m = m.copy()
    wrong_m[1] = m[0]
    for kw in (dict(h0=wrong_h0), dict(masks=wrong_m)):
        args = dict(h0=h0v, masks=m)
        args.update(kw)
        other = chain(s, "exact", flat, x, args["h0"], names, G, ys, dl=dl, arg=arg, masks=args["masks"])[0]["l1d0.w_hh"]
        assert np.abs(other - base).max() > 1e-3 * np.abs(base).max(), kw
