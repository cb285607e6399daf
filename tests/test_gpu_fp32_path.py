"""The fp32 FFMA path (BIGRU_PREC_FP32: kernels_f32.cuh and the fp32 branches of forward_plan / backward_plan in api.cu)
against the exact fp64 oracle, tensor by tensor, at the tile, split-K and reduction edges of its kernels.

precision="auto" runs this path for every hidden size above 256, so it has to be as accurate as fp32 arithmetic allows.
An fp32 yardstick computed on the CPU says how accurate that is at each shape:
- for the free-running comparison, the same model in float32 on the CPU: oracle/bigru_oracle.py's torch nn.GRU (one
  nn.GRU per layer, so that every layer's output is visible) routed through forward_routed;
- for the one-step comparison, gru_driver.stepwise evaluated in float32 from the kernel's own state.
For every tensor, the kernel's distance from the exact answer must be at most kappa x the yardstick's distance from the
exact answer, plus a small floor (TOL, per class).  So the bound scales with each shape by itself, and a kernel that
drops a k-tile, a split, a row of a reduction or the dropout mask, or evaluates a transcendental coarsely, lands far
above it while the loose bounds of test_gpu_parity.py (1e-4 on logits, 1e-3 on gradients) still pass.

The C ABI is driven directly with a fixed seed per shape.  Compared, each on its own: Y per layer, direction and step; hn;
logits; every parameter gradient by name (each bias on its own); dx; dh0.  The oracle's backward routes the max-pool
gradient the way the kernel did, and every routing disagreement must be a tie.  The second half checks every parameter
gradient with dropout active, on all three precisions, against the masks rebuilt on the host.

Run on an H100:  python -m pytest tests/test_gpu_fp32_path.py -m gpu -q
(BIGRU_FP32_REPORT=path.jsonl appends every measured distance to that file; tests/FP32_PATH.md holds the measurements.)"""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

import oracle_c
from gru_driver import abi_names, dist, dropout_mask, kernel, kernel_steps, stepwise, tensors
from oracle import bigru_oracle as bo
from test_gpu_parity import TOL as PARITY_TOL
from test_gpu_rounding_model import TOL as ROUNDING_TOL

NSM = 132                  # SMs of an H100 SXM: what sgemm_launch (kernels_f32.cuh) aims its tile choice at


def cdiv(a, b):
    return -(-a // b)


# ---------------------------------------------------------------------------------------------------------------------
# the launch rules of the fp32 path, restated
# ---------------------------------------------------------------------------------------------------------------------
def sgemm_variant(M, N, batch, splitk):
    """sgemm_launch's tile choice: (BM, BK) of the 128x128x16 variant when there are enough tiles to fill the SMs, else the
    32x32x32 one."""
    big = cdiv(M, 128) * cdiv(N, 128) * batch * splitk >= NSM and M >= 64 and N >= 64
    return (128, 16) if big else (32, 32)


def split_lengths(K, splitk, bk):
    """Reduction length of each split of sgemm_kernel: kchunk = K / splitk rounded up to whole k-tiles."""
    kchunk = cdiv(cdiv(K, splitk), bk) * bk
    return kchunk, [max(0, min(K, (z + 1) * kchunk) - z * kchunk) for z in range(splitk)]


def dw_splitk(s):
    """backward_plan's split-K of the fp32 weight-gradient GEMMs."""
    return min(64, max(1, s["B"] * s["T"] // 512))


def colsum_chunks(rows):
    """colsum_launch's (rows_per_block, chunk count)."""
    rpb = max(256, cdiv(rows, 64))
    return rpb, cdiv(rows, rpb)


def gemms(s):
    """Every sgemm_launch of one forward + backward, by role: dict(role, layer, M, N, K, batch, splitk, bm, bk, kchunk,
    splits).  gh0 is the step-0 recurrent GEMM: K = H from h0, or the masked K = 1 pure-bias GEMM without h0."""
    B, T, F, H, L, C_, D = (s[k] for k in "BTFHLCD")
    BT, out = B * T, []

    def add(role, l, M, N, K, batch=1, splitk=1):
        bm, bk = sgemm_variant(M, N, batch, splitk)
        kchunk, splits = split_lengths(K, splitk, bk)
        out.append(dict(role=role, layer=l, M=M, N=N, K=K, batch=batch, splitk=splitk, bm=bm, bk=bk, kchunk=kchunk,
                        splits=splits))

    sk = dw_splitk(s)
    for l in range(L):
        I = F if l == 0 else D * H
        add("projection", l, BT, 3 * H, I, D)
        add("gh0", l, B, 3 * H, H if s["h0"] else 1, D)
        if T > 1:
            add("gh", l, B, 3 * H, H, D)
        add("dhc", l, B, H, 3 * H, D)
        for _ in range(D):
            add("dW_ih", l, 3 * H, I, BT, 1, sk)
            if T > 1:
                add("dW_hh", l, 3 * H, H, BT, 1, sk)
            if s["h0"]:
                add("w0", l, 3 * H, H, B)
            add("dX", l, BT, I, 3 * H)
    add("lin", L, B, C_, 3 * H)
    add("dcat", L, B, 3 * H, C_)
    add("dlin_w", L, C_, 3 * H, B)
    return out


def oracle_macs(s):
    """Multiply-adds of the fp64 oracle's forward and backward (every GEMM above once)."""
    return sum(g["M"] * g["N"] * g["K"] * g["batch"] for g in gemms(s))


def _roles(s, role):
    return [g for g in gemms(s) if g["role"] == role]


def _ragged_split(g):
    """The last non-empty split of g is not a whole number of k-tiles, and it is not the split's first k-tile."""
    last = [n for n in g["splits"] if n > 0][-1]
    return last % g["bk"] != 0 and last > g["bk"]


# the regimes where the fp32 kernels go wrong, and how a shape proves it is in one
REGIMES = {
    # the 128x128 variant with whole k-tiles followed by a ragged one in the projection
    "proj_big_ragged_k": lambda s: any(g["bm"] == 128 and g["K"] % 16 != 0 and g["K"] > 16 for g in _roles(s, "projection")),
    # the recurrent GEMM with the strided A (sam = T*D*H) and direction 1's zA offset, on big tiles
    "gh_big_d2": lambda s: s["D"] == 2 and any(g["bm"] == 128 for g in _roles(s, "gh")),
    "dhc_big": lambda s: any(g["bm"] == 128 for g in _roles(s, "dhc")),
    # split-K on dW_ih and dW_hh, a ragged last split (on big tiles for one of them), chunks that cut through sequences
    "dw_splitk_ragged": lambda s: all(g["splitk"] > 1 and _ragged_split(g) and g["kchunk"] % s["T"] != 0
                                      for g in _roles(s, "dW_ih") + _roles(s, "dW_hh"))
                                  and any(g["bm"] == 128 for g in _roles(s, "dW_ih") + _roles(s, "dW_hh")),
    "splitk_cap": lambda s: s["B"] * s["T"] // 512 > 64 and dw_splitk(s) == 64,
    # the bias colsums: 64 chunks of more than 256 rows; several chunks, the last one short
    "colsum_64_chunks": lambda s: (lambda rpb, n: n == 64 and rpb > 256)(*colsum_chunks(s["B"] * s["T"])),
    "colsum_ragged_chunks": lambda s: (lambda rpb, n: n > 1 and s["B"] * s["T"] % rpb != 0)(*colsum_chunks(s["B"] * s["T"])),
    # hidden sizes precision="auto" sends to this path, and tiny ones
    "H257": lambda s: s["H"] == 257, "H300": lambda s: s["H"] == 300, "H384": lambda s: s["H"] == 384,
    "H512": lambda s: s["H"] == 512, "H1": lambda s: s["H"] == 1, "H7": lambda s: s["H"] == 7, "H33": lambda s: s["H"] == 33,
    "T1": lambda s: s["T"] == 1 and not _roles(s, "dW_hh"), "T2": lambda s: s["T"] == 2,
    "h0": lambda s: s["h0"], "no_h0": lambda s: not s["h0"] and all(g["K"] == 1 for g in _roles(s, "gh0")),
    "D1": lambda s: s["D"] == 1, "D2": lambda s: s["D"] == 2, "L3": lambda s: s["L"] == 3,
    "F_gt_DH": lambda s: s["F"] > s["D"] * s["H"], "F_lt_DH": lambda s: s["F"] < s["D"] * s["H"],
    "C_gt32": lambda s: s["C"] > 32, "B1": lambda s: s["B"] == 1,
    "DBH_not_256": lambda s: s["D"] * s["B"] * s["H"] % 256 != 0,
}

SHAPES = {
    "h384_proj_f20": dict(B=64, T=64, F=20, H=384, L=1, C=3, D=2, h0=False,
                          regimes=("proj_big_ragged_k", "H384", "F_lt_DH", "no_h0", "D2")),
    "h384_gh_big_h0": dict(B=1024, T=3, F=13, H=384, L=1, C=3, D=2, h0=True, regimes=("gh_big_d2", "H384", "h0")),
    "h512_dhc_big": dict(B=2176, T=2, F=8, H=512, L=1, C=3, D=2, h0=False, regimes=("dhc_big", "H512", "T2", "no_h0")),
    "h300_splitk": dict(B=33, T=125, F=40, H=300, L=1, C=5, D=2, h0=True,
                        regimes=("dw_splitk_ragged", "colsum_ragged_chunks", "H300", "h0", "DBH_not_256")),
    "splitk_cap": dict(B=520, T=64, F=8, H=40, L=1, C=3, D=1, h0=True,
                       regimes=("splitk_cap", "colsum_64_chunks", "D1", "DBH_not_256")),
    "h257_l2": dict(B=8, T=4, F=16, H=257, L=2, C=3, D=2, h0=False, regimes=("H257", "F_lt_DH", "DBH_not_256")),
    "h512_l2_h0": dict(B=4, T=6, F=24, H=512, L=2, C=3, D=2, h0=True, regimes=("H512", "h0")),
    "h1_t1_b1": dict(B=1, T=1, F=5, H=1, L=1, C=2, D=2, h0=False, regimes=("H1", "T1", "B1", "F_gt_DH", "no_h0")),
    "h7_l3_c40": dict(B=3, T=5, F=9, H=7, L=3, C=40, D=2, h0=True, regimes=("H7", "L3", "C_gt32", "F_lt_DH", "h0")),
    "h33_d1_t2": dict(B=5, T=2, F=70, H=33, L=2, C=4, D=1, h0=True, regimes=("H33", "D1", "T2", "F_gt_DH", "h0")),
}

# what the fp64 oracle may cost per shape (multiply-adds of all its GEMMs; 8 CPU threads run 1e10 in about 10 s) and in all
ORACLE_BUDGET = 2e10
ORACLE_BUDGET_TOTAL = 5e10

# Per class: (kappa, floor rel-L2, floor max-abs / max |ref|).  A tensor passes when, in both measures, the kernel's distance
# from the exact answer is at most kappa x the fp32 yardstick's distance plus the floor.  kappa is about 4x the worst ratio
# of the two distances measured on an H100 80GB HBM3 (SXM, 700 W power limit) over the shapes and dropout cases here; the
# floors, two to four float32 ulps, admit a kernel that is off by an ulp where the yardstick happens to be exact.  The
# measurements are in tests/FP32_PATH.md.  Free-running classes: y (every layer, direction and step), hn, logits, w (w_ih,
# w_hh, lin_w gradients), b (bias gradients), dx, dh0.  One-step classes (stepwise from the kernel's state): y_step,
# logits_step, w_step (the lin_w gradient).  The logits classes have the widest kappa: with B x C a dozen values the
# float32 yardstick is sometimes unusually close, and the kernel sums the 3H-long head GEMM in one sequential FFMA chain.
FLOOR = (2e-7, 4e-7)
TOL = {"y_step": (11, *FLOOR), "logits_step": (20, *FLOOR), "w_step": (10, *FLOOR),
       "y": (11, *FLOOR), "hn": (8, *FLOOR), "logits": (22, *FLOOR),
       "w": (17, *FLOOR), "b": (14, *FLOOR), "dx": (7, *FLOOR), "dh0": (7, *FLOOR)}


def test_shapes_are_in_the_regimes_they_claim():
    covered = set()
    for name, s in SHAPES.items():
        for r in s["regimes"]:
            assert REGIMES[r](s), (name, r)
        covered |= set(s["regimes"])
    assert covered == set(REGIMES), set(REGIMES) - covered


def test_launch_rules_at_the_edges():
    """The restated rules at the shapes the regimes hinge on (kernels_f32.cuh / api.cu)."""
    g = {x["role"]: x for x in gemms(SHAPES["h300_splitk"])}
    assert dw_splitk(SHAPES["h300_splitk"]) == 8
    assert (g["dW_hh"]["bm"], g["dW_hh"]["kchunk"], g["dW_hh"]["splits"][-1]) == (128, 528, 4125 - 7 * 528)
    assert (g["dW_ih"]["bm"], g["dW_ih"]["kchunk"], g["dW_ih"]["splits"][-1]) == (32, 544, 4125 - 7 * 544)
    assert colsum_chunks(4125) == (256, 17) and colsum_chunks(16384) == (256, 64) and colsum_chunks(33280) == (520, 64)
    assert {x["role"]: x["bm"] for x in gemms(SHAPES["h512_dhc_big"])}["dhc"] == 128
    assert {x["role"]: x["bm"] for x in gemms(dict(SHAPES["h512_dhc_big"], B=2048))}["dhc"] == 32
    assert split_lengths(20, 1, 16) == (32, [20])


@pytest.mark.parametrize("name", list(SHAPES))
def test_oracle_cost_is_within_budget(name):
    assert oracle_macs(SHAPES[name]) <= ORACLE_BUDGET, oracle_macs(SHAPES[name])
    assert sum(oracle_macs(s) for s in SHAPES.values()) <= ORACLE_BUDGET_TOTAL


# ---------------------------------------------------------------------------------------------------------------------
# references
# ---------------------------------------------------------------------------------------------------------------------
def _inputs(s, seed=0):
    B, T, F, H, L, C_, D = (s[k] for k in "BTFHLCD")
    rng = np.random.default_rng([B, T, F, H, L, D, seed])
    k = 1 / np.sqrt(H)                                          # nn.GRU / nn.Linear initialisation scale
    flat = rng.uniform(-k, k, oracle_c.lib().bigru_ref_param_count(F, H, L, C_, D)).astype(np.float32)
    x = rng.standard_normal((B, T, F)).astype(np.float32)
    h0 = (0.5 * rng.standard_normal((L * D, B, H))).astype(np.float32) if s["h0"] else None
    dl = rng.standard_normal((B, C_)).astype(np.float32)
    return flat, x, h0, dl


def _oracle(s, flat, x, h0, dl, arg):
    """The exact C oracle, its backward routed through the max-pool choice `arg`."""
    B, T, H, L, C_, D = (s[k] for k in "BTHLCD")
    logits, hn, stash = oracle_c.forward(flat, x, H, L, C_, D, h0, keep=True)
    oracle_c.set_routing(stash, arg)
    grads, dx, dh0 = oracle_c.backward(flat, x, stash, dl, H, L, C_, D)
    f64 = lambda a: None if a is None else a.astype(np.float64)  # noqa: E731
    return dict(logits=f64(logits), hn=f64(hn), ys=[y.copy() for y in oracle_c.layer_outputs(stash, B, T, H, L, D)],
                grads=f64(grads), dx=f64(dx), dh0=f64(dh0) if h0 is not None else None)


class _LayerStack(nn.Module):
    """nn.GRU's multi-layer recurrence as one nn.GRU per layer: keeps every layer's output, and applies the inter-layer
    dropout masks (the factors dropout_kernel multiplies by) when given."""

    def __init__(self, layers, masks):
        super().__init__()
        self.layers, self.masks, self.outs, self.hn = nn.ModuleList(layers), masks, [], None

    def forward(self, x, hidden=None):
        D = 2 if self.layers[0].bidirectional else 1
        inp, hns, self.outs = x, [], []
        for l, g in enumerate(self.layers):
            if l > 0 and self.masks is not None:
                inp = inp * self.masks[l]
            out, hn = g(inp, None if hidden is None else hidden[l * D:(l + 1) * D])
            self.outs.append(out)
            hns.append(hn)
            inp = out
        self.hn = torch.cat(hns, 0)
        return inp, self.hn


def torch_model(s, flat, x, h0, dl, arg, dtype, masks=None):
    """oracle/bigru_oracle.py's model (torch nn.GRU on the CPU) at `dtype`, max-pool routed through `arg`
    (forward_routed), with the dropout factors `masks` (per layer, [B, T, I_l]) when given.  Returns what gru_driver.kernel
    returns."""
    B, T, F, H, L, C_, D = (s[k] for k in "BTFHLCD")
    names = abi_names(s)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dtype)   # noqa: E731
    m = bo.OracleBiGRU(H, F, C_, L, 50, 0.0, False, D == 2).to(dtype)
    layers = [nn.GRU(F if l == 0 else D * H, H, batch_first=True, bidirectional=D == 2).to(dtype) for l in range(L)]
    blocks = []
    for l in range(L):
        for d in range(D):
            sfx = "_l0" + ("_reverse" if d else "")
            for nm, tn in (("w_ih", "weight_ih"), ("w_hh", "weight_hh"), ("b_ih", "bias_ih"), ("b_hh", "bias_hh")):
                blocks.append((names[f"l{l}d{d}.{nm}"], getattr(layers[l], tn + sfx)))
    blocks += [(names["lin_w"], m.linear.weight), (names["lin_b"], m.linear.bias)]
    with torch.no_grad():
        for (o, k), prm in blocks:
            prm.copy_(t(flat[o:o + k]).view_as(prm))
    m.gru = _LayerStack(layers, None if masks is None else [t(mk) for mk in masks])
    xr = t(x).requires_grad_(True)
    hr = None if h0 is None else t(h0).requires_grad_(True)
    xin = xr if masks is None else xr * t(masks[0])
    logits, _ = bo.forward_routed(m, xin, hr, torch.from_numpy(arg))
    logits.backward(t(dl))
    grads = np.zeros(flat.size)
    for (o, k), prm in blocks:
        grads[o:o + k] = prm.grad.double().numpy().ravel()
    f64 = lambda a: a.detach().double().numpy()                 # noqa: E731
    return dict(logits=f64(logits), hn=f64(m.gru.hn), ys=[f64(o) for o in m.gru.outs], grads=grads, dx=f64(xr.grad),
                dh0=None if hr is None else f64(hr.grad))


def _routing_ties(s, got, ref):
    """Where the kernel's max-pool picked another step than the reference, the two must tie to within the kernel's own
    deviation from the reference.  Returns the number of flips."""
    H, D = s["H"], s["D"]
    pool = lambda ys: ys[-1][..., :H] + ys[-1][..., H:] if D == 2 else ys[-1]   # noqa: E731
    sk, sr = pool(got["ys"]), pool(ref["ys"])
    own = sr.argmax(1)                                          # first maximum, the kernels' rule
    flips = got["arg"] != own
    if flips.any():
        bi, ji = np.nonzero(flips)
        gap = sr[bi, own[bi, ji], ji] - sr[bi, got["arg"][bi, ji], ji]
        assert gap.max() <= 2 * np.abs(sk - sr).max(), (int(flips.sum()), float(gap.max()))
    return int(flips.sum())


def _report(rows):
    out = os.environ.get("BIGRU_FP32_REPORT")
    if out:
        with open(out, "a") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")


def _against_yardstick(case, tk, te, ty):
    """kernel-vs-exact against kappa x yardstick-vs-exact + floor, tensor by tensor.  Returns the failures."""
    rows, bad = [], []
    for key in tk:
        tname, cls = key
        ke, ye = dist(tk[key], te[key]), dist(ty[key], te[key])
        rows.append(dict(case=case, tensor=tname, cls=cls, ke_l2=ke[0], ke_max=ke[1], ye_l2=ye[0], ye_max=ye[1]))
        kap, f2, fm = TOL[cls]
        if not (ke[0] <= kap * ye[0] + f2 and ke[1] <= kap * ye[1] + fm):
            bad.append((tname, ke, ye))
    _report(rows)
    worst = {}
    for r in rows:
        w = worst.setdefault(r["cls"], [0.0, 0.0])
        w[0] = max(w[0], r["ke_l2"] / (r["ye_l2"] + 1e-30))
        w[1] = max(w[1], r["ke_l2"])
    print(f"\n{case} " + " ".join(f"{c}: ke/ye {w[0]:.2g} ke {w[1]:.1e}" for c, w in worst.items()))
    return bad


# ---------------------------------------------------------------------------------------------------------------------
# CPU checks of the references
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["h7_l3_c40", "h33_d1_t2", "h1_t1_b1"])
def test_yardstick_lands_near_the_oracle(name):
    """The torch restatement is the oracle's model: in float64 it reproduces the oracle, in float32 (the yardstick) it lands
    within fp32 noise of it.  The one-step yardstick, fed the oracle's own state, does the same."""
    s = SHAPES[name]
    flat, x, h0, dl = _inputs(s)
    B, T, H, L, C_, D = (s[k] for k in "BTHLCD")
    _, _, stash = oracle_c.forward(flat, x, H, L, C_, D, h0, keep=True)
    arg = oracle_c.routing(stash, B, H)
    ref = _oracle(s, flat, x, h0, dl, arg)
    names = abi_names(s)
    t64, t32 = torch_model(s, flat, x, h0, dl, arg, torch.float64), torch_model(s, flat, x, h0, dl, arg, torch.float32)
    tr, ta, tb = tensors(ref, s, names), tensors(t64, s, names), tensors(t32, s, names)
    for key in tr:
        assert dist(ta[key], tr[key])[1] <= 2e-7, key          # the oracle returns logits and gradients as float32
        assert dist(tb[key], tr[key])[1] <= 1e-5, key
    e, f = stepwise(s, "exact", flat, x, h0, dl, ref, names), stepwise(s, "fp32", flat, x, h0, dl, ref, names)
    want = kernel_steps(ref, s, names)
    for key, v in want.items():
        assert dist(e[key], v)[1] <= (1e-12 if key[1] == "y_step" else 2e-7), key
        assert dist(f[key], v)[1] <= 1e-5, key


def test_dropout_masks_restated():
    """The host masks: about p of the elements dropped, the rest scaled by the float32 1/(1-p); spatial masks are one
    draw per (row, feature), shared over T."""
    m = dropout_mask(7, 0, 64, 9, 20, 0.3)
    assert abs((m == 0).mean() - 0.3) < 0.02 and set(np.unique(m)) == {0, np.float32(1) / np.float32(0.7)}
    sp = dropout_mask(7, 0, 64, 9, 20, 0.3, spatial=True)
    assert (sp == sp[:, :1]).all() and not (sp == sp[:1]).all()


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the fp32 path free-running and one step from its own state
# ---------------------------------------------------------------------------------------------------------------------
def _need_h100():
    import financial_market_data_analysis_b200 as pkg
    if pkg._lib.load().bigru_device_check(0) != 0:
        pytest.fail("no H100: " + pkg._lib.load().bigru_last_error().decode())


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SHAPES))
def test_fp32_path_against_exact_oracle(name):
    _need_h100()
    s = SHAPES[name]
    flat, x, h0, dl = _inputs(s)
    got, names = kernel(s, "fp32", flat, x, h0, dl)
    exact = _oracle(s, flat, x, h0, dl, got["arg"])
    flips = _routing_ties(s, got, exact)
    yard = torch_model(s, flat, x, h0, dl, got["arg"], torch.float32)
    tk, te, ty = tensors(got, s, names), tensors(exact, s, names), tensors(yard, s, names)
    tk.update(kernel_steps(got, s, names))
    te.update(stepwise(s, "exact", flat, x, h0, dl, got, names))
    ty.update(stepwise(s, "fp32", flat, x, h0, dl, got, names))
    bad = _against_yardstick(f"{name} flips={flips}", tk, te, ty)
    assert not bad, bad[:10]


# ---------------------------------------------------------------------------------------------------------------------
# GPU: weight gradients under dropout
# ---------------------------------------------------------------------------------------------------------------------
DROP_P, DROP_SEED = 0.3, 1234
DROP_L1 = {"fp32": dict(B=40, T=9, F=13, H=48, L=1, C=3, D=2, h0=True),
           "bf16": dict(B=32, T=6, F=20, H=128, L=1, C=3, D=2, h0=False),
           "bf16x3": dict(B=32, T=6, F=20, H=128, L=1, C=3, D=2, h0=True)}
DROP_L2 = {"fp32": dict(B=24, T=7, F=11, H=40, L=2, C=3, D=2, h0=False),
           "bf16": dict(B=32, T=5, F=16, H=128, L=2, C=3, D=2, h0=False),
           "bf16x3": dict(B=32, T=5, F=16, H=128, L=2, C=3, D=2, h0=False)}


@pytest.mark.gpu
@pytest.mark.parametrize("spatial", [False, True], ids=["elementwise", "spatial"])
@pytest.mark.parametrize("prec", ["fp32", "bf16", "bf16x3"])
def test_input_dropout_weight_gradients(prec, spatial):
    """L = 1: x' = x * mask formed on the host exactly as dropout_kernel forms it, fed to the oracle.  fp32 is held to this
    file's tolerances against the exact oracle; the tensor-core paths to test_gpu_rounding_model.py's tolerances against
    their rounding model, because to_planes_kernel rounds the dropped input.  dx must be mask * dx'."""
    _need_h100()
    s = DROP_L1[prec]
    flat, x, h0, dl = _inputs(s, seed=1)
    got, names = kernel(s, prec, flat, x, h0, dl, p=DROP_P, spatial=spatial, seed=DROP_SEED)
    mask = dropout_mask(DROP_SEED, 0, s["B"], s["T"], s["F"], DROP_P, spatial)
    xd = x * mask                                               # float32, as the kernel
    ref = _oracle(s, flat, xd, h0, dl, got["arg"]) if prec == "fp32" else None
    if prec == "fp32":
        _routing_ties(s, got, ref)
        yard = torch_model(s, flat, xd, h0, dl, got["arg"], torch.float32)
        ref["dx"], yard["dx"] = ref["dx"] * mask, yard["dx"] * mask
        tk, te, ty = tensors(got, s, names), tensors(ref, s, names), tensors(yard, s, names)
        tk.update(kernel_steps(got, s, names))
        te.update(stepwise(s, "exact", flat, xd, h0, dl, got, names))
        ty.update(stepwise(s, "fp32", flat, xd, h0, dl, got, names))
        bad = _against_yardstick(f"dropout-l1-{prec}-{'spatial' if spatial else 'elementwise'}", tk, te, ty)
        assert not bad, bad[:10]
        return
    B, T, H, L, C_, D = (s[k] for k in "BTHLCD")
    logits, hn, stash = oracle_c.forward(flat, xd, H, L, C_, D, h0, keep=True, prec=oracle_c.PRECISION[prec])
    oracle_c.set_routing(stash, got["arg"])
    grads, dx, dh0 = oracle_c.backward(flat, xd, stash, dl, H, L, C_, D, prec=oracle_c.PRECISION[prec])
    model = dict(logits=logits.astype(np.float64), hn=hn.astype(np.float64), grads=grads.astype(np.float64),
                 ys=[y.copy() for y in oracle_c.layer_outputs(stash, B, T, H, L, D)], dx=dx.astype(np.float64) * mask,
                 dh0=None if h0 is None else dh0.astype(np.float64))
    _routing_ties(s, got, model)
    tk, tm = tensors(got, s, names), tensors(model, s, names)
    tk.update(kernel_steps(got, s, names))
    tm.update(stepwise(s, prec, flat, xd, h0, dl, got, names))
    bad = []
    for key in tk:
        km, tol = dist(tk[key], tm[key]), ROUNDING_TOL[prec][key[1]]
        if km[0] > tol[0] or km[1] > tol[1]:
            bad.append((key[0], km, tol))
    assert not bad, bad[:10]
    assert ((got["dx"] == 0) == (mask == 0)).all()


@pytest.mark.gpu
@pytest.mark.parametrize("spatial", [False, True], ids=["elementwise", "spatial"])
@pytest.mark.parametrize("prec", ["fp32", "bf16", "bf16x3"])
def test_interlayer_dropout_weight_gradients(prec, spatial):
    """L = 2: input dropout and nn.GRU's inter-layer dropout, against the torch restatement in float64 with the host masks.
    dW_ih of layer 1 must come from the dropped layer-0 output.  fp32 is held to this file's tolerances (the restatement in
    float32 is the yardstick); the tensor-core paths to the per-tensor bounds of test_gpu_parity.py's TOL."""
    _need_h100()
    s = DROP_L2[prec]
    B, T, F, H, L, C_, D = (s[k] for k in "BTFHLCD")
    flat, x, h0, dl = _inputs(s, seed=2)
    got, names = kernel(s, prec, flat, x, h0, dl, p=DROP_P, spatial=spatial, seed=DROP_SEED)
    masks = [dropout_mask(DROP_SEED, 0, B, T, F, DROP_P, spatial), dropout_mask(DROP_SEED, 1, B, T, D * H, DROP_P)]
    ref = torch_model(s, flat, x, h0, dl, got["arg"], torch.float64, masks)
    _routing_ties(s, got, ref)
    tk, te = tensors(got, s, names), tensors(ref, s, names)
    if prec == "fp32":
        ty = tensors(torch_model(s, flat, x, h0, dl, got["arg"], torch.float32, masks), s, names)
        bad = _against_yardstick(f"dropout-l2-{prec}-{'spatial' if spatial else 'elementwise'}", tk, te, ty)
        assert not bad, bad[:10]
        return
    tol = PARITY_TOL[prec]
    bad = []
    for key in tk:
        if key[1] in ("w", "b", "dx"):
            e = dist(tk[key], te[key])[0]
            if e >= tol["grads"]:
                bad.append((key[0], e))
    e = dist(tk[("logits", "logits")], te[("logits", "logits")])[1]
    assert e < tol["logits"], e
    assert not bad, bad
    assert ((got["dx"] == 0) == (masks[0] == 0)).all()
