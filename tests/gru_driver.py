"""Drives the library's C ABI on one plan and takes the result apart tensor by tensor.  Test infrastructure, shared by
test_gpu_rounding_model.py and test_gpu_fp32_path.py.

A shape is a dict with B, T, F, H, L, C, D (1 or 2) and h0 (bool).  `kernel` runs bigru_forward and bigru_backward at a
precision ("fp32", "bf16" or "bf16x3"), optionally with dropout, and returns every layer's output, hn, the max-pool
routing, the flat gradient, dx and dh0 in float64.  `tensors` / `kernel_steps` split such a result into the per-tensor
comparisons, `stepwise` recomputes one step from the kernel's own state, `dist` measures two tensors."""
import ctypes as C

import numpy as np
import torch

CODE = {"fp32": 0, "bf16": 1, "bf16x3": 2}      # BIGRU_PREC_* of include/bigru_b200.h


def _pkg():
    import financial_market_data_analysis_b200 as pkg
    return pkg


def bigru_uniform(seed, stream, idx):
    """common.cuh bigru_uniform restated: splitmix64 finaliser over (seed, stream, element index) -> [0, 1)."""
    idx = np.asarray(idx, np.uint64)
    with np.errstate(over="ignore"):
        z = np.uint64(seed) + np.uint64(0x9E3779B97F4A7C15) * (idx + np.uint64(1)) + (np.uint64(stream) << np.uint64(40)) * np.uint64(0xD1B54A32D192ED03)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
    return (z >> np.uint64(40)).astype(np.float64) * (1.0 / 16777216.0)


def dropout_mask(seed, layer, B, T, I, p, spatial=False):
    """The float32 factor dropout_kernel (kernels_f32.cuh) multiplies layer `layer`'s input [B, T, I] by: 0 where the
    element is dropped, else 1/(1-p) rounded to float32.  spatial: one draw per (b, feature), shared over T."""
    bi, ti, fi = np.meshgrid(np.arange(B), np.arange(T), np.arange(I), indexing="ij")
    key = bi * I + fi if spatial else (bi * T + ti) * I + fi
    p32 = np.float32(p)
    scale = np.float32(1) / (np.float32(1) - p32)
    return np.where(bigru_uniform(seed, layer, key).astype(np.float32) < p32, np.float32(0), scale).astype(np.float32)


def param_names(plan, s):
    """name -> (offset, size) of every parameter block, from bigru_param_offset."""
    lib = _pkg()._lib.load()
    out = {}
    off, rows, cols = C.c_int64(), C.c_int64(), C.c_int64()
    for l in range(s["L"] + 1):
        for d in range(s["D"] if l < s["L"] else 1):
            for which, nm in enumerate(("w_ih", "w_hh", "b_ih", "b_hh")):
                if l == s["L"] and which in (1, 3):
                    continue
                assert lib.bigru_param_offset(plan, l, d, which, C.byref(off), C.byref(rows), C.byref(cols)) == 0
                name = ("lin_w" if which == 0 else "lin_b") if l == s["L"] else f"l{l}d{d}.{nm}"
                out[name] = (off.value, rows.value * cols.value)
    return out


def abi_names(s):
    """param_names without a plan: the C-ABI order (per layer and direction w_ih, w_hh, b_ih, b_hh; then lin_w, lin_b)."""
    names, o = {}, 0
    H, D = s["H"], s["D"]
    for l in range(s["L"]):
        for d in range(D):
            for nm, n in (("w_ih", 3 * H * (s["F"] if l == 0 else D * H)), ("w_hh", 3 * H * H), ("b_ih", 3 * H), ("b_hh", 3 * H)):
                names[f"l{l}d{d}.{nm}"] = (o, n)
                o += n
    names["lin_w"], names["lin_b"] = (o, s["C"] * 3 * H), (o + s["C"] * 3 * H, s["C"])
    return names


def kernel(s, prec, flat, x, h0, dl, p=0.0, spatial=False, seed=0):
    """bigru_forward + bigru_backward of shape s at precision prec; dropout p (training mode) when p > 0."""
    pkg = _pkg()
    lib, L_ = pkg._lib.load(), pkg._lib
    B, T, F, H, L, C_, D = (s[k] for k in "BTFHLCD")
    plan = C.c_void_p()
    L_.check(lib.bigru_plan_create(B, T, F, H, L, C_, int(D == 2), CODE[prec], C.byref(plan)), "plan_create")
    try:
        sb, cb = C.c_size_t(), C.c_size_t()
        L_.check(lib.bigru_workspace_bytes(plan, C.byref(sb), C.byref(cb)), "workspace_bytes")
        dev = torch.device("cuda")
        stash = torch.zeros(sb.value // 4, dtype=torch.float32, device=dev)
        scratch = torch.zeros(cb.value // 4, dtype=torch.float32, device=dev)
        pd, xd = torch.from_numpy(flat).to(dev), torch.from_numpy(x).to(dev)
        h0d = None if h0 is None else torch.from_numpy(h0).to(dev)
        logits = torch.zeros(B, C_, device=dev)
        hn = torch.zeros(L * D, B, H, device=dev)
        st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        ptr = L_.ptr
        train = int(p > 0)
        L_.check(lib.bigru_forward(plan, ptr(pd), ptr(xd), ptr(h0d), p, int(spatial), train, seed, ptr(stash), ptr(scratch),
                                   ptr(logits), ptr(hn), st), "forward")
        off = C.c_size_t()
        ys = []
        for l in range(L):
            L_.check(lib.bigru_stash_output_offset(plan, l, C.byref(off)), "stash_output_offset")
            ys.append(stash[off.value // 4: off.value // 4 + B * T * D * H].view(B, T, D * H).cpu().numpy().astype(np.float64))
        L_.check(lib.bigru_stash_argmax_offset(plan, C.byref(off)), "stash_argmax_offset")
        arg = stash.view(torch.int32)[off.value // 4: off.value // 4 + B * H].view(B, H).cpu().numpy().astype(np.int64)
        grads = torch.zeros(flat.size, device=dev)
        dx = torch.zeros(B, T, F, device=dev)
        dh0 = torch.zeros(L * D, B, H, device=dev) if h0 is not None else None
        dld = torch.from_numpy(dl).to(dev)                      # alive until the synchronize below: the backward reads it
        L_.check(lib.bigru_backward(plan, ptr(pd), ptr(xd), ptr(h0d), p, int(spatial), train, seed, ptr(stash), ptr(scratch),
                                    ptr(dld), ptr(grads), ptr(dx), ptr(dh0), st), "backward")
        torch.cuda.synchronize()
        names = param_names(plan, s)
    finally:
        lib.bigru_plan_destroy(plan)
    f64 = lambda t: None if t is None else t.cpu().numpy().astype(np.float64)   # noqa: E731
    return dict(logits=f64(logits), hn=f64(hn), ys=ys, arg=arg, grads=f64(grads), dx=f64(dx), dh0=f64(dh0)), names


def bf16(v32):
    """Round float32 to the nearest bf16 (ties to even), returned as float32."""
    u = np.ascontiguousarray(v32, np.float32).view(np.uint32)
    u = (u + np.uint32(0x7FFF) + ((u >> np.uint32(16)) & np.uint32(1))) & np.uint32(0xFFFF0000)
    return u.view(np.float32)


def mm(a, b, prec):
    """a[M,K] b[N,K]^T.  exact: float64.  fp32: float32 operands and arithmetic.  bf16 / bf16x3: float64 with both operands
    rounded as the kernels store them (fp32, then bf16 or a bf16 pair): ah bf + al bh = ah bh + ah bl + al bh, the rule
    of oracle/bigru_ref.c."""
    if prec == "exact":
        return a @ b.T
    if prec == "fp32":
        return a.astype(np.float32) @ b.astype(np.float32).T
    def split(v):
        v32 = v.astype(np.float32)
        hi = bf16(v32)
        lo = bf16(v32 - hi) if prec == "bf16x3" else np.zeros_like(hi)
        return hi.astype(np.float64) + lo, hi.astype(np.float64), lo.astype(np.float64)
    _, ah, al = split(a)
    bf, bh, _ = split(b)
    return ah @ bf.T + al @ bh.T


def stepwise(s, prec, flat, x, h0, dl, got, names):
    """The model at `prec` (mm's) run one step at a time from the kernel's own state: every step of every layer starts
    from the kernel's h_{t-1} (its Y, or h0) and the kernel's layer input (x, or the previous layer's Y), the head from
    the kernel's top-layer Y.  Rounding flips cannot compound, so what is left of the kernel's distance is the arithmetic
    of one step.  At "fp32" every operation is float32.  Returns (name, class) -> array like `tensors`: Y per layer,
    direction and step, the logits and the lin_w gradient."""
    B, T, H, L, C_, D = (s[k] for k in "BTHLCD")
    dt = np.float32 if prec == "fp32" else np.float64
    one = dt(1)
    out = {}
    sig = lambda v: one / (one + np.exp(-v))                    # noqa: E731
    inp = x.astype(dt)
    for l in range(L):
        Y = got["ys"][l].astype(dt)
        I = inp.shape[2]
        for d in range(D):
            o = names[f"l{l}d{d}.w_ih"][0]
            w_ih = flat[o:o + 3 * H * I].reshape(3 * H, I).astype(dt); o += 3 * H * I
            w_hh = flat[o:o + 3 * H * H].reshape(3 * H, H).astype(dt); o += 3 * H * H
            b_ih, b_hh = flat[o:o + 3 * H].astype(dt), flat[o + 3 * H:o + 6 * H].astype(dt)
            y = Y[:, :, d * H:(d + 1) * H]
            start = np.zeros((B, H), dt) if h0 is None else h0[l * D + d].astype(dt)
            if d == 0:
                hp = np.concatenate([start[:, None], y[:, :-1]], 1)
            else:
                hp = np.concatenate([y[:, 1:], start[:, None]], 1)
            gi = (mm(inp.reshape(B * T, I), w_ih, prec) + b_ih).reshape(B, T, 3 * H)
            gh = (mm(hp.reshape(B * T, H), w_hh, prec) + b_hh).reshape(B, T, 3 * H)
            r = sig(gi[..., :H] + gh[..., :H])
            z = sig(gi[..., H:2 * H] + gh[..., H:2 * H])
            n = np.tanh(gi[..., 2 * H:] + r * gh[..., 2 * H:])
            h = (one - z) * n + z * hp
            for t in range(T):
                out[(f"step:y[l{l}d{d},t{t}]", "y_step")] = h[:, t].astype(np.float64)
        inp = Y
    top = got["ys"][-1].astype(dt)
    pooled = top[..., :H] + top[..., H:] if D == 2 else top
    last = top[:, T - 1, :H] + (top[:, 0, H:] if D == 2 else 0)
    cat = np.concatenate([last, pooled.max(1), pooled.sum(1) / dt(T)], 1)
    o = names["lin_w"][0]
    lin_w = flat[o:o + C_ * 3 * H].reshape(C_, 3 * H).astype(dt)
    lin_b = flat[names["lin_b"][0]:names["lin_b"][0] + C_].astype(dt)
    out[("step:logits", "logits_step")] = (mm(cat, lin_w, prec) + lin_b).astype(np.float64)
    out[("step:grad:lin_w", "w_step")] = mm(dl.astype(dt).T, cat.T, prec).ravel().astype(np.float64)
    return out


def kernel_steps(got, s, names):
    """The kernel's side of stepwise."""
    H = s["H"]
    out = {}
    for l, y in enumerate(got["ys"]):
        for d in range(s["D"]):
            for t in range(s["T"]):
                out[(f"step:y[l{l}d{d},t{t}]", "y_step")] = y[:, t, d * H:(d + 1) * H]
    out[("step:logits", "logits_step")] = got["logits"]
    o, k = names["lin_w"]
    out[("step:grad:lin_w", "w_step")] = got["grads"][o:o + k]
    return out


def tensors(r, s, names):
    """(name, class) -> array of every compared tensor; y per layer and time step, hn and dh0 per layer and direction."""
    out = {("logits", "logits"): r["logits"], ("dx", "dx"): r["dx"]}
    H, T = s["H"], s["T"]
    for l, y in enumerate(r["ys"]):
        for d in range(s["D"]):
            for t in range(T):
                out[(f"y[l{l}d{d},t{t}]", "y")] = y[:, t, d * H:(d + 1) * H]
    for i in range(s["L"] * s["D"]):
        out[(f"hn[l{i // s['D']}d{i % s['D']}]", "hn")] = r["hn"][i]
        if r["dh0"] is not None:
            out[(f"dh0[l{i // s['D']}d{i % s['D']}]", "dh0")] = r["dh0"][i]
    for n, (o, k) in names.items():
        out[(f"grad:{n}", "b" if n.split(".")[-1] in ("b_ih", "b_hh", "lin_b") else "w")] = r["grads"][o:o + k]
    return out


def dist(a, b):
    """(rel-L2, max-abs / max |b|); a reference of zeros admits only zeros."""
    nb, mb = np.linalg.norm(b), np.abs(b).max()
    d = a - b
    if mb == 0:
        return (0.0, 0.0) if not d.any() else (np.inf, np.inf)
    return float(np.linalg.norm(d) / nb), float(np.abs(d).max() / mb)
