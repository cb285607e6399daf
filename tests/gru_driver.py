"""Drives the library's C ABI on one plan and takes the result apart tensor by tensor.  Test infrastructure, shared by
test_gpu_rounding_model.py, test_gpu_fp32_path.py, test_gpu_tc_steps.py, test_gpu_scan_tiles.py, test_gpu_rd_steps.py,
test_gpu_gru_steps.py and test_gpu_layer_steps.py.

A shape is a dict with B, T, F, H, L, C, D (1 or 2) and h0 (bool).  `kernel` runs bigru_forward and bigru_backward at a
precision ("fp32", "bf16" or "bf16x3"), optionally with dropout, recurrent dropout and per-sequence lengths, and returns
every layer's output, hn, the max-pool routing, the flat gradient, dx and dh0 in float64 (with regions=True also the
backward's intermediates, read through bigru_workspace_region).  `tensors` / `kernel_steps` split such a result into the per-tensor comparisons, `stepwise`
recomputes one forward step from the kernel's own state, `backward_steps` / `gemm_steps` each backward step of layer 0
and each backward GEMM from the kernel's own operands, `plane_checks` the bf16 planes bit for bit, `dist` measures two
tensors.  The models take optional recurrent-dropout masks and lengths (DESIGN.md §4.8, §4.5); without them they are the
models of the plain path, operation for operation.  With head=False the plan is a head-less one (bigru_gru_*, the nn.GRU
drop-in): the top layer's output and upstream gradient are the caller's y and dy, each layer's carry starts from the
caller's dhn, and there are no logits, pooling routing, dcat or head GEMMs.  With layer=l (kernel: the backward stops after
layer l) the backward models are those of layer l, fed that layer's operands."""
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


def param_names(plan, s, head=True):
    """name -> (offset, size) of every parameter block, from bigru_param_offset (head=False: a plan without lin_w, lin_b)."""
    lib = _pkg()._lib.load()
    out = {}
    off, rows, cols = C.c_int64(), C.c_int64(), C.c_int64()
    for l in range(s["L"] + int(head)):
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


# BIGRU_WS_* of include/bigru_b200.h
WS = dict(GATES=0, Y_PLANES=1, IN_PLANES=2, DGI=3, DGH=4, DGI_PLANES=5, DGH_PLANES=6, DY=7, DHC=8, DCAT=9)
WS_RD = dict(RD_MASK=10, RD_STATE=11)           # the regions of plans with recurrent dropout only
PLANE_REGIONS = ("Y_PLANES", "IN_PLANES", "DGI_PLANES", "DGH_PLANES")


def region(plan, which, layer):
    """bigru_workspace_region: (rc, in_scratch, byte offset, lo byte offset, pitch)."""
    lib = _pkg()._lib.load()
    sc, off, lo, pitch = C.c_int(), C.c_size_t(), C.c_size_t(), C.c_int64()
    rc = lib.bigru_workspace_region(plan, {**WS, **WS_RD}[which], layer, C.byref(sc), C.byref(off), C.byref(lo), C.byref(pitch))
    return rc, sc.value, off.value, lo.value, pitch.value


def _bits_to_f32(u16):
    """bf16 bit patterns -> the float32 values they stand for."""
    return (u16.astype(np.uint32) << np.uint32(16)).view(np.float32)


def dy_layers(L, layer):
    """The layers whose upstream gradient survives a backward stopped at `layer` (BIGRU_WS_DY of include/bigru_b200.h):
    the two ping-pong buffers hold layers 0 and 1 at stop 0, layers layer-1 and layer above it."""
    lo = layer - 1 if layer > 0 else 0
    return [l for l in (lo, lo + 1) if l < L]


def _workspace(plan, s, prec, stash, scratch, rd=False, head=True, layer=0):
    """The backward's operands and intermediates (bigru_workspace_region) as host arrays: fp32 regions as float32, planes
    as (hi, lo) pairs of bf16 bit patterns (uint16; lo None at bf16; both None at fp32, which keeps no planes).  Rows are
    split into [B, T] (and a leading D where there is one).  rd: also every layer's recurrent-dropout masks RDM [D, B, H]
    and masked state RDS [B, T, D*H] (planes, or float32 at fp32).  head=False: DCAT and the top layer's DY, which a
    head-less plan refuses (its top layer's upstream gradient is the caller's dy), are None.  layer: the layer the backward
    stopped at, whose dgi, dgh, their planes and dh_{-1} the scratch holds; XP is that layer's own input planes and DY[l]
    is None for every layer but those of dy_layers."""
    B, T, F, H, L, D = (s[k] for k in "BTFHLD")
    bufs = (stash, scratch)

    def f32(which, layer, shape):
        _, sc, off, _, _ = region(plan, which, layer)
        n = int(np.prod(shape))
        return bufs[sc][off // 4: off // 4 + n].view(*shape).cpu().numpy()

    def planes(which, layer, shape):
        if prec == "fp32":
            return None, None
        _, sc, off, lo, _ = region(plan, which, layer)
        n = int(np.prod(shape))
        v = bufs[sc].view(torch.int16)
        get = lambda o: v[o // 2: o // 2 + n].view(*shape).cpu().numpy().view(np.uint16)   # noqa: E731
        return get(off), (get(lo) if prec == "bf16x3" else None)

    pitch = region(plan, "IN_PLANES", layer)[4]
    keep = dy_layers(L, layer)
    ws = dict(G=[f32("GATES", l, (D, B, T, 4 * H)) for l in range(L)],
              YP=[planes("Y_PLANES", l, (B, T, D * H)) for l in range(L)],
              XP=planes("IN_PLANES", layer, (B, T, pitch)),
              DGI=f32("DGI", layer, (D, B, T, 3 * H)), DGH=f32("DGH", layer, (D, B, T, 3 * H)),
              DGIP=planes("DGI_PLANES", layer, (D, B, T, 3 * H)), DGHP=planes("DGH_PLANES", layer, (D, B, T, 3 * H)),
              DY=[f32("DY", l, (B, T, D * H)) if l in keep and (head or l < L - 1) else None
                  for l in range(L if layer else min(L, 2))],
              DHC=f32("DHC", layer, (D, B, H)), DCAT=f32("DCAT", L, (B, 3 * H)) if head else None)
    if rd:
        ws["RDM"] = [f32("RD_MASK", l, (D, B, H)) for l in range(L)]
        ws["RDS"] = [(f32("RD_STATE", l, (B, T, D * H)), None) if prec == "fp32" else planes("RD_STATE", l, (B, T, D * H))
                     for l in range(L)]
    return ws


def kernel(s, prec, flat, x, h0, dl, p=0.0, spatial=False, seed=0, regions=False, rd_p=0.0, lens=None, head=True, dy=None,
           dhn=None, layer=0):
    """bigru_forward_lengths + bigru_backward_lengths of shape s at precision prec on a bigru_plan_create_rd plan (p = 0:
    bigru_plan_create's plan); dropout p and recurrent dropout rd_p (training mode when either is on); lens: per-row
    lengths [B] or None.  regions: the result also holds "ws", the intermediates of _workspace.  layer > 0: the backward
    stops after that layer (bigru_plan_set_backward_stop), so that "ws" holds its intermediates; the gradients of the
    layers below are 0, and dx and their dh0 slices stay zero.
    head=False: bigru_gru_forward + bigru_gru_backward on a bigru_gru_plan_create_rd plan (flat is the recurrent prefix, dl
    and spatial are unused, p drops only between layers).  dy [B, T, D*H] is the gradient of the top layer's output (None:
    zeros, as GRU passes it), dhn [L*D, B, H] that of h_n (None: no gradient).  ys then takes the top layer from d_y, and
    the result has no logits and no arg."""
    pkg = _pkg()
    lib, L_ = pkg._lib.load(), pkg._lib
    B, T, F, H, L, C_, D = (s[k] for k in "BTFHLCD")
    plan = C.c_void_p()
    if head:
        L_.check(lib.bigru_plan_create_rd(B, T, F, H, L, C_, int(D == 2), CODE[prec], rd_p, C.byref(plan)), "plan_create")
    else:
        L_.check(lib.bigru_gru_plan_create_rd(B, T, F, H, L, int(D == 2), CODE[prec], rd_p, C.byref(plan)), "gru_plan_create")
    try:
        if layer:
            L_.check(lib.bigru_plan_set_backward_stop(plan, layer), "plan_set_backward_stop")
        sb, cb = C.c_size_t(), C.c_size_t()
        L_.check(lib.bigru_workspace_bytes(plan, C.byref(sb), C.byref(cb)), "workspace_bytes")
        dev = torch.device("cuda")
        stash = torch.zeros(sb.value // 4, dtype=torch.float32, device=dev)
        scratch = torch.zeros(cb.value // 4, dtype=torch.float32, device=dev)
        pd, xd = torch.from_numpy(flat).to(dev), torch.from_numpy(x).to(dev)
        h0d = None if h0 is None else torch.from_numpy(h0).to(dev)
        logits = torch.zeros(B, C_, device=dev) if head else None
        y = None if head else torch.zeros(B, T, D * H, device=dev)
        hn = torch.zeros(L * D, B, H, device=dev)
        st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        ptr = L_.ptr
        train = int(p > 0 or rd_p > 0)
        lend = None if lens is None else torch.from_numpy(np.asarray(lens, np.int32)).to(dev)
        if head:
            L_.check(lib.bigru_forward_lengths(plan, ptr(pd), ptr(xd), ptr(h0d), p, int(spatial), train, seed, ptr(stash),
                                               ptr(scratch), ptr(logits), ptr(hn), ptr(lend), st), "forward")
        else:
            L_.check(lib.bigru_gru_forward(plan, ptr(pd), ptr(xd), ptr(h0d), p, train, seed, ptr(stash), ptr(scratch), ptr(y),
                                           ptr(hn), ptr(lend), st), "gru_forward")
        off = C.c_size_t()
        ys = []
        for l in range(L if head else L - 1):
            L_.check(lib.bigru_stash_output_offset(plan, l, C.byref(off)), "stash_output_offset")
            ys.append(stash[off.value // 4: off.value // 4 + B * T * D * H].view(B, T, D * H).cpu().numpy().astype(np.float64))
        arg = None
        if head:
            L_.check(lib.bigru_stash_argmax_offset(plan, C.byref(off)), "stash_argmax_offset")
            arg = stash.view(torch.int32)[off.value // 4: off.value // 4 + B * H].view(B, H).cpu().numpy().astype(np.int64)
        else:
            ys.append(y.cpu().numpy().astype(np.float64))
        grads = torch.zeros(flat.size, device=dev)
        dx = torch.zeros(B, T, F, device=dev)
        dh0 = torch.zeros(L * D, B, H, device=dev) if h0 is not None else None
        if head:
            dld = torch.from_numpy(dl).to(dev)                  # alive until the synchronize below: the backward reads it
            L_.check(lib.bigru_backward_lengths(plan, ptr(pd), ptr(xd), ptr(h0d), p, int(spatial), train, seed, ptr(stash),
                                                ptr(scratch), ptr(dld), ptr(grads), ptr(dx), ptr(dh0), ptr(lend), st), "backward")
        else:
            dyd = torch.zeros(B, T, D * H, device=dev) if dy is None else torch.from_numpy(np.asarray(dy, np.float32)).to(dev)
            dhnd = None if dhn is None else torch.from_numpy(np.asarray(dhn, np.float32)).to(dev)
            L_.check(lib.bigru_gru_backward(plan, ptr(pd), ptr(xd), ptr(h0d), p, train, seed, ptr(stash), ptr(scratch), ptr(y),
                                            ptr(dyd), ptr(dhnd), ptr(grads), ptr(dx), ptr(dh0), ptr(lend), st), "gru_backward")
        torch.cuda.synchronize()
        names = param_names(plan, s, head)
        ws = _workspace(plan, s, prec, stash, scratch, rd=rd_p > 0, head=head, layer=layer) if regions else None
        del stash, scratch
    finally:
        lib.bigru_plan_destroy(plan)
    f64 = lambda t: None if t is None else t.cpu().numpy().astype(np.float64)   # noqa: E731
    out = dict(logits=f64(logits), hn=f64(hn), ys=ys, arg=arg, grads=f64(grads), dx=f64(dx), dh0=f64(dh0))
    if regions:
        out["ws"] = ws
    return out, names


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


def split(v, prec):
    """An operand as the tensor-core kernels read it, as a (hi, lo) pair of float64 arrays: exact -> (v, None); bf16 ->
    (rn_bf16(fp32 v), None); bf16x3 -> split_bf16 of tc_hopper.cuh, hi = rn_bf16(v), lo = rn_bf16(v - hi), from fp32 v."""
    if prec == "exact":
        return np.asarray(v, np.float64), None
    v32 = np.asarray(v, np.float32)
    hi = bf16(v32)
    return hi.astype(np.float64), (bf16(v32 - hi).astype(np.float64) if prec == "bf16x3" else None)


def pmm(a, b):
    """a @ b of split operands (hi, lo) in float64: ah bh + ah bl + al bh (lo None: absent), the products the bf16x3
    kernels issue; the dropped lo*lo is what split_bf16's model drops too."""
    out = a[0] @ b[0]
    if b[1] is not None:
        out += a[0] @ b[1]
    if a[1] is not None:
        out += a[1] @ b[0]
    return out


def tr(p):
    """Transpose of a split operand."""
    return p[0].T, (None if p[1] is None else p[1].T)


def f64(a):
    """float64 values of an operand array: bf16 bit patterns (uint16, a kernel's plane) or floating-point values."""
    return _bits_to_f32(a).astype(np.float64) if a.dtype == np.uint16 else np.asarray(a, np.float64)


def rows64(p, sl, cols=slice(None)):
    """Rows `sl` (and columns `cols`) of a (hi, lo) operand pair as a float64 split operand."""
    return f64(p[0][sl, cols]), (None if p[1] is None else f64(p[1][sl, cols]))


def _masked(m, v, prec):
    """m * v as the kernels form the masked state: a float32 product (in float64 at "exact")."""
    if prec == "exact":
        return np.asarray(m, np.float64) * v
    return (np.asarray(m, np.float32) * np.asarray(v, np.float32)).astype(np.float64)


def stepwise(s, prec, flat, x, h0, dl, got, names, rows=None, gates=False, masks=None, lens=None, drops=None, head=True):
    """The model at `prec` (mm's) run one step at a time from the kernel's own state: every step of every layer starts
    from the kernel's h_{t-1} (its Y, or h0) and the kernel's layer input (x, or the previous layer's Y), the head from
    the kernel's top-layer Y.  Rounding flips cannot compound, so what is left of the kernel's distance is the arithmetic
    of one step.  At "fp32" every operation is float32.  Returns (name, class) -> array like `tensors`: Y per layer,
    direction and step, the logits and the lin_w gradient.  rows: the batch rows the layers are stepped for (all when
    None; the head always takes all).  gates: also G per layer, direction and step (class g_step), the model's r, z, n and
    W_hn h_{t-1} + b_hn, which the forward scan stashes for the backward.
    masks: recurrent-dropout masks per layer [D, B, H] (DESIGN.md §4.8): gh and the carry take m * h_{t-1} (_masked).
    lens: per-row lengths [B]: a padded (row, t) has Y = 0 and no G (0 in the zeroed stash); the head pools valid steps.
    drops: per layer None or the float32 factor dropout_kernel multiplies that layer's input by.  head=False: no logits and
    no lin_w gradient (dl is unused)."""
    B, T, H, L, C_, D = (s[k] for k in "BTHLCD")
    rows = np.arange(B) if rows is None else np.asarray(rows)
    B = len(rows)
    valid = None if lens is None else (np.arange(T)[None, :] < np.asarray(lens)[rows][:, None])[..., None]
    dt = np.float32 if prec == "fp32" else np.float64
    one = dt(1)
    out = {}
    sig = lambda v: one / (one + np.exp(-v))                    # noqa: E731
    inp = x[rows].astype(dt)
    for l in range(L):
        Y = got["ys"][l][rows].astype(dt)
        if drops is not None and drops[l] is not None:
            inp = (inp.astype(np.float32) * drops[l][rows]).astype(dt)
        I = inp.shape[2]
        for d in range(D):
            o = names[f"l{l}d{d}.w_ih"][0]
            w_ih = flat[o:o + 3 * H * I].reshape(3 * H, I).astype(dt); o += 3 * H * I
            w_hh = flat[o:o + 3 * H * H].reshape(3 * H, H).astype(dt); o += 3 * H * H
            b_ih, b_hh = flat[o:o + 3 * H].astype(dt), flat[o + 3 * H:o + 6 * H].astype(dt)
            y = Y[:, :, d * H:(d + 1) * H]
            start = np.zeros((B, H), dt) if h0 is None else h0[l * D + d][rows].astype(dt)
            if d == 0:
                hp = np.concatenate([start[:, None], y[:, :-1]], 1)
            else:
                hp = np.concatenate([y[:, 1:], start[:, None]], 1)
            if masks is not None:
                hp = _masked(masks[l][d][rows][:, None, :], hp, prec).astype(dt)
            gi = (mm(inp.reshape(B * T, I), w_ih, prec) + b_ih).reshape(B, T, 3 * H)
            gh = (mm(hp.reshape(B * T, H), w_hh, prec) + b_hh).reshape(B, T, 3 * H)
            r = sig(gi[..., :H] + gh[..., :H])
            z = sig(gi[..., H:2 * H] + gh[..., H:2 * H])
            n = np.tanh(gi[..., 2 * H:] + r * gh[..., 2 * H:])
            h = (one - z) * n + z * hp
            if valid is not None:
                h = np.where(valid, h, dt(0))
            for t in range(T):
                out[(f"step:y[l{l}d{d},t{t}]", "y_step")] = h[:, t].astype(np.float64)
                if gates:
                    g = np.concatenate([r[:, t], z[:, t], n[:, t], gh[:, t, 2 * H:]], 1).astype(np.float64)
                    out[(f"step:g[l{l}d{d},t{t}]", "g_step")] = g if valid is None else np.where(valid[:, t], g, 0.0)
        inp = Y
    if not head:
        return out
    top = got["ys"][-1].astype(dt)
    pooled = top[..., :H] + top[..., H:] if D == 2 else top
    if lens is None:
        last = top[:, T - 1, :H] + (top[:, 0, H:] if D == 2 else 0)
        cat = np.concatenate([last, pooled.max(1), pooled.sum(1) / dt(T)], 1)
    else:
        # head_pool_kernel: the forward direction's last valid step, max and mean over the valid steps (padded Y is 0)
        n_b = np.asarray(lens)
        ok = (np.arange(T)[None, :] < n_b[:, None])[..., None]
        last = top[np.arange(len(n_b)), n_b - 1, :H] + (top[:, 0, H:] if D == 2 else 0)
        cat = np.concatenate([last, np.where(ok, pooled, -np.inf).max(1), pooled.sum(1) / n_b[:, None].astype(dt)], 1)
    o = names["lin_w"][0]
    lin_w = flat[o:o + C_ * 3 * H].reshape(C_, 3 * H).astype(dt)
    lin_b = flat[names["lin_b"][0]:names["lin_b"][0] + C_].astype(dt)
    out[("step:logits", "logits_step")] = (mm(cat, lin_w, prec) + lin_b).astype(np.float64)
    out[("step:grad:lin_w", "w_step")] = mm(dl.astype(dt).T, cat.T, prec).ravel().astype(np.float64)
    return out


def kernel_steps(got, s, names, rows=None, gates=False, head=True):
    """The kernel's side of stepwise."""
    H = s["H"]
    rows = np.arange(s["B"]) if rows is None else np.asarray(rows)
    out = {}
    for l, y in enumerate(got["ys"]):
        for d in range(s["D"]):
            for t in range(s["T"]):
                out[(f"step:y[l{l}d{d},t{t}]", "y_step")] = y[rows, t, d * H:(d + 1) * H]
                if gates:
                    out[(f"step:g[l{l}d{d},t{t}]", "g_step")] = got["ws"]["G"][l][d][rows, t].astype(np.float64)
    if not head:
        return out
    out[("step:logits", "logits_step")] = got["logits"]
    o, k = names["lin_w"]
    out[("step:grad:lin_w", "w_step")] = got["grads"][o:o + k]
    return out


def _block(flat, names, name, shape):
    o = names[name][0]
    return flat[o:o + int(np.prod(shape))].reshape(shape)


def head_dcat(s, prec, flat, dl, names):
    """d cat [B, 3H] = dlogits lin_w, operands split as tc_pack_kernel splits them."""
    return pmm(split(dl, prec), split(_block(flat, names, "lin_w", (s["C"], 3 * s["H"])), prec))


def head_dy(s, dcat, arg, lens=None):
    """The top layer's upstream gradient [B, T, D*H] from d cat and the max-pool routing, as head_bwd_dy_kernel routes it:
    the mean's share at every step plus the max's at the arg-max step, the same for both directions.  (The `last` share
    is the carry into the layer's last step, dcat[:, :H].)  lens: the mean's share is over len valid steps, and padded
    steps get 0 (the `last` share passes through them to t = len - 1 in the backward scan)."""
    B, T, H, D = (s[k] for k in "BTHD")
    if lens is None:
        v = np.broadcast_to(dcat[:, None, 2 * H:] / T, (B, T, H)).copy()
    else:
        v = np.broadcast_to(dcat[:, None, 2 * H:] / np.asarray(lens)[:, None, None], (B, T, H)).copy()
    v += np.where(arg[:, None, :] == np.arange(T)[None, :, None], dcat[:, None, H:2 * H], 0.0)
    if lens is not None:
        v[np.arange(T)[None, :] >= np.asarray(lens)[:, None]] = 0.0
    return np.concatenate([v] * D, 2)


def backward_steps(s, prec, flat, h0, ws, ys, names, own=False, masks=None, lens=None, head=True, dy=None, dhn=None,
                   layer=0):
    """Layer 0's backward recurrence one step at a time in float64, following gru_scan_bwd_kernel (tc_hopper.cuh), per
    direction in the kernel's step order.  Each step takes the kernel's own operands: its dY (ws["DY"][0]), its gates
    (ws["G"][0]) and its h_{t-1} (ys[0], or h0), and
        dh_t = dY_t + dh_{t+1} z_{t+1} + P_{t+1},   P_{t+1} = dgh_{t+1} W_hh  with both operands split at `prec`,
    where dgh_{t+1} is the kernel's fp32 dgh (ws["DGH"]; not its planes, which are zero at the first step, where the
    recurrence still reads the real tile).  The carry dh itself stays float64: no rounding separates it from the kernel's,
    so rounding flips cannot compound.  It starts from the head's `last` share of the kernel's dcat when layer 0 is the
    top layer, else from zero.  own: P takes the model's own dgh instead, which makes this the oracle's free-running
    backward again.  Yields ("dg", d, t, dgi, dgh) per step ([B, 3H] each: dgi's n gate is dan, dgh's is dan r) and
    ("dh0", d, None, dh_{-1}, None) after each direction's last step.
    masks: layer 0's recurrent-dropout masks [D, B, H] (DESIGN.md §4.8): the gate math takes m * h_{t-1} (_masked), and
    the carry leaving a valid step is m (dh z + P).  The dh0 item then ends in the carry before the last step's mask (the
    fp32 path masks it into dh0 later; the scans' dh_{-1} is masked).  lens: a padded step has dgi = dgh = 0 and passes the
    carry on unchanged and unmasked.
    head=False (a head-less plan): the carry of direction d starts from the caller's dhn[0*D + d] (None: zero), and when
    layer 0 is the top layer (L = 1) its dY is the caller's dy (None: zero) rather than a workspace region.
    layer: the same for layer l: its dY ws["DY"][l] (on a head-less plan's top layer the caller's dy), its gates ws["G"][l],
    its h_{t-1} from ys[l] or h0[l*D + d], W_hh of layer l; the carry starts from the head's `last` share when l = L-1, from
    dhn[l*D + d] on a head-less plan, else from zero.  masks are then layer l's."""
    B, T, H, L, D = (s[k] for k in "BTHLD")
    if head or layer < L - 1:
        dYall = ws["DY"][layer]
    else:
        dYall = np.zeros((B, T, D * H)) if dy is None else dy
    for d in range(D):
        w = split(_block(flat, names, f"l{layer}d{d}.w_hh", (3 * H, H)), prec)   # P[b, k] = sum_q dgh[b, q] W[q, k]
        G, y, dY = ws["G"][layer][d], ys[layer][:, :, d * H:(d + 1) * H], dYall[:, :, d * H:(d + 1) * H]
        if not head:
            carry = np.zeros((B, H)) if dhn is None else np.asarray(dhn[layer * D + d], np.float64)
        else:
            carry = ws["DCAT"][:, :H].astype(np.float64) if layer == L - 1 else np.zeros((B, H))
        start = np.zeros((B, H)) if h0 is None else h0[layer * D + d].astype(np.float64)
        raw = None
        for st in range(T):
            t = T - 1 - st if d == 0 else st
            first = t == (0 if d == 0 else T - 1)
            g = G[:, t].astype(np.float64)
            r, z, n, hnv = g[:, :H], g[:, H:2 * H], g[:, 2 * H:3 * H], g[:, 3 * H:]
            hp = start if first else y[:, t - 1 if d == 0 else t + 1].astype(np.float64)
            if masks is not None:
                hp = _masked(masks[d], hp, prec)
            dh = carry + dY[:, t]
            dan = dh * (1 - z) * (1 - n * n)
            dar = dan * hnv * r * (1 - r)
            daz = dh * (hp - n) * z * (1 - z)
            dgi = np.concatenate([dar, daz, dan], 1)
            dgh = np.concatenate([dar, daz, dan * r], 1)
            ok = None if lens is None else (np.asarray(lens) > t)[:, None]
            if ok is not None:
                dgi, dgh = np.where(ok, dgi, 0.0), np.where(ok, dgh, 0.0)
            yield "dg", d, t, dgi, dgh
            new = dh * z + pmm(split(dgh if own else ws["DGH"][d][:, t], prec), w)
            if masks is not None:
                raw, new = new, masks[d].astype(np.float64) * new
            if ok is not None:
                new = np.where(ok, new, carry)
                raw = None if raw is None else np.where(ok, raw, carry)
            carry = new
        yield "dh0", d, None, carry, raw


def gemm_steps(s, prec, flat, dl, h0, ops, names, arg, masks=None, lens=None, head=True, layer=0, drop=None):
    """Every backward GEMM of layer 0 and of the head in float64, from the operands the kernels read: `ops` holds the dgi
    and dgh planes (DGIP, DGHP: (hi, lo) [D, B, T, 3H]), the layer input's planes (XP [B, T, pitch]), the Y planes of layer
    0 (YP [B, T, D*H]), fp32 dgi and dgh (DGI, DGH [D, B, T, 3H]) and the kernel's dcat.  Returns (name, "gemm_step") ->
      grad:l0d{d}.w_ih   dgi planes^T input planes;
      grad:l0d{d}.w_hh   dgh planes^T Y planes shifted by one row against the step order, plus the w0 term from fp32 dgh
                         at each sequence's first step and h0 (both split as tc_pack_kernel splits them);
      grad:l0d{d}.b_ih, .b_hh   column sums of fp32 dgi, dgh;
      dx                 sum over d of dgi planes W_ih[d] (the kcat GEMM);
      dcat               dlogits lin_w;
      dy[l{L-1}]         the top layer's upstream gradient from the kernel's dcat and `arg` (when it survives the backward:
                         layers 0 and 1).
    masks: layer 0's recurrent-dropout masks [D, B, H]: dW_hh takes the masked-state planes ops["RDS"] instead of the Y
    planes, and its w0 term m * h0 (_masked).  lens: as head_dy.  head=False: no dcat and no head dy (dl, arg and
    ops["DCAT"] are unused); the top layer's upstream gradient is the caller's.
    layer: the GEMMs of layer l: XP is then its input's planes (the Y planes of layer l-1 [B, T, D*H], or its own input
    planes when its input was dropped), YP (or RDS) layer l's, h0 the whole [L*D, B, H] state (its slices l*D + d enter
    the w0 term) and masks layer l's.  Its dX is grad "dy[l{l-1}]" instead of dx.  drop: the float32 factor dropout_kernel
    multiplied the layer's input by (dropout_mask), or None: the dX GEMM's result is multiplied by it, as the in-place
    dropout backward does.  The head's dy[l{L-1}] is compared only when that layer is one of dy_layers."""
    B, T, F, H, L, D = (s[k] for k in "BTFHLD")
    BT = B * T
    I = F if layer == 0 else D * H
    flat2 = lambda p, d=None: tuple(None if a is None else (a if d is None else a[d]).reshape(BT, -1) for a in p)   # noqa: E731
    xp, yp = flat2(ops["XP"]), flat2(ops["YP"] if masks is None else ops["RDS"])
    t_of = np.arange(BT) % T
    dx = np.zeros((BT, I))
    out = {}
    for d in range(D):
        gi, gh = flat2(ops["DGIP"], d), flat2(ops["DGHP"], d)
        w_ih = split(_block(flat, names, f"l{layer}d{d}.w_ih", (3 * H, I)), prec)
        dwih, dwhh = np.zeros((3 * H, I)), np.zeros((3 * H, H))
        # K = B*T in chunks of rows, so that no float64 copy of a whole plane is made
        for r0 in range(0, BT, 8192):
            sl = slice(r0, min(BT, r0 + 8192))
            a, c = rows64(gi, sl), rows64(gh, sl)
            dwih += pmm(tr(a), rows64(xp, sl, slice(0, I)))
            # H_prev(b, t) = Y(b, t - 1) forward, Y(b, t + 1) reverse: rows shifted by one; where that leaves the sequence
            # the dgh planes are zero (and so is H_prev here)
            src = np.arange(sl.start, sl.stop) + (-1 if d == 0 else 1)
            keep = (t_of[sl] != (0 if d == 0 else T - 1))[:, None]
            hp = rows64(yp, np.clip(src, 0, BT - 1), slice(d * H, (d + 1) * H))
            dwhh += pmm(tr(c), tuple(None if v is None else v * keep for v in hp))
            dx[sl] += pmm(a, w_ih)
        if h0 is not None:
            tf = 0 if d == 0 else T - 1
            h0l = h0[layer * D + d]
            h0d = h0l if masks is None else _masked(masks[d], h0l, prec)
            dwhh += pmm(tr(split(ops["DGH"][d][:, tf], prec)), split(h0d, prec))
        pre = f"gemm:grad:l{layer}d{d}"
        out[(f"{pre}.w_ih", "gemm_step")] = dwih.ravel()
        out[(f"{pre}.w_hh", "gemm_step")] = dwhh.ravel()
        out[(f"{pre}.b_ih", "gemm_step")] = ops["DGI"][d].reshape(BT, 3 * H).astype(np.float64).sum(0)
        out[(f"{pre}.b_hh", "gemm_step")] = ops["DGH"][d].reshape(BT, 3 * H).astype(np.float64).sum(0)
    dx = dx.reshape(B, T, I)
    if drop is not None:
        dx = dx * drop
    out[(_dx_name(layer), "gemm_step")] = dx
    if not head:
        return out
    out[("gemm:dcat", "gemm_step")] = head_dcat(s, prec, flat, dl, names)
    if L - 1 in dy_layers(L, layer):
        out[(f"gemm:dy[l{L - 1}]", "gemm_step")] = head_dy(s, ops["DCAT"].astype(np.float64), arg, lens)
    return out


def _dx_name(layer):
    """The gradient layer l's dX GEMM writes: dx at layer 0, else the upstream gradient of layer l-1."""
    return "gemm:dx" if layer == 0 else f"gemm:dy[l{layer - 1}]"


def kernel_gemm_steps(got, s, names, head=True, layer=0):
    """The kernel's side of gemm_steps."""
    out = {}
    L = s["L"]
    for d in range(s["D"]):
        for nm in ("w_ih", "w_hh", "b_ih", "b_hh"):
            o, k = names[f"l{layer}d{d}.{nm}"]
            out[(f"gemm:grad:l{layer}d{d}.{nm}", "gemm_step")] = got["grads"][o:o + k]
    out[(_dx_name(layer), "gemm_step")] = got["dx"] if layer == 0 else got["ws"]["DY"][layer - 1].astype(np.float64)
    if not head:
        return out
    out[("gemm:dcat", "gemm_step")] = got["ws"]["DCAT"].astype(np.float64)
    if L - 1 in dy_layers(L, layer):
        out[(f"gemm:dy[l{L - 1}]", "gemm_step")] = got["ws"]["DY"][L - 1].astype(np.float64)
    return out


def _split_bits(v32, prec):
    """split_bf16 of float32 values as bf16 bit patterns (uint16): hi, and lo at bf16x3."""
    bits = lambda v: (v.view(np.uint32) >> np.uint32(16)).astype(np.uint16)     # noqa: E731
    hi = bf16(v32)
    return bits(hi), (bits(bf16(v32 - hi)) if prec == "bf16x3" else None)


def dropped(v, factor):
    """dropout_kernel's output restated: +0 where the element is dropped (factor 0), else the float32 product v * factor."""
    v32 = np.asarray(v, np.float32)
    return np.where(factor == 0, np.float32(0), v32 * factor).astype(np.float32)


def plane_checks(got, s, prec, x, masks=None, lens=None, drop=False, layer=0):
    """Elements (hi and lo together) where a plane the kernels wrote differs bitwise from split_bf16 of its fp32 source:
    the Y planes of every layer; layer 0's input planes (x, zero-padded to the pitch; the dropped x under dropout with a
    head, the undropped x on a head-less plan, whose dropout never touches x: pass that x); the dgi
    planes; the dgh planes, zero at each sequence's first step.  name -> count; all must be 0.
    layer: the layer the backward stopped at (kernel's layer): the dgi / dgh planes are that layer's, and its input planes
    are checked against x, the layer's dropped input dropped(Y[l-1], factor), when the layer owns them (x None: it reads
    the Y planes of layer l-1 and has none).  With h0 (got["dh0"]) the scratch's dh_{-1} must equal the caller's
    dh0[l*D + d] bit for bit.
    masks: the host restatement of the recurrent-dropout masks [L, D, B, H] (rd_masks).  Then the masks in the stash must
    equal them, RDS[l] must be split_bf16 of fp32(m * Y) (at fp32 the float32 product itself; only these two at fp32), and
    the Y planes exist only for a layer below the top whose next layer reads them (to_planes_kernel): not where that layer
    owns its input planes, as every layer above 0 does under dropout (drop).  lens: the dgi and dgh planes are zero at
    padded steps."""
    ws, T, F, H, D = got["ws"], s["T"], s["F"], s["H"], s["D"]
    bad = lambda a, b: int((a != b).sum())                                       # noqa: E731

    def cmp(pl, want):
        n = bad(pl[0], want[0])
        return n + (bad(pl[1], want[1]) if prec == "bf16x3" else 0)

    out = {}
    if masks is not None:
        for l, y in enumerate(got["ys"]):
            out[f"RD_MASK[l{l}]"] = bad(ws["RDM"][l].view(np.uint32), np.asarray(masks[l], np.float32).view(np.uint32))
            r = np.concatenate([np.asarray(masks[l][d], np.float32)[:, None, :] * y[..., d * H:(d + 1) * H].astype(np.float32)
                                for d in range(D)], 2)
            if prec == "fp32":
                out[f"RD_STATE[l{l}]"] = bad(ws["RDS"][l][0].view(np.uint32), r.view(np.uint32))
            else:
                out[f"RD_STATE[l{l}]"] = cmp(ws["RDS"][l], _split_bits(r, prec))
    if prec == "fp32":                                          # fp32 keeps no planes
        return out
    for l, y in enumerate(got["ys"]):
        if masks is None or (l + 1 < s["L"] and not drop):
            out[f"Y_PLANES[l{l}]"] = cmp(ws["YP"][l], _split_bits(y.astype(np.float32), prec))
    if x is not None:
        xw = np.zeros(ws["XP"][0].shape, np.float32)
        xw[..., :x.shape[2]] = x
        hi, lo = _split_bits(xw, prec)
        out[f"IN_PLANES[l{layer}]"] = cmp(ws["XP"], (hi, lo))
    if got["dh0"] is not None:
        out[f"DHC=dh0[l{layer}]"] = bad(ws["DHC"].astype(np.float64), got["dh0"][layer * D:(layer + 1) * D])
    padded = None if lens is None else np.arange(T)[None, :] >= np.asarray(lens)[:, None]
    want = [p.copy() if p is not None else None for p in _split_bits(ws["DGI"], prec)]
    if padded is not None:
        for p in want:
            if p is not None:
                p[:, padded] = 0
    out["DGI_PLANES"] = cmp(ws["DGIP"], want)
    want = [p.copy() if p is not None else None for p in _split_bits(ws["DGH"], prec)]
    for p in want:
        if p is not None:
            p[0, :, 0] = 0
            if s["D"] == 2:
                p[1, :, T - 1] = 0
            if padded is not None:
                p[:, padded] = 0
    out["DGH_PLANES"] = cmp(ws["DGHP"], want)
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
