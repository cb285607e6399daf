// api.cu - extern "C" entry points of libbigru_b200.so (see include/bigru_b200.h).
#include "common.cuh"
#include "kernels_f32.cuh"
#include "tc_hopper.cuh"
#include "features.cuh"
#include "infer_small.cuh"

#include <cstring>
#include <new>

static thread_local char g_err[512] = "";
void bigru_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

extern "C" const char* bigru_last_error(void) { return g_err; }
extern "C" int bigru_version(void) { return 204; }

extern "C" int bigru_device_check(int dev) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0 || dev >= n) {
        cudaGetLastError();
        bigru_set_error("no CUDA device %d (libbigru_b200 has no CPU fallback)", dev);
        return BIGRU_ERR_DEVICE;
    }
    cudaDeviceProp p;
    CUDA_TRY(cudaGetDeviceProperties(&p, dev));
    if (p.major != 9 || p.minor != 0) {
        bigru_set_error("device %d is sm_%d%d; libbigru_b200 is built for sm_90a (H100) only", dev, p.major, p.minor);
        return BIGRU_ERR_DEVICE;
    }
    return BIGRU_OK;
}

// ------------------------------------------------------------------------------------------
// workspace carve-up (fp32 path).  Offsets in floats.
// ------------------------------------------------------------------------------------------
// Tensor-core precisions add bf16 planes of the GEMM operands (hi, and lo at bf16x3; see tc_hopper.cuh) in their
// producers' layouts.  Plane offsets are rounded to 64 floats: TMA needs 16-byte aligned bases.
struct StashF32 {       // kept forward -> backward
    int64_t Y[16], G[16], X[16];   // per layer: output [B*T*D*H], gates [D][B*T][4H], dropped input [B*T*I_l]
    int64_t YP[16], XP[16];        // per layer: planes of Y [B*T][D*H] and of the layer input [B*T][in_pitch(l)]
    int64_t cat, arg, total;
};
struct ScratchF32 {
    int64_t gi, gh, dgi, dgh, dYa, dYb, dhc, dcat, csum, dgiP, dghP, tcw, part, total;
};
static inline int64_t in_pitch(const bigru_plan& p, int l) { return rup(p.in_size(l), 8); }
// floats taken by n bf16 elements per plane
static inline int64_t plane_floats(const bigru_plan& p, int64_t n) {
    return p.prec == BIGRU_PREC_FP32 ? 0 : rup((p.prec == BIGRU_PREC_BF16X3 ? 2 : 1) * n, 128) / 2;
}
static StashF32 stash_layout(const bigru_plan& p) {
    StashF32 s{};
    int64_t o = 0;
    const int64_t BT = (int64_t)p.B * p.T;
    for (int l = 0; l < p.L; ++l) {
        s.Y[l] = o; o += BT * p.D * p.H;
        s.G[l] = o; o += (int64_t)p.D * BT * 4 * p.H;
        s.X[l] = o; o += BT * p.in_size(l);
        o = rup(o, 64);
        s.YP[l] = o; o += plane_floats(p, BT * p.D * p.H);
        s.XP[l] = o; o += plane_floats(p, BT * in_pitch(p, l));
    }
    s.cat = o; o += (int64_t)p.B * 3 * p.H;
    s.arg = o; o += (int64_t)p.B * p.H;
    s.total = o;
    return s;
}
// split-K partials of the weight-gradient GEMMs of layer l (floats): dW_ih [splits][D][3H][I], dW_hh [splits][D][3H][H]
static int64_t dw_part_floats(const bigru_plan& p, int l, int64_t N) {
    const int64_t BT = (int64_t)p.B * p.T, M = 3LL * p.H;
    const int s = wg_splits(cdiv64(M, htc::WG_BM) * cdiv64(N, htc::WG_BN) * p.D, cdiv64(BT, htc::WG_BK));
    return s > 1 ? (int64_t)s * p.D * M * N : 0;
}
static ScratchF32 scratch_layout(const bigru_plan& p) {
    ScratchF32 s{};
    int64_t o = 0;
    const int64_t BT = (int64_t)p.B * p.T;
    const int64_t wide = p.D * p.H > p.F ? p.D * p.H : p.F;
    s.gi = o; o += (int64_t)p.D * BT * 3 * p.H;
    s.gh = o; o += (int64_t)p.D * p.B * 3 * p.H;
    s.dgi = o; o += (int64_t)p.D * BT * 3 * p.H;
    s.dgh = o; o += (int64_t)p.D * BT * 3 * p.H;
    s.dYa = o; o += BT * wide;
    s.dYb = o; o += BT * wide;
    s.dhc = o; o += (int64_t)p.D * p.B * p.H;
    s.dcat = o; o += (int64_t)p.B * 3 * p.H;
    s.csum = o; o += (int64_t)COLSUM_MAX_CHUNKS * (3 * p.H > p.C ? 3 * p.H : p.C);   // colsum_launch partials
    o = rup(o, 64);
    s.dgiP = o; o += plane_floats(p, (int64_t)p.D * BT * 3 * p.H);                     // planes of dgi, dgh
    s.dghP = o; o += plane_floats(p, (int64_t)p.D * BT * 3 * p.H);
    s.tcw = o;                                                                           // packed weights / head operands
    s.part = o;
    if (p.prec != BIGRU_PREC_FP32) {
        const int64_t H3 = 3LL * p.H, B = p.B, C = p.C, D = p.D;
        int64_t need = 0, part = 0;
        for (int l = 0; l < p.L; ++l) {
            const int64_t I = p.in_size(l);
            need = std::max(need, tc_pack_elems(H3, I, D, p.prec));             // W_ih, projection
            need = std::max(need, tc_pack_elems(I, H3, D, p.prec));             // W_ih^T, dX
            part = std::max(part, std::max(dw_part_floats(p, l, I), dw_part_floats(p, l, p.H)));
        }
        const int64_t h[4] = {tc_gemm_ws_elems(B, C, H3, 1, p.prec), tc_gemm_ws_elems(B, H3, C, 1, p.prec),
                              tc_gemm_ws_elems(C, H3, B, 1, p.prec), tc_gemm_ws_elems(H3, p.H, B, 1, p.prec)};   // head, w0
        for (int64_t v : h) need = std::max(need, v);
        o += plane_floats(p, need);
        s.part = o; o += part;
    }
    s.total = o;
    return s;
}

// Shapes the tensor-core scans take: 64-unit slices per CTA (clusters of H/64), 16-row batch tiles.  bf16x3 needs hi/lo
// weight pairs, which fit the 227 KB of shared memory per block up to H = 256; bf16 goes to H = 512.  The batch multiples
// are those the Python mirror pads to.
static int tc_plan_check(const bigru_plan& p) {
    if (p.prec == BIGRU_PREC_BF16X3 && ((p.H != 128 && p.H != 256) || p.B % 32 != 0)) {
        bigru_set_error("BIGRU_PREC_BF16X3 supports hidden_size 128 or 256 and batch %% 32 == 0 (got H=%d B=%d; the Python mirror pads "
                        "other batch sizes with zero rows); use BIGRU_PREC_FP32 for other shapes", p.H, p.B);
        return BIGRU_ERR_UNSUPPORTED;
    }
    if (p.prec == BIGRU_PREC_BF16 && !(((p.H == 128 || p.H == 256) && p.B % 16 == 0) || (p.H == 512 && p.B % 32 == 0))) {
        bigru_set_error("BIGRU_PREC_BF16 supports hidden_size 128 or 256 with batch %% 16 == 0 and hidden_size 512 with batch %% 32 == 0 "
                        "(got H=%d B=%d; the Python mirror pads other batch sizes with zero rows); use BIGRU_PREC_FP32 for other shapes", p.H, p.B);
        return BIGRU_ERR_UNSUPPORTED;
    }
    return BIGRU_OK;
}

// GEMMs of a plan: FFMA on the fp32 path, tensor cores (bf16 or split bf16x3 operands) on the others
static int plan_gemm(const bigru_plan& p, const GemmArgs& g, int cls, float* scratch, cudaStream_t st) {
    return p.prec == BIGRU_PREC_FP32 ? sgemm_launch(g, st)
                                     : tc_gemm_launch(g, p.prec, cls, reinterpret_cast<htc::bf16_t*>(scratch + scratch_layout(p).tcw), st);
}

// planes [depth][rows][pitch] at float offset off of buf (lo follows hi at bf16x3)
static Planes plan_planes(const bigru_plan& p, const float* buf, int64_t off, int64_t cols, int64_t rows, int64_t depth,
                          int64_t pitch) {
    const htc::bf16_t* hi = reinterpret_cast<const htc::bf16_t*>(buf + off);
    return Planes{hi, p.prec == BIGRU_PREC_BF16X3 ? hi + depth * rows * pitch : nullptr, cols, rows, depth, pitch};
}
// the layer input's planes as the projection and dW_ih read them: its own (layer 0, dropout) or the previous layer's Y
static Planes input_planes(const bigru_plan& p, const float* stash, int l, bool own) {
    const StashF32 S = stash_layout(p);
    const int64_t BT = (int64_t)p.B * p.T;
    return own ? plan_planes(p, stash, S.XP[l], p.in_size(l), BT, 1, in_pitch(p, l))
               : plan_planes(p, stash, S.YP[l - 1], (int64_t)p.D * p.H, BT, 1, (int64_t)p.D * p.H);
}
static htc::bf16_t* mut(const Planes& q) { return const_cast<htc::bf16_t*>(q.hi); }
static htc::bf16_t* mut_lo(const Planes& q) { return const_cast<htc::bf16_t*>(q.lo); }

extern "C" int bigru_plan_create(int B, int T, int F, int H, int L, int C, int bidirectional, int precision,
                                 bigru_plan** out) {
    if (!out) { bigru_set_error("plan_create: out is null"); return BIGRU_ERR_ARG; }
    if (B <= 0 || T <= 0 || F <= 0 || H <= 0 || L <= 0 || L > 16 || C <= 0) {
        bigru_set_error("plan_create: bad shape B=%d T=%d F=%d H=%d L=%d C=%d", B, T, F, H, L, C);
        return BIGRU_ERR_ARG;
    }
    if (precision != BIGRU_PREC_FP32 && precision != BIGRU_PREC_BF16 && precision != BIGRU_PREC_BF16X3) {
        bigru_set_error("plan_create: unknown precision %d", precision);
        return BIGRU_ERR_ARG;
    }
    bigru_plan* p = new (std::nothrow) bigru_plan();
    if (!p) { bigru_set_error("plan_create: out of host memory"); return BIGRU_ERR_ARG; }
    p->B = B; p->T = T; p->F = F; p->H = H; p->L = L; p->C = C; p->D = bidirectional ? 2 : 1; p->prec = precision;
    p->nparams = p->off_linb() + C;
    if (precision != BIGRU_PREC_FP32) {
        int rc = tc_plan_check(*p);
        if (rc != BIGRU_OK) { delete p; return rc; }
    }
    p->stash_bytes = (size_t)stash_layout(*p).total * sizeof(float);
    p->scratch_bytes = (size_t)scratch_layout(*p).total * sizeof(float);
    *out = p;
    return BIGRU_OK;
}

extern "C" int bigru_plan_destroy(bigru_plan* plan) { delete plan; return BIGRU_OK; }
extern "C" int64_t bigru_param_count(const bigru_plan* plan) { return plan ? plan->nparams : -1; }

extern "C" int bigru_param_offset(const bigru_plan* p, int layer, int dir, int which, int64_t* offset,
                                  int64_t* rows, int64_t* cols) {
    if (!p || !offset || !rows || !cols || layer < 0 || layer > p->L || dir < 0 || dir >= p->D || which < 0 || which > 3) {
        bigru_set_error("param_offset: bad argument");
        return BIGRU_ERR_ARG;
    }
    if (layer == p->L) {
        if (which == 0) { *offset = p->off_linw(); *rows = p->C; *cols = 3 * p->H; }
        else if (which == 2) { *offset = p->off_linb(); *rows = p->C; *cols = 1; }
        else { bigru_set_error("param_offset: linear has which 0 (weight) or 2 (bias)"); return BIGRU_ERR_ARG; }
        return BIGRU_OK;
    }
    switch (which) {
        case 0: *offset = p->off_wih(layer, dir); *rows = 3 * p->H; *cols = p->in_size(layer); break;
        case 1: *offset = p->off_whh(layer, dir); *rows = 3 * p->H; *cols = p->H; break;
        case 2: *offset = p->off_bih(layer, dir); *rows = 3 * p->H; *cols = 1; break;
        default: *offset = p->off_bhh(layer, dir); *rows = 3 * p->H; *cols = 1; break;
    }
    return BIGRU_OK;
}

extern "C" int bigru_workspace_bytes(const bigru_plan* p, size_t* stash_bytes, size_t* scratch_bytes) {
    if (!p || !stash_bytes || !scratch_bytes) { bigru_set_error("workspace_bytes: null argument"); return BIGRU_ERR_ARG; }
    *stash_bytes = p->stash_bytes;
    *scratch_bytes = p->scratch_bytes;
    return BIGRU_OK;
}

// where the head keeps argmax_t of the pooled output (int32 [B][H]) inside the stash of the last forward
extern "C" int bigru_stash_argmax_offset(const bigru_plan* p, size_t* byte_offset) {
    if (!p || !byte_offset) { bigru_set_error("stash_argmax_offset: null argument"); return BIGRU_ERR_ARG; }
    *byte_offset = (size_t)stash_layout(*p).arg * sizeof(float);
    return BIGRU_OK;
}

// where the forward keeps layer l's output Y[B][T][D*H] (fp32) inside the stash
extern "C" int bigru_stash_output_offset(const bigru_plan* p, int layer, size_t* byte_offset) {
    if (!p || !byte_offset || layer < 0 || layer >= p->L) { bigru_set_error("stash_output_offset: bad argument"); return BIGRU_ERR_ARG; }
    *byte_offset = (size_t)stash_layout(*p).Y[layer] * sizeof(float);
    return BIGRU_OK;
}

static inline unsigned nblk(int64_t n, int bs) { return (unsigned)cdiv64(n, bs); }

// ------------------------------------------------------------------------------------------
// forward (all precisions share the layout; the recurrence and the GEMMs run on tensor cores except at fp32)
// ------------------------------------------------------------------------------------------
static int forward_plan(const bigru_plan& p, const float* params, const float* x, const float* h0, float drop,
                        int spatial, int training, uint64_t seed, float* stash, float* scratch, float* logits,
                        float* hn, cudaStream_t st) {
    if (p.prec == BIGRU_PREC_BF16 && h0) {
        bigru_set_error("BIGRU_PREC_BF16: an initial hidden state is not supported; use BIGRU_PREC_FP32 or BIGRU_PREC_BF16X3");
        return BIGRU_ERR_UNSUPPORTED;
    }
    const StashF32 S = stash_layout(p);
    const ScratchF32 W = scratch_layout(p);
    const int B = p.B, T = p.T, H = p.H, D = p.D;
    const int64_t BT = (int64_t)B * T;
    const bool do_drop = training && drop > 0.f;
    const float* inp = x;
    for (int l = 0; l < p.L; ++l) {
        const int I = (int)p.in_size(l);
        if (do_drop && (l == 0 || p.L > 1)) {
            // l == 0: input dropout (elementwise or per-channel); l > 0: nn.GRU inter-layer dropout
            float* xd = stash + S.X[l];
            KLAUNCH(KC_MISC, 0.0, 0.0, st, dropout_kernel<<<132 * 8, 256, 0, st>>>(inp, xd, BT * I, T, I, l == 0 ? spatial : 0, drop, seed, (uint32_t)l));
            inp = xd;
        }
        float* Y = stash + S.Y[l];
        float* G = stash + S.G[l];
        const float* h0l = h0 ? h0 + (int64_t)l * D * B * H : nullptr;
        float* hnl = hn ? hn + (int64_t)l * D * B * H : nullptr;
        if (p.prec != BIGRU_PREC_FP32) {
            const bool own = l == 0 || do_drop;
            const Planes xp = input_planes(p, stash, l, own);
            if (own)
                KLAUNCH(KC_PACK, 0.0, 0.0, st, htc::to_planes_kernel<<<132 * 8, 256, 0, st>>>(inp, BT, I, (int)xp.pitch, mut(xp), mut_lo(xp)));
            // gi[d] = X W_ih[d]^T + b_ih[d]   for both directions
            Planes wp;
            TRY(tc_pack(params + p.off_wih(l, 0), I, 1, p.ld_block(l), 3 * H, I, D, p.prec, reinterpret_cast<htc::bf16_t*>(scratch + W.tcw),
                        &wp, st));
            {
                ProfScope ps(KC_TC_GEMM, 2.0 * BT * 3 * H * (double)I * D, 0.0, st);
                htc::WgJob j = wg_job(scratch + W.gi, (int)BT, 3 * H, 3 * H, D, cdiv64(I, htc::WG_BK));
                j.bias = params + p.off_bih(l, 0); j.zBias = p.ld_block(l); j.zC = BT * 3 * H;
                j.b.zsel = 1;
                TRY(wg_gemm(j, xp, false, wp, false, p.prec, st));
            }
            const Planes yp = plan_planes(p, stash, S.YP[l], (int64_t)D * H, BT, 1, (int64_t)D * H);
            TRY(tc_scan_fwd(p, l, scratch + W.gi, params + p.off_whh(l, 0), params + p.off_bhh(l, 0), h0l, Y, G, hnl, mut(yp), mut_lo(yp), st));
            inp = Y;
            continue;
        }
        // gi[d] = X W_ih[d]^T + b_ih[d]   for both directions
        GemmArgs g = gemm_args(inp, params + p.off_wih(l, 0), scratch + W.gi, (int)BT, 3 * H, I, I, 1, I, 1, 3 * H);
        g.bias = params + p.off_bih(l, 0);
        g.batch = D; g.zA = 0; g.zB = p.ld_block(l); g.zBias = p.ld_block(l); g.zC = BT * 3 * H;
        TRY(plan_gemm(p, g, KC_TC_GEMM, scratch, st));
        for (int s = 0; s < T; ++s) {
            // gh[d] = h_prev[d] W_hh[d]^T + b_hh[d];  h_prev rows live in Y (or h0 at s == 0)
            const float* hp; int64_t sam, zA;
            if (s == 0) { hp = h0l; sam = H; zA = (int64_t)B * H; }
            else {
                // direction 0 reads t = s-1, direction 1 reads t = T-s; express via base pointer + batch stride
                hp = Y + (int64_t)(s - 1) * D * H;
                sam = (int64_t)T * D * H;
                zA = D == 2 ? ((int64_t)(T - s) - (s - 1)) * D * H + H : 0;
            }
            GemmArgs r = gemm_args(hp, params + p.off_whh(l, 0), scratch + W.gh, B, 3 * H, hp ? H : 0, sam, 1, H, 1, 3 * H);
            r.bias = params + p.off_bhh(l, 0);
            r.batch = D; r.zA = zA; r.zB = p.ld_block(l); r.zBias = p.ld_block(l); r.zC = (int64_t)B * 3 * H;
            if (hp) { TRY(sgemm_launch(r, st)); }
            else {
                // zero initial state: gh = b_hh
                r.A = params; r.K = 1; r.sam = 0; r.sak = 1; r.zA = 0;       // dummy operand, masked out below
                r.mask_period = 1; r.mask_skip = 0;                           // every k masked -> pure bias
                TRY(sgemm_launch(r, st));
            }
            KLAUNCH(KC_GATES_FWD, 0.0, 0.0, st, gru_gates_fwd_kernel<<<nblk((int64_t)D * B * H, 256), 256, 0, st>>>(scratch + W.gi, scratch + W.gh, h0l, Y, G,
                                                                              hnl, B, T, H, D, s));
        }
        inp = Y;
    }
    const float* Ytop = stash + S.Y[p.L - 1];
    KLAUNCH(KC_HEAD, 0.0, 0.0, st, head_pool_kernel<<<nblk((int64_t)B * H, 128), 128, 0, st>>>(Ytop, stash + S.cat, (int*)(stash + S.arg), B, T, H, D));
    GemmArgs lin = gemm_args(stash + S.cat, params + p.off_linw(), logits, B, p.C, 3 * H, 3 * H, 1, 3 * H, 1, p.C);
    lin.bias = params + p.off_linb();
    TRY(plan_gemm(p, lin, KC_HEAD, scratch, st));
    return BIGRU_OK;
}

// ------------------------------------------------------------------------------------------
// backward: the head, then layers L-1 .. 0.  The upstream gradient of layer l lives in dYa when L-1-l is even, else in dYb.
// ------------------------------------------------------------------------------------------
static int backward_plan(const bigru_plan& p, const float* params, const float* x, const float* h0, float drop,
                         int spatial, int training, uint64_t seed, const float* stash, float* scratch,
                         const float* dlogits, float* grads, float* dx, float* dh0, cudaStream_t st) {
    if (p.prec == BIGRU_PREC_BF16 && (h0 || dh0)) {
        bigru_set_error("BIGRU_PREC_BF16: initial hidden state / its gradient are not supported");
        return BIGRU_ERR_UNSUPPORTED;
    }
    const StashF32 S = stash_layout(p);
    const ScratchF32 W = scratch_layout(p);
    const int B = p.B, T = p.T, H = p.H, D = p.D, C = p.C;
    const int64_t BT = (int64_t)B * T, H3 = 3LL * H;
    const bool do_drop = training && drop > 0.f;
    const bool tc = p.prec != BIGRU_PREC_FP32;
    float* dhc = scratch + W.dhc;
    CUDA_TRY(cudaMemsetAsync(grads, 0, sizeof(float) * p.nparams, st));
    // head: dcat = dlogits lin_w ; dlin_w = dlogits^T cat ; dlin_b = colsum(dlogits)
    GemmArgs a = gemm_args(dlogits, params + p.off_linw(), scratch + W.dcat, B, 3 * H, C, C, 1, 1, 3 * H, 3 * H);
    TRY(plan_gemm(p, a, KC_HEAD, scratch, st));
    GemmArgs w = gemm_args(dlogits, stash + S.cat, grads + p.off_linw(), C, 3 * H, B, 1, C, 1, 3 * H, 3 * H);
    TRY(plan_gemm(p, w, KC_HEAD, scratch, st));
    TRY(colsum_launch(dlogits, grads + p.off_linb(), B, C, C, 1, 0, 0, scratch + W.csum, st));
    KLAUNCH(KC_HEAD, 0.0, 0.0, st, head_bwd_dy_kernel<<<nblk(BT * H, 256), 256, 0, st>>>(scratch + W.dcat, (const int*)(stash + S.arg), scratch + W.dYa, dhc, B, T, H, D));
    for (int l = p.L - 1; l >= 0; --l) {
        const int I = (int)p.in_size(l);
        const bool even = (p.L - 1 - l) % 2 == 0;
        const bool drop_l = do_drop && (l == 0 || p.L > 1);
        float* dY = scratch + (even ? W.dYa : W.dYb);
        float* dYnext = scratch + (even ? W.dYb : W.dYa);
        const float* Y = stash + S.Y[l];
        const float* G = stash + S.G[l];
        const float* h0l = h0 ? h0 + (int64_t)l * D * B * H : nullptr;
        float* dgi = scratch + W.dgi;
        float* dgh = scratch + W.dgh;
        if (l != p.L - 1) CUDA_TRY(cudaMemsetAsync(dhc, 0, sizeof(float) * D * B * H, st));
        const Planes gip = plan_planes(p, scratch, W.dgiP, H3, BT, D, H3);
        const Planes ghp = plan_planes(p, scratch, W.dghP, H3, BT, D, H3);
        // recurrence: dgi, dgh [D][B*T][3H] and dh0 in dhc
        if (tc) {
            TRY(tc_scan_bwd(p, l, G, Y, h0l, dY, dhc, dgi, dgh, params + p.off_whh(l, 0), mut(gip), mut_lo(gip), mut(ghp), mut_lo(ghp), st));
        } else {
            for (int s = 0; s < T; ++s) {
                KLAUNCH(KC_GATES_BWD, 0.0, 0.0, st, gru_gates_bwd_kernel<<<nblk((int64_t)D * B * H, 256), 256, 0, st>>>(G, Y, h0l, dY, dhc, dgi, dgh, B, T, H, D, s));
                // dhc[d] += dgh_t[d] W_hh[d]   (rows t: dir0 -> T-1-s, dir1 -> s)
                const int t0 = T - 1 - s, t1 = s;
                GemmArgs r = gemm_args(dgh + (int64_t)t0 * 3 * H, params + p.off_whh(l, 0), dhc, B, H, 3 * H,
                                       (int64_t)T * 3 * H, 1, 1, H, H);
                r.beta = 1; r.batch = D;
                r.zA = BT * 3 * H + (int64_t)(t1 - t0) * 3 * H; r.zB = p.ld_block(l); r.zC = (int64_t)B * H;
                TRY(sgemm_launch(r, st));
            }
        }
        if (dh0) CUDA_TRY(cudaMemcpyAsync(dh0 + (int64_t)l * D * B * H, dhc, sizeof(float) * D * B * H,
                                          cudaMemcpyDeviceToDevice, st));
        // dW_ih[d] = dgi[d]^T X and dW_hh[d] = dgh[d]^T H_prev, H_prev(b,t) = Y[b,t-1] (dir 0) / Y[b,t+1] (dir 1), the columns
        // of direction d.  The first step's h_prev is h0: its term is the w0 GEMM below.
        if (tc) {
            const int64_t kb = cdiv64(BT, htc::WG_BK);
            float* part = scratch + W.part;
            {
                ProfScope ps(KC_TC_GEMM_DWIH, 2.0 * H3 * I * (double)BT * D, 0.0, st);
                htc::WgJob j = wg_job(grads + p.off_wih(l, 0), (int)H3, I, I, D, kb);
                j.zC = p.ld_block(l); j.a.zsel = 1; j.part = part;
                j.splits = wg_splits(cdiv64(H3, htc::WG_BM) * cdiv64(I, htc::WG_BN) * D, kb);
                TRY(wg_gemm(j, gip, true, input_planes(p, stash, l, l == 0 || do_drop), true, p.prec, st));
            }
            // the dgh planes are zero at each sequence's first step, so the ±1-row shift needs no mask
            if (T > 1) {
                ProfScope ps(KC_TC_GEMM_DWHH, 2.0 * H3 * H * (double)BT * D, 0.0, st);
                htc::WgJob j = wg_job(grads + p.off_whh(l, 0), (int)H3, H, H, D, kb);
                j.zC = p.ld_block(l); j.a.zsel = 1; j.part = part;
                j.b.coff = H; j.b.kshift[0] = -1; j.b.kshift[1] = 1;
                j.splits = wg_splits(cdiv64(H3, htc::WG_BM) * cdiv64(H, htc::WG_BN) * D, kb);
                TRY(wg_gemm(j, ghp, true, plan_planes(p, stash, S.YP[l], (int64_t)D * H, BT, 1, (int64_t)D * H), true, p.prec, st));
            }
        } else {
            // the layer input as the projection saw it (the dropped copy when dropout was applied)
            const float* inp = drop_l ? stash + S.X[l] : l == 0 ? x : stash + S.Y[l - 1];
            const int splitk = (int)min((int64_t)64, max((int64_t)1, BT / 512));
            for (int d = 0; d < D; ++d) {
                const float* dgi_d = dgi + (int64_t)d * BT * 3 * H;
                const float* dgh_d = dgh + (int64_t)d * BT * 3 * H;
                GemmArgs wi = gemm_args(dgi_d, inp, grads + p.off_wih(l, d), 3 * H, I, (int)BT, 1, 3 * H, 1, I, I);
                wi.splitk = splitk;
                TRY(sgemm_launch(wi, st));
                if (T > 1) {
                    const float* hp = Y + (int64_t)d * H + (d == 0 ? -(int64_t)D * H : (int64_t)D * H);
                    GemmArgs wh = gemm_args(dgh_d, hp, grads + p.off_whh(l, d), 3 * H, H, (int)BT, 1, 3 * H, 1,
                                            (int64_t)D * H, H);
                    wh.splitk = splitk; wh.mask_period = T; wh.mask_skip = d == 0 ? 0 : T - 1;
                    TRY(sgemm_launch(wh, st));
                }
            }
        }
        // dW_hh[d] += dgh[d]_first^T h0[d]; bias gradients are column sums of dgi and dgh
        for (int d = 0; d < D; ++d) {
            const float* dgi_d = dgi + (int64_t)d * BT * 3 * H;
            const float* dgh_d = dgh + (int64_t)d * BT * 3 * H;
            if (h0l) {
                const int tf = d == 0 ? 0 : T - 1;
                GemmArgs w0 = gemm_args(dgh_d + (int64_t)tf * 3 * H, h0l + (int64_t)d * B * H, grads + p.off_whh(l, d),
                                        3 * H, H, B, 1, (int64_t)T * 3 * H, 1, H, H);
                w0.beta = 1;
                TRY(plan_gemm(p, w0, KC_TC_GEMM_DWHH, scratch, st));
            }
            TRY(colsum_launch(dgi_d, grads + p.off_bih(l, d), BT, 3 * H, 3 * H, 1, 0, 0, scratch + W.csum, st));
            TRY(colsum_launch(dgh_d, grads + p.off_bhh(l, d), BT, 3 * H, 3 * H, 1, 0, 0, scratch + W.csum, st));
        }
        // dX = sum_d dgi[d] W_ih[d]
        float* dxo = l == 0 ? dx : dYnext;
        if (!dxo) continue;
        if (tc) {
            // one K loop over direction 0, then direction 1
            Planes wp;
            TRY(tc_pack(params + p.off_wih(l, 0), 1, I, p.ld_block(l), I, 3 * H, D, p.prec, reinterpret_cast<htc::bf16_t*>(scratch + W.tcw),
                        &wp, st));
            ProfScope ps(KC_TC_GEMM_DX, 2.0 * BT * I * (double)H3 * D, 0.0, st);
            htc::WgJob j = wg_job(dxo, (int)BT, I, I, 1, D * (H3 / htc::WG_BK));
            j.kbd = (int)(H3 / htc::WG_BK); j.kcat = 1; j.a.zsel = 1; j.b.zsel = 1;
            TRY(wg_gemm(j, gip, false, wp, false, p.prec, st));
        } else {
            for (int d = 0; d < D; ++d) {
                GemmArgs gx = gemm_args(dgi + (int64_t)d * BT * 3 * H, params + p.off_wih(l, d), dxo, (int)BT, I, 3 * H,
                                        3 * H, 1, 1, I, I);
                gx.beta = d;
                TRY(sgemm_launch(gx, st));
            }
        }
        // d(dropout): the same mask, in place (dropout_kernel multiplies by mask / (1 - p))
        if (drop_l)
            KLAUNCH(KC_MISC, 0.0, 0.0, st, dropout_kernel<<<132 * 8, 256, 0, st>>>(dxo, dxo, BT * I, T, I, l == 0 ? spatial : 0, drop, seed, (uint32_t)l));
    }
    return BIGRU_OK;
}

// ------------------------------------------------------------------------------------------
// exported compute entry points
// ------------------------------------------------------------------------------------------
extern "C" int bigru_forward(const bigru_plan* plan, const float* d_params, const float* d_x, const float* d_h0,
                             float dropout_p, int spatial, int training, uint64_t seed, void* d_stash,
                             void* d_scratch, float* d_logits, float* d_hn, void* stream) {
    if (!plan || !d_params || !d_x || !d_stash || !d_scratch || !d_logits) {
        bigru_set_error("forward: null argument");
        return BIGRU_ERR_ARG;
    }
    if (dropout_p < 0.f || dropout_p >= 1.f) { bigru_set_error("forward: dropout_p must be in [0,1)"); return BIGRU_ERR_ARG; }
    return forward_plan(*plan, d_params, d_x, d_h0, dropout_p, spatial, training, seed, (float*)d_stash,
                        (float*)d_scratch, d_logits, d_hn, (cudaStream_t)stream);
}

extern "C" int bigru_backward(const bigru_plan* plan, const float* d_params, const float* d_x, const float* d_h0,
                              float dropout_p, int spatial, int training, uint64_t seed, const void* d_stash,
                              void* d_scratch, const float* d_dlogits, float* d_grads, float* d_dx, float* d_dh0,
                              void* stream) {
    if (!plan || !d_params || !d_x || !d_stash || !d_scratch || !d_dlogits || !d_grads) {
        bigru_set_error("backward: null argument");
        return BIGRU_ERR_ARG;
    }
    return backward_plan(*plan, d_params, d_x, d_h0, dropout_p, spatial, training, seed, (const float*)d_stash,
                         (float*)d_scratch, d_dlogits, d_grads, d_dx, d_dh0, (cudaStream_t)stream);
}

extern "C" int bigru_chunk_minmax(const float* d_table, int64_t N, int F, int64_t row_lo, int64_t row_hi, float* d_min,
                                  float* d_max, void* stream) {
    if (!d_table || !d_min || !d_max || F <= 0 || row_lo < 0 || row_hi > N || row_lo >= row_hi) {
        bigru_set_error("chunk_minmax: bad argument");
        return BIGRU_ERR_ARG;
    }
    KLAUNCH(KC_GATHER, 0.0, 4.0 * (row_hi - row_lo) * F, (cudaStream_t)stream,
            chunk_minmax_kernel<<<(F + 31) / 32, dim3(32, 8), 0, (cudaStream_t)stream>>>(d_table, F, row_lo, row_hi, d_min, d_max));
    return BIGRU_OK;
}

extern "C" int bigru_window_features(const float* d_close, const float* d_high, const float* d_low, const float* d_volume,
                                     const float* d_delta, int64_t n, const int* vol_periods, int n_vol, const int* price_periods,
                                     int n_price, const int* delta_periods, int n_delta, int bb_period, float bb_std, int stochastic,
                                     float n1, float n2, float* d_out, float* d_targets, int* n_out, void* stream) {
    if (n_vol < 0 || n_vol > 8 || n_price < 0 || n_price > 8 || n_delta < 0 || n_delta > 8 || bb_period < 0 || n < 0 ||
        (n_vol && !vol_periods) || (n_price && !price_periods) || (n_delta && !delta_periods)) {
        bigru_set_error("window_features: bad argument (at most 8 periods per list)");
        return BIGRU_ERR_ARG;
    }
    FeatureCfg cfg{};
    cfg.n_vol = n_vol; cfg.n_price = n_price; cfg.n_delta = n_delta;
    for (int i = 0; i < n_vol; ++i) cfg.vol_p[i] = vol_periods[i];
    for (int i = 0; i < n_price; ++i) cfg.price_p[i] = price_periods[i];
    for (int i = 0; i < n_delta; ++i) cfg.delta_p[i] = delta_periods[i];
    for (int i = 0; i < 8; ++i)
        if ((i < n_vol && cfg.vol_p[i] < 1) || (i < n_price && cfg.price_p[i] < 1) || (i < n_delta && cfg.delta_p[i] < 1)) {
            bigru_set_error("window_features: periods must be >= 1");
            return BIGRU_ERR_ARG;
        }
    cfg.bb_period = bb_period; cfg.bb_std = bb_std; cfg.stochastic = stochastic ? 1 : 0; cfg.n1 = n1; cfg.n2 = n2;
    cfg.n_out = (bb_period > 0 ? 2 : 0) + n_vol + n_price + n_delta + (stochastic ? 1 : 0) + 2;
    if (n_out) *n_out = cfg.n_out;
    if (!d_out || n == 0) return BIGRU_OK;
    if (!d_close || !d_high || !d_low || (n_vol && !d_volume) || (n_delta && !d_delta)) {
        bigru_set_error("window_features: null column");
        return BIGRU_ERR_ARG;
    }
    int halo = 14;
    for (int i = 0; i < n_vol; ++i) halo = std::max(halo, cfg.vol_p[i] - 1);
    for (int i = 0; i < n_price; ++i) halo = std::max(halo, cfg.price_p[i] - 1);
    for (int i = 0; i < n_delta; ++i) halo = std::max(halo, cfg.delta_p[i] - 1);
    halo = std::max(halo, bb_period - 1);
    if (halo > 4095) { bigru_set_error("window_features: periods above 4096 rows are not supported"); return BIGRU_ERR_UNSUPPORTED; }
    const int span = FEAT_TR + halo;
    const size_t smem = sizeof(float) * ((size_t)4 * span + 16 + (size_t)FEAT_TR * (cfg.n_out + 4));
    // the reference's own configuration (config.py:40-49) runs with compile-time periods
    const bool fast = n_vol == 2 && cfg.vol_p[0] == 6 && cfg.vol_p[1] == 20 && n_price == 1 && cfg.price_p[0] == 20 && n_delta == 1 &&
                      cfg.delta_p[0] == 12 && bb_period == 20 && stochastic;
    if (smem > 48 * 1024)        // per-device opt-in, set on every call (no process-wide cache: a second GPU would miss it)
        CUDA_TRY(fast ? cudaFuncSetAttribute(window_features_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)
                      : cudaFuncSetAttribute(window_features_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const unsigned blocks = (unsigned)std::min<int64_t>((n + FEAT_TR - 1) / FEAT_TR, 132 * 8);
    if (fast)
        KLAUNCH(KC_GATHER, 0.0, 4.0 * n * (5 + cfg.n_out + 4), (cudaStream_t)stream,
                window_features_kernel<true><<<blocks, FEAT_TR, smem, (cudaStream_t)stream>>>(d_close, d_high, d_low, d_volume, d_delta, n, cfg,
                                                                                              halo, d_out, d_targets));
    else
        KLAUNCH(KC_GATHER, 0.0, 4.0 * n * (5 + cfg.n_out + 4), (cudaStream_t)stream,
                window_features_kernel<false><<<blocks, FEAT_TR, smem, (cudaStream_t)stream>>>(d_close, d_high, d_low, d_volume, d_delta, n, cfg,
                                                                                               halo, d_out, d_targets));
    return BIGRU_OK;
}

extern "C" int bigru_infer_window(const float* d_params, const float* d_x, const float* d_xmin, const float* d_xmax, int B, int T,
                                  int F, int H, int L, int C, int bidirectional, float* d_logits, float* d_probs, void* stream) {
    if (!d_params || !d_x || !d_logits || B <= 0 || T <= 0 || F <= 0 || H <= 0 || L <= 0 || C <= 0 || ((d_xmin == nullptr) != (d_xmax == nullptr))) {
        bigru_set_error("infer_window: bad argument");
        return BIGRU_ERR_ARG;
    }
    const int D = bidirectional ? 2 : 1, DH = D * H, W = F > DH ? F : DH;
    const size_t smem = sizeof(float) * ((size_t)T * W + (size_t)T * DH + 2 * (size_t)DH + 3 * (size_t)H);
    if (DH > 1024 || smem > 200 * 1024) {
        bigru_set_error("infer_window: window too large for the single-CTA path (D*H=%d, %zu bytes of shared memory); use bigru_forward", DH, smem);
        return BIGRU_ERR_UNSUPPORTED;
    }
    if (smem > 48 * 1024)
        CUDA_TRY(cudaFuncSetAttribute(infer_window_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int threads = std::max(32, ((DH + 31) / 32) * 32);
    KLAUNCH(KC_MISC, 0.0, 0.0, (cudaStream_t)stream,
            infer_window_kernel<<<B, threads, smem, (cudaStream_t)stream>>>(d_params, d_x, d_xmin, d_xmax, T, F, H, L, C, D, d_logits, d_probs));
    return BIGRU_OK;
}

extern "C" int bigru_loss(int kind, const float* d_logits, const void* d_target, const float* d_weight,
                          const float* d_pos_weight, int B, int C, double denom, float* d_loss, float* d_dlogits,
                          void* stream) {
    if (!d_logits || !d_target || !d_loss || B <= 0 || C <= 0 || denom <= 0 || kind < 0 || kind > 2) {
        bigru_set_error("loss: bad argument");
        return BIGRU_ERR_ARG;
    }
    cudaStream_t st = (cudaStream_t)stream;
    CUDA_TRY(cudaMemsetAsync(d_loss, 0, sizeof(float), st));
    if (kind == BIGRU_LOSS_MLSM) { d_weight = nullptr; d_pos_weight = nullptr; }
    KLAUNCH(KC_LOSS, 0.0, 0.0, st, loss_kernel<<<1, 256, 0, st>>>(kind, d_logits, d_target, d_weight, d_pos_weight, B, C,
                                             (float)(1.0 / denom), d_loss, d_dlogits));
    return BIGRU_OK;
}

extern "C" int bigru_sqnorm(const float* d_g, int64_t n, float* d_out, float* d_ws, void* stream) {
    if (!d_g || !d_out || !d_ws || n < 0) { bigru_set_error("sqnorm: bad argument"); return BIGRU_ERR_ARG; }
    if (n == 0) return BIGRU_OK;
    const int blocks = (int)min((int64_t)BIGRU_SQNORM_WS, cdiv64(n, 256));
    KLAUNCH(KC_OPTIM, 0.0, 0.0, (cudaStream_t)stream, sqnorm_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(d_g, n, d_ws));
    KLAUNCH(KC_OPTIM, 0.0, 0.0, (cudaStream_t)stream, sqnorm_finish_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(d_ws, blocks, d_out));
    return BIGRU_OK;
}

extern "C" int bigru_adam_tick(int* d_step, float* d_sqnorm, void* stream) {
    if (!d_step || !d_sqnorm) { bigru_set_error("adam_tick: null argument"); return BIGRU_ERR_ARG; }
    KLAUNCH(KC_OPTIM, 0.0, 0.0, (cudaStream_t)stream, adam_tick_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(d_step, d_sqnorm));
    return BIGRU_OK;
}

extern "C" int bigru_clip_adam_step_dev(float* d_params, float* d_grads, float* d_m, float* d_v, int64_t n,
                                        const float* d_sqnorm, float clip, float lr, float b1, float b2, float eps,
                                        const int* d_step, float grad_scale, void* stream) {
    if (!d_params || !d_grads || !d_m || !d_v || !d_sqnorm || !d_step || n <= 0) {
        bigru_set_error("clip_adam_step_dev: bad argument");
        return BIGRU_ERR_ARG;
    }
    const unsigned blocks = (unsigned)min((int64_t)132 * 8, cdiv64(n, 256));
    KLAUNCH(KC_OPTIM, 0.0, 0.0, (cudaStream_t)stream, clip_adam_dev_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(d_params, d_grads, d_m, d_v, n, d_sqnorm, clip,
                                                                    lr, b1, b2, eps, d_step, grad_scale));
    return BIGRU_OK;
}

extern "C" int bigru_window_gather_norm(const float* d_src, const float* d_xmin, const float* d_xmax, int64_t start,
                                        int64_t N, int B, int T, int F, float* d_out, void* stream) {
    if (B == 0 && T > 0 && F > 0 && start >= 0) return BIGRU_OK;          // empty batch: nothing to write
    if (!d_src || !d_out || B < 0 || T <= 0 || F <= 0 || start < 0 || (B > 0 && start + B + T - 1 > N) ||
        ((d_xmin == nullptr) != (d_xmax == nullptr))) {
        bigru_set_error("window_gather_norm: bad argument (start=%lld B=%d T=%d N=%lld)", (long long)start, B, T, (long long)N);
        return BIGRU_ERR_ARG;
    }
    cudaStream_t st = (cudaStream_t)stream;
    const bool vec = F % 4 == 0 && ((uintptr_t)d_src % 16 == 0) && ((uintptr_t)d_out % 16 == 0) &&
                     (!d_xmin || (((uintptr_t)d_xmin % 16 == 0) && ((uintptr_t)d_xmax % 16 == 0)));
    const int64_t total = (int64_t)B * T * (vec ? F / 4 : F);
    const unsigned blocks = (unsigned)min((int64_t)132 * 16, cdiv64(total, 256));
    // algorithmic bytes: write B*T*F floats, read the (B+T-1)*F source rows once (SURVEY.md 8(d))
    const double bytes = 4.0 * ((double)B * T * F + (double)(B + T - 1) * F);
    if (vec) KLAUNCH(KC_GATHER, 0.0, bytes, st, window_gather_kernel<4><<<blocks, 256, 0, st>>>(d_src, d_xmin, d_xmax, start, B, T, F, d_out));
    else KLAUNCH(KC_GATHER, 0.0, bytes, st, window_gather_kernel<1><<<blocks, 256, 0, st>>>(d_src, d_xmin, d_xmax, start, B, T, F, d_out));
    return BIGRU_OK;
}

extern "C" int bigru_window_targets(const float* d_y, int64_t start, int64_t N, int B, int T, int C, float* d_out,
                                    void* stream) {
    if (B == 0 && T > 0 && C > 0 && start >= 0) return BIGRU_OK;
    if (!d_y || !d_out || B < 0 || T <= 0 || C <= 0 || start < 0 || (B > 0 && start + B + T - 1 > N)) {
        bigru_set_error("window_targets: bad argument");
        return BIGRU_ERR_ARG;
    }
    if (B == 0) return BIGRU_OK;
    KLAUNCH(KC_GATHER, 0.0, 0.0, (cudaStream_t)stream, window_targets_kernel<<<nblk((int64_t)B * C, 256), 256, 0, (cudaStream_t)stream>>>(d_y, start, B, T, C, d_out));
    return BIGRU_OK;
}

extern "C" int bigru_multilabel_counts(const float* d_logits, const float* d_target, int B, int C,
                                       long long* d_counts, void* stream) {
    if (!d_logits || !d_target || !d_counts || B <= 0 || C <= 0) { bigru_set_error("multilabel_counts: bad argument"); return BIGRU_ERR_ARG; }
    KLAUNCH(KC_MISC, 0.0, 0.0, (cudaStream_t)stream, multilabel_counts_kernel<<<nblk(B, 128), 128, 0, (cudaStream_t)stream>>>(d_logits, d_target, B, C,
                                                                            (unsigned long long*)d_counts));
    return BIGRU_OK;
}

// ------------------------------------------------------------------------------------------
// measurement hooks (bench.py): launch counter and per-kernel-class CUDA-event timing
// ------------------------------------------------------------------------------------------
extern "C" long long bigru_launch_count(void) { return profiler().launches.load(); }
// kernels replayed through a captured CUDA graph do not pass the launch macros: the caller reports them (n per replay)
extern "C" void bigru_launch_count_add(long long n) { profiler().launches.fetch_add(n, std::memory_order_relaxed); }

extern "C" int bigru_prof_enable(int on) {
    Profiler& p = profiler();
    std::lock_guard<std::mutex> g(p.mu);
    for (auto& r : p.recs) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
    p.recs.clear();
    p.enabled.store(on ? 1 : 0);
    return BIGRU_OK;
}

extern "C" int bigru_prof_classes(void) { return KC_COUNT; }
extern "C" const char* bigru_prof_class_name(int cls) { return cls >= 0 && cls < KC_COUNT ? kKClassNames[cls] : ""; }

// Sums the recorded launches of class `cls` (synchronises on their events).
extern "C" int bigru_prof_report(int cls, double* ms, long long* launches, double* flops, double* bytes) {
    if (cls < 0 || cls >= KC_COUNT || !ms || !launches || !flops || !bytes) { bigru_set_error("prof_report: bad argument"); return BIGRU_ERR_ARG; }
    Profiler& p = profiler();
    std::lock_guard<std::mutex> g(p.mu);
    *ms = 0; *launches = 0; *flops = 0; *bytes = 0;
    for (auto& r : p.recs) {
        if (r.cls != cls) continue;
        CUDA_TRY(cudaEventSynchronize(r.b));
        float t = 0.f;
        CUDA_TRY(cudaEventElapsedTime(&t, r.a, r.b));
        *ms += t; *launches += 1; *flops += r.flops; *bytes += r.bytes;
    }
    return BIGRU_OK;
}
