// kernels_f32.cuh - the fp32 (FFMA) path: strided SGEMM, GRU gate math forward/backward,
// pooling head, losses, clip+Adam, window gather, dropout.  This is the parity path
// (BIGRU_PREC_FP32); the tensor-core precisions reuse the layout, head, loss and optimiser kernels.
#pragma once
#include "common.cuh"

// ------------------------------------------------------------------------------------------
// Generic strided SGEMM:  C[z][m,n] (+)= sum_k A(m,k) * B(n,k) (+ bias[n])
//   A(m,k) = A[m*sam + k*sak],  B(n,k) = B[n*sbn + k*sbk]; covers NT / NN / TN by strides.
//   splitk > 1: partial sums are atomically added (C pre-initialised by the caller).
//   mask_period > 0: reduction rows k with (k % mask_period) == mask_skip contribute nothing and
//   are never loaded (used for the time-shifted h_{t-1} operand of dW_hh).
// ------------------------------------------------------------------------------------------
struct GemmArgs {
    const float* A; const float* B; float* C; const float* bias;
    int M, N, K;
    int64_t sam, sak, sbn, sbk, ldc;
    int64_t zA, zB, zC, zBias;
    int batch, splitk, beta;
    int mask_period, mask_skip;
};

template <int BM, int BN, int BK, int TM, int TN>
__global__ void __launch_bounds__((BM / TM) * (BN / TN)) sgemm_kernel(GemmArgs g) {
    constexpr int NT = (BM / TM) * (BN / TN);
    __shared__ float As[BK][BM + 4];
    __shared__ float Bs[BK][BN + 4];
    const int zb = blockIdx.z / g.splitk, zs = blockIdx.z % g.splitk;
    const float* __restrict__ A = g.A + zb * g.zA;
    const float* __restrict__ B = g.B + zb * g.zB;
    float* __restrict__ C = g.C + zb * g.zC;
    const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
    const int kchunk = ((g.K + g.splitk - 1) / g.splitk + BK - 1) / BK * BK;
    const int kbeg = zs * kchunk;
    const int kend = min(g.K, kbeg + kchunk);
    const int tid = threadIdx.x;
    const int ty = tid / (BN / TN), tx = tid % (BN / TN);
    float acc[TM][TN];
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

    for (int k0 = kbeg; k0 < kend; k0 += BK) {
#pragma unroll 4
        for (int i = tid; i < BM * BK; i += NT) {
            int m, k;
            if (g.sak == 1) { m = i / BK; k = i % BK; } else { k = i / BM; m = i % BM; }
            const int gm = m0 + m, gk = k0 + k;
            float v = 0.f;
            if (gm < g.M && gk < kend && !(g.mask_period && (gk % g.mask_period) == g.mask_skip))
                v = A[(int64_t)gm * g.sam + (int64_t)gk * g.sak];
            As[k][m] = v;
        }
#pragma unroll 4
        for (int i = tid; i < BN * BK; i += NT) {
            int n, k;
            if (g.sbk == 1) { n = i / BK; k = i % BK; } else { k = i / BN; n = i % BN; }
            const int gn = n0 + n, gk = k0 + k;
            float v = 0.f;
            if (gn < g.N && gk < kend && !(g.mask_period && (gk % g.mask_period) == g.mask_skip))
                v = B[(int64_t)gn * g.sbn + (int64_t)gk * g.sbk];
            Bs[k][n] = v;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            float a[TM], b[TN];
#pragma unroll
            for (int i = 0; i < TM; ++i) a[i] = As[k][ty * TM + i];
#pragma unroll
            for (int j = 0; j < TN; ++j) b[j] = Bs[k][tx * TN + j];
#pragma unroll
            for (int i = 0; i < TM; ++i)
#pragma unroll
                for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
    }
    const float* bias = g.bias ? g.bias + zb * g.zBias : nullptr;
#pragma unroll
    for (int i = 0; i < TM; ++i) {
        const int gm = m0 + ty * TM + i;
        if (gm >= g.M) continue;
#pragma unroll
        for (int j = 0; j < TN; ++j) {
            const int gn = n0 + tx * TN + j;
            if (gn >= g.N) continue;
            float v = acc[i][j];
            if (bias && zs == 0) v += bias[gn];
            float* c = C + (int64_t)gm * g.ldc + gn;
            if (g.splitk > 1) atomicAdd(c, v);
            else if (g.beta) *c += v;
            else *c = v;
        }
    }
}

static inline GemmArgs gemm_args(const float* A, const float* B, float* C, int M, int N, int K,
                                 int64_t sam, int64_t sak, int64_t sbn, int64_t sbk, int64_t ldc) {
    GemmArgs g{};
    g.A = A; g.B = B; g.C = C; g.bias = nullptr; g.M = M; g.N = N; g.K = K;
    g.sam = sam; g.sak = sak; g.sbn = sbn; g.sbk = sbk; g.ldc = ldc;
    g.zA = g.zB = g.zC = g.zBias = 0; g.batch = 1; g.splitk = 1; g.beta = 0;
    g.mask_period = 0; g.mask_skip = 0;
    return g;
}

static int sgemm_launch(const GemmArgs& g, cudaStream_t st) {
    if (g.M <= 0 || g.N <= 0 || g.K <= 0) return BIGRU_OK;
    ProfScope ps(KC_SGEMM, 2.0 * g.M * g.N * (double)g.K * g.batch, 0.0, st);
    const int64_t big_tiles = cdiv64(g.M, 128) * cdiv64(g.N, 128) * g.batch * g.splitk;
    const bool big = big_tiles >= 132 && g.M >= 64 && g.N >= 64;  // enough 128x128 tiles to fill 132 SMs
    if (big) {
        dim3 grid((g.N + 127) / 128, (g.M + 127) / 128, g.batch * g.splitk);
        sgemm_kernel<128, 128, 16, 8, 8><<<grid, 256, 0, st>>>(g);
    } else {
        dim3 grid((g.N + 31) / 32, (g.M + 31) / 32, g.batch * g.splitk);
        sgemm_kernel<32, 32, 32, 2, 2><<<grid, 256, 0, st>>>(g);
    }
    LAUNCH_CHECK();
    return BIGRU_OK;
}

// column sums: out[z][c] += sum_r A[z][r*ld + c], in a fixed order so that a gradient is the same from run to run (a step
// replayed from a CUDA graph matches plain launches bit for bit): block (x, y, z) sums its row chunk into ws, then
// colsum_finish_kernel adds the chunks in chunk order.  ws holds COLSUM_MAX_CHUNKS * cols * batch floats.
constexpr int COLSUM_MAX_CHUNKS = 64;
__global__ void colsum_kernel(const float* __restrict__ A, float* __restrict__ ws, int64_t rows, int cols,
                              int64_t ld, int64_t zA, int rows_per_block) {
    __shared__ float sm[8][33];
    const float* a = A + blockIdx.z * zA;
    const int c = blockIdx.x * 32 + threadIdx.x;
    const int64_t r0 = (int64_t)blockIdx.y * rows_per_block;
    const int64_t r1 = min(rows, r0 + rows_per_block);
    float s = 0.f;
    if (c < cols)
        for (int64_t r = r0 + threadIdx.y; r < r1; r += 8) s += a[r * ld + c];
    sm[threadIdx.y][threadIdx.x] = s;
    __syncthreads();
    if (threadIdx.y == 0 && c < cols) {
        float t = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) t += sm[i][threadIdx.x];
        ws[((int64_t)blockIdx.z * gridDim.y + blockIdx.y) * cols + c] = t;
    }
}
__global__ void colsum_finish_kernel(const float* __restrict__ ws, float* __restrict__ out, int nchunks, int cols, int batch,
                                     int64_t zOut) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)cols * batch) return;
    const int c = i % cols, z = i / cols;
    float t = 0.f;
    for (int k = 0; k < nchunks; ++k) t += ws[((int64_t)z * nchunks + k) * cols + c];
    out[z * zOut + c] += t;
}
static int colsum_launch(const float* A, float* out, int64_t rows, int cols, int64_t ld, int batch, int64_t zA,
                         int64_t zOut, float* ws, cudaStream_t st) {
    ProfScope ps(KC_MISC, 0.0, 4.0 * rows * cols * batch, st);
    const int rpb = (int)max((int64_t)256, cdiv64(rows, COLSUM_MAX_CHUNKS));
    const int nchunks = (int)cdiv64(rows, rpb);
    dim3 grid((cols + 31) / 32, nchunks, batch);
    colsum_kernel<<<grid, dim3(32, 8), 0, st>>>(A, ws, rows, cols, ld, zA, rpb);
    LAUNCH_CHECK();
    colsum_finish_kernel<<<(unsigned)cdiv64((int64_t)cols * batch, 256), 256, 0, st>>>(ws, out, nchunks, cols, batch, zOut);
    LAUNCH_CHECK();
    return BIGRU_OK;
}

// ------------------------------------------------------------------------------------------
// GRU pointwise: forward gates for one time step of both directions.
//   gi [D][B*T][3H] (input projection + b_ih), gh [D][B][3H] (h_prev W_hh^T + b_hh)
//   Y [B][T][D*H] layer output; G [D][B*T][4H] stash of (r, z, n, gh_n)
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ float sigmoid_f(float x) { return 1.f / (1.f + expf(-x)); }

__global__ void gru_gates_fwd_kernel(const float* __restrict__ gi, const float* __restrict__ gh,
                                     const float* __restrict__ h0, float* __restrict__ Y, float* __restrict__ G,
                                     float* __restrict__ hn_out, int B, int T, int H, int D, int s) {
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t total = (int64_t)D * B * H;
    if (idx >= total) return;
    const int j = idx % H;
    const int b = (idx / H) % B;
    const int d = idx / ((int64_t)H * B);
    const int t = d == 0 ? s : T - 1 - s;
    const int64_t row = (int64_t)b * T + t;
    const float* gir = gi + ((int64_t)d * B * T + row) * 3 * H;
    const float* ghr = gh + ((int64_t)d * B + b) * 3 * H;
    float hp;
    if (s == 0) hp = h0 ? h0[((int64_t)d * B + b) * H + j] : 0.f;
    else hp = Y[((int64_t)b * T + (d == 0 ? t - 1 : t + 1)) * D * H + d * H + j];
    const float r = sigmoid_f(gir[j] + ghr[j]);
    const float z = sigmoid_f(gir[H + j] + ghr[H + j]);
    const float hn = ghr[2 * H + j];
    const float n = tanhf(gir[2 * H + j] + r * hn);
    const float h = (1.f - z) * n + z * hp;
    Y[row * D * H + d * H + j] = h;
    float* g = G + ((int64_t)d * B * T + row) * 4 * H;
    g[j] = r; g[H + j] = z; g[2 * H + j] = n; g[3 * H + j] = hn;
    if (hn_out && s == T - 1) hn_out[((int64_t)d * B + b) * H + j] = h;
}

// backward gates for one step: consumes dh carry + dY_t, emits dgi/dgh rows and dh*z
__global__ void gru_gates_bwd_kernel(const float* __restrict__ G, const float* __restrict__ Y,
                                     const float* __restrict__ h0, const float* __restrict__ dY,
                                     float* __restrict__ dhc, float* __restrict__ dgi, float* __restrict__ dgh,
                                     int B, int T, int H, int D, int s) {
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t total = (int64_t)D * B * H;
    if (idx >= total) return;
    const int j = idx % H;
    const int b = (idx / H) % B;
    const int d = idx / ((int64_t)H * B);
    const int t = d == 0 ? T - 1 - s : s;
    const int64_t row = (int64_t)b * T + t;
    const float* g = G + ((int64_t)d * B * T + row) * 4 * H;
    const float r = g[j], z = g[H + j], n = g[2 * H + j], hn = g[3 * H + j];
    const bool first = d == 0 ? t == 0 : t == T - 1;
    float hp;
    if (first) hp = h0 ? h0[((int64_t)d * B + b) * H + j] : 0.f;
    else hp = Y[((int64_t)b * T + (d == 0 ? t - 1 : t + 1)) * D * H + d * H + j];
    const int64_t ci = ((int64_t)d * B + b) * H + j;
    const float dh = dhc[ci] + dY[row * D * H + d * H + j];
    const float dan = dh * (1.f - z) * (1.f - n * n);
    const float dar = dan * hn * r * (1.f - r);
    const float daz = dh * (hp - n) * z * (1.f - z);
    float* a = dgi + ((int64_t)d * B * T + row) * 3 * H;
    float* c = dgh + ((int64_t)d * B * T + row) * 3 * H;
    a[j] = dar; a[H + j] = daz; a[2 * H + j] = dan;
    c[j] = dar; c[H + j] = daz; c[2 * H + j] = dan * r;
    dhc[ci] = dh * z;
}

// ------------------------------------------------------------------------------------------
// Head (biGRU_model.py:111-133): direction sum, last hidden, max / mean pooling over T.
// ------------------------------------------------------------------------------------------
__global__ void head_pool_kernel(const float* __restrict__ Y, float* __restrict__ cat, int* __restrict__ arg,
                                 int B, int T, int H, int D) {
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (int64_t)B * H) return;
    const int j = idx % H, b = idx / H;
    const float* y = Y + (int64_t)b * T * D * H;
    float last = y[(int64_t)(T - 1) * D * H + j];
    if (D == 2) last += y[H + j];
    float mx = -INFINITY, sum = 0.f;
    int am = 0;
    for (int t = 0; t < T; ++t) {
        float s = y[(int64_t)t * D * H + j];
        if (D == 2) s += y[(int64_t)t * D * H + H + j];
        if (s > mx) { mx = s; am = t; }
        sum += s;
    }
    float* c = cat + (int64_t)b * 3 * H;
    c[j] = last; c[H + j] = mx; c[2 * H + j] = sum / (float)T;
    arg[idx] = am;
}

// dY of the top layer from d(concat): mean + routed max;  dhc (carry) = d(last_hidden) for both dirs
__global__ void head_bwd_dy_kernel(const float* __restrict__ dcat, const int* __restrict__ arg,
                                   float* __restrict__ dY, float* __restrict__ dhc, int B, int T, int H, int D) {
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (int64_t)B * T * H) return;
    const int j = idx % H;
    const int t = (idx / H) % T;
    const int b = idx / ((int64_t)H * T);
    const float* dc = dcat + (int64_t)b * 3 * H;
    const float v = dc[2 * H + j] / (float)T + (arg[(int64_t)b * H + j] == t ? dc[H + j] : 0.f);
    float* o = dY + ((int64_t)b * T + t) * D * H;
    o[j] = v;
    if (D == 2) o[H + j] = v;
    if (t == 0) {
        dhc[(int64_t)b * H + j] = dc[j];
        if (D == 2) dhc[((int64_t)B + b) * H + j] = dc[j];
    }
}

// ------------------------------------------------------------------------------------------
// Losses: value (mean over `denom`) + dlogits.  One block: each thread sums its rows in order, then a fixed-order block
// reduction, so the loss is bit-reproducible (B x C is small).
// ------------------------------------------------------------------------------------------
__global__ void loss_kernel(int kind, const float* __restrict__ logits, const void* __restrict__ target,
                            const float* __restrict__ weight, const float* __restrict__ pos_weight, int B, int C,
                            float inv_denom, float* __restrict__ loss, float* __restrict__ dlogits) {
    float l = 0.f;
    for (int b = threadIdx.x; b < B; b += blockDim.x) {
        const float* lg = logits + (int64_t)b * C;
        if (kind == BIGRU_LOSS_CE) {
            // a target outside [0, C) (torch's ignore_index -100 included) is never read through: its row's loss and dlogits
            // are NaN, so the mismatch with torch, which would skip the row, cannot pass unnoticed
            const long long tg = ((const long long*)target)[b];
            const bool valid = tg >= 0 && tg < C;
            float m = lg[0];
            for (int c = 1; c < C; ++c) m = fmaxf(m, lg[c]);
            float s = 0.f;
            for (int c = 0; c < C; ++c) s += expf(lg[c] - m);
            const float lse = m + logf(s);
            l += lse - (valid ? lg[tg] : nanf(""));
            if (dlogits)
                for (int c = 0; c < C; ++c)
                    dlogits[(int64_t)b * C + c] = valid ? (expf(lg[c] - lse) - (c == tg ? 1.f : 0.f)) * inv_denom : nanf("");
        } else {
            const float* tg = (const float*)target + (int64_t)b * C;
            for (int c = 0; c < C; ++c) {
                const float x = lg[c], y = tg[c];
                const float pw = pos_weight ? pos_weight[c] : 1.f, w = weight ? weight[c] : 1.f;
                const float spn = fmaxf(-x, 0.f) + log1pf(expf(-fabsf(x)));
                const float lw = 1.f + (pw - 1.f) * y;
                l += w * ((1.f - y) * x + lw * spn);
                if (dlogits) {
                    const float sg = 1.f / (1.f + expf(-x));
                    dlogits[(int64_t)b * C + c] = w * ((1.f - y) - lw * (1.f - sg)) * inv_denom;
                }
            }
        }
    }
    // block reduce
    __shared__ float sm[32];
    for (int o = 16; o > 0; o >>= 1) l += __shfl_xor_sync(0xffffffffu, l, o);
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = l;
    __syncthreads();
    if (threadIdx.x < 32) {
        float v = threadIdx.x < (blockDim.x >> 5) ? sm[threadIdx.x] : 0.f;
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (threadIdx.x == 0) *loss += v * inv_denom;
    }
}

// ------------------------------------------------------------------------------------------
// clip_grad_norm_ + Adam over the flat buffers
// ------------------------------------------------------------------------------------------
// sum(g^2): each block reduces its grid-stride share in a fixed order into ws[block]; sqnorm_finish_kernel then adds the
// block sums in a fixed order into *out (no atomics: bit-reproducible for a given n)
__global__ void sqnorm_kernel(const float* __restrict__ g, int64_t n, float* __restrict__ ws) {
    float s = 0.f;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const float v = g[i];
        s = fmaf(v, v, s);
    }
    __shared__ float sm[32];
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x < 32) {
        float v = threadIdx.x < (blockDim.x >> 5) ? sm[threadIdx.x] : 0.f;
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (threadIdx.x == 0) ws[blockIdx.x] = v;
    }
}
// one warp: lane l adds ws[l], ws[l + 32], ... in order, then a fixed butterfly
__global__ void sqnorm_finish_kernel(const float* __restrict__ ws, int nblocks, float* __restrict__ out) {
    float v = 0.f;
    for (int i = threadIdx.x; i < nblocks; i += 32) v += ws[i];
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (threadIdx.x == 0) *out += v;
}

// device-resident step counter (CUDA-graph friendly: nothing about the step number is baked into the launch):
// adam_tick increments *step and clears the squared-norm accumulator; the update kernel forms the bias corrections itself
__global__ void adam_tick_kernel(int* __restrict__ step, float* __restrict__ sqnorm) {
    if (threadIdx.x == 0 && blockIdx.x == 0) { *step += 1; *sqnorm = 0.f; }
}
__global__ void clip_adam_dev_kernel(float* __restrict__ p, float* __restrict__ g, float* __restrict__ m,
                                     float* __restrict__ v, int64_t n, const float* __restrict__ sqnorm, float clip,
                                     float lr, float b1, float b2, float eps, const int* __restrict__ step_p, float gscale) {
    const int step_i = *step_p;
    const float bc1 = (float)(1.0 - pow((double)b1, (double)step_i));
    const float bc2_sqrt = (float)sqrt(1.0 - pow((double)b2, (double)step_i));
    const float norm = sqrtf(*sqnorm) * gscale;
    const float coef = fminf(1.f, clip / (norm + 1e-6f)) * gscale;
    const float step = lr / bc1;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const float gq = g[i] * coef;
        g[i] = gq;
        const float mi = m[i] + (gq - m[i]) * (1.f - b1);        // lerp, as torch.optim.Adam does
        const float vi = v[i] * b2 + (1.f - b2) * gq * gq;
        m[i] = mi; v[i] = vi;
        const float denom = sqrtf(vi) / bc2_sqrt + eps;
        p[i] = p[i] - step * (mi / denom);
    }
}

// ------------------------------------------------------------------------------------------
// Window collation (sql_pytorch_dataloader.py:239-245): coalesced, float4 when F % 4 == 0
// ------------------------------------------------------------------------------------------
template <int VEC>
__global__ void window_gather_kernel(const float* __restrict__ src, const float* __restrict__ xmin,
                                     const float* __restrict__ xmax, int64_t start, int B, int T, int F,
                                     float* __restrict__ out) {
    const int FV = F / VEC;
    const int64_t total = (int64_t)B * T * FV;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int fv = i % FV;
        const int64_t bt = i / FV;
        const int t = bt % T;
        const int64_t b = bt / T;
        const int64_t srow = start + b + t;
        if (VEC == 4) {
            float4 v = *reinterpret_cast<const float4*>(src + srow * F + fv * 4);
            if (xmin) {
                const float4 mn = *reinterpret_cast<const float4*>(xmin + fv * 4);
                const float4 mx = *reinterpret_cast<const float4*>(xmax + fv * 4);
                v.x = (v.x - mn.x) / (mx.x - mn.x); v.y = (v.y - mn.y) / (mx.y - mn.y);
                v.z = (v.z - mn.z) / (mx.z - mn.z); v.w = (v.w - mn.w) / (mx.w - mn.w);
            }
            __stcs(reinterpret_cast<float4*>(out + bt * F + fv * 4), v);
        } else {
            float v = src[srow * F + fv];
            if (xmin) v = (v - xmin[fv]) / (xmax[fv] - xmin[fv]);
            out[bt * F + fv] = v;
        }
    }
}

__global__ void window_targets_kernel(const float* __restrict__ y, int64_t start, int B, int T, int C,
                                      float* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)B * C) return;
    const int c = i % C;
    const int64_t b = i / C;
    out[i] = y[(start + b + T - 1) * C + c];
}

// ------------------------------------------------------------------------------------------
// Dropout (biGRU_model.py:87-94 and the inter-layer dropout of nn.GRU, :55)
//   spatial: one Bernoulli per (b, f), shared over T (Dropout2d on the permuted tensor)
// ------------------------------------------------------------------------------------------
__global__ void dropout_kernel(const float* __restrict__ in, float* __restrict__ out, int64_t n, int T, int F,
                               int spatial, float p, uint64_t seed, uint32_t stream) {
    const float scale = 1.f / (1.f - p);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        uint64_t key = i;
        if (spatial) { const int f = i % F; const int64_t b = i / ((int64_t)F * T); key = b * F + f; }
        const float u = bigru_uniform(seed, stream, key);
        out[i] = u < p ? 0.f : in[i] * scale;
    }
}

// ------------------------------------------------------------------------------------------
// Multi-label metric counts (biGRU_model.py:213-221 without the sklearn round trip)
// ------------------------------------------------------------------------------------------
__global__ void multilabel_counts_kernel(const float* __restrict__ logits, const float* __restrict__ target, int B,
                                         int C, unsigned long long* __restrict__ counts) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    int mism = 0;
    for (int c = 0; c < C; ++c) {
        // fp32 sigmoid as torch.sigmoid evaluates it on the GPU: it rounds to exactly 0.5 for positive x below about 1e-7,
        // so the test is not the same as x > 0
        const bool pred = 1.f / (1.f + expf(-logits[(int64_t)b * C + c])) > 0.5f;
        const bool tru = target[(int64_t)b * C + c] > 0.5f;
        if (pred != tru) ++mism;
        if (pred && tru) atomicAdd(counts + 2 + 3 * c, 1ull);
        if (pred && !tru) atomicAdd(counts + 3 + 3 * c, 1ull);
        if (!pred && tru) atomicAdd(counts + 4 + 3 * c, 1ull);
    }
    if (mism == 0) atomicAdd(counts, 1ull);
    if (mism) atomicAdd(counts + 1, (unsigned long long)mism);
}

// per-feature min / max over table rows [lo, hi); NaN (SQL NULL) ignored.  One block = 32 features x 8 row lanes.
__global__ void chunk_minmax_kernel(const float* __restrict__ tab, int F, int64_t lo, int64_t hi, float* __restrict__ mn,
                                    float* __restrict__ mx) {
    __shared__ float smn[8][33], smx[8][33];
    const int f = blockIdx.x * 32 + threadIdx.x;
    float a = INFINITY, b = -INFINITY;
    if (f < F)
        for (int64_t r = lo + threadIdx.y; r < hi; r += 8) {
            const float v = tab[r * F + f];
            a = fminf(a, v); b = fmaxf(b, v);            // fminf/fmaxf return the non-NaN operand
        }
    smn[threadIdx.y][threadIdx.x] = a; smx[threadIdx.y][threadIdx.x] = b;
    __syncthreads();
    if (threadIdx.y == 0 && f < F) {
        for (int i = 1; i < 8; ++i) { a = fminf(a, smn[i][threadIdx.x]); b = fmaxf(b, smx[i][threadIdx.x]); }
        mn[f] = a; mx[f] = b;
    }
}

__global__ void fill_kernel(float* __restrict__ p, int64_t n, float v) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) p[i] = v;
}
