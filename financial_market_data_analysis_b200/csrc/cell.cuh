// cell.cuh - torch.nn.GRUCell on sm_90a: one step, no carried state, no plan (DESIGN.md §4.7).
//
// Parameters are nn.GRUCell's own vector  w_ih[3H][I] w_hh[3H][H] b_ih[3H] b_hh[3H]  (gate rows r | z | n), i.e. the layer-0,
// direction-0 block of the flat order in bigru_b200.h.  Activations are row-major: x [B][I], h [B][H].
//
// Forward, one launch:
//   * tensor-core precisions (gru_cell_fwd_tc_kernel): mma.sync m16n8k16 bf16 -> fp32 with the weight rows on M and the batch
//     rows on N ("swap-AB", as in the scans).  A CTA owns CELL_U = 16 hidden units (their r, z and n rows) and 8 * NBLK batch
//     rows; its CELL_W warps take the k16 steps of [W_ih x | W_hh h] round-robin, and their partial sums meet in shared memory,
//     added in warp order.  Fragments are read from the fp32 operands in global memory and split into bf16 (hi, and lo at
//     bf16x3) in registers, so there is no pack launch and no padded copy: ragged units, batch rows and k are zero-filled.
//     Four accumulators per element: r and z sum both products, W_in x and W_hn h stay apart (SURVEY.md §7.2).
//   * fp32 (gru_cell_fwd_f32_kernel): FFMA, a warp per (unit, 8 batch rows); lanes stride over k and a fixed xor-butterfly
//     adds the lanes.
//   Each output element is a fixed sequence over k that depends on neither the batch size, nor the row's position, nor whether
//   the stash G [B][4H] = r, z, n, W_hn h + b_hn (the scans' gate-stash row) is written.  A null h is the zero state: the W_hh
//   product is skipped and gh = b_hh.
// Backward, three launches (two when neither dx nor dh is wanted), nothing memset:
//   1. gru_cell_bwd_gates_kernel: dgi = (dar, daz, dan), dgh = (dar, daz, dan * r), gru_scan_bwd_tile's formulas, into scratch;
//   2. dx = dgi W_ih and dh = dh' z + dgh W_hh: gru_cell_bwd_dxh_tc_kernel (tensor cores, the forward's tiling with the output
//      column on M) or gru_cell_bwd_dxh_f32_kernel (FFMA, a thread per output);
//   3. gru_cell_bwd_dw_kernel, every precision: dW_ih = dgi^T x, dW_hh = dgh^T h, db_ih = sum_b dgi, db_hh = sum_b dgh as one
//      fp32 FFMA product [3H] x [I + H + 2] over the batch, b = 0, 1, ... in order (no atomics, no split): every gradient
//      element is written exactly once and a backward is bitwise reproducible.
#pragma once
#include "common.cuh"
#include "kernels_f32.cuh"
#include "tc_hopper.cuh"

namespace cell {

constexpr int CELL_U = 16;                 // hidden units (or dx / dh columns) per tensor-core CTA: one m16 tile per gate
constexpr int CELL_W = 4;                  // warps per tensor-core CTA, splitting the k16 steps
constexpr int CELL_THREADS = CELL_W * 32;
constexpr int F32_ROWS = 8;                // batch rows per warp of the fp32 forward
constexpr int F32_WARPS = 8;               // units (warps) per CTA of the fp32 forward
constexpr int DW_T = 32;                   // tile of the weight-gradient kernel: 32 gate rows x 32 columns x 32 batch rows

// two consecutive-k values as packed bf16x2: hi, and lo = the rounding error of hi (bf16x3 only), as split_bf16
template <int NS>
__device__ __forceinline__ void split2(float a, float b, uint32_t& hi, uint32_t& lo) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    hi = *reinterpret_cast<const uint32_t*>(&h);
    lo = 0u;
    if (NS != 1) {
        const __nv_bfloat162 l = __floats2bfloat162_rn(a - __low2float(h), b - __high2float(h));
        lo = *reinterpret_cast<const uint32_t*>(&l);
    }
}
// A fragment (16 x 16, row-major) of m16n8k16 from ld(m, k), k from k0
template <int NS, class F>
__device__ __forceinline__ void frag_a(const F& ld, int k0, int lane, uint32_t (&hi)[4], uint32_t (&lo)[4]) {
    const int g = lane >> 2, t = k0 + (lane & 3) * 2;
    split2<NS>(ld(g, t), ld(g, t + 1), hi[0], lo[0]);
    split2<NS>(ld(g + 8, t), ld(g + 8, t + 1), hi[1], lo[1]);
    split2<NS>(ld(g, t + 8), ld(g, t + 9), hi[2], lo[2]);
    split2<NS>(ld(g + 8, t + 8), ld(g + 8, t + 9), hi[3], lo[3]);
}
// B fragment (16 x 8, stored [n][k]) from ld(n, k), columns n0 .. n0 + 7
template <int NS, class F>
__device__ __forceinline__ void frag_b(const F& ld, int n0, int k0, int lane, uint32_t (&hi)[2], uint32_t (&lo)[2]) {
    const int n = n0 + (lane >> 2), t = k0 + (lane & 3) * 2;
    split2<NS>(ld(n, t), ld(n, t + 1), hi[0], lo[0]);
    split2<NS>(ld(n, t + 8), ld(n, t + 9), hi[1], lo[1]);
}
// c += a b: hi*lo + lo*hi + hi*hi at bf16x3 (the scans' order), hi*hi at bf16
template <int NS>
__device__ __forceinline__ void mma3(float (&c)[4], const uint32_t (&ah)[4], const uint32_t (&al)[4], const uint32_t (&bh)[2],
                                     const uint32_t (&bl)[2]) {
    if (NS != 1) {
        htc::mma_bf16(c, ah, bl[0], bl[1]);
        htc::mma_bf16(c, al, bh[0], bh[1]);
    }
    htc::mma_bf16(c, ah, bh[0], bh[1]);
}
// accumulator e of n8 block j: row (M) and column (N) inside the CTA tile
__device__ __forceinline__ int acc_m(int lane, int e) { return (lane >> 2) + (e >= 2 ? 8 : 0); }
__device__ __forceinline__ int acc_n(int lane, int j, int e) { return j * 8 + (lane & 3) * 2 + (e & 1); }

// ---- forward ------------------------------------------------------------------------------------------------------------
// Grid (cdiv(H, 16), cdiv(B, 8 * NBLK)).  hout must not overlap x or h: every CTA reads all of h.
template <int NS, int NBLK>
__global__ void __launch_bounds__(CELL_THREADS)
gru_cell_fwd_tc_kernel(const float* __restrict__ P, const float* __restrict__ x, const float* __restrict__ h,
                       float* __restrict__ hout, float* __restrict__ G, int B, int I, int H) {
    constexpr int NBT = NBLK * 8;
    __shared__ float red[CELL_W][4][NBT][CELL_U + 1];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int u0 = blockIdx.x * CELL_U, b0 = blockIdx.y * NBT;
    const int64_t H3 = 3LL * H;
    const float* Wih = P;
    const float* Whh = P + H3 * I;
    const float* bih = Whh + H3 * H;
    const float* bhh = bih + H3;
    float acc[4][NBLK][4];
#pragma unroll
    for (int g = 0; g < 4; ++g)
#pragma unroll
        for (int j = 0; j < NBLK; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[g][j][e] = 0.f;
    const int KI = (I + 15) / 16, KH = h ? (H + 15) / 16 : 0;
    for (int s = warp; s < KI + KH; s += CELL_W) {
        const bool xs = s < KI;                               // a step of W_ih x, else of W_hh h
        const float* W = xs ? Wih : Whh;
        const float* A = xs ? x : h;
        const int K = xs ? I : H, k0 = (xs ? s : s - KI) * 16;
        uint32_t bh[NBLK][2], bl[NBLK][2];
#pragma unroll
        for (int j = 0; j < NBLK; ++j)
            frag_b<NS>([&](int n, int k) { return n < B && k < K ? A[(int64_t)n * K + k] : 0.f; }, b0 + j * 8, k0, lane, bh[j], bl[j]);
#pragma unroll
        for (int gte = 0; gte < 3; ++gte) {
            uint32_t ah[4], al[4];
            frag_a<NS>([&](int m, int k) { const int u = u0 + m; return u < H && k < K ? W[(gte * H + u) * (int64_t)K + k] : 0.f; },
                       k0, lane, ah, al);
#pragma unroll
            for (int j = 0; j < NBLK; ++j) {
                if (gte < 2) mma3<NS>(acc[gte][j], ah, al, bh[j], bl[j]);
                else if (xs) mma3<NS>(acc[2][j], ah, al, bh[j], bl[j]);
                else mma3<NS>(acc[3][j], ah, al, bh[j], bl[j]);
            }
        }
    }
#pragma unroll
    for (int g = 0; g < 4; ++g)
#pragma unroll
        for (int j = 0; j < NBLK; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) red[warp][g][acc_n(lane, j, e)][acc_m(lane, e)] = acc[g][j][e];
    __syncthreads();
    // gate math, units fastest (coalesced stores); the warps' partial sums are added in warp order
    for (int i = threadIdx.x; i < NBT * CELL_U; i += CELL_THREADS) {
        const int n = i / CELL_U, m = i % CELL_U, u = u0 + m, b = b0 + n;
        if (u >= H || b >= B) continue;
        float a[4];
#pragma unroll
        for (int g = 0; g < 4; ++g) {
            float v = red[0][g][n][m];
#pragma unroll
            for (int w = 1; w < CELL_W; ++w) v += red[w][g][n][m];
            a[g] = v;
        }
        const float r = sigmoid_f(a[0] + bih[u] + bhh[u]);
        const float z = sigmoid_f(a[1] + bih[H + u] + bhh[H + u]);
        const float ghn = a[3] + bhh[2 * H + u];
        const float nn = tanhf(a[2] + bih[2 * H + u] + r * ghn);
        const int64_t o = (int64_t)b * H + u;
        const float hp = h ? h[o] : 0.f;
        hout[o] = (1.f - z) * nn + z * hp;
        if (G) {
            float* gs = G + (int64_t)b * 4 * H + u;
            gs[0] = r; gs[H] = z; gs[2 * H] = nn; gs[3 * H] = ghn;
        }
    }
}

// Grid (cdiv(H, F32_WARPS), cdiv(B, F32_ROWS)), F32_WARPS warps: warp w owns unit blockIdx.x * F32_WARPS + w
__global__ void __launch_bounds__(F32_WARPS * 32)
gru_cell_fwd_f32_kernel(const float* __restrict__ P, const float* __restrict__ x, const float* __restrict__ h,
                        float* __restrict__ hout, float* __restrict__ G, int B, int I, int H) {
    const int lane = threadIdx.x & 31, u = blockIdx.x * F32_WARPS + (threadIdx.x >> 5), b0 = blockIdx.y * F32_ROWS;
    if (u >= H) return;
    const int64_t H3 = 3LL * H;
    const float* Wih = P;
    const float* Whh = P + H3 * I;
    const float* bih = Whh + H3 * H;
    const float* bhh = bih + H3;
    float acc[4][F32_ROWS];
#pragma unroll
    for (int g = 0; g < 4; ++g)
#pragma unroll
        for (int r = 0; r < F32_ROWS; ++r) acc[g][r] = 0.f;
    for (int k = lane; k < I; k += 32) {
        const float w0 = Wih[(int64_t)u * I + k], w1 = Wih[(int64_t)(H + u) * I + k], w2 = Wih[(int64_t)(2 * H + u) * I + k];
#pragma unroll
        for (int r = 0; r < F32_ROWS; ++r) {
            const float v = b0 + r < B ? x[(int64_t)(b0 + r) * I + k] : 0.f;
            acc[0][r] = fmaf(w0, v, acc[0][r]); acc[1][r] = fmaf(w1, v, acc[1][r]); acc[2][r] = fmaf(w2, v, acc[2][r]);
        }
    }
    if (h) {
        for (int k = lane; k < H; k += 32) {
            const float w0 = Whh[(int64_t)u * H + k], w1 = Whh[(int64_t)(H + u) * H + k], w2 = Whh[(int64_t)(2 * H + u) * H + k];
#pragma unroll
            for (int r = 0; r < F32_ROWS; ++r) {
                const float v = b0 + r < B ? h[(int64_t)(b0 + r) * H + k] : 0.f;
                acc[0][r] = fmaf(w0, v, acc[0][r]); acc[1][r] = fmaf(w1, v, acc[1][r]); acc[3][r] = fmaf(w2, v, acc[3][r]);
            }
        }
    }
    // xor butterfly: every lane ends with the same sums (a + b == b + a), whatever the batch
#pragma unroll
    for (int off = 16; off > 0; off >>= 1)
#pragma unroll
        for (int g = 0; g < 4; ++g)
#pragma unroll
            for (int r = 0; r < F32_ROWS; ++r) acc[g][r] += __shfl_xor_sync(0xffffffffu, acc[g][r], off);
#pragma unroll
    for (int r = 0; r < F32_ROWS; ++r) {
        const int b = b0 + r;
        if (lane != r || b >= B) continue;
        const float rg = sigmoid_f(acc[0][r] + bih[u] + bhh[u]);
        const float z = sigmoid_f(acc[1][r] + bih[H + u] + bhh[H + u]);
        const float ghn = acc[3][r] + bhh[2 * H + u];
        const float nn = tanhf(acc[2][r] + bih[2 * H + u] + rg * ghn);
        const int64_t o = (int64_t)b * H + u;
        const float hp = h ? h[o] : 0.f;
        hout[o] = (1.f - z) * nn + z * hp;
        if (G) {
            float* gs = G + (int64_t)b * 4 * H + u;
            gs[0] = rg; gs[H] = z; gs[2 * H] = nn; gs[3 * H] = ghn;
        }
    }
}

// ---- backward -----------------------------------------------------------------------------------------------------------
// 1. gate gradients from the forward's stash: dgi, dgh [B][3H] (grid-stride over B * H)
__global__ void gru_cell_bwd_gates_kernel(const float* __restrict__ G, const float* __restrict__ h, const float* __restrict__ dhout,
                                          float* __restrict__ dgi, float* __restrict__ dgh, int B, int H) {
    const int64_t n = (int64_t)B * H;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t b = i / H;
        const int j = (int)(i % H);
        const float* gs = G + b * 4 * H + j;
        const float r = gs[0], z = gs[H], nn = gs[2 * H], hnv = gs[3 * H];
        const float hp = h ? h[i] : 0.f, dh = dhout[i];
        const float dan = dh * (1.f - z) * (1.f - nn * nn);
        const float dar = dan * hnv * r * (1.f - r);
        const float daz = dh * (hp - nn) * z * (1.f - z);
        float* a = dgi + b * 3 * H + j;
        float* c = dgh + b * 3 * H + j;
        a[0] = dar; a[H] = daz; a[2 * H] = dan;
        c[0] = dar; c[H] = daz; c[2 * H] = dan * r;
    }
}

// 2. dx [B][I] = dgi W_ih and dh [B][H] = dh' z + dgh W_hh on tensor cores: A(m, k) = W[k][m] (the output column on M), B(n, k)
//    = dg[n][k], k over the 3H gate rows.  Grid (mx + mh, cdiv(B, 8 * NBLK)): the first mx column tiles are dx's (mx = 0 without
//    dx), the next mh dh's (mh = 0 without dh).
template <int NS, int NBLK>
__global__ void __launch_bounds__(CELL_THREADS)
gru_cell_bwd_dxh_tc_kernel(const float* __restrict__ P, const float* __restrict__ G, const float* __restrict__ dhout,
                           const float* __restrict__ dgi, const float* __restrict__ dgh, float* __restrict__ dx,
                           float* __restrict__ dh, int B, int I, int H, int mx) {
    constexpr int NBT = NBLK * 8;
    __shared__ float red[CELL_W][NBT][CELL_U + 1];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const bool isx = (int)blockIdx.x < mx;
    const int m0 = (isx ? blockIdx.x : blockIdx.x - mx) * CELL_U, M = isx ? I : H, b0 = blockIdx.y * NBT;
    const int K = 3 * H;
    const float* W = isx ? P : P + 3LL * H * I;             // [3H][M]
    const float* Dg = isx ? dgi : dgh;                       // [B][3H]
    float acc[NBLK][4];
#pragma unroll
    for (int j = 0; j < NBLK; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[j][e] = 0.f;
    for (int s = warp; s < (K + 15) / 16; s += CELL_W) {
        const int k0 = s * 16;
        uint32_t ah[4], al[4];
        frag_a<NS>([&](int m, int k) { return m0 + m < M && k < K ? W[(int64_t)k * M + m0 + m] : 0.f; }, k0, lane, ah, al);
#pragma unroll
        for (int j = 0; j < NBLK; ++j) {
            uint32_t bh[2], bl[2];
            frag_b<NS>([&](int n, int k) { return n < B && k < K ? Dg[(int64_t)n * K + k] : 0.f; }, b0 + j * 8, k0, lane, bh, bl);
            mma3<NS>(acc[j], ah, al, bh, bl);
        }
    }
#pragma unroll
    for (int j = 0; j < NBLK; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) red[warp][acc_n(lane, j, e)][acc_m(lane, e)] = acc[j][e];
    __syncthreads();
    for (int i = threadIdx.x; i < NBT * CELL_U; i += CELL_THREADS) {
        const int n = i / CELL_U, m = i % CELL_U, c = m0 + m, b = b0 + n;
        if (c >= M || b >= B) continue;
        float v = red[0][n][m];
#pragma unroll
        for (int w = 1; w < CELL_W; ++w) v += red[w][n][m];
        if (isx) dx[(int64_t)b * I + c] = v;
        else dh[(int64_t)b * H + c] = dhout[(int64_t)b * H + c] * G[(int64_t)b * 4 * H + H + c] + v;
    }
}

// 2. at fp32: a thread per output column c (dx's I columns, then dh's H; cx = I with dx, 0 without), grid (cdiv(cols, 256), B)
__global__ void __launch_bounds__(256)
gru_cell_bwd_dxh_f32_kernel(const float* __restrict__ P, const float* __restrict__ G, const float* __restrict__ dhout,
                            const float* __restrict__ dgi, const float* __restrict__ dgh, float* __restrict__ dx,
                            float* __restrict__ dh, int B, int I, int H, int cx, int cols) {
    const int c = blockIdx.x * 256 + threadIdx.x, b = blockIdx.y;
    if (c >= cols) return;
    const bool isx = c < cx;
    const int m = isx ? c : c - cx, M = isx ? I : H, K = 3 * H;
    const float* W = (isx ? P : P + 3LL * H * I) + m;
    const float* dg = (isx ? dgi : dgh) + (int64_t)b * K;
    float v = 0.f;
    for (int k = 0; k < K; ++k) v = fmaf(dg[k], W[(int64_t)k * M], v);
    if (isx) dx[(int64_t)b * I + m] = v;
    else dh[(int64_t)b * H + m] = dhout[(int64_t)b * H + m] * G[(int64_t)b * 4 * H + H + m] + v;
}

// 3. weight and bias gradients: grads[q][c] over the virtual columns c of [x | h | 1 | 1] (I + H + 2), q over the 3H gate rows,
//    summed over b in order.  Column c pairs with dgi (x, and the first 1: db_ih) or dgh (h, and the second 1: db_hh); without
//    h, dW_hh is written as zeros.  Grid (cdiv(I + H + 2, 32), cdiv(3H, 32)), block (32, 8): 4 gate rows per thread.
__global__ void __launch_bounds__(256)
gru_cell_bwd_dw_kernel(const float* __restrict__ x, const float* __restrict__ h, const float* __restrict__ dgi,
                       const float* __restrict__ dgh, float* __restrict__ grads, int B, int I, int H) {
    __shared__ float sg[2][DW_T][DW_T + 1];                  // [dgi | dgh][b][q]
    __shared__ float ss[DW_T][DW_T + 1];                     // [b][c]
    const int tx = threadIdx.x, ty = threadIdx.y, tid = ty * DW_T + tx;
    const int c0 = blockIdx.x * DW_T, q0 = blockIdx.y * DW_T, K = 3 * H, NC = I + H + 2;
    const int c = c0 + tx;
    const int sel = c < I || c == I + H ? 0 : 1;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int bb0 = 0; bb0 < B; bb0 += DW_T) {
        for (int i = tid; i < DW_T * DW_T; i += DW_T * 8) {
            const int r = i / DW_T, cc = i % DW_T, b = bb0 + r, q = q0 + cc, col = c0 + cc;
            const bool in = b < B;
            sg[0][r][cc] = in && q < K ? dgi[(int64_t)b * K + q] : 0.f;
            sg[1][r][cc] = in && q < K ? dgh[(int64_t)b * K + q] : 0.f;
            float v = 0.f;
            if (in && col < NC) {
                if (col < I) v = x[(int64_t)b * I + col];
                else if (col < I + H) v = h ? h[(int64_t)b * H + col - I] : 0.f;
                else v = 1.f;
            }
            ss[r][cc] = v;
        }
        __syncthreads();
#pragma unroll 8
        for (int r = 0; r < DW_T; ++r) {
            const float v = ss[r][tx];
#pragma unroll
            for (int k = 0; k < 4; ++k) acc[k] = fmaf(sg[sel][r][ty + 8 * k], v, acc[k]);
        }
        __syncthreads();
    }
    if (c >= NC) return;
    const int64_t H3 = K, ob = H3 * I + H3 * H;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int q = q0 + ty + 8 * k;
        if (q >= K) continue;
        float* o = c < I ? grads + (int64_t)q * I + c
                 : c < I + H ? grads + H3 * I + (int64_t)q * H + (c - I)
                 : grads + ob + (c == I + H ? 0 : H3) + q;
        *o = acc[k];
    }
}

}  // namespace cell

// ---- host side ------------------------------------------------------------------------------------------------------------
// shape limits of the cell (bigru_b200.h): grid extents and 32-bit row counts stay in range below them
constexpr int CELL_MAX_B = 32768, CELL_MAX_DIM = 65536;

static inline int cell_nblk(int B) { return B <= 8 ? 1 : B <= 16 ? 2 : 4; }

static int cell_fwd_launch(int B, int I, int H, int prec, const float* P, const float* x, const float* h, float* hout, float* G,
                           cudaStream_t st) {
    using namespace cell;
    const double flops = 2.0 * B * 3.0 * H * (I + (h ? H : 0));
    const double bytes = 4.0 * (3.0 * H * (I + H) + 6.0 * H + (double)B * (I + (h ? 2 : 1) * H) + (G ? 4.0 * B * H : 0.0));
    if (prec == BIGRU_PREC_FP32) {
        const dim3 grid((unsigned)cdiv64(H, F32_WARPS), (unsigned)cdiv64(B, F32_ROWS));
        KLAUNCH(KC_CELL_FWD, flops, bytes, st, gru_cell_fwd_f32_kernel<<<grid, F32_WARPS * 32, 0, st>>>(P, x, h, hout, G, B, I, H));
        return BIGRU_OK;
    }
    const int nb = cell_nblk(B);
    const dim3 grid((unsigned)cdiv64(H, CELL_U), (unsigned)cdiv64(B, 8 * nb));
#define CELL_FWD(NS, NB) KLAUNCH(KC_CELL_FWD, flops, bytes, st, gru_cell_fwd_tc_kernel<NS, NB><<<grid, CELL_THREADS, 0, st>>>(P, x, h, hout, G, B, I, H))
    if (prec == BIGRU_PREC_BF16X3) {
        if (nb == 1) CELL_FWD(3, 1); else if (nb == 2) CELL_FWD(3, 2); else CELL_FWD(3, 4);
    } else {
        if (nb == 1) CELL_FWD(1, 1); else if (nb == 2) CELL_FWD(1, 2); else CELL_FWD(1, 4);
    }
#undef CELL_FWD
    return BIGRU_OK;
}

// scratch: dgi, dgh [B][3H] fp32
static int cell_bwd_launch(int B, int I, int H, int prec, const float* P, const float* x, const float* h, const float* G,
                           const float* dhout, float* grads, float* dx, float* dh, float* scratch, cudaStream_t st) {
    using namespace cell;
    const int64_t H3 = 3LL * H;
    float* dgi = scratch;
    float* dgh = scratch + (int64_t)B * H3;
    const int64_t n = (int64_t)B * H;
    KLAUNCH(KC_CELL_BWD, 0.0, 4.0 * (double)n * (4 + 2 + 6), st,
            gru_cell_bwd_gates_kernel<<<(unsigned)std::min<int64_t>(cdiv64(n, 256), 132 * 16), 256, 0, st>>>(G, h, dhout, dgi, dgh, B, H));
    if (dx || dh) {
        const int cx = dx ? I : 0, ch = dh ? H : 0;
        const double flops = 2.0 * B * H3 * (cx + ch);
        if (prec == BIGRU_PREC_FP32) {
            const dim3 grid((unsigned)cdiv64(cx + ch, 256), (unsigned)B);
            KLAUNCH(KC_CELL_BWD, flops, 0.0, st, gru_cell_bwd_dxh_f32_kernel<<<grid, 256, 0, st>>>(P, G, dhout, dgi, dgh, dx, dh, B, I, H, cx, cx + ch));
        } else {
            const int nb = cell_nblk(B), mx = dx ? (int)cdiv64(I, CELL_U) : 0, mh = dh ? (int)cdiv64(H, CELL_U) : 0;
            const dim3 grid((unsigned)(mx + mh), (unsigned)cdiv64(B, 8 * nb));
#define CELL_DXH(NS, NB) KLAUNCH(KC_CELL_BWD, flops, 0.0, st, gru_cell_bwd_dxh_tc_kernel<NS, NB><<<grid, CELL_THREADS, 0, st>>>(P, G, dhout, dgi, dgh, dx, dh, B, I, H, mx))
            if (prec == BIGRU_PREC_BF16X3) {
                if (nb == 1) CELL_DXH(3, 1); else if (nb == 2) CELL_DXH(3, 2); else CELL_DXH(3, 4);
            } else {
                if (nb == 1) CELL_DXH(1, 1); else if (nb == 2) CELL_DXH(1, 2); else CELL_DXH(1, 4);
            }
#undef CELL_DXH
        }
    }
    const dim3 grid((unsigned)cdiv64(I + H + 2, DW_T), (unsigned)cdiv64(H3, DW_T));
    KLAUNCH(KC_CELL_BWD, 2.0 * B * H3 * (I + H + 2), 0.0, st,
            gru_cell_bwd_dw_kernel<<<grid, dim3(DW_T, 8), 0, st>>>(x, h, dgi, dgh, grads, B, I, H));
    return BIGRU_OK;
}
