// tc_hopper.cuh - the tensor-core pieces of BIGRU_PREC_BF16 and BIGRU_PREC_BF16X3 on sm_90a (H100).
//
// Both precisions share the data layout and step composition of the fp32 path (api.cu): time steps of the recurrence and
// all GEMMs read and write the same fp32 buffers.  What changes is where the arithmetic runs:
//   * tc_gemm_launch      - the strided GEMM of kernels_f32.cuh (same GemmArgs: NT / NN / TN by strides, batches, split-K,
//                           bias, accumulate, the h_{t-1} row mask): operands packed once into K-major bf16 images, then a
//                           TMA + mbarrier pipelined wgmma kernel (wg_gemm_kernel).
//   * gru_scan_fwd_kernel - one layer's whole forward recurrence in one launch: a thread-block cluster per (direction,
//                           16-row batch tile); CTA c of the cluster owns hidden units [64c, 64c+64) and keeps their W_hh
//                           rows (3 gates x 64 units x H) resident in shared memory for all T steps.  Each step it multiplies
//                           them with h_{t-1} of the tile, runs the gate math in registers and writes its slice of h_t into
//                           the shared memory of every CTA of the cluster (distributed shared memory), then a cluster barrier.
//   * gru_scan_bwd_kernel - the backward recurrence, reduction-partitioned: CTA c keeps W_hh^T restricted to its own units'
//                           gate rows (H x 192), multiplies it with its local dgh tile and sends each peer the fp32 partial
//                           sums of dh_{t-1} for the peer's units; the owner adds them up.
// Precision: NS = 1 (bf16) uses single bf16 operands; NS = 3 (bf16x3) splits every operand x = hi + lo (both bf16, |lo| <=
// 2^-9 |x|) and adds hi*hi + hi*lo + lo*hi (the dropped lo*lo term is below 2^-16 relative), all with fp32 accumulation:
// fp32-class results on the tensor cores.  State, gate math, stash and gradients are fp32 in both.
// H100 budget that shapes the scans: 227 KB of shared memory per block holds a 64-unit slice of W_hh at H = 256 as hi/lo
// pairs (192 KB) or at H = 512 in bf16 (192 KB); clusters of H/64 <= 8 CTAs stay within the portable cluster size.
#pragma once
#include "common.cuh"
#include "kernels_f32.cuh"
#include <cuda.h>
#include <cuda_bf16.h>

namespace htc {

typedef __nv_bfloat16 bf16_t;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void split_bf16(float x, bf16_t& hi, bf16_t& lo) {
    hi = __float2bfloat16(x);
    lo = __float2bfloat16(x - __bfloat162float(hi));
}

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t (&r)[4]) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x2(uint32_t addr, uint32_t (&r)[2]) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x2.shared.b16 {%0, %1}, [%2];" : "=r"(r[0]), "=r"(r[1]) : "r"(addr));
}
// D (16x8, fp32) += A (16x16, bf16, row-major) * B (16x8, bf16, "col": stored as [n][k])
__device__ __forceinline__ void mma_bf16(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
                 "{%0, %1, %2, %3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// byte offset of bf16 element (row, k) in a tile whose rows are PITCH bytes (a multiple of 128): the 16-byte chunk index is
// XORed with row % 8, so the eight row addresses of one ldmatrix land in eight different bank groups
template <int PITCH>
__device__ __forceinline__ uint32_t swz(int row, int k) {
    return (uint32_t)(row * PITCH + ((((k >> 3) ^ (row & 7))) << 4) + ((k & 7) << 1));
}

// ---- cluster / distributed shared memory ------------------------------------------------------------
__device__ __forceinline__ uint32_t mapa(uint32_t local_addr, uint32_t cta) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_addr), "r"(cta));
    return r;
}
__device__ __forceinline__ void st_cluster_b16(uint32_t addr, bf16_t v) {
    asm volatile("st.shared::cluster.b16 [%0], %1;" ::"r"(addr), "h"(__bfloat16_as_ushort(v)) : "memory");
}
__device__ __forceinline__ void st_cluster_f32(uint32_t addr, float v) {
    asm volatile("st.shared::cluster.f32 [%0], %1;" ::"r"(addr), "f"(v) : "memory");
}
__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire;" ::: "memory"); }
__device__ __forceinline__ uint32_t cluster_rank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}

// ------------------------------------------------------------------------------------------------------
// GEMM: C[z][m,n] (+)= sum_k A(m,k) B(n,k) (+ bias[n]), the contract of sgemm_kernel (kernels_f32.cuh), in two passes:
//   tc_pack_kernel  - each operand is read once (any strides, the dW_hh row mask) and written as a zero-padded K-major bf16
//                     image [batch][rows / 128 * 128][K / 64 * 64]: one plane at bf16, hi and lo planes at bf16x3;
//   wg_gemm_kernel  - 128 x 128 output tiles, warp-specialised: one thread streams 64-deep k-blocks of every plane into a
//                     STAGES-deep shared-memory ring with TMA (128-byte swizzle) and mbarrier completion, two consumer
//                     warpgroups (64 rows each) multiply them with wgmma.m64n128k16 (fp32 accumulation) and release the
//                     slot; bf16x3 issues hi*hi + hi*lo + lo*hi per k-step.  Epilogue: bias, accumulate, split-K atomics.
// ------------------------------------------------------------------------------------------------------
constexpr int WG_BM = 128, WG_BN = 128, WG_BK = 64;

__global__ void tc_pack_kernel(const float* __restrict__ src, int64_t s_r, int64_t s_k, int64_t zsrc, int R, int K, int Rp, int Kp,
                               int mask_period, int mask_skip, bf16_t* __restrict__ hi, bf16_t* __restrict__ lo) {
    __shared__ float tile[32][33];
    const int z = blockIdx.z, r0 = blockIdx.y * 32, k0 = blockIdx.x * 32;
    const float* a = src + z * zsrc;
    const bool kfast = s_k == 1;
    for (int j = threadIdx.y; j < 32; j += 8) {
        const int r = r0 + (kfast ? j : threadIdx.x), k = k0 + (kfast ? threadIdx.x : j);
        float v = 0.f;
        if (r < R && k < K && !(mask_period && (k % mask_period) == mask_skip)) v = a[(int64_t)r * s_r + (int64_t)k * s_k];
        if (kfast) tile[j][threadIdx.x] = v; else tile[threadIdx.x][j] = v;
    }
    __syncthreads();
    for (int j = threadIdx.y; j < 32; j += 8) {
        const int r = r0 + j, k = k0 + threadIdx.x;
        const int64_t o = ((int64_t)z * Rp + r) * Kp + k;
        bf16_t h, l;
        split_bf16(tile[j][threadIdx.x], h, l);
        hi[o] = h;
        if (lo) lo[o] = l;
    }
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
// a wait that has not completed after 5 s of wall clock means the pipeline protocol is broken: stop the kernel (the launch
// reports an error) rather than occupy the GPU
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    uint64_t t0, t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
    for (uint32_t i = 0;; ++i) {
        if (mbar_try_wait(bar, parity)) return;
        if ((i & 1023u) == 1023u) {
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
            if (t - t0 > 5000000000ull) __trap();
        }
    }
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
// wgmma shared-memory descriptor of a K-major tile with 128-byte swizzle: rows of 64 bf16, 8-row groups 1024 B apart
__device__ __forceinline__ uint64_t wg_desc(uint32_t saddr) {
    return (uint64_t)((saddr & 0x3FFFF) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t da, uint64_t db) {
    asm volatile("wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, 1, 1, 1, 0, 0;"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "l"(da), "l"(db));
}

struct WgOut {
    float* C; const float* bias;
    int M, N, kblocks, Mp, Np, splitk, beta;
    int64_t ldc, zC, zBias;
};

template <int NS, int STAGES>
__global__ void __launch_bounds__(384, 1)
wg_gemm_kernel(const __grid_constant__ CUtensorMap ta_hi, const __grid_constant__ CUtensorMap ta_lo,
               const __grid_constant__ CUtensorMap tb_hi, const __grid_constant__ CUtensorMap tb_lo, WgOut o) {
    constexpr int NH = NS == 1 ? 1 : 2;
    constexpr int PLANE = WG_BM * WG_BK * 2;                  // 16 KB: one 128 x 64 bf16 tile
    constexpr int STAGE = 2 * NH * PLANE;                     // A planes, then B planes
    extern __shared__ __align__(1024) uint8_t wg_smem_raw[];
    uint8_t* sm = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(wg_smem_raw) + 1023) & ~(uintptr_t)1023);
    uint64_t* full = reinterpret_cast<uint64_t*>(sm + STAGES * STAGE);
    uint64_t* empty = full + STAGES;
    const int wgi = threadIdx.x / 128, tid = threadIdx.x % 128;
    const int zb = blockIdx.z / o.splitk, zs = blockIdx.z % o.splitk;
    const int m0 = blockIdx.y * WG_BM, n0 = blockIdx.x * WG_BN;
    const int per = (o.kblocks + o.splitk - 1) / o.splitk;
    const int kb0 = zs * per, kb1 = min(o.kblocks, kb0 + per);
    if (threadIdx.x == 0) {
        for (int i = 0; i < STAGES; ++i) { mbar_init(full + i, 1); mbar_init(empty + i, 2); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (wgi == 0) {                                           // producer
        if (tid == 0) {
            for (int kb = kb0, i = 0; kb < kb1; ++kb, ++i) {
                const int st = i % STAGES;
                if (i >= STAGES) mbar_wait(empty + st, ((i / STAGES) - 1) & 1);
                uint8_t* base = sm + st * STAGE;
                mbar_arrive_expect_tx(full + st, STAGE);
                const int kc = kb * WG_BK, ra = zb * o.Mp + m0, rb = zb * o.Np + n0;
                tma_load_2d(base, &ta_hi, full + st, kc, ra);
                if (NH == 2) tma_load_2d(base + PLANE, &ta_lo, full + st, kc, ra);
                tma_load_2d(base + NH * PLANE, &tb_hi, full + st, kc, rb);
                if (NH == 2) tma_load_2d(base + (NH + 1) * PLANE, &tb_lo, full + st, kc, rb);
            }
        }
        return;
    }
    const int cg = wgi - 1;                                   // consumer warpgroup: rows cg*64 .. +64 of the tile
    float d[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) d[i] = 0.f;
    for (int kb = kb0, i = 0; kb < kb1; ++kb, ++i) {
        const int st = i % STAGES;
        mbar_wait(full + st, (i / STAGES) & 1);
        const uint32_t base = smem_u32(sm + st * STAGE);
        const uint32_t a_hi = base + cg * 64 * 128, a_lo = a_hi + PLANE;
        const uint32_t b_hi = base + NH * PLANE, b_lo = b_hi + PLANE;
        asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
        for (int ks = 0; ks < WG_BK / 16; ++ks) {
            wgmma_m64n128k16(d, wg_desc(a_hi + ks * 32), wg_desc(b_hi + ks * 32));
            if (NS != 1) {
                wgmma_m64n128k16(d, wg_desc(a_hi + ks * 32), wg_desc(b_lo + ks * 32));
                wgmma_m64n128k16(d, wg_desc(a_lo + ks * 32), wg_desc(b_hi + ks * 32));
            }
        }
        asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
        asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
        if (tid == 0) mbar_arrive(empty + st);
    }
    const int w = tid / 32, l = tid % 32;
    float* C = o.C + zb * o.zC;
    const float* bias = o.bias ? o.bias + zb * o.zBias : nullptr;
#pragma unroll
    for (int i = 0; i < 16; ++i)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int gm = m0 + cg * 64 + w * 16 + (l >> 2) + (e >= 2 ? 8 : 0);
            const int gn = n0 + 8 * i + 2 * (l & 3) + (e & 1);
            if (gm >= o.M || gn >= o.N) continue;
            float v = d[4 * i + e];
            if (bias && zs == 0) v += bias[gn];
            float* c = C + (int64_t)gm * o.ldc + gn;
            if (o.splitk > 1) atomicAdd(c, v);
            else if (o.beta) *c += v;
            else *c = v;
        }
}

// ------------------------------------------------------------------------------------------------------
// Forward recurrence of one layer, both directions.  Layouts are those of gru_gates_fwd_kernel:
//   gi [D][B*T][3H] (x W_ih^T + b_ih), Y [B][T][D*H], G [D][B*T][4H] = (r, z, n, W_hn h + b_hn), hn [D][B][H].
// Grid (CS, B/16, D), cluster (CS, 1, 1), 256 threads.  Warp w owns units 16*(w/2) .. +16 of the CTA's slice and batch
// columns 8*(w%2) .. +8: its r, z and n accumulators hold the same (unit, column) pairs, so the gate math needs no exchange.
// ------------------------------------------------------------------------------------------------------
constexpr int SCAN_U = 64, SCAN_NB = 16, SCAN_THREADS = 256;

template <int H, int NS>
struct FwdSmem {
    static constexpr int NH = NS == 1 ? 1 : 2;
    static constexpr int WP = H * 2;                        // W row pitch (bytes): K = H
    static constexpr int WBYTES = 3 * SCAN_U * WP;          // one of hi / lo
    static constexpr int HBYTES = SCAN_NB * H * 2;          // h tile, one of hi / lo
    static constexpr int TOTAL = NH * WBYTES + 2 * NH * HBYTES;
};

template <int H, int NS>
__global__ void __launch_bounds__(SCAN_THREADS, 1)
gru_scan_fwd_kernel(const float* __restrict__ gi, const float* __restrict__ Whh, const float* __restrict__ bhh, int64_t zW,
                    const float* __restrict__ h0, float* __restrict__ Y, float* __restrict__ G, float* __restrict__ hn_out,
                    int B, int T, int D) {
    using S = FwdSmem<H, NS>;
    constexpr int U = SCAN_U, CS = H / U, NH = S::NH;
    extern __shared__ __align__(128) uint8_t smem[];
    uint8_t* Wsm = smem;                                     // [NH][3U rows][H]
    uint8_t* Hsm = smem + NH * S::WBYTES;                    // [2 buffers][NH][NB rows][H]
    const int c = (int)cluster_rank(), tile = blockIdx.y, d = blockIdx.z;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int bt0 = tile * SCAN_NB;
    const float* W = Whh + d * zW;

    for (int i = tid; i < 3 * U * H; i += SCAN_THREADS) {
        const int q = i / H, k = i % H, gte = q / U, u = q % U;
        const float v = W[(int64_t)(gte * H + c * U + u) * H + k];
        bf16_t hi, lo;
        split_bf16(v, hi, lo);
        *reinterpret_cast<bf16_t*>(Wsm + swz<S::WP>(q, k)) = hi;
        if (NH == 2) *reinterpret_cast<bf16_t*>(Wsm + S::WBYTES + swz<S::WP>(q, k)) = lo;
    }
    for (int i = tid; i < SCAN_NB * H; i += SCAN_THREADS) {
        const int b = i / H, k = i % H;
        const float v = h0 ? h0[((int64_t)d * B + bt0 + b) * H + k] : 0.f;
        bf16_t hi, lo;
        split_bf16(v, hi, lo);
        *reinterpret_cast<bf16_t*>(Hsm + swz<H * 2>(b, k)) = hi;
        if (NH == 2) *reinterpret_cast<bf16_t*>(Hsm + S::HBYTES + swz<H * 2>(b, k)) = lo;
    }

    const int ug = warp >> 1, nt = warp & 1;
    int unit[2], bcol[2];
    unit[0] = ug * 16 + (lane >> 2); unit[1] = unit[0] + 8;
    bcol[0] = nt * 8 + 2 * (lane & 3); bcol[1] = bcol[0] + 1;
    float bias[3][2], hp[4];
#pragma unroll
    for (int gte = 0; gte < 3; ++gte)
#pragma unroll
        for (int j = 0; j < 2; ++j) bias[gte][j] = bhh[d * zW + gte * H + c * U + unit[j]];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const int b = bt0 + bcol[e & 1], j = c * U + unit[e >> 1];
        hp[e] = h0 ? h0[((int64_t)d * B + b) * H + j] : 0.f;
    }
    // every CTA of the cluster has started and staged its tiles before any distributed-shared-memory store
    cluster_arrive();
    cluster_wait();

    const int DH = D * H;
    for (int s = 0; s < T; ++s) {
        const int t = d == 0 ? s : T - 1 - s;
        const int buf = s & 1;
        float giv[3][4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int64_t row = (int64_t)(bt0 + bcol[e & 1]) * T + t;
            const float* gr = gi + ((int64_t)d * B * T + row) * 3 * H + c * U + unit[e >> 1];
#pragma unroll
            for (int gte = 0; gte < 3; ++gte) giv[gte][e] = gr[gte * H];
        }
        float acc[3][4];
#pragma unroll
        for (int gte = 0; gte < 3; ++gte)
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[gte][e] = 0.f;
        const uint32_t hbase = smem_u32(Hsm + buf * NH * S::HBYTES);
        const uint32_t wbase = smem_u32(Wsm);
#pragma unroll 4
        for (int ks = 0; ks < H / 16; ++ks) {
            uint32_t bh[NH][2];
            const int brow = nt * 8 + (lane & 7), bk = ks * 16 + ((lane >> 3) & 1) * 8;
#pragma unroll
            for (int h = 0; h < NH; ++h) ldsm_x2(hbase + h * S::HBYTES + swz<H * 2>(brow, bk), bh[h]);
#pragma unroll
            for (int gte = 0; gte < 3; ++gte) {
                const int arow = gte * U + ug * 16 + (lane & 15), ak = ks * 16 + (lane >> 4) * 8;
                uint32_t a[NH][4];
#pragma unroll
                for (int h = 0; h < NH; ++h) ldsm_x4(wbase + h * S::WBYTES + swz<S::WP>(arow, ak), a[h]);
                if (NS != 1) {
                    mma_bf16(acc[gte], a[0], bh[NH - 1][0], bh[NH - 1][1]);
                    mma_bf16(acc[gte], a[NH - 1], bh[0][0], bh[0][1]);
                }
                mma_bf16(acc[gte], a[0], bh[0][0], bh[0][1]);
            }
        }
        const int nbuf = buf ^ 1;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int b = bt0 + bcol[e & 1], ul = unit[e >> 1], j = c * U + ul;
            const float r = sigmoid_f(giv[0][e] + acc[0][e] + bias[0][e >> 1]);
            const float z = sigmoid_f(giv[1][e] + acc[1][e] + bias[1][e >> 1]);
            const float hnv = acc[2][e] + bias[2][e >> 1];
            const float n = tanhf(giv[2][e] + r * hnv);
            const float h = (1.f - z) * n + z * hp[e];
            hp[e] = h;
            const int64_t row = (int64_t)b * T + t;
            Y[row * DH + d * H + j] = h;
            float* gs = G + ((int64_t)d * B * T + row) * 4 * H + j;
            gs[0] = r; gs[H] = z; gs[2 * H] = n; gs[3 * H] = hnv;
            if (hn_out && s == T - 1) hn_out[((int64_t)d * B + b) * H + j] = h;
            if (s + 1 < T) {
                bf16_t hi, lo;
                split_bf16(h, hi, lo);
                const uint32_t off = swz<H * 2>(bcol[e & 1], j);
                const uint32_t la = smem_u32(Hsm + nbuf * NH * S::HBYTES) + off;
#pragma unroll
                for (int p = 0; p < CS; ++p) {
                    st_cluster_b16(mapa(la, p), hi);
                    if (NH == 2) st_cluster_b16(mapa(la + S::HBYTES, p), lo);
                }
            }
        }
        cluster_arrive();
        cluster_wait();
    }
}

// ------------------------------------------------------------------------------------------------------
// Backward recurrence of one layer, both directions.  Layouts are those of gru_gates_bwd_kernel: G, Y, h0 as in the
// forward; dY [B][T][D*H]; dhc [D][B][H] carries dh into the layer's last step (head / zero) and returns dh_{-1};
// dgi, dgh [D][B*T][3H].  Shared memory: W^T rows (H) x own gate rows (192) | dgh tile [16][192] | receive slots of the
// peers' partial sums [CS-1][16][64] fp32 (this CTA's own partial goes into the dgh tile's space, which is free by then).
// Cluster barrier phases per step: (1) partials of the step have landed; (2) every CTA has read its receive slots, so
// the next step's partials may be written.
// ------------------------------------------------------------------------------------------------------
template <int H, int NS>
struct BwdSmem {
    static constexpr int NH = NS == 1 ? 1 : 2;
    static constexpr int Q = 3 * SCAN_U;                   // own gate rows
    static constexpr int WP = Q * 2;                        // W^T row pitch (bytes)
    static constexpr int WBYTES = H * WP;
    static constexpr int DBYTES = SCAN_NB * Q * 2;
    static constexpr int SLOT = SCAN_NB * SCAN_U * 4;
    static constexpr int TOTAL = NH * WBYTES + NH * DBYTES + (H / SCAN_U - 1) * SLOT;
    static_assert(NH * DBYTES >= SLOT, "own partial sums alias the dgh tile");
};

template <int H, int NS>
__global__ void __launch_bounds__(SCAN_THREADS, 1)
gru_scan_bwd_kernel(const float* __restrict__ G, const float* __restrict__ Y, const float* __restrict__ h0,
                    const float* __restrict__ dY, float* __restrict__ dhc, float* __restrict__ dgi, float* __restrict__ dgh,
                    const float* __restrict__ Whh, int64_t zW, int B, int T, int D) {
    using S = BwdSmem<H, NS>;
    constexpr int U = SCAN_U, CS = H / U, NH = S::NH, Q = S::Q, NB = SCAN_NB;
    constexpr int MT = H / 16 / 8;                           // m-tiles (16 rows of W^T) per warp
    constexpr int PAIRS = NB * U / SCAN_THREADS;             // (unit, column) pairs per thread in the gate math
    extern __shared__ __align__(128) uint8_t smem[];
    uint8_t* Wsm = smem;                                     // [NH][H rows][Q]
    uint8_t* Dsm = smem + NH * S::WBYTES;                    // [NH][NB rows][Q]; also this CTA's own partial [NB][U] fp32
    float* recv = reinterpret_cast<float*>(Dsm + NH * S::DBYTES);   // [CS-1][NB][U]
    const int c = (int)cluster_rank(), tile = blockIdx.y, d = blockIdx.z;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int bt0 = tile * NB;
    const float* W = Whh + d * zW;
    float* own = reinterpret_cast<float*>(Dsm);
    auto slot = [&](int src) -> float* { return src == c ? own : recv + (src < c ? src : src - 1) * NB * U; };

    for (int i = tid; i < Q * H; i += SCAN_THREADS) {
        const int q = i / H, k = i % H, gte = q / U, u = q % U;
        const float v = W[(int64_t)(gte * H + c * U + u) * H + k];
        bf16_t hi, lo;
        split_bf16(v, hi, lo);
        *reinterpret_cast<bf16_t*>(Wsm + swz<S::WP>(k, q)) = hi;
        if (NH == 2) *reinterpret_cast<bf16_t*>(Wsm + S::WBYTES + swz<S::WP>(k, q)) = lo;
    }
    float dhr[PAIRS], dhz[PAIRS];
#pragma unroll
    for (int i = 0; i < PAIRS; ++i) {
        const int p = tid + i * SCAN_THREADS, u = p % U, b = p / U;
        dhr[i] = dhc[((int64_t)d * B + bt0 + b) * H + c * U + u];
        dhz[i] = 0.f;
    }
    cluster_arrive();
    cluster_wait();

    const int DH = D * H;
    for (int s = 0; s < T; ++s) {
        const int t = d == 0 ? T - 1 - s : s;
        const bool first = d == 0 ? t == 0 : t == T - 1;
        if (s > 0) {
#pragma unroll
            for (int i = 0; i < PAIRS; ++i) {
                const int p = tid + i * SCAN_THREADS;
                float v = dhz[i];
#pragma unroll
                for (int src = 0; src < CS; ++src) v += slot(src)[p];
                dhr[i] = v;
            }
        }
        cluster_arrive();                                    // phase (2): this CTA's receive slots are read
        __syncthreads();                                     // own partial read before the dgh tile is rewritten
#pragma unroll
        for (int i = 0; i < PAIRS; ++i) {
            const int p = tid + i * SCAN_THREADS, u = p % U, bl = p / U, b = bt0 + bl, j = c * U + u;
            const int64_t row = (int64_t)b * T + t;
            const float* gs = G + ((int64_t)d * B * T + row) * 4 * H + j;
            const float r = gs[0], z = gs[H], n = gs[2 * H], hnv = gs[3 * H];
            float hpv;
            if (first) hpv = h0 ? h0[((int64_t)d * B + b) * H + j] : 0.f;
            else hpv = Y[((int64_t)b * T + (d == 0 ? t - 1 : t + 1)) * DH + d * H + j];
            const float dh = dhr[i] + dY[row * DH + d * H + j];
            const float dan = dh * (1.f - z) * (1.f - n * n);
            const float dar = dan * hnv * r * (1.f - r);
            const float daz = dh * (hpv - n) * z * (1.f - z);
            const float dgn = dan * r;
            float* a = dgi + ((int64_t)d * B * T + row) * 3 * H + j;
            float* cg = dgh + ((int64_t)d * B * T + row) * 3 * H + j;
            a[0] = dar; a[H] = daz; a[2 * H] = dan;
            cg[0] = dar; cg[H] = daz; cg[2 * H] = dgn;
            dhz[i] = dh * z;
            const float gv[3] = {dar, daz, dgn};
#pragma unroll
            for (int gte = 0; gte < 3; ++gte) {
                bf16_t hi, lo;
                split_bf16(gv[gte], hi, lo);
                *reinterpret_cast<bf16_t*>(Dsm + swz<S::WP>(bl, gte * U + u)) = hi;
                if (NH == 2) *reinterpret_cast<bf16_t*>(Dsm + S::DBYTES + swz<S::WP>(bl, gte * U + u)) = lo;
            }
        }
        __syncthreads();
        // partial dh_{t-1}[k, b] = sum over this CTA's gate rows q of W[q, k] dgh[b, q], for all H units k
        float acc[MT][2][4];
#pragma unroll
        for (int m = 0; m < MT; ++m)
#pragma unroll
            for (int n = 0; n < 2; ++n)
#pragma unroll
                for (int e = 0; e < 4; ++e) acc[m][n][e] = 0.f;
        const uint32_t wbase = smem_u32(Wsm), dbase = smem_u32(Dsm);
#pragma unroll 2
        for (int ks = 0; ks < Q / 16; ++ks) {
            uint32_t bv[NH][4];
            const int brow = (lane & 7) + ((lane >> 4) << 3), bk = ks * 16 + ((lane >> 3) & 1) * 8;
#pragma unroll
            for (int h = 0; h < NH; ++h) ldsm_x4(dbase + h * S::DBYTES + swz<S::WP>(brow, bk), bv[h]);
#pragma unroll
            for (int m = 0; m < MT; ++m) {
                const int arow = (warp + 8 * m) * 16 + (lane & 15), ak = ks * 16 + (lane >> 4) * 8;
                uint32_t a[NH][4];
#pragma unroll
                for (int h = 0; h < NH; ++h) ldsm_x4(wbase + h * S::WBYTES + swz<S::WP>(arow, ak), a[h]);
#pragma unroll
                for (int n = 0; n < 2; ++n) {
                    if (NS != 1) {
                        mma_bf16(acc[m][n], a[0], bv[NH - 1][2 * n], bv[NH - 1][2 * n + 1]);
                        mma_bf16(acc[m][n], a[NH - 1], bv[0][2 * n], bv[0][2 * n + 1]);
                    }
                    mma_bf16(acc[m][n], a[0], bv[0][2 * n], bv[0][2 * n + 1]);
                }
            }
        }
        __syncthreads();                                     // dgh tile consumed: its space takes the own partial
        cluster_wait();                                      // phase (2) complete: peers' receive slots are free
#pragma unroll
        for (int m = 0; m < MT; ++m)
#pragma unroll
            for (int n = 0; n < 2; ++n)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int k = (warp + 8 * m) * 16 + (lane >> 2) + (e >= 2 ? 8 : 0);
                    const int bl = n * 8 + 2 * (lane & 3) + (e & 1);
                    const int dst = k / U, kl = k % U;
                    if (dst == c) {
                        own[bl * U + kl] = acc[m][n][e];
                    } else {
                        // at CTA dst, the slot of source c is (c < dst ? c : c - 1)
                        const float* rs = recv + (c < dst ? c : c - 1) * NB * U + bl * U + kl;
                        st_cluster_f32(mapa(smem_u32(rs), dst), acc[m][n][e]);
                    }
                }
        cluster_arrive();                                    // phase (1): this step's partial sums are delivered
        cluster_wait();
    }
#pragma unroll
    for (int i = 0; i < PAIRS; ++i) {
        const int p = tid + i * SCAN_THREADS, u = p % U, b = p / U;
        float v = dhz[i];
#pragma unroll
        for (int src = 0; src < CS; ++src) v += slot(src)[p];
        dhc[((int64_t)d * B + bt0 + b) * H + c * U + u] = v;
    }
}

}  // namespace htc

// ---- host launchers ----------------------------------------------------------------------------------------
static inline int64_t rup(int64_t v, int64_t m) { return (v + m - 1) / m * m; }
// bf16 elements of the packed operand images of one GEMM (what tc_gemm_launch needs in its workspace)
static inline int64_t tc_gemm_ws_elems(int64_t M, int64_t N, int64_t K, int64_t batch, int prec) {
    const int nh = prec == BIGRU_PREC_BF16X3 ? 2 : 1;
    return nh * batch * (rup(M, htc::WG_BM) + rup(N, htc::WG_BN)) * rup(K, htc::WG_BK);
}

typedef CUresult (*PFN_encodeTiled_t)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                      const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                      CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
// tensor map over a packed image [rows][Kp] bf16: boxes of 64 (K) x 128 rows with 128-byte swizzle
static int make_pack_map(CUtensorMap* m, const void* base, int64_t rows, int64_t Kp) {
    static PFN_encodeTiled_t enc = nullptr;
    if (!enc) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) {
            bigru_set_error("tc_gemm: cuTensorMapEncodeTiled is unavailable");
            return BIGRU_ERR_CUDA;
        }
        enc = (PFN_encodeTiled_t)p;
    }
    const cuuint64_t dims[2] = {(cuuint64_t)Kp, (cuuint64_t)rows};
    const cuuint64_t strides[1] = {(cuuint64_t)Kp * 2};
    const cuuint32_t box[2] = {(cuuint32_t)htc::WG_BK, 128u}, es[2] = {1u, 1u};
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { bigru_set_error("tc_gemm: cuTensorMapEncodeTiled failed (%d)", (int)r); return BIGRU_ERR_CUDA; }
    return BIGRU_OK;
}

// prec: BIGRU_PREC_BF16 (NS = 1) or BIGRU_PREC_BF16X3 (NS = 3); ws: tc_gemm_ws_elems(...) bf16 elements
static int tc_gemm_launch(const GemmArgs& g, int prec, int cls, htc::bf16_t* ws, cudaStream_t st) {
    if (g.M <= 0 || g.N <= 0 || g.K <= 0) return BIGRU_OK;
    const bool x3 = prec == BIGRU_PREC_BF16X3;
    ProfScope ps(cls, 2.0 * g.M * g.N * (double)g.K * g.batch, 0.0, st);
    const int Mp = (int)rup(g.M, htc::WG_BM), Np = (int)rup(g.N, htc::WG_BN), Kp = (int)rup(g.K, htc::WG_BK);
    const int64_t asz = (int64_t)g.batch * Mp * Kp, bsz = (int64_t)g.batch * Np * Kp;
    htc::bf16_t* a_hi = ws;
    htc::bf16_t* a_lo = x3 ? a_hi + asz : nullptr;
    htc::bf16_t* b_hi = a_hi + (x3 ? 2 : 1) * asz;
    htc::bf16_t* b_lo = x3 ? b_hi + bsz : nullptr;
    htc::tc_pack_kernel<<<dim3(Kp / 32, Mp / 32, g.batch), dim3(32, 8), 0, st>>>(g.A, g.sam, g.sak, g.zA, g.M, g.K, Mp, Kp, g.mask_period,
                                                                                g.mask_skip, a_hi, a_lo);
    LAUNCH_CHECK();
    htc::tc_pack_kernel<<<dim3(Kp / 32, Np / 32, g.batch), dim3(32, 8), 0, st>>>(g.B, g.sbn, g.sbk, g.zB, g.N, g.K, Np, Kp, g.mask_period,
                                                                                g.mask_skip, b_hi, b_lo);
    LAUNCH_CHECK();
    CUtensorMap ta_hi, ta_lo, tb_hi, tb_lo;
    TRY(make_pack_map(&ta_hi, a_hi, (int64_t)g.batch * Mp, Kp));
    TRY(make_pack_map(&tb_hi, b_hi, (int64_t)g.batch * Np, Kp));
    if (x3) {
        TRY(make_pack_map(&ta_lo, a_lo, (int64_t)g.batch * Mp, Kp));
        TRY(make_pack_map(&tb_lo, b_lo, (int64_t)g.batch * Np, Kp));
    } else {
        ta_lo = ta_hi; tb_lo = tb_hi;
    }
    htc::WgOut o{g.C, g.bias, g.M, g.N, Kp / htc::WG_BK, Mp, Np, g.splitk, g.beta, g.ldc, g.zC, g.zBias};
    dim3 grid(Np / htc::WG_BN, Mp / htc::WG_BM, g.batch * g.splitk);
    constexpr int X3_STAGES = 3, BF_STAGES = 4;
    if (x3) {
        const int smem = X3_STAGES * 2 * 2 * 16384 + 1024 + 2 * X3_STAGES * 8;
        CUDA_TRY(cudaFuncSetAttribute(htc::wg_gemm_kernel<3, X3_STAGES>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        htc::wg_gemm_kernel<3, X3_STAGES><<<grid, 384, smem, st>>>(ta_hi, ta_lo, tb_hi, tb_lo, o);
    } else {
        const int smem = BF_STAGES * 2 * 16384 + 1024 + 2 * BF_STAGES * 8;
        CUDA_TRY(cudaFuncSetAttribute(htc::wg_gemm_kernel<1, BF_STAGES>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        htc::wg_gemm_kernel<1, BF_STAGES><<<grid, 384, smem, st>>>(ta_hi, ta_lo, tb_hi, tb_lo, o);
    }
    LAUNCH_CHECK();
    return BIGRU_OK;
}

template <typename... KArgs, typename... Args>
static int launch_cluster(void (*kernel)(KArgs...), int cs, int ntiles, int D, int smem, cudaStream_t st, Args... args) {
    CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(cs, ntiles, D);
    cfg.blockDim = dim3(htc::SCAN_THREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = cs; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    CUDA_TRY(cudaLaunchKernelEx(&cfg, kernel, args...));
    return BIGRU_OK;
}

// one layer's forward recurrence; shapes were validated by the plan (H in {128, 256, 512}, B % 16 == 0)
static int tc_scan_fwd(const bigru_plan& p, int l, const float* gi, const float* Whh, const float* bhh, const float* h0,
                       float* Y, float* G, float* hn, cudaStream_t st) {
    const int H = p.H, D = p.D, B = p.B, T = p.T, cs = H / htc::SCAN_U, nt = B / htc::SCAN_NB;
    const int64_t zW = p.ld_block(l);
    ProfScope ps(KC_TC_SCAN_FWD, 2.0 * D * B * (double)T * 3 * H * H, 0.0, st);
#define FWD(HH, NS) return launch_cluster(htc::gru_scan_fwd_kernel<HH, NS>, cs, nt, D, htc::FwdSmem<HH, NS>::TOTAL, st, gi, Whh, bhh, zW, h0, Y, G, hn, B, T, D)
    if (p.prec == BIGRU_PREC_BF16X3) {
        if (H == 128) FWD(128, 3);
        if (H == 256) FWD(256, 3);
    } else {
        if (H == 128) FWD(128, 1);
        if (H == 256) FWD(256, 1);
        if (H == 512) FWD(512, 1);
    }
#undef FWD
    bigru_set_error("tc_scan_fwd: no kernel for H=%d at precision %d", H, p.prec);
    return BIGRU_ERR_UNSUPPORTED;
}

static int tc_scan_bwd(const bigru_plan& p, int l, const float* G, const float* Y, const float* h0, const float* dY, float* dhc,
                       float* dgi, float* dgh, const float* Whh, cudaStream_t st) {
    const int H = p.H, D = p.D, B = p.B, T = p.T, cs = H / htc::SCAN_U, nt = B / htc::SCAN_NB;
    const int64_t zW = p.ld_block(l);
    ProfScope ps(KC_TC_SCAN_BWD, 2.0 * D * B * (double)T * 3 * H * H, 0.0, st);
#define BWD(HH, NS) return launch_cluster(htc::gru_scan_bwd_kernel<HH, NS>, cs, nt, D, htc::BwdSmem<HH, NS>::TOTAL, st, G, Y, h0, dY, dhc, dgi, dgh, Whh, zW, B, T, D)
    if (p.prec == BIGRU_PREC_BF16X3) {
        if (H == 128) BWD(128, 3);
        if (H == 256) BWD(256, 3);
    } else {
        if (H == 128) BWD(128, 1);
        if (H == 256) BWD(256, 1);
        if (H == 512) BWD(512, 1);
    }
#undef BWD
    bigru_set_error("tc_scan_bwd: no kernel for H=%d at precision %d", H, p.prec);
    return BIGRU_ERR_UNSUPPORTED;
}
