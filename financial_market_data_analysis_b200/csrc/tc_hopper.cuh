// tc_hopper.cuh - the tensor-core pieces of BIGRU_PREC_BF16 and BIGRU_PREC_BF16X3 on sm_90a (H100).
//
// Both precisions share the data layout and step composition of the fp32 path (api.cu): time steps of the recurrence and
// all GEMMs read and write the same fp32 buffers.  What changes is where the arithmetic runs:
//   * wg_gemm             - a persistent TMA + mbarrier pipelined wgmma GEMM (wg_gemm_kernel) over bf16 operand planes that
//                           the scans and to_planes_kernel write next to the fp32 activations; deterministic split-K.
//                           tc_gemm_launch keeps the GemmArgs contract for the small head / h0 GEMMs (operands packed).
//   * gru_scan_fwd_kernel - one layer's whole forward recurrence in one launch: a thread-block cluster per direction and
//                           one or, at bf16x3, two 16-row batch tiles (how many take two follows from how many clusters
//                           the device holds at once: scan_geometry); CTA c of the cluster owns hidden units [64c, 64c+64) and keeps
//                           their W_hh rows (3 gates x 64 units x H) resident in shared memory for all T steps.  Each step it
//                           multiplies them with h_{t-1} of the tile, runs the gate math in registers and bulk-copies its
//                           slice of h_t into the shared memory of every CTA of the cluster (distributed shared memory),
//                           where an mbarrier counts the bytes in.
//   * gru_scan_bwd_kernel - the backward recurrence, reduction-partitioned: CTA c keeps W_hh^T restricted to its own units'
//                           gate rows (H x 192), multiplies it with its local dgh tile and sends each peer the fp32 partial
//                           sums of dh_{t-1} for the peer's units; the owner adds them up.  One 16-row tile per cluster, or 8
//                           rows in a short last round (scan_bwd_geometry).
// Precision: NS = 1 (bf16) uses single bf16 operands; NS = 3 (bf16x3) splits every operand x = hi + lo (both bf16, |lo| <=
// 2^-9 |x|) and adds hi*hi + hi*lo + lo*hi (the dropped lo*lo term is below 2^-16 relative), all with fp32 accumulation:
// fp32-class results on the tensor cores.  State, gate math, stash and gradients are fp32 in both.
// H100 budget that shapes the scans: 227 KB of shared memory per block holds a 64-unit slice of W_hh at H = 256 as hi/lo
// pairs (192 KB) or at H = 512 in bf16 (192 KB), next to the forward's h tile (one 32-row buffer at bf16x3); clusters of
// H/64 <= 8 CTAs stay within the portable cluster size.
#pragma once
#include "common.cuh"
#include "kernels_f32.cuh"
#include <algorithm>
#include <map>
#include <mutex>
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
__device__ __forceinline__ void st_cluster_v2_f32(uint32_t addr, float2 v) {
    asm volatile("st.shared::cluster.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(v.x), "f"(v.y) : "memory");
}
__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire;" ::: "memory"); }
__device__ __forceinline__ uint32_t cluster_rank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}

// ------------------------------------------------------------------------------------------------------
// GEMM: C[z][m,n] (+)= sum_k A(m,k) B(n,k) (+ bias[n]) on bf16 planes (hi, and lo at bf16x3) that TMA reads straight from
// where their producers left them: the scans write Y, dgi and dgh planes next to their fp32 copies, the layer input gets
// planes from to_planes_kernel, and the small weight operands are packed per call by tc_pack_kernel.
//   * operands are K-major (box 64 K x 128 rows) or MN-major (two boxes 64 MN x 64 K rows; the k = b*t reduction of the
//     weight gradients runs down the rows of the activations), all with 128-byte swizzle; TMA's out-of-bounds zero fill
//     covers ragged M, N and K edges, and the +-1 row shift of h_{t-1} in dW_hh;
//   * persistent: at most one CTA per SM strides over (tile, split) units.  One thread streams 64-deep k-blocks through a
//     STAGES-deep mbarrier ring and runs ahead across unit boundaries; two consumer warpgroups (64 rows each) multiply with
//     wgmma.m64n128k16 (fp32 accumulation), keep one wgmma group in flight and release the previous stage;
//     bf16x3 issues hi*hi + hi*lo + lo*hi per k-step;
//   * split-K units write fp32 partials; splitk_reduce_kernel adds them in split order (no atomics: bit-reproducible);
//   * jobs that overwrite a 16-byte-aligned C with rows of whole 16-byte chunks (WgJob::cmap) stage each warpgroup's
//     64 x 128 result, bias added, in shared memory as 64 x 32 boxes and send them with bulk tensor stores that drain while
//     the next unit's mainloop runs; the others (beta accumulation, unaligned C, N % 4 != 0) store straight from registers.
// ------------------------------------------------------------------------------------------------------
constexpr int WG_BM = 128, WG_BN = 128, WG_BK = 64;
constexpr int WG_CBOX = 64 * 32 * 4;                          // one staging box: 64 rows x 32 fp32 (128-byte rows)
// staging boxes per consumer warpgroup: a whole 64 x 128 result at bf16; at bf16x3 the 3-stage ring leaves room for two
__host__ __device__ constexpr int wg_cboxes(int ns) { return ns == 1 ? 4 : 2; }
__host__ __device__ constexpr int wg_smem_bytes(int ns, int stages) {
    return 1024 + stages * 2 * (ns == 1 ? 1 : 2) * WG_BM * WG_BK * 2 + 2 * wg_cboxes(ns) * WG_CBOX + 2 * stages * 8;
}

// packs a small fp32 operand (weights, head activations) into a zero-padded K-major image [batch][Rp][Kp], hi and lo planes
__global__ void tc_pack_kernel(const float* __restrict__ src, int64_t s_r, int64_t s_k, int64_t zsrc, int R, int K, int Rp, int Kp,
                               bf16_t* __restrict__ hi, bf16_t* __restrict__ lo) {
    __shared__ float tile[32][33];
    const int z = blockIdx.z, r0 = blockIdx.y * 32, k0 = blockIdx.x * 32;
    const float* a = src + z * zsrc;
    const bool kfast = s_k == 1;
    for (int j = threadIdx.y; j < 32; j += 8) {
        const int r = r0 + (kfast ? j : threadIdx.x), k = k0 + (kfast ? threadIdx.x : j);
        float v = 0.f;
        if (r < R && k < K) v = a[(int64_t)r * s_r + (int64_t)k * s_k];
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

// bf16 planes of a row-major fp32 matrix [rows][cols]; row pitch `pitch` elements (a multiple of 8: 16-byte TMA strides)
__global__ void to_planes_kernel(const float* __restrict__ src, int64_t rows, int cols, int pitch, bf16_t* __restrict__ hi,
                                 bf16_t* __restrict__ lo) {
    const int64_t n = rows * cols;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / cols, c = i % cols, o = r * pitch + c;
        bf16_t h, l;
        split_bf16(src[i], h, l);
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
// the same with acquire at cluster scope: the phase's bytes were written by peer CTAs' bulk copies
__device__ __forceinline__ bool mbar_try_wait_cluster(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
// a wait that has not completed after 5 s of wall clock means the pipeline protocol is broken: stop the kernel (the launch
// reports an error) rather than occupy the GPU
template <bool CLUSTER = false>
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    auto ready = [&] { return CLUSTER ? mbar_try_wait_cluster(bar, parity) : mbar_try_wait(bar, parity); };
    if (ready()) return;
    uint64_t t0, t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
    for (uint32_t i = 0;; ++i) {
        if (ready()) return;
        if ((i & 1023u) == 1023u) {
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
            if (t - t0 > 5000000000ull) __trap();
        }
    }
}
// bytes from this CTA's shared memory at src to CTA `cta` of the cluster at dst (an offset in this CTA's shared window,
// mapped to the peer's); completes on that CTA's mbarrier.  Only the peer's mbarrier tracks the copy: no bulk group does, so
// the source may be rewritten only once the peer has reported the phase complete
__device__ __forceinline__ void bulk_copy_to_peer_at(uint32_t dst, uint32_t src, uint32_t bytes, uint64_t* bar, uint32_t cta) {
    asm volatile("cp.async.bulk.shared::cluster.shared::cta.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(mapa(dst, cta)), "r"(src), "r"(bytes), "r"(mapa(smem_u32(bar), cta)) : "memory");
}
// the same at the same offset in the peer
__device__ __forceinline__ void bulk_copy_to_peer(uint32_t src, uint32_t bytes, uint64_t* bar, uint32_t cta) {
    bulk_copy_to_peer_at(src, src, bytes, bar, cta);
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
                 ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
// one box from shared memory to global; TMA clips the rows and columns that fall outside the map
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* m, uint32_t src, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
                 ::"l"(reinterpret_cast<uint64_t>(m)), "r"(src), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// at most N of this thread's bulk groups still read shared memory
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void named_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
// wgmma shared-memory descriptor, 128-byte swizzle.  K-major: rows of 64 bf16 (128 B), 8-row groups 1024 B apart.
// MN-major: lines of 64 MN elements per k, 8-k groups 1024 B apart (stride byte offset), 64-element MN blocks 8 KB apart
// (leading byte offset: one 64 x 64 TMA box).
__device__ __forceinline__ uint64_t wg_desc(uint32_t saddr, uint32_t lbo) {
    return (uint64_t)((saddr & 0x3FFFF) >> 4) | ((uint64_t)(lbo >> 4) << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
// TA / TB: 1 = MN-major ("transposed") shared-memory operand
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t da, uint64_t db) {
    asm volatile("wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, 1, 1, 1, %66, %67;"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "l"(da), "l"(db), "n"(TA), "n"(TB));
}

// one operand of a GEMM: tensor maps are 3-D [depth][rows][cols] (cols innermost).  For the k-block of direction dz:
// K-major coordinates (k, r0, dz * zsel); MN-major (r0 + dz * coff, k + kshift[dz], dz * zsel)
struct WgOp {
    int zsel, coff, kshift[2];
};
struct WgJob {
    WgOp a, b;
    float* C; const float* bias; float* part;  // part: [splits][batch][M][N] fp32 partials when splits > 1
    int M, N, tm, tn, batch, splits;
    int kblocks, kbd;                           // k-blocks per unit's full K range; per direction when kcat
    int kcat;                                   // 1: the K loop runs over direction 0, then direction 1 (dz = kb / kbd)
    int beta;
    int cmap;                                   // 1: C (or part) goes out through the C tensor map, staged in shared memory
    int64_t ldc, zC, zBias;
};

template <int NS, int STAGES, int AMN, int BMN>
__global__ void __launch_bounds__(384, 1)
wg_gemm_kernel(const __grid_constant__ CUtensorMap ta_hi, const __grid_constant__ CUtensorMap ta_lo,
               const __grid_constant__ CUtensorMap tb_hi, const __grid_constant__ CUtensorMap tb_lo,
               const __grid_constant__ CUtensorMap tc, const WgJob j) {
    constexpr int NH = NS == 1 ? 1 : 2;
    constexpr int PLANE = WG_BM * WG_BK * 2;                  // 16 KB: one 128 x 64 bf16 tile
    constexpr int STAGE = 2 * NH * PLANE;                     // A planes, then B planes
    constexpr int CB = wg_cboxes(NS);
    extern __shared__ __align__(1024) uint8_t wg_smem_raw[];
    uint8_t* sm = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(wg_smem_raw) + 1023) & ~(uintptr_t)1023);
    uint64_t* full = reinterpret_cast<uint64_t*>(sm + STAGES * STAGE + 2 * CB * WG_CBOX);
    uint64_t* empty = full + STAGES;
    const int wgi = threadIdx.x / 128, tid = threadIdx.x % 128;
    const int units = j.tm * j.tn * j.batch * j.splits;
    const int per = (j.kblocks + j.splits - 1) / j.splits;
    if (threadIdx.x == 0) {
        for (int i = 0; i < STAGES; ++i) { mbar_init(full + i, 1); mbar_init(empty + i, 2); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    // unit u: split fastest, then n tile, m tile, batch (consecutive units share the A rows of a tile row)
    auto decode = [&](int u, int& s, int& zb, int& m0, int& n0) {
        s = u % j.splits; u /= j.splits;
        n0 = (u % j.tn) * WG_BN; u /= j.tn;
        m0 = (u % j.tm) * WG_BM; zb = u / j.tm;
    };

    if (wgi == 0) {                                           // producer
        if (tid == 0) {
            uint32_t it = 0;
            for (int u = blockIdx.x; u < units; u += gridDim.x) {
                int s, zb, m0, n0;
                decode(u, s, zb, m0, n0);
                const int kb1 = min(j.kblocks, (s + 1) * per);
                for (int kb = s * per; kb < kb1; ++kb, ++it) {
                    const int st = it % STAGES;
                    if (it >= STAGES) mbar_wait(empty + st, ((it / STAGES) - 1) & 1);
                    const uint32_t base = smem_u32(sm + st * STAGE);
                    mbar_arrive_expect_tx(full + st, STAGE);
                    const int dz = j.kcat ? kb / j.kbd : zb, kc = (j.kcat ? kb % j.kbd : kb) * WG_BK;
#pragma unroll
                    for (int h = 0; h < NH; ++h) {
                        const CUtensorMap* ma = h ? &ta_lo : &ta_hi;
                        const CUtensorMap* mb = h ? &tb_lo : &tb_hi;
                        const uint32_t da = base + h * PLANE, db = base + (NH + h) * PLANE;
                        if (AMN) {
                            const int k = kc + (dz ? j.a.kshift[1] : j.a.kshift[0]), r = m0 + dz * j.a.coff;
                            tma_load_3d(da, ma, full + st, r, k, dz * j.a.zsel);
                            tma_load_3d(da + PLANE / 2, ma, full + st, r + 64, k, dz * j.a.zsel);
                        } else {
                            tma_load_3d(da, ma, full + st, kc, m0, dz * j.a.zsel);
                        }
                        if (BMN) {
                            const int k = kc + (dz ? j.b.kshift[1] : j.b.kshift[0]), r = n0 + dz * j.b.coff;
                            tma_load_3d(db, mb, full + st, r, k, dz * j.b.zsel);
                            tma_load_3d(db + PLANE / 2, mb, full + st, r + 64, k, dz * j.b.zsel);
                        } else {
                            tma_load_3d(db, mb, full + st, kc, n0, dz * j.b.zsel);
                        }
                    }
                }
            }
        }
        return;
    }
    const int cg = wgi - 1;                                   // consumer warpgroup: rows cg*64 .. +64 of the tile
    const int w = tid / 32, l = tid % 32;
    // per k-step (16 deep) address advance: 32 B along a K-major row, 16 lines of 128 B down an MN-major box
    constexpr uint32_t AKS = AMN ? 2048 : 32, BKS = BMN ? 2048 : 32;
    constexpr uint32_t ALBO = AMN ? PLANE / 2 : 16, BLBO = BMN ? PLANE / 2 : 16;
    uint32_t it = 0;
    for (int u = blockIdx.x; u < units; u += gridDim.x) {
        int s, zb, m0, n0;
        decode(u, s, zb, m0, n0);
        const int kb1 = min(j.kblocks, (s + 1) * per);
        float d[64];
#pragma unroll
        for (int i = 0; i < 64; ++i) d[i] = 0.f;
        int prev = -1;
        for (int kb = s * per; kb < kb1; ++kb, ++it) {
            const int st = it % STAGES;
            mbar_wait(full + st, (it / STAGES) & 1);
            const uint32_t base = smem_u32(sm + st * STAGE);
            const uint32_t a_hi = base + cg * (PLANE / 2), a_lo = a_hi + PLANE;
            const uint32_t b_hi = base + NH * PLANE, b_lo = b_hi + PLANE;
            asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
            for (int ks = 0; ks < WG_BK / 16; ++ks) {
                wgmma_m64n128k16<AMN, BMN>(d, wg_desc(a_hi + ks * AKS, ALBO), wg_desc(b_hi + ks * BKS, BLBO));
                if (NS != 1) {
                    wgmma_m64n128k16<AMN, BMN>(d, wg_desc(a_hi + ks * AKS, ALBO), wg_desc(b_lo + ks * BKS, BLBO));
                    wgmma_m64n128k16<AMN, BMN>(d, wg_desc(a_lo + ks * AKS, ALBO), wg_desc(b_hi + ks * BKS, BLBO));
                }
            }
            asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
            asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory");   // the previous k-block's group is done
            if (prev >= 0 && tid == 0) mbar_arrive(empty + prev);
            prev = st;
        }
        asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
        if (prev >= 0 && tid == 0) mbar_arrive(empty + prev);
        if (j.cmap) {
            // box c holds columns 32c .. +32 of the warpgroup's 64 rows in staging slot c % CB.  Row r's 16-byte chunk k sits
            // at chunk k ^ (r % 8), the 128-byte swizzle of the map, so a warp's v2 stores (8 rows x 32 B) hit every bank twice
            const float* bias = j.splits == 1 && j.bias ? j.bias + zb * j.zBias : nullptr;
            const int zc = j.splits > 1 ? s * j.batch + zb : zb;
            const int q = l & 3, r8 = l >> 2;
            float bv[32];
#pragma unroll
            for (int i = 0; i < 16; ++i)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int gn = n0 + 8 * i + 2 * q + e;
                    bv[2 * i + e] = bias && gn < j.N ? bias[gn] : 0.f;
                }
            uint8_t* stg = sm + STAGES * STAGE + cg * CB * WG_CBOX;
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                const uint32_t box = smem_u32(stg + (c % CB) * WG_CBOX);
                if (tid == 0) bulk_wait_read<CB - 1>();       // the store that last read this slot is done with it
                named_sync(1 + cg, 128);
#pragma unroll
                for (int ii = 0; ii < 4; ++ii) {
                    const int i = 4 * c + ii;
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        float v0 = d[4 * i + 2 * h], v1 = d[4 * i + 2 * h + 1];
                        if (bias) { v0 += bv[2 * i]; v1 += bv[2 * i + 1]; }
                        const uint32_t a = box + (w * 16 + r8 + 8 * h) * 128 + (((2 * ii + (q >> 1)) ^ r8) << 4) + (q & 1) * 8;
                        asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a), "f"(v0), "f"(v1) : "memory");
                    }
                }
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // the writes, visible to the bulk copy
                named_sync(1 + cg, 128);
                if (tid == 0) {
                    if (n0 + 32 * c < j.N) tma_store_3d(&tc, box, n0 + 32 * c, m0 + cg * 64, zc);
                    bulk_commit();
                }
            }
            continue;
        }
        // direct stores from registers: the only path for jobs that add to C (beta), for a C whose base or row pitch is not
        // 16-byte aligned, which a tensor map cannot describe, and for rows that end inside a 16-byte chunk (e.g. N = 13
        // features), which a bulk tensor store would overrun
        float* C;
        int64_t ldc;
        const float* bias = nullptr;
        if (j.splits > 1) {
            C = j.part + ((int64_t)s * j.batch + zb) * j.M * j.N;
            ldc = j.N;
        } else {
            C = j.C + zb * j.zC;
            ldc = j.ldc;
            if (j.bias) bias = j.bias + zb * j.zBias;
        }
#pragma unroll
        for (int i = 0; i < 16; ++i)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int gm = m0 + cg * 64 + w * 16 + (l >> 2) + (e >= 2 ? 8 : 0);
                const int gn = n0 + 8 * i + 2 * (l & 3) + (e & 1);
                if (gm >= j.M || gn >= j.N) continue;
                float v = d[4 * i + e];
                if (bias) v += bias[gn];
                float* c = C + (int64_t)gm * ldc + gn;
                if (j.beta && j.splits == 1) *c += v;
                else *c = v;
            }
    }
    if (j.cmap && tid == 0) bulk_wait_all();
}

// C[z][m][n] (+)= sum over s = 0, 1, ... of part[s][z][m][n]: the split-K partial sums in a fixed order
__global__ void splitk_reduce_kernel(const float* __restrict__ part, int splits, int batch, int M, int N, float* __restrict__ C,
                                     int64_t ldc, int64_t zC, int beta) {
    const int64_t per = (int64_t)M * N, n = per * batch;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        float v = 0.f;
        for (int s = 0; s < splits; ++s) v += part[(int64_t)s * n + i];
        const int64_t z = i / per, r = i % per;
        float* c = C + z * zC + (r / N) * ldc + r % N;
        *c = beta ? *c + v : v;
    }
}

// ------------------------------------------------------------------------------------------------------
// Forward recurrence of one layer, both directions.  Layouts are those of gru_gates_fwd_kernel:
//   gi [D][B*T][3H] (x W_ih^T + b_ih), Y [B][T][D*H], G [D][B*T][4H] = (r, z, n, W_hn h + b_hn), hn [D][B][H].
// Y also goes out as bf16 planes (yh, and yl at bf16x3) in Y's layout: the next layer's projection and the weight gradients
// read them.
// Grid (CS, clusters, 1), cluster (CS, 1, 1), 256 threads.  A cluster takes one or two (bf16x3 only) 16-row batch tiles of
// one direction (scan_tile): nb = 16 or 32 rows.  Warp w owns units 16*(w/2) .. +16 of the CTA's slice and nb/2 batch columns from
// (w%2)*nb/2, one or two n8 blocks: each W fragment it loads feeds every block, so a 32-row tile reads W from shared memory
// as often as a 16-row one.  Its r, z and n accumulators hold the same (unit, column) pairs, so the gate math needs no
// exchange.  Every output element comes from the same MMA sequence over k whatever the tile size: a row's bits do not
// depend on its cluster's tile.
// The h tile is laid out [NBUF][NH][CS][nb rows][64 units] in one region that holds two 16-row buffers or one 32-row
// buffer (NBUF = 2 or 1): CTA c's part of a plane is one block at the same offset in every CTA.  Each step a CTA writes its h_t into its own block, and one thread sends that block to every peer with a bulk
// copy, which completes on the peer's "full" mbarrier of that buffer.  Before its next multiply a CTA waits on that barrier
// for the (CS - 1) blocks of its peers.  With one buffer (bf16x3, 32 rows) a CTA also arrives on every peer's "empty"
// mbarrier after its multiply: its reads of the tile are done.  There is no cluster barrier per step.
// OUT selects at compile time which of Y, G and the Y planes are written (hn_out is written whenever it is non-null): the
// training forward keeps all three for the backward; inference writes the planes of a lower layer (the next projection reads
// them) and the fp32 Y of the top layer (the pooling head reads it).  The h arithmetic is the same in every instantiation.
// LEN: per-sequence lengths (lens [B], 1 <= len <= T).  A padded (row, t >= len) keeps its state (hp and the h tile) and skips
// G; its Y row and Y plane rows are 0, so the reverse direction stays at the zero state until t = len - 1 and hn is the state
// after the row's last valid step.  Without LEN the kernel is the one without lengths, instruction for instruction.
// ------------------------------------------------------------------------------------------------------
constexpr int SCAN_U = 64, SCAN_NB = 16, SCAN_THREADS = 256;
constexpr int SCAN_Y = 1, SCAN_G = 2, SCAN_PLANES = 4;
constexpr int SCAN_TRAIN = SCAN_Y | SCAN_G | SCAN_PLANES, SCAN_INFER_LOWER = SCAN_PLANES, SCAN_INFER_TOP = SCAN_Y;

template <int H, int NS>
struct FwdSmem {
    static constexpr int NH = NS == 1 ? 1 : 2;
    // rows of the largest tile a cluster takes: 32 at bf16x3, where a CTA has its SM to itself; 16 at bf16, where a 32-row
    // body's registers would keep a second CTA off the SM (H <= 256) or its tile would not fit (H = 512)
    static constexpr int NBMAX = NS == 1 ? SCAN_NB : 2 * SCAN_NB;
    // buffers of the largest tile: a double-buffered 32-row tile does not fit.  The same bytes hold two 16-row buffers, so
    // 16-row tiles are double-buffered at every precision
    static constexpr int NBUF = NBMAX == SCAN_NB ? 2 : 1;
    static constexpr int WP = H * 2;                        // W row pitch (bytes): K = H
    static constexpr int WBYTES = 3 * SCAN_U * WP;          // one of hi / lo
    static constexpr int HBYTES = NBMAX * H * 2;            // h tile, one of hi / lo
    static constexpr int SLICE = NBMAX * SCAN_U * 2;        // one CTA's block of one h plane: NBMAX rows x 128 B
    static constexpr int TOTAL = NH * WBYTES + NBUF * NH * HBYTES + 2 * 8;   // + two full barriers, or full and empty
};

// the batch tile of cluster q (blockIdx.y): the first D * m2 clusters take 32 rows, m2 per direction; the others 16.  ntd:
// 16-row tiles per direction (B / 16)
__device__ __forceinline__ void scan_tile(int q, int m2, int ntd, int D, int& d, int& bt0, int& nb) {
    if (q < D * m2) {
        d = q / m2; bt0 = (q % m2) * 2 * SCAN_NB; nb = 2 * SCAN_NB;
    } else {
        const int r = q - D * m2, o = ntd - 2 * m2;
        d = r / o; bt0 = (2 * m2 + r % o) * SCAN_NB; nb = SCAN_NB;
    }
}

// byte offset of h element (row b, unit k) in one plane of the forward h tile: 128-byte rows within the block of the units'
// CTA, chunks XOR-swizzled as in swz
template <int NBMAX>
__device__ __forceinline__ uint32_t hsw(int b, int k) {
    return (uint32_t)((k / SCAN_U) * (NBMAX * SCAN_U * 2)) + swz<SCAN_U * 2>(b, k % SCAN_U);
}

__device__ __forceinline__ void mbar_arrive_peer(uint64_t* bar, uint32_t cta) {
    asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(mapa(smem_u32(bar), cta)) : "memory");
}

// the scan of one cluster whose tile has JN * 16 rows from bt0, direction d.  RD: recurrent dropout with the layer's masks
// `mask` [D][B][H] (DESIGN.md §4.8): the h tile holds m * h (staged from m * h0), the carry is z * (m * h_{t-1}), and the own
// block's copy (yh, yl) is the masked state; Y, hn and the carried hp stay unmasked
template <int H, int NS, int OUT, bool LEN, int JN, bool RD = false>
__device__ __forceinline__ void gru_scan_fwd_tile(const float* __restrict__ gi, const float* __restrict__ Whh,
                                                  const float* __restrict__ bhh, int64_t zW, const float* __restrict__ h0,
                                                  float* __restrict__ Y, float* __restrict__ G, float* __restrict__ hn_out,
                                                  bf16_t* __restrict__ yh, bf16_t* __restrict__ yl, int B, int T, int D,
                                                  const int* __restrict__ lens, int d, int bt0,
                                                  const float* __restrict__ mask = nullptr) {
    using S = FwdSmem<H, NS>;
    constexpr int U = SCAN_U, CS = H / U, NH = S::NH, JMAX = JN, jn = JN, nb = JN * SCAN_NB;   // jn n8 blocks per warp
    // the h region holds two 16-row buffers or one 32-row buffer: a 16-row tile is double-buffered, a 32-row tile is not
    constexpr int NBMAX = nb, NBUF = S::NBUF * S::NBMAX / nb;
    constexpr int HBYTES = nb * H * 2, SLICE = nb * U * 2;  // one buffer of one h plane; one CTA's block of it
    static_assert(NBUF * HBYTES == S::NBUF * S::HBYTES, "both tile sizes fill the h region");
    static_assert(SCAN_THREADS % (nb * (U / 8)) == 0, "a thread copies the same Y plane row in every pass");
    extern __shared__ __align__(128) uint8_t smem[];
    uint8_t* Wsm = smem;                                     // [NH][3U rows][H]
    uint8_t* Hsm = smem + NH * S::WBYTES;                    // [NBUF][NH][CS][NBMAX rows][U]
    uint64_t* full = reinterpret_cast<uint64_t*>(Hsm + NBUF * NH * HBYTES);   // [2]: two buffers' full, or full and empty
    uint64_t* empty = full + 1;                              // NBUF == 1
    const int c = (int)cluster_rank();
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const float* W = Whh + d * zW;

    for (int i = tid; i < 3 * U * H; i += SCAN_THREADS) {
        const int q = i / H, k = i % H, gte = q / U, u = q % U;
        const float v = W[(int64_t)(gte * H + c * U + u) * H + k];
        bf16_t hi, lo;
        split_bf16(v, hi, lo);
        *reinterpret_cast<bf16_t*>(Wsm + swz<S::WP>(q, k)) = hi;
        if (NH == 2) *reinterpret_cast<bf16_t*>(Wsm + S::WBYTES + swz<S::WP>(q, k)) = lo;
    }
    for (int i = tid; i < nb * H; i += SCAN_THREADS) {
        const int b = i / H, k = i % H;
        float v = h0 ? h0[((int64_t)d * B + bt0 + b) * H + k] : 0.f;
        if constexpr (RD) v *= mask[((int64_t)d * B + bt0 + b) * H + k];
        bf16_t hi, lo;
        split_bf16(v, hi, lo);
        *reinterpret_cast<bf16_t*>(Hsm + hsw<NBMAX>(b, k)) = hi;
        if (NH == 2) *reinterpret_cast<bf16_t*>(Hsm + HBYTES + hsw<NBMAX>(b, k)) = lo;
    }
    if (tid == 0) {
        mbar_init(full, 1);
        mbar_init(full + 1, NBUF == 2 ? 1 : CS - 1);     // the second buffer's full, or empty
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }

    const int ug = warp >> 1, nt = warp & 1;
    int unit[2], bcol[JMAX][2];
    unit[0] = ug * 16 + (lane >> 2); unit[1] = unit[0] + 8;
#pragma unroll
    for (int j = 0; j < JMAX; ++j) {
        bcol[j][0] = (nt * jn + j) * 8 + 2 * (lane & 3); bcol[j][1] = bcol[j][0] + 1;
    }
    float bias[3][2], hp[JMAX][4], mk[RD ? JMAX : 1][4];
#pragma unroll
    for (int gte = 0; gte < 3; ++gte)
#pragma unroll
        for (int i = 0; i < 2; ++i) bias[gte][i] = bhh[d * zW + gte * H + c * U + unit[i]];
    // lengths of this thread's batch columns, and of the row it copies to the Y planes (the same row in every pass of the
    // copy loop: SCAN_THREADS is a multiple of nb * U / 8)
    int len[JMAX][2], rlen = T;
#pragma unroll
    for (int j = 0; j < JMAX; ++j) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int b = bt0 + bcol[j][e & 1], k = c * U + unit[e >> 1];
            hp[j][e] = h0 ? h0[((int64_t)d * B + b) * H + k] : 0.f;
            if constexpr (RD) mk[j][e] = mask[((int64_t)d * B + b) * H + k];
        }
        len[j][0] = len[j][1] = T;
        if (LEN) { len[j][0] = lens[bt0 + bcol[j][0]]; len[j][1] = lens[bt0 + bcol[j][1]]; }
    }
    if (LEN) rlen = lens[bt0 + (tid / (U / 8)) % nb];
    // every CTA of the cluster has started, staged its tiles and initialised its barriers before any bulk copy or arrive
    cluster_arrive();
    cluster_wait();

    // Step s multiplies with buffer buf (h_{s-1}; h0 at s = 0) and produces h_s in buffer nbuf: with two buffers buf = s & 1
    // and nbuf = buf ^ 1, and each buffer's full barrier completes every other step (phase (s - 1) / 2 is awaited at step
    // s); with one buffer both are 0, and full and empty complete once per step (phase s).  The last step sends nothing:
    // only its own block is read (Y planes).
    // Two buffers, write after read: a peer sends its h_{s+1} into this CTA's buffer buf (the one step s reads) only after
    // its own full barrier for h_s has completed, which needs this CTA's h_s, which this CTA sends only after the
    // __syncthreads that follows its step-s multiply.  The own block of a buffer is rewritten at step s + 2 only after this
    // CTA's full barrier for h_{s+1} completed, which needs every peer's h_{s+1}, which each peer computed after receiving
    // all of this CTA's step-s copy: the bulk copies that read it are done.
    // One buffer, write after read on a peer's block: a peer sends h_s into this CTA's tile only after its empty barrier of
    // step s has completed, which needs this CTA's arrive, which follows the __syncthreads that ends this CTA's step-s
    // multiply.  On the own block: this CTA rewrites it with h_s only after its own empty barrier of step s has completed.
    // Each peer arrived there after its step-s multiply, which followed its full barrier of step s - 1, which completed when
    // this CTA's copy of h_{s-1} out of the own block had landed.
    // The Y planes read the own block before the __syncthreads that ends the next multiply.  Arrives release and waits
    // acquire at cluster scope; the copies' complete_tx does the same.
    const int DH = D * H;
    for (int s = 0; s < T; ++s) {
        const int t = d == 0 ? s : T - 1 - s;
        const int buf = NBUF == 2 ? s & 1 : 0, nbuf = NBUF == 2 ? buf ^ 1 : 0;
        // the peers' blocks of h_{s-1} have landed; and the barrier of the buffer this step fills expects theirs of h_s
        if (s > 0) mbar_wait<true>(full + buf, (NBUF == 2 ? (s - 1) >> 1 : s - 1) & 1);
        if (tid == 0 && s + 1 < T) mbar_arrive_expect_tx(full + nbuf, (CS - 1) * NH * nb * U * 2);
        float giv[3][JMAX][4];
#pragma unroll
        for (int j = 0; j < JMAX; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int64_t row = (int64_t)(bt0 + bcol[j][e & 1]) * T + t;
                const float* gr = gi + ((int64_t)d * B * T + row) * 3 * H + c * U + unit[e >> 1];
#pragma unroll
                for (int gte = 0; gte < 3; ++gte) giv[gte][j][e] = gr[gte * H];
            }
        float acc[3][JMAX][4];
#pragma unroll
        for (int gte = 0; gte < 3; ++gte)
#pragma unroll
            for (int j = 0; j < JMAX; ++j)
#pragma unroll
                for (int e = 0; e < 4; ++e) acc[gte][j][e] = 0.f;
        const uint32_t hbase = smem_u32(Hsm + buf * NH * HBYTES);
        const uint32_t wbase = smem_u32(Wsm);
#pragma unroll 4
        for (int ks = 0; ks < H / 16; ++ks) {
            uint32_t bh[JMAX][NH][2];
            const int bk = ks * 16 + ((lane >> 3) & 1) * 8;
#pragma unroll
            for (int j = 0; j < JMAX; ++j)
#pragma unroll
                for (int h = 0; h < NH; ++h)
                    ldsm_x2(hbase + h * HBYTES + hsw<NBMAX>((nt * jn + j) * 8 + (lane & 7), bk), bh[j][h]);
#pragma unroll
            for (int gte = 0; gte < 3; ++gte) {
                const int arow = gte * U + ug * 16 + (lane & 15), ak = ks * 16 + (lane >> 4) * 8;
                uint32_t a[NH][4];
#pragma unroll
                for (int h = 0; h < NH; ++h) ldsm_x4(wbase + h * S::WBYTES + swz<S::WP>(arow, ak), a[h]);
#pragma unroll
                for (int j = 0; j < JMAX; ++j) {
                    if (NS != 1) {
                        mma_bf16(acc[gte][j], a[0], bh[j][NH - 1][0], bh[j][NH - 1][1]);
                        mma_bf16(acc[gte][j], a[NH - 1], bh[j][0][0], bh[j][0][1]);
                    }
                    mma_bf16(acc[gte][j], a[0], bh[j][0][0], bh[j][0][1]);
                }
            }
        }
        if (NBUF == 1) {
            // this CTA's reads of the tile are done: tell every peer (threads 0 .. CS - 2, one peer each)
            __syncthreads();
            if (tid < CS - 1) mbar_arrive_peer(empty, (c + 1 + tid) % CS);
        }
        float hv[JMAX][4];
#pragma unroll
        for (int j = 0; j < JMAX; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int b = bt0 + bcol[j][e & 1], ul = unit[e >> 1], k = c * U + ul;
                const float r = sigmoid_f(giv[0][j][e] + acc[0][j][e] + bias[0][e >> 1]);
                const float z = sigmoid_f(giv[1][j][e] + acc[1][j][e] + bias[1][e >> 1]);
                const float hnv = acc[2][j][e] + bias[2][e >> 1];
                const float n = tanhf(giv[2][j][e] + r * hnv);
                const bool pad = LEN && t >= len[j][e & 1];
                float h;
                if constexpr (RD) h = pad ? hp[j][e] : (1.f - z) * n + z * (mk[j][e] * hp[j][e]);
                else h = pad ? hp[j][e] : (1.f - z) * n + z * hp[j][e];
                hp[j][e] = h;
                if constexpr (RD) hv[j][e] = mk[j][e] * h;
                else hv[j][e] = h;
                const int64_t row = (int64_t)b * T + t;
                if (OUT & SCAN_Y) Y[row * DH + d * H + k] = pad ? 0.f : h;
                if ((OUT & SCAN_G) && !pad) {
                    float* gs = G + ((int64_t)d * B * T + row) * 4 * H + k;
                    gs[0] = r; gs[H] = z; gs[2 * H] = n; gs[3 * H] = hnv;
                }
                if (hn_out && s == T - 1) hn_out[((int64_t)d * B + b) * H + k] = h;
            }
        // every peer has multiplied with h_{s-1}, so this CTA's copies of it out of the own block are done
        if (NBUF == 1) mbar_wait<true>(empty, s & 1);
#pragma unroll
        for (int j = 0; j < JMAX; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                bf16_t hi, lo;
                split_bf16(hv[j][e], hi, lo);
                uint8_t* la = Hsm + nbuf * NH * HBYTES + hsw<NBMAX>(bcol[j][e & 1], c * U + unit[e >> 1]);
                *reinterpret_cast<bf16_t*>(la) = hi;
                if (NH == 2) *reinterpret_cast<bf16_t*>(la + HBYTES) = lo;
            }
        // the own block of h_s is complete; make it visible to the bulk copies (async proxy), then send it to every peer
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncthreads();
        const uint32_t own = smem_u32(Hsm + nbuf * NH * HBYTES + c * SLICE);
        if (tid == 0 && s + 1 < T) {
#pragma unroll
            for (int p = 1; p < CS; ++p) {
                const uint32_t dst = (c + p) % CS;
#pragma unroll
                for (int h = 0; h < NH; ++h) bulk_copy_to_peer(own + h * HBYTES, nb * U * 2, full + nbuf, dst);
            }
        }
        // the Y planes of this CTA's units from its own block, 16-byte stores, while the copies are in flight.  A padded
        // row's tile holds the carried state: its plane rows are zeros.
        if (OUT & SCAN_PLANES) {
            for (int i = tid; i < NH * nb * (U / 8); i += SCAN_THREADS) {
                const int h = i / (nb * U / 8), r = (i / (U / 8)) % nb, kl = (i % (U / 8)) * 8;
                uint4 v = *reinterpret_cast<const uint4*>(Hsm + (nbuf * NH + h) * HBYTES + c * SLICE + swz<U * 2>(r, kl));
                if (LEN && t >= rlen) v = make_uint4(0u, 0u, 0u, 0u);
                *reinterpret_cast<uint4*>((h ? yl : yh) + ((int64_t)(bt0 + r) * T + t) * DH + d * H + c * U + kl) = v;
            }
        }
    }
    // no CTA leaves while a bulk copy or an arrive into or out of its shared memory may be in flight
    cluster_arrive();
    cluster_wait();
}

// RD: recurrent dropout, in the training forward only (SCAN_TRAIN outputs): yh, yl receive the masked state, not Y.  mask is
// null without RD
template <int H, int NS, int OUT, bool LEN, bool RD>
__global__ void __launch_bounds__(SCAN_THREADS, 1)
gru_scan_fwd_kernel(const float* __restrict__ gi, const float* __restrict__ Whh, const float* __restrict__ bhh, int64_t zW,
                    const float* __restrict__ h0, float* __restrict__ Y, float* __restrict__ G, float* __restrict__ hn_out,
                    bf16_t* __restrict__ yh, bf16_t* __restrict__ yl, int B, int T, int D, int m2, const int* __restrict__ lens,
                    const float* __restrict__ mask) {
    static_assert(!RD || OUT == SCAN_TRAIN, "recurrent dropout runs in the training forward only");
    int d, bt0, nb;
    scan_tile(blockIdx.y, m2, B / SCAN_NB, D, d, bt0, nb);
    if constexpr (FwdSmem<H, NS>::NBMAX == 2 * SCAN_NB) {
        if (nb == 2 * SCAN_NB) {
            gru_scan_fwd_tile<H, NS, OUT, LEN, 2, RD>(gi, Whh, bhh, zW, h0, Y, G, hn_out, yh, yl, B, T, D, lens, d, bt0, mask);
            return;
        }
    }
    gru_scan_fwd_tile<H, NS, OUT, LEN, 1, RD>(gi, Whh, bhh, zW, h0, Y, G, hn_out, yh, yl, B, T, D, lens, d, bt0, mask);
}

// ------------------------------------------------------------------------------------------------------
// Backward recurrence of one layer, both directions.  Layouts are those of gru_gates_bwd_kernel: G, Y, h0 as in the
// forward; dY [B][T][D*H]; dhc [D][B][H] carries dh into the layer's last step (head / zero) and returns dh_{-1};
// dgi, dgh [D][B*T][3H], and their bf16 planes gih/gil, ghh/ghl in the same layout for the GEMMs.  The dgh planes hold
// zeros at each sequence's first step (t = 0 for d = 0, t = T-1 for d = 1): that row pairs with h0 (covered from fp32 dgh),
// so dW_hh = dgh^T H_prev needs no row mask.  Shared memory: W^T rows (H) x own gate rows (192) | region X | receive slots of
// the peers' partial sums [CS-1][64][16] fp32 (k-major, xslot) | (BULK) full and empty mbarriers.  X holds the dgh tile
// [NH][16][192] bf16 from the gate math to the multiply, then the step's partial sums.
// BULK (H <= 256): X holds this CTA's partial for every owner CTA, block X[dst] = [U][NB] fp32 in xslot order (the own one
// at X[c]), written with local stores; one thread sends block X[dst] to dst's receive slot of source c with one bulk copy
// per peer, completing on dst's "full" mbarrier, and a CTA waits on its own full before it reads its slots.  After reading
// them, threads 0 .. CS - 2 each arrive on one peer's "empty" mbarrier; a CTA waits on its own empty (phase s - 1 at step
// s) after the gate math, before it writes the dgh tile into X.  There is no cluster barrier per step.
//   * No peer copies into a receive slot that is still being read: a peer's step-s copy into this CTA follows the peer's
//     empty wait of phase s - 1, which needs this CTA's arrive, which follows the __syncthreads after which every thread of
//     this CTA has read its step-(s - 1) slots.
//   * No complete_tx lands in the wrong phase of full: this CTA waits on phase s - 1 and then (thread 0) arms phase s
//     with its (CS - 1) * SLOT bytes before that __syncthreads and arrive, so every step-s copy into this CTA is issued
//     after phase s - 1 completed and phase s expects it.  Phase 0 is armed before the starting cluster barrier.
//   * X is rewritten only after the copies out of it are done: those copies are tracked by the peers' full barriers alone
//     (no bulk group), so the empty wait before the dgh tile write is what shows it: every peer arrived after its full
//     wait of phase s - 1, which completed when this CTA's step-(s - 1) copy into it had landed.  The own block X[c] is read
//     before the __syncthreads that precedes that write.
//   Arrives release and waits acquire at cluster scope; the copies' complete_tx does the same.
// At H = 512 the 28 KB of receive slots and 32 KB of outgoing blocks next to the 192 KB of W^T exceed the 227 KB a block may
// use, so there the partials go out as remote stores and two cluster barrier phases per step keep order: (1) partials of
// the step have landed; (2) every CTA has read its receive slots, so the next step's partials may be written.  The own
// partial then sits at the start of X.
// LEN: at a padded (row, t >= lens[b]) dgi and dgh are 0 (fp32 and planes) and dh passes through unchanged: its dgh row
// adds exact zeros to the partial sums.  The barriers and the exchange are those of every step.
// ------------------------------------------------------------------------------------------------------
template <int H, int NS>
struct BwdSmem {
    static constexpr int NH = NS == 1 ? 1 : 2;
    static constexpr int CS = H / SCAN_U;
    static constexpr int Q = 3 * SCAN_U;                   // own gate rows
    static constexpr int WP = Q * 2;                        // W^T row pitch (bytes)
    static constexpr int WBYTES = H * WP;
    static constexpr int DBYTES = SCAN_NB * Q * 2;
    static constexpr int SLOT = SCAN_NB * SCAN_U * 4;
    static constexpr bool BULK = H <= 256;                  // outgoing blocks in X fit next to W^T (see above)
    static constexpr int XBYTES = BULK && CS * SLOT > NH * DBYTES ? CS * SLOT : NH * DBYTES;
    static constexpr int TOTAL = NH * WBYTES + XBYTES + (CS - 1) * SLOT + (BULK ? 2 * 8 : 0);
    static_assert(NH * DBYTES >= SLOT, "own partial sums alias the dgh tile");
    static_assert(TOTAL <= 232448, "an H100 block's shared memory");
};

// float index of the partial sum for (unit kl, batch column b) in a receive slot: k-major [U][NB], so a thread's two
// accumulators of adjacent columns (b even, b + 1) are one 8-byte store.  The column pair is XORed with a function of kl
// that keeps each half-warp's 8-byte stores conflict-free and leaves the owner's reads (32 consecutive units, one column)
// at two lanes per bank.
__device__ __forceinline__ int xslot(int kl, int b) {
    static_assert(SCAN_NB == 16, "eight column pairs per unit");
    const int g = ((kl >> 1) & 1) * 4 + ((kl >> 2) & 3);
    return kl * SCAN_NB + (((b >> 1) ^ g) << 1) + (b & 1);
}

// the scan of one cluster whose tile has NR (16 or 8) rows from bt0, direction d; the shared-memory layout is that of 16.
// RD: recurrent dropout with the forward's masks `mask` [D][B][H] (DESIGN.md §4.8): the gate math reads m * h_{t-1}, and the
// gradient leaving a valid step is dh_{t-1} = m * (dh z + sum of the partials); a padded step passes it unmasked
template <int H, int NS, bool LEN, int NR, bool RD = false>
__device__ __forceinline__ void gru_scan_bwd_tile(const float* __restrict__ G, const float* __restrict__ Y,
                                                  const float* __restrict__ h0, const float* __restrict__ dY,
                                                  float* __restrict__ dhc, float* __restrict__ dgi, float* __restrict__ dgh,
                                                  const float* __restrict__ Whh, int64_t zW, bf16_t* __restrict__ gih,
                                                  bf16_t* __restrict__ gil, bf16_t* __restrict__ ghh, bf16_t* __restrict__ ghl,
                                                  int B, int T, int D, const int* __restrict__ lens, int d, int bt0,
                                                  const float* __restrict__ mask = nullptr) {
    using S = BwdSmem<H, NS>;
    constexpr int U = SCAN_U, CS = H / U, NH = S::NH, Q = S::Q, NB = SCAN_NB;
    constexpr int MT = H / 16 / 8;                           // m-tiles (16 rows of W^T) per warp
    constexpr int PAIRS = NR * U / SCAN_THREADS;             // (unit, column) pairs per thread in the gate math
    constexpr int NBLK = NR / 8;                             // n8 blocks of the tile
    extern __shared__ __align__(128) uint8_t smem[];
    uint8_t* Wsm = smem;                                     // [NH][H rows][Q]
    uint8_t* Dsm = smem + NH * S::WBYTES;                    // X: [NH][NB rows][Q] dgh tile; then partials [CS or 1][U][NB] fp32
    float* recv = reinterpret_cast<float*>(Dsm + S::XBYTES);   // [CS-1][U][NB] (xslot)
    uint64_t* full = reinterpret_cast<uint64_t*>(recv + (CS - 1) * NB * U);   // BULK
    uint64_t* empty = full + 1;
    const int c = (int)cluster_rank();
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const float* W = Whh + d * zW;
    float* own = reinterpret_cast<float*>(Dsm + (S::BULK ? c * S::SLOT : 0));
    auto slot = [&](int src) -> float* { return src == c ? own : recv + (src < c ? src : src - 1) * NB * U; };

    for (int i = tid; i < Q * H; i += SCAN_THREADS) {
        const int q = i / H, k = i % H, gte = q / U, u = q % U;
        const float v = W[(int64_t)(gte * H + c * U + u) * H + k];
        bf16_t hi, lo;
        split_bf16(v, hi, lo);
        *reinterpret_cast<bf16_t*>(Wsm + swz<S::WP>(k, q)) = hi;
        if (NH == 2) *reinterpret_cast<bf16_t*>(Wsm + S::WBYTES + swz<S::WP>(k, q)) = lo;
    }
    float dhr[PAIRS], dhz[PAIRS], mk[RD ? PAIRS : 1];
    int plen[PAIRS];
#pragma unroll
    for (int i = 0; i < PAIRS; ++i) {
        const int p = tid + i * SCAN_THREADS, u = p % U, b = p / U;
        dhr[i] = dhc[((int64_t)d * B + bt0 + b) * H + c * U + u];
        dhz[i] = 0.f;
        plen[i] = LEN ? lens[bt0 + b] : T;
        if constexpr (RD) mk[i] = mask[((int64_t)d * B + bt0 + b) * H + c * U + u];
    }
    if (S::BULK && tid == 0) {
        mbar_init(full, 1);
        mbar_init(empty, CS - 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        mbar_arrive_expect_tx(full, (CS - 1) * S::SLOT);     // phase 0: step 0's partials
    }
    // every CTA of the cluster has started and initialised its barriers before any remote store, bulk copy or arrive
    cluster_arrive();
    cluster_wait();

    const int DH = D * H;
    // the step's operands from global memory: G (r, z, n, W_hn h + b_hn), h_{t-1} (Y, or h0 at the first step) and dY.
    // Step s + 1's are loaded during step s, so their latency hides behind the rest of the step and the dgh tile waits only
    // for the incoming dh.  They are issued right after the gate math at both precisions: at configs[1] on an H100 that
    // ran the backward scan 0.03 ms faster at bf16x3 than issuing them after the multiply, and 0.2 ms faster at bf16.
    float gr[PAIRS], gz[PAIRS], gn[PAIRS], ghn[PAIRS], hprev[PAIRS], dyv[PAIRS];
    auto load_step = [&](int s) {
        const int t = d == 0 ? T - 1 - s : s;
        const bool first = d == 0 ? t == 0 : t == T - 1;
#pragma unroll
        for (int i = 0; i < PAIRS; ++i) {
            const int p = tid + i * SCAN_THREADS, u = p % U, b = bt0 + p / U, j = c * U + u;
            const int64_t row = (int64_t)b * T + t;
            const float* gs = G + ((int64_t)d * B * T + row) * 4 * H + j;
            gr[i] = gs[0]; gz[i] = gs[H]; gn[i] = gs[2 * H]; ghn[i] = gs[3 * H];
            if (first) hprev[i] = h0 ? h0[((int64_t)d * B + b) * H + j] : 0.f;
            else hprev[i] = Y[((int64_t)b * T + (d == 0 ? t - 1 : t + 1)) * DH + d * H + j];
            dyv[i] = dY[row * DH + d * H + j];
            if constexpr (RD) hprev[i] *= mk[i];
        }
    };
    load_step(0);
    for (int s = 0; s < T; ++s) {
        const int t = d == 0 ? T - 1 - s : s;
        const bool first = d == 0 ? t == 0 : t == T - 1;
        if (s > 0) {
            if constexpr (S::BULK) {
                mbar_wait<true>(full, (s - 1) & 1);          // the peers' partials of step s - 1 have landed
                if (tid == 0) mbar_arrive_expect_tx(full, (CS - 1) * S::SLOT);   // phase s: this step's
            }
#pragma unroll
            for (int i = 0; i < PAIRS; ++i) {
                const int p = tid + i * SCAN_THREADS, x = xslot(p % U, p / U);
                float v = dhz[i];
#pragma unroll
                for (int src = 0; src < CS; ++src) v += slot(src)[x];
                // the previous step (t + 1 forward, t - 1 reverse) applied a cell to the masked state unless it was padded
                if constexpr (RD) v = LEN && (d == 0 ? t + 1 : t - 1) >= plen[i] ? v : mk[i] * v;
                dhr[i] = v;
            }
        }
        if constexpr (!S::BULK) cluster_arrive();            // phase (2): this CTA's receive slots are read
        __syncthreads();                                     // own partial read before the dgh tile is rewritten
        // this CTA's receive slots are read: tell every peer (threads 0 .. CS - 2, one peer each)
        if (S::BULK && s > 0 && tid < CS - 1) mbar_arrive_peer(empty, (c + 1 + tid) % CS);
        float gv[PAIRS][3];
#pragma unroll
        for (int i = 0; i < PAIRS; ++i) {
            const int p = tid + i * SCAN_THREADS, u = p % U, bl = p / U, b = bt0 + bl, j = c * U + u;
            const int64_t row = (int64_t)b * T + t;
            const float r = gr[i], z = gz[i], n = gn[i], hnv = ghn[i], hpv = hprev[i];
            const float dh = dhr[i] + dyv[i];
            float dan = dh * (1.f - z) * (1.f - n * n);
            float dar = dan * hnv * r * (1.f - r);
            float daz = dh * (hpv - n) * z * (1.f - z);
            float dgn = dan * r;
            const bool pad = LEN && t >= plen[i];
            if (pad) dan = dar = daz = dgn = 0.f;
            float* a = dgi + ((int64_t)d * B * T + row) * 3 * H + j;
            float* cg = dgh + ((int64_t)d * B * T + row) * 3 * H + j;
            a[0] = dar; a[H] = daz; a[2 * H] = dan;
            cg[0] = dar; cg[H] = daz; cg[2 * H] = dgn;
            dhz[i] = pad ? dhr[i] : dh * z;
            gv[i][0] = dar; gv[i][1] = daz; gv[i][2] = dgn;
            // dgi's n gate is dan (dgh's is dgn = dan * r); its r and z gates equal dgh's and leave from the dgh tile below
            bf16_t hi, lo;
            split_bf16(dan, hi, lo);
            const int64_t po = ((int64_t)d * B * T + row) * 3 * H + 2 * H + j;
            gih[po] = hi;
            if (NH == 2) gil[po] = lo;
        }
        // every peer has read its slots of step s - 1, so this CTA's copies of that step out of X are done, and the
        // peers' slots are free for this step's
        if (S::BULK && s > 0) mbar_wait<true>(empty, (s - 1) & 1);
#pragma unroll
        for (int i = 0; i < PAIRS; ++i) {
            const int p = tid + i * SCAN_THREADS, u = p % U, bl = p / U;
#pragma unroll
            for (int gte = 0; gte < 3; ++gte) {
                bf16_t hi, lo;
                split_bf16(gv[i][gte], hi, lo);
                *reinterpret_cast<bf16_t*>(Dsm + swz<S::WP>(bl, gte * U + u)) = hi;
                if (NH == 2) *reinterpret_cast<bf16_t*>(Dsm + S::DBYTES + swz<S::WP>(bl, gte * U + u)) = lo;
            }
        }
        if (s + 1 < T) load_step(s + 1);
        __syncthreads();
        // planes of this step's rows from the dgh tile, 16-byte stores: dgh (zeros at a sequence's first step) and dgi's r, z
        for (int i = tid; i < NH * NR * (Q / 8); i += SCAN_THREADS) {
            const int h = i / (NR * Q / 8), r = (i / (Q / 8)) % NR, q = (i % (Q / 8)) * 8, gte = q / U;
            uint4 v = *reinterpret_cast<const uint4*>(Dsm + h * S::DBYTES + swz<S::WP>(r, q));
            const int64_t o = ((int64_t)d * B * T + (int64_t)(bt0 + r) * T + t) * 3 * H + gte * H + c * U + q % U;
            if (gte < 2) *reinterpret_cast<uint4*>((h ? gil : gih) + o) = v;
            if (first) v = make_uint4(0u, 0u, 0u, 0u);
            *reinterpret_cast<uint4*>((h ? ghl : ghh) + o) = v;
        }
        // partial dh_{t-1}[k, b] = sum over this CTA's gate rows q of W[q, k] dgh[b, q], for all H units k
        float acc[MT][2][4];
#pragma unroll
        for (int m = 0; m < MT; ++m)
#pragma unroll
            for (int n = 0; n < NBLK; ++n)
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
                for (int n = 0; n < NBLK; ++n) {
                    if (NS != 1) {
                        mma_bf16(acc[m][n], a[0], bv[NH - 1][2 * n], bv[NH - 1][2 * n + 1]);
                        mma_bf16(acc[m][n], a[NH - 1], bv[0][2 * n], bv[0][2 * n + 1]);
                    }
                    mma_bf16(acc[m][n], a[0], bv[0][2 * n], bv[0][2 * n + 1]);
                }
            }
        }
        __syncthreads();                                     // dgh tile consumed: its space takes the partials
        if constexpr (!S::BULK) cluster_wait();              // phase (2) complete: peers' receive slots are free
        // accumulators e = 0, 1 (and 2, 3) are adjacent batch columns of one unit: one 8-byte store each
#pragma unroll
        for (int m = 0; m < MT; ++m)
#pragma unroll
            for (int n = 0; n < NBLK; ++n)
#pragma unroll
                for (int e = 0; e < 4; e += 2) {
                    const int k = (warp + 8 * m) * 16 + (lane >> 2) + (e >= 2 ? 8 : 0);
                    const int bl = n * 8 + 2 * (lane & 3);
                    const int dst = k / U, x = xslot(k % U, bl);
                    const float2 v = make_float2(acc[m][n][e], acc[m][n][e + 1]);
                    if (S::BULK) {
                        *reinterpret_cast<float2*>(Dsm + dst * S::SLOT + x * 4) = v;
                    } else if (dst == c) {
                        *reinterpret_cast<float2*>(own + x) = v;
                    } else {
                        // at CTA dst, the slot of source c is (c < dst ? c : c - 1)
                        const float* rs = recv + (c < dst ? c : c - 1) * NB * U + x;
                        st_cluster_v2_f32(mapa(smem_u32(rs), dst), v);
                    }
                }
        if constexpr (S::BULK) {
            // the blocks of X are complete; make them visible to the bulk copies (async proxy), then send one to each peer:
            // all of its slot, also from an 8-row tile (xslot spreads its columns over all 16).  The last step's go to the
            // final dh_{-1} sum below
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncthreads();
            if (tid == 0) {
#pragma unroll
                for (int p = 1; p < CS; ++p) {
                    const int dst = (c + p) % CS;
                    bulk_copy_to_peer_at(smem_u32(recv + (c < dst ? c : c - 1) * NB * U), smem_u32(Dsm + dst * S::SLOT),
                                         S::SLOT, full, dst);
                }
            }
        } else {
            cluster_arrive();                                // phase (1): this step's partial sums are delivered
            cluster_wait();
        }
    }
    if constexpr (S::BULK) mbar_wait<true>(full, (T - 1) & 1);   // the peers' partials of the last step have landed
#pragma unroll
    for (int i = 0; i < PAIRS; ++i) {
        const int p = tid + i * SCAN_THREADS, u = p % U, b = p / U, x = xslot(u, b);
        float v = dhz[i];
#pragma unroll
        for (int src = 0; src < CS; ++src) v += slot(src)[x];
        if constexpr (RD) v = LEN && (d == 0 ? 0 : T - 1) >= plen[i] ? v : mk[i] * v;
        dhc[((int64_t)d * B + bt0 + b) * H + c * U + u] = v;
    }
    if constexpr (S::BULK) {
        // no CTA leaves while a bulk copy out of its shared memory may be in flight
        cluster_arrive();
        cluster_wait();
    }
}

// Grid (CS, clusters, 1), cluster (CS, 1, 1).  The first D * B / 16 - L8 clusters take one 16-row tile each, in (direction,
// tile) order; the last L8 tiles are split into two 8-row clusters each (scan_bwd_geometry), so a short last round of
// clusters takes less time.  An 8-row cluster multiplies one n8 block with the same MMA sequence per element: a row's bits
// do not depend on its tile.
// RD: the backward of the recurrent-dropout forward: Y is the unmasked output; the dgh planes pair with the masked-state
// planes.  mask is null without RD
template <int H, int NS, bool LEN, bool RD>
__global__ void __launch_bounds__(SCAN_THREADS, 1)
gru_scan_bwd_kernel(const float* __restrict__ G, const float* __restrict__ Y, const float* __restrict__ h0,
                    const float* __restrict__ dY, float* __restrict__ dhc, float* __restrict__ dgi, float* __restrict__ dgh,
                    const float* __restrict__ Whh, int64_t zW, bf16_t* __restrict__ gih, bf16_t* __restrict__ gil,
                    bf16_t* __restrict__ ghh, bf16_t* __restrict__ ghl, int B, int T, int D, int L8, const int* __restrict__ lens,
                    const float* __restrict__ mask) {
    const int ntd = B / SCAN_NB, n16 = D * ntd - L8, q = blockIdx.y;
    if (q < n16) {
        gru_scan_bwd_tile<H, NS, LEN, SCAN_NB, RD>(G, Y, h0, dY, dhc, dgi, dgh, Whh, zW, gih, gil, ghh, ghl, B, T, D, lens,
                                                    q / ntd, (q % ntd) * SCAN_NB, mask);
    } else {
        const int f = n16 + (q - n16) / 2;
        gru_scan_bwd_tile<H, NS, LEN, SCAN_NB / 2, RD>(G, Y, h0, dY, dhc, dgi, dgh, Whh, zW, gih, gil, ghh, ghl, B, T, D, lens,
                                                        f / ntd, (f % ntd) * SCAN_NB + ((q - n16) & 1) * (SCAN_NB / 2), mask);
    }
}

}  // namespace htc

// ---- host launchers ----------------------------------------------------------------------------------------
static inline int64_t rup(int64_t v, int64_t m) { return (v + m - 1) / m * m; }
// bf16 elements of a zero-padded K-major image [batch][rup(R, 128)][rup(K, 64)] written by tc_pack_kernel (hi and lo planes)
static inline int64_t tc_pack_elems(int64_t R, int64_t K, int64_t batch, int prec) {
    return (prec == BIGRU_PREC_BF16X3 ? 2 : 1) * batch * rup(R, htc::WG_BM) * rup(K, htc::WG_BK);
}
// bf16 elements of both packed operands of tc_gemm_launch
static inline int64_t tc_gemm_ws_elems(int64_t M, int64_t N, int64_t K, int64_t batch, int prec) {
    return tc_pack_elems(M, K, batch, prec) + tc_pack_elems(N, K, batch, prec);
}
// Split-K count of a weight-gradient GEMM (K = B*T).  Four units per SM of a 132-SM H100 keep the spread of unit times
// (the last split is shorter, the tile count rarely divides 132) small next to the work per SM: dW_ih of layer 1 at
// configs[1] has 48 tiles -> 11 splits = 528 units; dW_hh 24 tiles -> 22 splits.  At least 8 k-blocks per split keep the
// pipeline fill small.  The count is fixed (not taken from the device) so that the summation order, and with it every
// bit of the result, depends on the shape only.
static inline int wg_splits(int64_t tiles, int64_t kblocks) {
    const int64_t s = std::min(cdiv64(4 * 132, tiles), kblocks / 8);
    if (s <= 1) return 1;
    const int64_t per = cdiv64(kblocks, s);
    return (int)cdiv64(kblocks, per);                 // no empty split
}

// bf16 planes [depth][rows][pitch] (cols <= pitch used; pitch % 8 == 0); lo is null at bf16
struct Planes {
    const htc::bf16_t* hi; const htc::bf16_t* lo;
    int64_t cols, rows, depth, pitch;
};

typedef CUresult (*PFN_encodeTiled_t)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                      const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                      CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
// 3-D tensor map [depth][rows][cols] with 128-byte swizzle; out-of-bounds elements read as zero and are not written
static int encode_map(CUtensorMap* m, CUtensorMapDataType type, int esize, const void* base, int64_t cols, int64_t rows,
                      int64_t depth, int64_t pitch, int64_t zstride, uint32_t box0, uint32_t box1) {
    static PFN_encodeTiled_t enc = nullptr;
    if (!enc) {
        void* f = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) {
            bigru_set_error("tc_gemm: cuTensorMapEncodeTiled is unavailable");
            return BIGRU_ERR_CUDA;
        }
        enc = (PFN_encodeTiled_t)f;
    }
    const cuuint64_t dims[3] = {(cuuint64_t)cols, (cuuint64_t)rows, (cuuint64_t)depth};
    const cuuint64_t strides[2] = {(cuuint64_t)(pitch * esize), (cuuint64_t)(zstride * esize)};
    const cuuint32_t box[3] = {box0, box1, 1u}, es[3] = {1u, 1u, 1u};
    CUresult r = enc(m, type, 3, const_cast<void*>(base), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { bigru_set_error("tc_gemm: cuTensorMapEncodeTiled failed (%d)", (int)r); return BIGRU_ERR_CUDA; }
    return BIGRU_OK;
}

// one plane: boxes of 64 (K) x 128 rows for a K-major operand, 64 (MN) x 64 (K) rows for an MN-major one
static int make_plane_map(CUtensorMap* m, const htc::bf16_t* base, const Planes& p, bool mn) {
    return encode_map(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, base, p.cols, p.rows, p.depth, p.pitch, p.pitch * p.rows, 64u,
                      mn ? 64u : 128u);
}

template <int NS, int AMN, int BMN>
static int wg_launch(const CUtensorMap (&tm)[5], const htc::WgJob& j, int grid, cudaStream_t st) {
    constexpr int STAGES = NS == 1 ? 4 : 3;
    constexpr int smem = htc::wg_smem_bytes(NS, STAGES);
    static_assert(smem <= 232448, "wg_gemm_kernel: more shared memory than an sm_90 block may have");
    auto k = htc::wg_gemm_kernel<NS, STAGES, AMN, BMN>;
    CUDA_TRY(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    k<<<grid, 384, smem, st>>>(tm[0], tm[1], tm[2], tm[3], tm[4], j);
    LAUNCH_CHECK();
    return BIGRU_OK;
}

// what wg_gemm refuses before it touches the device.  A bias with split-K: neither epilogue adds it to the partials and
// splitk_reduce_kernel has no bias, so the result would silently lack it (no plan asks for the combination)
static int wg_job_check(const htc::WgJob& j) {
    if (j.bias && j.splits > 1) {
        bigru_set_error("tc_gemm: a bias together with split-K (%d splits) is not supported", j.splits);
        return BIGRU_ERR_ARG;
    }
    return BIGRU_OK;
}

// runs j (M, N, batch, kblocks, kbd, kcat, C, bias, beta, ldc, zC, zBias, a/b coordinates set; tm, tn, part filled here)
// over planes A and B; split-K partials (j.splits > 1) go to j.part and are reduced into C in split order.  staged (nullable)
// receives j.cmap, the epilogue the kernel runs
static int wg_gemm(htc::WgJob j, const Planes& A, bool amn, const Planes& B, bool bmn, int prec, cudaStream_t st,
                   int* staged = nullptr) {
    TRY(wg_job_check(j));
    if (j.M <= 0 || j.N <= 0) return BIGRU_OK;
    const bool x3 = prec == BIGRU_PREC_BF16X3;
    if (x3 != (A.lo != nullptr) || x3 != (B.lo != nullptr) || amn != bmn) {
        bigru_set_error("tc_gemm: operand planes do not match the precision / majors");
        return BIGRU_ERR_ARG;
    }
    j.tm = (int)cdiv64(j.M, htc::WG_BM);
    j.tn = (int)cdiv64(j.N, htc::WG_BN);
    CUtensorMap tm[5];
    TRY(make_plane_map(&tm[0], A.hi, A, amn));
    TRY(make_plane_map(&tm[2], B.hi, B, bmn));
    if (x3) {
        TRY(make_plane_map(&tm[1], A.lo, A, amn));
        TRY(make_plane_map(&tm[3], B.lo, B, bmn));
    } else {
        tm[1] = tm[0]; tm[3] = tm[2];
    }
    // the kernel's output: part [splits * batch][M][N] for split jobs, else C [batch][M][ldc] with batch stride zC.  It goes
    // through a tensor map when the job overwrites it, its base and strides are 16-byte aligned (a map's requirement) and
    // its rows are whole 16-byte chunks: the bulk tensor store clips a box at the map's column extent only to 16 bytes, so
    // N = 13 at ldc = 16 would overwrite columns 13..15 of every row (seen on the H100; tests/test_gpu_tc_gemm.py)
    const bool split = j.splits > 1;
    float* const cbase = split ? j.part : j.C;
    const int64_t depth = split ? (int64_t)j.splits * j.batch : j.batch, ldc = split ? j.N : j.ldc;
    const int64_t zc = depth == 1 ? j.M * ldc : split ? (int64_t)j.M * j.N : j.zC;
    j.cmap = (split || !j.beta) && reinterpret_cast<uintptr_t>(cbase) % 16 == 0 && ldc % 4 == 0 && zc % 4 == 0 && j.N % 4 == 0;
    if (j.cmap) TRY(encode_map(&tm[4], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, cbase, j.N, j.M, depth, ldc, zc, 32u, 64u));
    else tm[4] = tm[0];
    if (staged) *staged = j.cmap;
    int dev = 0, nsm = 132;
    CUDA_TRY(cudaGetDevice(&dev));
    CUDA_TRY(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev));
    const int64_t units = (int64_t)j.tm * j.tn * j.batch * j.splits;
    const int grid = (int)std::min<int64_t>(units, nsm);
    const int rc = amn ? (x3 ? wg_launch<3, 1, 1>(tm, j, grid, st) : wg_launch<1, 1, 1>(tm, j, grid, st))
                       : (x3 ? wg_launch<3, 0, 0>(tm, j, grid, st) : wg_launch<1, 0, 0>(tm, j, grid, st));
    TRY(rc);
    if (j.splits > 1) {
        const int64_t n = (int64_t)j.batch * j.M * j.N;
        htc::splitk_reduce_kernel<<<(unsigned)std::min<int64_t>(cdiv64(n, 256), 132 * 8), 256, 0, st>>>(j.part, j.splits, j.batch, j.M,
                                                                                                        j.N, j.C, j.ldc, j.zC, j.beta);
        LAUNCH_CHECK();
    }
    return BIGRU_OK;
}

static htc::WgJob wg_job(float* C, int M, int N, int64_t ldc, int batch, int64_t kblocks) {
    htc::WgJob j{};
    j.C = C; j.M = M; j.N = N; j.ldc = ldc; j.batch = batch; j.kblocks = (int)kblocks; j.kbd = (int)kblocks; j.splits = 1;
    return j;
}

// packs batch x [R][K] fp32 (element (r, k) at src[z * zsrc + r * s_r + k * s_k]) into K-major planes at ws (timed as pack_bf16)
static int tc_pack(const float* src, int64_t s_r, int64_t s_k, int64_t zsrc, int R, int K, int batch, int prec, htc::bf16_t* ws,
                   Planes* out, cudaStream_t st) {
    const bool x3 = prec == BIGRU_PREC_BF16X3;
    const int Rp = (int)rup(R, htc::WG_BM), Kp = (int)rup(K, htc::WG_BK);
    const int64_t sz = (int64_t)batch * Rp * Kp;
    *out = Planes{ws, x3 ? ws + sz : nullptr, Kp, Rp, batch, Kp};
    KLAUNCH(KC_PACK, 0.0, (4.0 + (x3 ? 4.0 : 2.0)) * batch * (double)R * K, st,
            htc::tc_pack_kernel<<<dim3(Kp / 32, Rp / 32, batch), dim3(32, 8), 0, st>>>(src, s_r, s_k, zsrc, R, K, Rp, Kp, ws,
                                                                                     x3 ? ws + sz : nullptr));
    return BIGRU_OK;
}

// the strided fp32 GEMM contract of sgemm_kernel (GemmArgs; no split-K, no row mask) for the small head and h0 GEMMs:
// both operands packed, then wg_gemm.  ws: tc_gemm_ws_elems(...) bf16 elements
static int tc_gemm_launch(const GemmArgs& g, int prec, int cls, htc::bf16_t* ws, cudaStream_t st) {
    if (g.M <= 0 || g.N <= 0 || g.K <= 0) return BIGRU_OK;
    if (g.splitk != 1 || g.mask_period) {
        bigru_set_error("tc_gemm_launch: split-K and row masks are not supported");
        return BIGRU_ERR_ARG;
    }
    Planes A, B;
    TRY(tc_pack(g.A, g.sam, g.sak, g.zA, g.M, g.K, g.batch, prec, ws, &A, st));
    TRY(tc_pack(g.B, g.sbn, g.sbk, g.zB, g.N, g.K, g.batch, prec, ws + tc_pack_elems(g.M, g.K, g.batch, prec), &B, st));
    ProfScope ps(cls, 2.0 * g.M * g.N * (double)g.K * g.batch, 0.0, st);
    htc::WgJob j = wg_job(g.C, g.M, g.N, g.ldc, g.batch, cdiv64(g.K, htc::WG_BK));
    j.bias = g.bias; j.beta = g.beta; j.zC = g.zC; j.zBias = g.zBias;
    j.a.zsel = 1; j.b.zsel = 1;
    return wg_gemm(j, A, false, B, false, prec, st);
}

template <typename K>
static cudaLaunchConfig_t cluster_config(K kernel, int cs, int ny, int nz, int smem, cudaStream_t st, cudaLaunchAttribute* attr) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(cs, ny, nz);
    cfg.blockDim = dim3(htc::SCAN_THREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = cs; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    return cfg;
}

template <typename... KArgs, typename... Args>
static int launch_cluster(void (*kernel)(KArgs...), int cs, int ny, int nz, int smem, cudaStream_t st, Args... args) {
    CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    cudaLaunchAttribute attr[1];
    const cudaLaunchConfig_t cfg = cluster_config(kernel, cs, ny, nz, smem, st, attr);
    CUDA_TRY(cudaLaunchKernelEx(&cfg, kernel, args...));
    return BIGRU_OK;
}

// R: clusters of `kernel` (cs CTAs, smem bytes each) that the current device holds at once, queried once per kernel and device
template <typename... KArgs>
static int cluster_residency(void (*kernel)(KArgs...), int cs, int smem, int* R) {
    static std::mutex mu;
    static std::map<std::pair<const void*, int>, int> cache;
    int dev = 0;
    CUDA_TRY(cudaGetDevice(&dev));
    const std::pair<const void*, int> key((const void*)kernel, dev);
    {
        std::lock_guard<std::mutex> g(mu);
        const auto it = cache.find(key);
        if (it != cache.end()) { *R = it->second; return BIGRU_OK; }
    }
    CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    cudaLaunchAttribute attr[1];
    const cudaLaunchConfig_t cfg = cluster_config(kernel, cs, 1, 1, smem, 0, attr);
    int n = 0;
    CUDA_TRY(cudaOccupancyMaxActiveClusters(&n, (void*)kernel, &cfg));
    if (n <= 0) { bigru_set_error("scan: no %d-CTA cluster with %d bytes of shared memory fits on this device", cs, smem); return BIGRU_ERR_DEVICE; }
    {
        std::lock_guard<std::mutex> g(mu);
        cache[key] = n;
    }
    *R = n;
    return BIGRU_OK;
}

// Forward scan geometry.  n = D * B / 16 tiles; R clusters fit at once.  rounds = ceil(n / 2R) rounds of clusters; the
// n2 = n - rounds * R clusters beyond rounds * R one-tile clusters take two tiles (rounded up to a multiple of D: a
// cluster's tiles share a direction), so at most rounds * R clusters run.  R >= n / 2 gives one round of two-tile
// clusters; R >= n gives n one-tile clusters, and so does a kernel without 32-row tiles (two = false).  Results do not
// depend on the geometry.  Returns m2 = n2 / D, the two-tile clusters per direction, and the cluster count.
static void scan_geometry(int R, bool two, int B, int D, int* m2, int* clusters) {
    const int ntd = B / htc::SCAN_NB, n = D * ntd;
    int n2 = 0;
    if (two) {
        const int rounds = (n + 2 * R - 1) / (2 * R);
        n2 = std::max(0, n - rounds * R);
        n2 = std::min((n2 + D - 1) / D * D, D * (ntd / 2));
    }
    *m2 = n2 / D;
    *clusters = n - n2;
}

// Backward scan geometry.  n = D * B / 16 tiles; R clusters fit at once.  With rounds = ceil(n / R) > 1, the last round
// holds L = n - (rounds - 1) * R tiles; when 2L <= R they run as 2L clusters of 8 rows, which take less time than L of 16.
// Results do not depend on the geometry.  Returns L8 = the split tiles and the cluster count.
static void scan_bwd_geometry(int R, int B, int D, int* L8, int* clusters) {
    const int n = D * (B / htc::SCAN_NB), rounds = (n + R - 1) / R, L = n - (rounds - 1) * R;
    *L8 = rounds > 1 && 2 * L <= R ? L : 0;
    *clusters = n + *L8;
}

// the scan kernels of one (precision, H, forward outputs, lengths, recurrent dropout).  All instantiations of a direction
// share one signature: the mask operand is null without recurrent dropout
typedef decltype(&htc::gru_scan_fwd_kernel<128, 1, htc::SCAN_TRAIN, false, false>) ScanFwdFn;
typedef decltype(&htc::gru_scan_bwd_kernel<128, 1, false, false>) ScanBwdFn;
struct ScanKernels {
    ScanFwdFn fwd; int fwd_smem; bool two;   // two: the forward has 32-row tiles
    ScanBwdFn bwd; int bwd_smem;
};

template <int HH, int NS, bool LEN>
static ScanKernels scan_instance(int out, bool rd) {
    using namespace htc;
    const ScanFwdFn fwd = rd                        ? gru_scan_fwd_kernel<HH, NS, SCAN_TRAIN, LEN, true>
                          : out == SCAN_TRAIN       ? gru_scan_fwd_kernel<HH, NS, SCAN_TRAIN, LEN, false>
                          : out == SCAN_INFER_LOWER ? gru_scan_fwd_kernel<HH, NS, SCAN_INFER_LOWER, LEN, false>
                                                    : gru_scan_fwd_kernel<HH, NS, SCAN_INFER_TOP, LEN, false>;
    const ScanBwdFn bwd = rd ? gru_scan_bwd_kernel<HH, NS, LEN, true> : gru_scan_bwd_kernel<HH, NS, LEN, false>;
    return {fwd, FwdSmem<HH, NS>::TOTAL, FwdSmem<HH, NS>::NBMAX == 2 * SCAN_NB, bwd, BwdSmem<HH, NS>::TOTAL};
}

// the scan kernels of plan p whose forward writes the outputs `out` (the backward's are those of SCAN_TRAIN); shapes were
// validated by the plan (H in {128, 256, 512}, B % 16 == 0)
static int scan_kernels(const bigru_plan& p, int out, bool len, bool rd, ScanKernels* k) {
    using namespace htc;
    if (rd && out != SCAN_TRAIN) { bigru_set_error("tc_scan: recurrent dropout runs in the training forward only"); return BIGRU_ERR_ARG; }
    if (out != SCAN_TRAIN && out != SCAN_INFER_LOWER && out != SCAN_INFER_TOP) {
        bigru_set_error("tc_scan: no kernel writes this set of outputs (Y %d, G %d, planes %d)", (out & SCAN_Y) != 0,
                        (out & SCAN_G) != 0, (out & SCAN_PLANES) != 0);
        return BIGRU_ERR_ARG;
    }
    const bool x3 = p.prec == BIGRU_PREC_BF16X3;
    if (x3 && p.H == 128) *k = len ? scan_instance<128, 3, true>(out, rd) : scan_instance<128, 3, false>(out, rd);
    else if (x3 && p.H == 256) *k = len ? scan_instance<256, 3, true>(out, rd) : scan_instance<256, 3, false>(out, rd);
    else if (!x3 && p.H == 128) *k = len ? scan_instance<128, 1, true>(out, rd) : scan_instance<128, 1, false>(out, rd);
    else if (!x3 && p.H == 256) *k = len ? scan_instance<256, 1, true>(out, rd) : scan_instance<256, 1, false>(out, rd);
    else if (!x3 && p.H == 512) *k = len ? scan_instance<512, 1, true>(out, rd) : scan_instance<512, 1, false>(out, rd);
    else {
        bigru_set_error("tc_scan: no kernel for H=%d at precision %d", p.H, p.prec);
        return BIGRU_ERR_UNSUPPORTED;
    }
    return BIGRU_OK;
}

// the operands of one layer's forward recurrence.  A null Y, G or yh: that output is not written (the instantiations: all
// three, planes only, Y only).  len: per-row lengths [B] or null.  mask: the layer's recurrent-dropout masks [D][B][H]
// (training outputs only; yh, yl then get the masked state) or null
struct ScanFwdOps {
    const float *gi, *Whh, *bhh, *h0;
    float *Y, *G, *hn;
    htc::bf16_t *yh, *yl;
    const int* len;
    const float* mask;
};

static int tc_scan_fwd(const bigru_plan& p, int l, const ScanFwdOps& o, cudaStream_t st) {
    using namespace htc;
    const int out = (o.Y ? SCAN_Y : 0) | (o.G ? SCAN_G : 0) | (o.yh ? SCAN_PLANES : 0);
    ScanKernels k;
    TRY(scan_kernels(p, out, o.len != nullptr, o.mask != nullptr, &k));
    const int cs = p.H / SCAN_U;
    int R = 0, m2 = 0, clusters = 0;
    TRY(cluster_residency(k.fwd, cs, k.fwd_smem, &R));
    scan_geometry(R, k.two, p.B, p.D, &m2, &clusters);
    ProfScope ps(KC_TC_SCAN_FWD, 2.0 * p.D * p.B * (double)p.T * 3 * p.H * p.H, 0.0, st);
    return launch_cluster(k.fwd, cs, clusters, 1, k.fwd_smem, st, o.gi, o.Whh, o.bhh, p.ld_block(l), o.h0, o.Y, o.G, o.hn, o.yh,
                          o.yl, p.B, p.T, p.D, m2, o.len, o.mask);
}

// the operands of one layer's backward recurrence; len and mask as in ScanFwdOps
struct ScanBwdOps {
    const float *G, *Y, *h0, *dY;
    float *dhc, *dgi, *dgh;
    const float* Whh;
    htc::bf16_t *gih, *gil, *ghh, *ghl;
    const int* len;
    const float* mask;
};

static int tc_scan_bwd(const bigru_plan& p, int l, const ScanBwdOps& o, cudaStream_t st) {
    ScanKernels k;
    TRY(scan_kernels(p, htc::SCAN_TRAIN, o.len != nullptr, o.mask != nullptr, &k));
    const int cs = p.H / htc::SCAN_U;
    int R = 0, L8 = 0, clusters = 0;
    TRY(cluster_residency(k.bwd, cs, k.bwd_smem, &R));
    scan_bwd_geometry(R, p.B, p.D, &L8, &clusters);
    ProfScope ps(KC_TC_SCAN_BWD, 2.0 * p.D * p.B * (double)p.T * 3 * p.H * p.H, 0.0, st);
    return launch_cluster(k.bwd, cs, clusters, 1, k.bwd_smem, st, o.G, o.Y, o.h0, o.dY, o.dhc, o.dgi, o.dgh, o.Whh, p.ld_block(l),
                          o.gih, o.gil, o.ghh, o.ghl, p.B, p.T, p.D, L8, o.len, o.mask);
}

// plan p's layer scans without lengths, training outputs, with recurrent dropout when the plan has it (test support): the
// clusters R the device holds at once, and n_split, the tiles in two-tile clusters (scan 0, forward) or split into two
// 8-row clusters (scan 1, backward)
static int tc_scan_geometry(const bigru_plan& p, int scan, int* R, int* n_split) {
    ScanKernels k;
    TRY(scan_kernels(p, htc::SCAN_TRAIN, false, p.rp > 0.f, &k));
    const int cs = p.H / htc::SCAN_U;
    int r = 0, m2 = 0, clusters = 0;
    if (scan == 0) {
        TRY(cluster_residency(k.fwd, cs, k.fwd_smem, &r));
        scan_geometry(r, k.two, p.B, p.D, &m2, &clusters);
        *n_split = p.D * m2;
    } else {
        TRY(cluster_residency(k.bwd, cs, k.bwd_smem, &r));
        scan_bwd_geometry(r, p.B, p.D, n_split, &clusters);
    }
    *R = r;
    return BIGRU_OK;
}
