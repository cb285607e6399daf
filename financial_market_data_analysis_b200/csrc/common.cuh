// common.cuh - shared declarations for libbigru_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdarg>
#include "../../include/bigru_b200.h"
#include "prof.cuh"

void bigru_set_error(const char* fmt, ...);

#define CUDA_TRY(expr)                                                                     \
    do {                                                                                   \
        cudaError_t e__ = (expr);                                                          \
        if (e__ != cudaSuccess) {                                                          \
            bigru_set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__),       \
                            __FILE__, __LINE__);                                           \
            return BIGRU_ERR_CUDA;                                                         \
        }                                                                                  \
    } while (0)
#define LAUNCH_CHECK() CUDA_TRY(cudaGetLastError())
// launch with accounting: kernel class, algorithmic flops, algorithmic bytes
#define KLAUNCH(cls, flops, bytes, st, ...) \
    do { { ProfScope ps__(cls, flops, bytes, st); __VA_ARGS__; } LAUNCH_CHECK(); } while (0)
#define TRY(expr) do { int r__ = (expr); if (r__ != BIGRU_OK) return r__; } while (0)

static inline int64_t cdiv64(int64_t a, int64_t b) { return (a + b - 1) / b; }

// Shapes, flat-parameter offsets and workspace carve-up.  All sizes in elements unless noted.
struct bigru_plan {
    int B, T, F, H, L, C, D, prec;
    int64_t nparams;
    int64_t layer_dir_stride[8];   // unused for L>8; offsets are computed on demand
    size_t stash_bytes, scratch_bytes;

    __host__ int64_t in_size(int l) const { return l == 0 ? F : (int64_t)D * H; }
    __host__ int64_t ld_block(int l) const { return 3LL * H * in_size(l) + 3LL * H * H + 6LL * H; }
    __host__ int64_t ld_off(int l, int d) const {
        int64_t off = 0;
        for (int ll = 0; ll < l; ++ll) off += (int64_t)D * ld_block(ll);
        return off + (l < L ? (int64_t)d * ld_block(l) : 0);
    }
    __host__ int64_t off_wih(int l, int d) const { return ld_off(l, d); }
    __host__ int64_t off_whh(int l, int d) const { return ld_off(l, d) + 3LL * H * in_size(l); }
    __host__ int64_t off_bih(int l, int d) const { return off_whh(l, d) + 3LL * H * H; }
    __host__ int64_t off_bhh(int l, int d) const { return off_bih(l, d) + 3LL * H; }
    __host__ int64_t off_linw() const { return ld_off(L, 0); }
    __host__ int64_t off_linb() const { return off_linw() + 3LL * H * C; }
};

// counter-based uniform in [0,1): splitmix64 finaliser over (seed, stream, index)
__host__ __device__ inline float bigru_uniform(uint64_t seed, uint32_t stream, uint64_t idx) {
    uint64_t z = seed + 0x9E3779B97F4A7C15ull * (idx + 1) + ((uint64_t)stream << 40) * 0xD1B54A32D192ED03ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    z = z ^ (z >> 31);
    return (float)(z >> 40) * (1.0f / 16777216.0f);
}
