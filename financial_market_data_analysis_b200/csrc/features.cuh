// features.cuh - SURVEY.md 8(f) N4: the SQL window-function features of the reference (create_database.py:76-190) as one
// row-parallel kernel over the joined table's columns.  Every output row i depends on rows [i - w + 1, i] (moving
// averages, Bollinger bands, stochastic oscillator, ATR), on row i - 1 (price change) or on rows i + 8 / i + 15 (targets):
// block = 256 consecutive rows staged in shared memory with their halo, thread = row.  The SQL server evaluates AVG / STD
// of FLOAT columns in double; here the frame sums run in fp32 over DIFFERENCES to the current row (exact to ~1e-7 of the
// spread).  The targets are decided in fp32 where that provably gives the SQL's answer, and re-evaluated in fp64 as the
// SQL does on the rare rows near a tie (target_labels); that is the only FP64 in this kernel.  SQL NULL is NaN.
// HBM-bound: 4 * (5 + n_out + 4) bytes per row.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <math.h>

struct FeatureCfg {
    int n_vol, n_price, n_delta;
    int vol_p[8], price_p[8], delta_p[8];      // AVG(col) OVER (ROWS BETWEEN p-1 PRECEDING AND CURRENT ROW)
    int bb_period; float bb_std;               // 0: no Bollinger columns
    int stochastic;                            // ROWS BETWEEN 14 PRECEDING AND CURRENT ROW (15 rows)
    float n1, n2;                              // ATR factors of the targets
    int n_out;
};

constexpr int FEAT_TR = 256;            // table rows per block (= threads)

// mean of the staged column c over the frame [jlo, j], as c[j] + mean(c[k] - c[j]): the differences are small, so fp32
// sums keep ~1e-7 of the spread (not of the level).  (Non-tensor FP64 is a 1/64-rate pipe on this part: a double
// version of this kernel - and one with double prefix sums - measured 1.10 / 1.21 ms against 0.8 for fp32.)
__device__ __forceinline__ float frame_mean(const float* __restrict__ c, int jlo, int j) {
    const float ref = c[j];
    float s = 0.f;
#pragma unroll 4
    for (int k = jlo; k < j; ++k) s += c[k] - ref;
    return ref + s / (float)(j - jlo + 1);
}

// The four labels of row i (up1, up2, down1, down2): p_h >= p0 + n * ATR and p_h <= p0 - n * ATR for h = 8 / 15, as the
// reference's `target` view evaluates them in double: ATR = S / cnt with S the double sum of (high - low) over the 15-row
// frame [lo, i], n * ATR, then p0 +- that.  The fp32 decision d >= a (d = fl(p_h - p0), a = fl(n * atrf)) is kept when
// |d - a| exceeds a bound on the error of both sides; otherwise the label is recomputed in fp64 from global memory.
// Bound, with u = 2^-24, r_k = high_k - low_k exact, R = sum r_k, m = cnt <= 15 terms, A = n * R / m:
//   fl(high - low) = r_k (1 + e), |e| <= u; the recursive fp32 sum of m terms adds <= gamma_{m-1} = 14.01 u of sum |r_k|:
//   |sa - R| <= 15.02 u sum|r_k|.  atrf = sa * fl(1/15) (2 roundings) or sa / m (1), a = fl(n * atrf) (1 more):
//   |a - A| <= 18.1 u |n| sum|r_k| / m.  |d - (p_h - p0)| <= u |d| (0 when Sterbenz applies).
//   The SQL's double threshold p0 + n * S / m is within 2^-53 (|p0| + 17 |n| sum|r_k| / m) of p0 + A.
// So if |d - a| > E = 19.2 u (|d| + |n| sum|r_k| / m) + 2^-53 |p0|, then p_h - p0 - A is nonzero, has the sign of d - a
// and is larger than the SQL's own error: fp32 and SQL decide alike.  The kernel tests |d - a| > 2^-19 (|d| + |n| atra)
// + 2^-50 |p0| + 2^-126, with atra = atrf when every high - low staged for the tile is >= 0 (then sum |r_k| = R and
// atrf is within 18 u of R / m) and +inf otherwise, which sends every label of such a tile to fp64: 32 u against 19.2 u
// covers the fp32 rounding of the test itself, and 2^-126 covers underflow.  NaN margins (a NULL input) take the fp64
// path, where every comparison is false, as with SQL NULL.  Both instantiations use these two routines, so they agree
// at ties.
// Near ties are marked -1 in t[q] and t[2 + q], and resolve_ties recomputes them once the frames of the row are done.
// Returns whether there is one.
__device__ __forceinline__ bool target_labels(int64_t n, int64_t i, const float* __restrict__ sc, int j, float atrf, float atra,
                                              float n1, float n2, float* __restrict__ t) {
    const float p0 = sc[j];
    bool tie = false;
#pragma unroll
    for (int q = 0; q < 2; ++q) {
        const int h = q ? 15 : 8;
        const float nf = q ? n2 : n1;
        float up = 0.f, down = 0.f;
        if (i + h < n) {                          // LEAD(close, h) is NULL past the end, and a comparison with NULL is not true
            const float d = sc[j + h] - p0, a = nf * atrf;
            const float tol = 0x1p-19f * (fabsf(d) + fabsf(nf) * atra) + 0x1p-50f * fabsf(p0) + 0x1p-126f;
            if (fabsf(d - a) > tol && fabsf(d + a) > tol) {
                up = d >= a ? 1.f : 0.f;
                down = d <= -a ? 1.f : 0.f;
            } else {
                up = down = -1.f;
                tie = true;
            }
        }
        t[q] = up;
        t[2 + q] = down;
    }
    return tie;
}

// The marked labels in fp64, as the SQL evaluates them.  Called after the row's frames, so its doubles and its loop over
// global memory do not add to the registers the frames need (inlined into the frame code they took FAST from 40 to 64).
__device__ __forceinline__ void resolve_ties(const float* __restrict__ high, const float* __restrict__ low, int64_t i,
                                             const float* __restrict__ sc, int j, float n1, float n2, float* __restrict__ t) {
#pragma unroll 1
    for (int q = 0; q < 2; ++q) {
        if (t[q] >= 0.f) continue;
        const int cnt = i >= 14 ? 15 : (int)i + 1;
        const float *hp = high + (i + 1 - cnt), *lp = low + (i + 1 - cnt);
        double S = 0.0;
#pragma unroll 1
        for (int k = 0; k < cnt; ++k) S += (double)hp[k] - (double)lp[k];
        const double na = (double)(q ? n2 : n1) * (S / (double)cnt), p0 = sc[j], ph = sc[j + (q ? 15 : 8)];
        t[q] = ph >= p0 + na ? 1.f : 0.f;
        t[2 + q] = ph <= p0 - na ? 1.f : 0.f;
    }
}

// One block = FEAT_TR consecutive table rows: the columns of rows [r0 - halo, r0 + TR + 15) are staged in shared memory
// with coalesced loads, every thread forms the frames of its row from there, and the outputs leave through shared
// memory as coalesced rows.
// FAST: the periods are those of the reference's config.py:40-49 (vol 6 / 20, price 20, delta 12, Bollinger 20, stochastic
// on) as compile-time constants - the frames of every row past the head of the table are then straight-line code (the
// generic loops are instruction-issue bound: ~1200 instructions per row against ~350).
// FAST asks for 6 blocks per SM: that holds it at the 40 registers it had before the label routine (48 without the hint,
// which measured ~5 % slower on an H100); the generic kernel is faster without a hint.
template <bool FAST>
__global__ void __launch_bounds__(FEAT_TR, FAST ? 6 : 0) window_features_kernel(
        const float* __restrict__ close, const float* __restrict__ high, const float* __restrict__ low, const float* __restrict__ volume,
        const float* __restrict__ delta, int64_t n, FeatureCfg cfg, int halo, float* __restrict__ out, float* __restrict__ targets) {
    extern __shared__ float fsm[];
    const int span = FEAT_TR + halo;
    float* sc = fsm;                          // [span + 16] close, incl. the 15 rows the targets look ahead
    float* sh = sc + span + 16;               // [span] high - low
    float* sv = sh + span;                    // [span] volume
    float* sd = sv + span;                    // [span] delta
    float* so = sd + span;                    // [TR][n_out]
    float* st = so + FEAT_TR * cfg.n_out;     // [TR][4]
    const int tid = threadIdx.x;
    const int64_t ntiles = (n + FEAT_TR - 1) / FEAT_TR;
    for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int64_t r0 = tile * FEAT_TR, base = r0 - halo;      // staged index j <-> table row base + j
        int neg = 0;                              // a negative (or NaN) high - low in the tile: see target_labels
        for (int j = tid; j < span + 16; j += FEAT_TR) {
            const int64_t row = base + j;
            const bool ok = row >= 0 && row < n;
            sc[j] = ok ? close[row] : 0.f;
            if (j < span) {
                sh[j] = ok ? high[row] - low[row] : 0.f;
                neg |= !(sh[j] >= 0.f);
                sv[j] = (ok && volume) ? volume[row] : 0.f;
                sd[j] = (ok && delta) ? delta[row] : 0.f;
            }
        }
        neg = __syncthreads_or(neg);
        const int64_t i = r0 + tid;
        bool tie = false;
        if (i < n) {
            const int j = halo + tid;
            float* o = so + tid * cfg.n_out;
            int c = 0;
            const float pcf = sc[j];
            // frame [max(0, i - w + 1), i] -> first staged index
            auto first = [&](int w) { const int64_t lo = i - w + 1 < 0 ? 0 : i - w + 1; return j - (int)(i - lo); };
            float atrf;
            if (FAST && i >= 19) {
                // ---- straight-line frames (all 20 / 15 / 12 / 6 rows exist)
                float s1 = 0.f;
#pragma unroll
                for (int k = 1; k < 20; ++k) s1 += sc[j - k] - pcf;
                const float md = s1 * (1.f / 20.f);
                float v = md * md;
#pragma unroll
                for (int k = 1; k < 20; ++k) { const float d = (sc[j - k] - pcf) - md; v = fmaf(d, d, v); }
                const float sdv = sqrtf(v * (1.f / 20.f));
                o[c++] = md + cfg.bb_std * sdv;
                o[c++] = cfg.bb_std * sdv - md;
                const float vref = sv[j];
                float v6 = 0.f;
#pragma unroll
                for (int k = 1; k < 6; ++k) v6 += sv[j - k] - vref;
                float v20 = v6;
#pragma unroll
                for (int k = 6; k < 20; ++k) v20 += sv[j - k] - vref;
                o[c++] = vref + v6 * (1.f / 6.f);
                o[c++] = vref + v20 * (1.f / 20.f);
                o[c++] = pcf + md;                                                                   // price_MA20 = BB_avg
                const float dref = sd[j];
                float d12 = 0.f;
#pragma unroll
                for (int k = 1; k < 12; ++k) d12 += sd[j - k] - dref;
                o[c++] = dref + d12 * (1.f / 12.f);
                float mn = pcf, mx = pcf;
#pragma unroll
                for (int k = 1; k < 15; ++k) { mn = fminf(mn, sc[j - k]); mx = fmaxf(mx, sc[j - k]); }
                o[c++] = mx > mn ? (pcf - mn) / (mx - mn) : nanf("");
                float sa = 0.f;
#pragma unroll
                for (int k = 0; k < 15; ++k) sa += sh[j - k];
                atrf = sa * (1.f / 15.f);
                o[c++] = atrf;
            } else {
            float bb_mean = 0.f;
            if (cfg.bb_period > 0) {
                // (BB_avg + k * BB_std) - close, close - (BB_avg - k * BB_std); STD = population standard deviation.
                // With d_k = close[k] - close[i]: avg - close = mean(d), std = sqrt(mean((d - mean d)^2)) (two passes)
                const int jlo = first(cfg.bb_period);
                const float cnt = (float)(j - jlo + 1);
                float s1 = 0.f;
#pragma unroll 4
                for (int k = jlo; k < j; ++k) s1 += sc[k] - pcf;
                const float md = s1 / cnt;
                float v = md * md;                                 // the k == i term: (0 - md)^2
#pragma unroll 4
                for (int k = jlo; k < j; ++k) { const float d = (sc[k] - pcf) - md; v = fmaf(d, d, v); }
                const float sdv = sqrtf(v / cnt);
                o[c++] = md + cfg.bb_std * sdv;
                o[c++] = cfg.bb_std * sdv - md;
                bb_mean = pcf + md;
            }
            for (int q = 0; q < cfg.n_vol; ++q) o[c++] = frame_mean(sv, first(cfg.vol_p[q]), j);
            for (int q = 0; q < cfg.n_price; ++q)
                o[c++] = (cfg.price_p[q] == cfg.bb_period) ? bb_mean : frame_mean(sc, first(cfg.price_p[q]), j);
            for (int q = 0; q < cfg.n_delta; ++q) o[c++] = frame_mean(sd, first(cfg.delta_p[q]), j);
            const int j15 = first(15);
            if (cfg.stochastic) {
                float mn = sc[j15], mx = sc[j15];
#pragma unroll 4
                for (int k = j15 + 1; k <= j; ++k) { mn = fminf(mn, sc[k]); mx = fmaxf(mx, sc[k]); }
                o[c++] = mx > mn ? (pcf - mn) / (mx - mn) : nanf("");     // x / 0 is NULL in SQL; both differences are exact in fp32
            }
            float sa = 0.f;                                                                            // ATR = AVG(high - low), 15 rows
#pragma unroll 4
            for (int k = j15; k <= j; ++k) sa += sh[k];
            atrf = sa / (float)(j - j15 + 1);
            o[c++] = atrf;
            }
            o[c++] = i > 0 ? pcf - sc[j - 1] : nanf("");                                               // LAG(close, 1): NULL on the first row
            if (targets) tie = target_labels(n, i, sc, j, atrf, neg ? __int_as_float(0x7f800000) : atrf, cfg.n1, cfg.n2, st + tid * 4);
        }
        if (tie) resolve_ties(high, low, i, sc, halo + tid, cfg.n1, cfg.n2, st + tid * 4);
        __syncthreads();
        const int rows = (int)((n - r0) < FEAT_TR ? (n - r0) : FEAT_TR);
        for (int k = tid; k < rows * cfg.n_out; k += FEAT_TR) out[r0 * cfg.n_out + k] = so[k];
        if (targets)
            for (int k = tid; k < rows * 4; k += FEAT_TR) targets[r0 * 4 + k] = st[k];
        __syncthreads();
    }
}
