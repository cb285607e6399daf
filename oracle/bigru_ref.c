/* oracle/bigru_ref.c - plain-C CPU restatement of the biGRU hot path.
 *
 * TEST INFRASTRUCTURE ONLY: linked/loaded by tests/, __graft_entry__.smoke() and the
 * cpu_baseline leg of bench.py.  The product never calls into this file.
 *
 * Restates (float storage, double accumulation):
 *   - model forward        /root/reference/biGRU_model.py:63-138  (eval mode / dropout p=0)
 *     whose recurrent cell is torch.nn.GRU (third-party; /root/reference/requirements.txt:11
 *     pins torch==1.2.0).  Published cell equations, gate row order r|z|n:
 *        r = s(Wir x + bir + Whr h + bhr)      z = s(Wiz x + biz + Whz h + bhz)
 *        n = tanh(Win x + bin + r*(Whn h + bhn))   h' = (1-z)*n + z*h
 *   - its reverse-mode derivative (the reference gets it from autograd, biGRU_model.py:204)
 *   - clip_grad_norm_ + Adam   biGRU_model.py:208-210
 *   - sliding-window collation + min/max normalisation  sql_pytorch_dataloader.py:8-18,239-245
 *   - the three losses the reference's callers plug in (CE for the benchmark configs,
 *     BCEWithLogits notebook raw :1192, MultiLabelSoftMargin predict.py:94)
 *
 * Flat parameter order (shared with the product's C-ABI, include/bigru_b200.h):
 *   for l in [0,L): for d in [0,D): w_ih[3H,I_l] w_hh[3H,H] b_ih[3H] b_hh[3H] ; lin_w[C,3H] lin_b[C]
 *   I_0 = F, I_l = D*H.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct { int B, T, F, H, L, C, D; } dims_t;

static int64_t in_size(const dims_t* d, int l) { return l == 0 ? d->F : (int64_t)d->D * d->H; }

static int64_t layer_dir_offset(const dims_t* d, int l, int dir) {
    int64_t off = 0;
    for (int ll = 0; ll < d->L; ++ll)
        for (int dd = 0; dd < d->D; ++dd) {
            if (ll == l && dd == dir) return off;
            off += 3LL * d->H * in_size(d, ll) + 3LL * d->H * d->H + 6LL * d->H;
        }
    return off;
}

int64_t bigru_ref_param_count(int F, int H, int L, int C, int D) {
    dims_t d = {0, 0, F, H, L, C, D};
    return layer_dir_offset(&d, L, 0) + 3LL * H * C + C;
}

static double sigm(double a) { return 1.0 / (1.0 + exp(-a)); }

/* ---- rounding model of the tensor-core precisions ------------------------------------------------------------
 * prec 0 (BIGRU_REF_EXACT): every product in fp64; bigru_ref_forward / bigru_ref_backward are this mode.
 * prec 1 (BIGRU_REF_BF16) and 2 (BIGRU_REF_BF16X3) round the two operands of every matrix product where the CUDA path
 * (financial_market_data_analysis_b200/csrc/api.cu, tc_hopper.cuh) rounds them, and nothing else: sums, biases, gate
 * math, state, pooling and the carried gradients stay fp64.  An operand value v is first rounded to fp32 (what the
 * kernels store), then
 *   bf16:   v -> rn_bf16(v)                                                  (round to nearest even)
 *   bf16x3: v -> hi = rn_bf16(v), lo = rn_bf16(v - hi); a product is ah*bh + ah*bl + al*bh   (split_bf16, tc_hopper.cuh)
 * Rounding points (bit of `mask`; a cleared bit keeps that operand exact, which the CPU tests use to show each point is
 * wired):
 *   forward   0 PROJ_X    layer input of x W_ih^T (x, or the previous layer's Y)      [to_planes_kernel / Y planes]
 *             1 PROJ_W    W_ih of the projection; b_ih is added unrounded                 [tc_pack_kernel]
 *             2 REC_H     h_{t-1} of h_{t-1} W_hh^T for t past the first step             [gru_scan_fwd_kernel h tile]
 *             3 REC_W     W_hh of the recurrence; b_hh, z*h_{t-1} and the gate math unrounded  [scan's W slice]
 *             4 HEAD_CAT  pooled features cat of cat lin_w^T                               [tc_gemm_launch]
 *             5 HEAD_W    lin_w of the head; lin_b unrounded                               [tc_gemm_launch]
 *            18 REC_H0    h0 in the first step's recurrent product                         [gru_scan_fwd_kernel h tile]
 *   backward  6 HB_DL     dlogits in dcat = dlogits lin_w and dlin_w = dlogits^T cat; dlin_b unrounded
 *             7 HB_W      lin_w in dcat                                                    [tc_gemm_launch]
 *             8 HB_CAT    cat in dlin_w                                                    [tc_gemm_launch]
 *             9 BR_DGH    dgh in the backward recurrence W_hh^T dgh; the dh*z term unrounded  [gru_scan_bwd_kernel]
 *            10 BR_W      W_hh there                                                       [gru_scan_bwd_kernel]
 *            11 DWIH_DGI  dgi in dW_ih = dgi^T X                                           [dgi planes]
 *            12 DWIH_X    X there (the projection's input)                                 [input planes]
 *            13 DWHH_DGH  dgh in dW_hh = dgh^T H_prev                                      [dgh planes, h0 term packed]
 *            14 DWHH_Y    H_prev rows past each sequence's first step (the previous Y)    [Y planes]
 *            15 DWHH_H0   H_prev rows of the first step (h0; the h0 term of tc_gemm_launch) [tc_gemm_launch]
 *            16 DX_DGI    dgi in dX = dgi W_ih                                             [dgi planes]
 *            17 DX_W      W_ih there                                                       [tc_pack_kernel]
 *   Bias gradients are column sums of the unrounded dgi / dgh.
 * Each operand array is rounded once (weights once per call, activations once per layer or step). */
enum {
    RP_PROJ_X, RP_PROJ_W, RP_REC_H, RP_REC_W, RP_HEAD_CAT, RP_HEAD_W, RP_HB_DL, RP_HB_W, RP_HB_CAT, RP_BR_DGH, RP_BR_W,
    RP_DWIH_DGI, RP_DWIH_X, RP_DWHH_DGH, RP_DWHH_Y, RP_DWHH_H0, RP_DX_DGI, RP_DX_W, RP_REC_H0, RP_COUNT
};
int bigru_ref_rounding_points(void) { return RP_COUNT; }

static float rn_bf16(float v) {
    uint32_t u;
    memcpy(&u, &v, 4);
    if ((u & 0x7fffffffu) > 0x7f800000u) return v;          /* NaN stays NaN */
    u += 0x7fffu + ((u >> 16) & 1u);
    u &= 0xffff0000u;
    memcpy(&v, &u, 4);
    return v;
}

/* an operand array as the products read it: f = hi + lo (the rounded value), h = hi, l = lo (bf16x3 only, else NULL);
 * a product a*b is a.h*b.f + a.l*b.h, i.e. ah*bh + ah*bl + al*bh.  Exact: f = h = the value. */
typedef struct { double *f, *h, *l, *buf; } op_t;

static op_t op_alloc(int64_t n, int prec) {
    op_t o = {0};
    o.buf = (double*)malloc(sizeof(double) * (size_t)n * (prec == 2 ? 3 : 1));
    o.f = o.h = o.buf;
    if (prec == 2) { o.h = o.buf + n; o.l = o.buf + 2 * n; }
    return o;
}
static void op_put(op_t* o, int64_t i, int prec, double v) {
    if (prec == 0) { o->f[i] = v; return; }
    const float v32 = (float)v, hi = rn_bf16(v32);
    if (prec == 1) { o->f[i] = hi; return; }
    const float lo = rn_bf16(v32 - hi);
    o->h[i] = hi; o->l[i] = lo; o->f[i] = (double)hi + (double)lo;
}
static op_t op_of_d(const double* src, int64_t n, int prec) {
    if (prec == 0) { op_t o = {(double*)src, (double*)src, NULL, NULL}; return o; }
    op_t o = op_alloc(n, prec);
    for (int64_t i = 0; i < n; ++i) op_put(&o, i, prec, src[i]);
    return o;
}
static op_t op_of_f(const float* src, int64_t n, int prec) {
    op_t o = op_alloc(n, prec);
    for (int64_t i = 0; i < n; ++i) op_put(&o, i, prec, (double)src[i]);
    return o;
}
static void op_free(op_t* o) { free(o->buf); o->buf = NULL; }

/* acc + sum_k a[ia+k] * b[ib+k] */
static double dot(const op_t* a, int64_t ia, const op_t* b, int64_t ib, int64_t n, double acc) {
    for (int64_t k = 0; k < n; ++k) acc += a->h[ia + k] * b->f[ib + k];
    if (a->l) for (int64_t k = 0; k < n; ++k) acc += a->l[ia + k] * b->h[ib + k];
    return acc;
}
static double mul(const op_t* a, int64_t i, const op_t* b, int64_t j) {
    double p = a->h[i] * b->f[j];
    if (a->l) p += a->l[i] * b->h[j];
    return p;
}

/* Workspace the backward needs; allocated by forward when stash != NULL.
 * stash layout (doubles): per layer: out[B,T,D*H]; per (l,dir): r,z,n,hn,hprev each [B,T,H];
 * then cat[B,3H] and arg[B,H] (as double; a caller may overwrite arg with another max-pool routing before the backward). */
static int64_t stash_doubles(const dims_t* d) {
    int64_t BT = (int64_t)d->B * d->T;
    return (int64_t)d->L * (BT * d->D * d->H + (int64_t)d->D * 5 * BT * d->H) + (int64_t)d->B * 4 * d->H;
}
int64_t bigru_ref_stash_doubles(int B, int T, int F, int H, int L, int C, int D) {
    dims_t d = {B, T, F, H, L, C, D};
    return stash_doubles(&d);
}

/* forward: x[B,T,F], h0 (nullable) [L*D,B,H] -> logits[B,C], hn_out (nullable) [L*D,B,H].
 * prec: 0 exact, 1 bf16, 2 bf16x3; mask: rounding points (bits above) that prec applies to. */
int bigru_ref_forward_p(int B, int T, int F, int H, int L, int C, int D, int prec, unsigned mask,
                        const float* params, const float* x, const float* h0,
                        float* logits, float* hn_out, double* stash) {
    dims_t dm = {B, T, F, H, L, C, D};
    int64_t BT = (int64_t)B * T;
    if (prec < 0 || prec > 2) return -2;
#define PR(bit) (((mask >> (bit)) & 1u) ? prec : 0)
    int own = 0;
    if (!stash) { stash = (double*)malloc(sizeof(double) * stash_doubles(&dm)); own = 1; if (!stash) return -1; }
    double* sp = stash;
    const double* inp_d = NULL;   /* previous layer's output (double) */
    double* out = NULL;
    for (int l = 0; l < L; ++l) {
        int64_t I = in_size(&dm, l);
        out = sp; sp += BT * D * H;
        op_t X = l == 0 ? op_of_f(x, BT * F, PR(RP_PROJ_X)) : op_of_d(inp_d, BT * I, PR(RP_PROJ_X));
        for (int dir = 0; dir < D; ++dir) {
            const float* w_ih = params + layer_dir_offset(&dm, l, dir);
            const float* w_hh = w_ih + 3LL * H * I;
            const float* b_ih = w_hh + 3LL * H * H;
            const float* b_hh = b_ih + 3LL * H;
            op_t WI = op_of_f(w_ih, 3LL * H * I, PR(RP_PROJ_W)), WH = op_of_f(w_hh, 3LL * H * H, PR(RP_REC_W));
            double *R = sp, *Z = R + BT * H, *N = Z + BT * H, *HN = N + BT * H, *HP = HN + BT * H;
            sp += 5 * BT * H;
            #pragma omp parallel for schedule(static)
            for (int b = 0; b < B; ++b) {
                double* h = (double*)malloc(sizeof(double) * 2 * H);
                double* hnew = h + H;
                op_t hs = op_alloc(H, prec);
                for (int j = 0; j < H; ++j) h[j] = h0 ? (double)h0[((int64_t)(l * D + dir) * B + b) * H + j] : 0.0;
                for (int s = 0; s < T; ++s) {
                    int t = dir == 0 ? s : T - 1 - s;
                    int64_t row = (int64_t)b * T + t;
                    const int ph = s == 0 ? PR(RP_REC_H0) : PR(RP_REC_H);
                    for (int j = 0; j < H; ++j) op_put(&hs, j, ph, h[j]);
                    if (ph == 0 && hs.l) memset(hs.l, 0, sizeof(double) * H);
                    if (ph == 0 && hs.h != hs.f) memcpy(hs.h, hs.f, sizeof(double) * H);
                    for (int j = 0; j < H; ++j) {
                        double gi[3], gh[3];
                        for (int g = 0; g < 3; ++g) {
                            gi[g] = dot(&WI, (int64_t)(g * H + j) * I, &X, row * I, I, b_ih[g * H + j]);
                            gh[g] = dot(&WH, (int64_t)(g * H + j) * H, &hs, 0, H, b_hh[g * H + j]);
                        }
                        double r = sigm(gi[0] + gh[0]), z = sigm(gi[1] + gh[1]);
                        double n = tanh(gi[2] + r * gh[2]);
                        hnew[j] = (1.0 - z) * n + z * h[j];
                        R[row * H + j] = r; Z[row * H + j] = z; N[row * H + j] = n; HN[row * H + j] = gh[2];
                        HP[row * H + j] = h[j];
                    }
                    for (int j = 0; j < H; ++j) { h[j] = hnew[j]; out[row * D * H + dir * H + j] = hnew[j]; }
                }
                if (hn_out) for (int j = 0; j < H; ++j) hn_out[((int64_t)(l * D + dir) * B + b) * H + j] = (float)h[j];
                op_free(&hs);
                free(h);
            }
            op_free(&WI); op_free(&WH);
        }
        op_free(&X);
        inp_d = out;
    }
    /* head: biGRU_model.py:111-137 */
    double* cat = sp; double* arg = cat + (int64_t)B * 3 * H;
    const float* lin_w = params + layer_dir_offset(&dm, L, 0);
    const float* lin_b = lin_w + 3LL * H * C;
    for (int b = 0; b < B; ++b)
        for (int j = 0; j < H; ++j) {
            double last = out[((int64_t)b * T + (T - 1)) * D * H + j];
            if (D == 2) last += out[((int64_t)b * T + 0) * D * H + H + j];
            double mx = -INFINITY, sum = 0.0; int am = 0;
            for (int t = 0; t < T; ++t) {
                double s = out[((int64_t)b * T + t) * D * H + j];
                if (D == 2) s += out[((int64_t)b * T + t) * D * H + H + j];
                if (s > mx) { mx = s; am = t; }          /* strict >: first maximum wins */
                sum += s;
            }
            cat[(int64_t)b * 3 * H + j] = last;
            cat[(int64_t)b * 3 * H + H + j] = mx;
            cat[(int64_t)b * 3 * H + 2 * H + j] = sum / (double)T;
            arg[(int64_t)b * H + j] = (double)am;
        }
    op_t CW = op_of_f(lin_w, 3LL * H * C, PR(RP_HEAD_W)), CX = op_of_d(cat, (int64_t)B * 3 * H, PR(RP_HEAD_CAT));
    for (int b = 0; b < B; ++b)
        for (int c = 0; c < C; ++c)
            logits[(int64_t)b * C + c] = (float)dot(&CW, (int64_t)c * 3 * H, &CX, (int64_t)b * 3 * H, 3 * H, lin_b[c]);
    op_free(&CW); op_free(&CX);
    if (own) free(stash);
    return 0;
}

int bigru_ref_forward(int B, int T, int F, int H, int L, int C, int D,
                      const float* params, const float* x, const float* h0,
                      float* logits, float* hn_out, double* stash) {
    return bigru_ref_forward_p(B, T, F, H, L, C, D, 0, ~0u, params, x, h0, logits, hn_out, stash);
}

/* backward: needs the stash written by bigru_ref_forward_p with the same prec and mask.  grads: flat, same order as
 * params.  dx nullable [B,T,F]; dh0 nullable [L*D,B,H]. */
int bigru_ref_backward_p(int B, int T, int F, int H, int L, int C, int D, int prec, unsigned mask,
                         const float* params, const float* x, const double* stash,
                         const float* dlogits, float* grads, float* dx, float* dh0) {
    dims_t dm = {B, T, F, H, L, C, D};
    int64_t BT = (int64_t)B * T;
    if (prec < 0 || prec > 2) return -2;
    int64_t P = bigru_ref_param_count(F, H, L, C, D);
    double* g = (double*)calloc(P, sizeof(double));
    /* locate stash pieces */
    const double** outs = (const double**)malloc(sizeof(double*) * L);
    const double** gates = (const double**)malloc(sizeof(double*) * L * D);
    const double* sp = stash;
    for (int l = 0; l < L; ++l) {
        outs[l] = sp; sp += BT * D * H;
        for (int dir = 0; dir < D; ++dir) { gates[l * D + dir] = sp; sp += 5 * BT * H; }
    }
    const double* cat = sp; const double* arg = cat + (int64_t)B * 3 * H;
    int64_t lin_off = layer_dir_offset(&dm, L, 0);
    const float* lin_w = params + lin_off;
    double* dcat = (double*)calloc((size_t)B * 3 * H, sizeof(double));
    op_t DL = op_of_f(dlogits, (int64_t)B * C, PR(RP_HB_DL));
    op_t CW = op_of_f(lin_w, 3LL * H * C, PR(RP_HB_W)), CX = op_of_d(cat, (int64_t)B * 3 * H, PR(RP_HB_CAT));
    for (int b = 0; b < B; ++b)
        for (int c = 0; c < C; ++c) {
            double dl = dlogits[(int64_t)b * C + c];
            g[lin_off + 3LL * H * C + c] += dl;
            for (int k = 0; k < 3 * H; ++k) {
                g[lin_off + (int64_t)c * 3 * H + k] += mul(&DL, (int64_t)b * C + c, &CX, (int64_t)b * 3 * H + k);
                dcat[(int64_t)b * 3 * H + k] += mul(&DL, (int64_t)b * C + c, &CW, (int64_t)c * 3 * H + k);
            }
        }
    op_free(&DL); op_free(&CW); op_free(&CX);
    /* dout for the top layer */
    double* dout = (double*)calloc((size_t)BT * D * H, sizeof(double));
    for (int b = 0; b < B; ++b)
        for (int j = 0; j < H; ++j) {
            double dmax = dcat[(int64_t)b * 3 * H + H + j], davg = dcat[(int64_t)b * 3 * H + 2 * H + j] / (double)T;
            int am = (int)arg[(int64_t)b * H + j];
            for (int t = 0; t < T; ++t) {
                double v = davg + (t == am ? dmax : 0.0);
                for (int dir = 0; dir < D; ++dir) dout[((int64_t)b * T + t) * D * H + dir * H + j] = v;
            }
        }
    for (int l = L - 1; l >= 0; --l) {
        int64_t I = in_size(&dm, l);
        double* dinp = (double*)calloc((size_t)BT * I, sizeof(double));
        op_t XW = l == 0 ? op_of_f(x, BT * F, PR(RP_DWIH_X)) : op_of_d(outs[l - 1], BT * I, PR(RP_DWIH_X));
        for (int dir = 0; dir < D; ++dir) {
            int64_t off = layer_dir_offset(&dm, l, dir);
            const float* w_ih = params + off;
            const float* w_hh = w_ih + 3LL * H * I;
            int64_t o_wih = off, o_whh = off + 3LL * H * I, o_bih = o_whh + 3LL * H * H, o_bhh = o_bih + 3LL * H;
            const double *R = gates[l * D + dir], *Z = R + BT * H, *N = Z + BT * H, *HN = N + BT * H, *HP = HN + BT * H;
            double* dgi = (double*)malloc(sizeof(double) * BT * 3 * H);
            double* dgh = (double*)malloc(sizeof(double) * BT * 3 * H);
            op_t WH = op_of_f(w_hh, 3LL * H * H, PR(RP_BR_W));
            const int pg = PR(RP_BR_DGH);
            #pragma omp parallel for schedule(static)
            for (int b = 0; b < B; ++b) {
                double* dh = (double*)calloc(2 * (size_t)H, sizeof(double));
                double* dhn = dh + H;
                op_t gs = op_alloc(3LL * H, pg);
                if (l == L - 1) for (int j = 0; j < H; ++j) dh[j] = dcat[(int64_t)b * 3 * H + j];
                for (int s = 0; s < T; ++s) {
                    int t = dir == 0 ? T - 1 - s : s;
                    int64_t row = (int64_t)b * T + t;
                    for (int j = 0; j < H; ++j) {
                        double d = dh[j] + dout[row * D * H + dir * H + j];
                        double r = R[row * H + j], z = Z[row * H + j], n = N[row * H + j];
                        double hn = HN[row * H + j], hp = HP[row * H + j];
                        double dan = d * (1.0 - z) * (1.0 - n * n);
                        double dar = dan * hn * r * (1.0 - r);
                        double daz = d * (hp - n) * z * (1.0 - z);
                        dgi[row * 3 * H + j] = dar; dgi[row * 3 * H + H + j] = daz; dgi[row * 3 * H + 2 * H + j] = dan;
                        dgh[row * 3 * H + j] = dar; dgh[row * 3 * H + H + j] = daz; dgh[row * 3 * H + 2 * H + j] = dan * r;
                        dhn[j] = d * z;
                    }
                    for (int q = 0; q < 3 * H; ++q) op_put(&gs, q, pg, dgh[row * 3 * H + q]);
                    for (int k = 0; k < H; ++k) {
                        double a = dhn[k];
                        for (int q = 0; q < 3 * H; ++q) a += mul(&gs, q, &WH, (int64_t)q * H + k);
                        dh[k] = a;
                    }
                }
                if (dh0) for (int j = 0; j < H; ++j) dh0[((int64_t)(l * D + dir) * B + b) * H + j] = (float)dh[j];
                op_free(&gs);
                free(dh);
            }
            op_free(&WH);
            /* weight / bias / input gradients */
            op_t GI = op_of_d(dgi, BT * 3 * H, PR(RP_DWIH_DGI)), GH = op_of_d(dgh, BT * 3 * H, PR(RP_DWHH_DGH));
            op_t HW = op_alloc(BT * H, prec);          /* H_prev: Y rows and, at each sequence's first step, h0 rows */
            for (int64_t row = 0; row < BT; ++row) {
                const int t = (int)(row % T), first = dir == 0 ? t == 0 : t == T - 1;
                const int ph = first ? PR(RP_DWHH_H0) : PR(RP_DWHH_Y);
                for (int k = 0; k < H; ++k) {
                    const int64_t i = row * H + k;
                    op_put(&HW, i, ph, HP[i]);
                    if (ph == 0 && HW.h != HW.f) HW.h[i] = HP[i];
                    if (ph == 0 && HW.l) HW.l[i] = 0.0;
                }
            }
            #pragma omp parallel for schedule(static)
            for (int q = 0; q < 3 * H; ++q) {
                double sb_i = 0.0, sb_h = 0.0;
                for (int64_t row = 0; row < BT; ++row) {
                    double a = dgi[row * 3 * H + q], c = dgh[row * 3 * H + q];
                    sb_i += a; sb_h += c;
                    for (int k = 0; k < I; ++k) g[o_wih + (int64_t)q * I + k] += mul(&GI, row * 3 * H + q, &XW, row * I + k);
                    for (int k = 0; k < H; ++k) g[o_whh + (int64_t)q * H + k] += mul(&GH, row * 3 * H + q, &HW, row * H + k);
                }
                g[o_bih + q] = sb_i; g[o_bhh + q] = sb_h;
            }
            op_free(&GI); op_free(&GH); op_free(&HW);
            op_t GX = op_of_d(dgi, BT * 3 * H, PR(RP_DX_DGI)), WX = op_of_f(w_ih, 3LL * H * I, PR(RP_DX_W));
            #pragma omp parallel for schedule(static)
            for (int64_t row = 0; row < BT; ++row)
                for (int q = 0; q < 3 * H; ++q)
                    for (int k = 0; k < I; ++k) dinp[row * I + k] += mul(&GX, row * 3 * H + q, &WX, (int64_t)q * I + k);
            op_free(&GX); op_free(&WX);
            free(dgi); free(dgh);
        }
        op_free(&XW);
        free(dout);
        dout = dinp;
    }
    if (dx) for (int64_t i = 0; i < BT * F; ++i) dx[i] = (float)dout[i];
    free(dout);
    for (int64_t i = 0; i < P; ++i) grads[i] = (float)g[i];
    free(g); free(dcat); free(outs); free(gates);
    return 0;
#undef PR
}

int bigru_ref_backward(int B, int T, int F, int H, int L, int C, int D,
                       const float* params, const float* x, const double* stash,
                       const float* dlogits, float* grads, float* dx, float* dh0) {
    return bigru_ref_backward_p(B, T, F, H, L, C, D, 0, ~0u, params, x, stash, dlogits, grads, dx, dh0);
}

/* ---- losses: value (mean reduction) + dlogits --------------------------------------- */
double bigru_ref_loss_ce(int B, int C, const float* logits, const int64_t* target, float* dlogits, double scale) {
    double loss = 0.0;
    for (int b = 0; b < B; ++b) {
        const float* lg = logits + (int64_t)b * C;
        double m = lg[0]; for (int c = 1; c < C; ++c) if (lg[c] > m) m = lg[c];
        double s = 0.0; for (int c = 0; c < C; ++c) s += exp(lg[c] - m);
        double lse = m + log(s);
        loss += lse - lg[target[b]];
        if (dlogits) for (int c = 0; c < C; ++c)
            dlogits[(int64_t)b * C + c] = (float)((exp(lg[c] - lse) - (c == target[b] ? 1.0 : 0.0)) * scale);
    }
    return loss * scale;
}

/* torch.nn.BCEWithLogitsLoss(weight[C] nullable, pos_weight[C] nullable), mean over B*C */
double bigru_ref_loss_bce(int B, int C, const float* logits, const float* target, const float* weight,
                          const float* pos_weight, float* dlogits, double scale) {
    double loss = 0.0;
    for (int b = 0; b < B; ++b) for (int c = 0; c < C; ++c) {
        double x = logits[(int64_t)b * C + c], y = target[(int64_t)b * C + c];
        double pw = pos_weight ? pos_weight[c] : 1.0, w = weight ? weight[c] : 1.0;
        double sp_neg = (x > 0 ? 0.0 : -x) + log1p(exp(-fabs(x)));   /* softplus(-x) = -log sigmoid(x) */
        double lw = 1.0 + (pw - 1.0) * y;
        loss += w * ((1.0 - y) * x + lw * sp_neg);
        if (dlogits) {
            double s = sigm(x);
            dlogits[(int64_t)b * C + c] = (float)(w * ((1.0 - y) - lw * (1.0 - s)) * scale);
        }
    }
    return loss * scale;
}

/* torch.nn.MultiLabelSoftMarginLoss(): mean over classes, then mean over batch */
double bigru_ref_loss_mlsm(int B, int C, const float* logits, const float* target, float* dlogits, double scale) {
    return bigru_ref_loss_bce(B, C, logits, target, NULL, NULL, dlogits, scale);
}

/* ---- clip_grad_norm_ + Adam (biGRU_model.py:208-210; torch.optim.Adam defaults) ------- */
double bigru_ref_clip_adam(int64_t P, float* params, float* grads, float* m, float* v, double clip,
                           double lr, double b1, double b2, double eps, int step) {
    double ss = 0.0;
    for (int64_t i = 0; i < P; ++i) ss += (double)grads[i] * grads[i];
    double norm = sqrt(ss);
    double coef = clip / (norm + 1e-6);
    if (coef > 1.0) coef = 1.0;
    double bc1 = 1.0 - pow(b1, step), bc2 = 1.0 - pow(b2, step);
    for (int64_t i = 0; i < P; ++i) {
        float gq = (float)(grads[i] * (float)coef);
        grads[i] = gq;
        m[i] = (float)(b1 * m[i] + (1.0 - b1) * gq);
        v[i] = (float)(b2 * v[i] + (1.0 - b2) * (double)gq * gq);
        double denom = sqrt((double)v[i]) / sqrt(bc2) + eps;
        params[i] = (float)(params[i] - (lr / bc1) * (m[i] / denom));
    }
    return norm;
}

/* ---- window collation: out[b,t,:] = (src[start+b+t,:]-min)/(max-min)
 * sql_pytorch_dataloader.py:239 (normalise) and :8-18,:243-245 (stride-1 windows) */
void bigru_ref_window_gather_norm(const float* src, const float* xmin, const float* xmax,
                                  int64_t start, int B, int T, int F, float* out) {
    for (int b = 0; b < B; ++b)
        for (int t = 0; t < T; ++t)
            for (int f = 0; f < F; ++f) {
                float v = src[(start + b + t) * F + f];
                out[((int64_t)b * T + t) * F + f] = (v - xmin[f]) / (xmax[f] - xmin[f]);
            }
}
