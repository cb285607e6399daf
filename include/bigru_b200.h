/* bigru_b200.h - C ABI of libbigru_b200.so: the H100 (sm_90a) biGRU hot path.
 *
 * The reference (radoslawkrolikowski/financial-market-data-analysis) has no FFI layer of its
 * own: its hot path is the Python class surface of biGRU_model.py / sql_pytorch_dataloader.py,
 * with the arithmetic inside torch.nn.GRU.  Each entry point below names the reference
 * interface (file:line under /root/reference) whose work it replaces.  The Python mirror in
 * financial_market_data_analysis_b200/ binds these with ctypes; INTEGRATION.md shows the stub.
 *
 * Conventions
 *  - plain C types only; every pointer named d_* is a DEVICE pointer owned by the caller; the
 *    library never frees caller memory and keeps no reference to it after the call returns;
 *  - `stream` is a cudaStream_t passed as void*; all calls are asynchronous on that stream and
 *    never synchronise; a plan may be used from one stream at a time;
 *  - a d_* array needs only the alignment of its element type (4 bytes for float and int32): where a kernel has a
 *    vector or bulk-tensor path (the tensor-core GEMMs' staged epilogue, bigru_window_gather_norm) it checks the actual
 *    address and strides and otherwise stores element by element, with bitwise the same results.  The workspaces
 *    (d_stash, d_scratch, d_workspace) hold bf16 planes that TMA reads and must be 16-byte aligned (cudaMalloc: 256);
 *  - every function returns 0 on success, <0 on error (BIGRU_ERR_*); bigru_last_error() returns
 *    a thread-local message.  There is no CPU fallback anywhere: without an sm_90 (H100)
 *    device every compute call fails with BIGRU_ERR_DEVICE.
 *
 * Flat parameter vector ("params", "grads", Adam moments): float32, order
 *     for l in [0,L): for d in [0,D):  w_ih[3H,I_l]  w_hh[3H,H]  b_ih[3H]  b_hh[3H]
 *     lin_w[C,3H]  lin_b[C]                       with I_0 = F, I_l = D*H, gate rows r|z|n
 * i.e. torch.nn.GRU's own per-layer order (state_dict keys gru.weight_ih_l{l}[_reverse] ...,
 * biGRU_model.py:54-60), so the Python side exposes each block as an ordinary nn.Parameter view.
 */
#ifndef BIGRU_B200_H
#define BIGRU_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BIGRU_OK               0
#define BIGRU_ERR_ARG         -1   /* bad shape / null pointer / unsupported combination */
#define BIGRU_ERR_CUDA        -2   /* a CUDA runtime call failed (message has the reason) */
#define BIGRU_ERR_DEVICE      -3   /* no sm_90 (H100) device */
#define BIGRU_ERR_UNSUPPORTED -4   /* shape not supported by the requested precision path */

#define BIGRU_PREC_FP32 0          /* fp32 FFMA path: exact, any shape (<=1e-4 rel on logits) */
#define BIGRU_PREC_BF16 1          /* bf16 operands on tensor cores, fp32 accumulate/state.
                                      hidden_size 128 or 256 with batch % 16 == 0, hidden_size 512 with batch % 32 == 0
                                      (BASELINE.json configs[4]); no initial hidden state */
#define BIGRU_PREC_BF16X3 2        /* fp32-class on tensor cores: (hi, lo) bf16 operand pairs, 3 products per term,
                                      fp32 accumulate / gate math / stash; meets the 1e-4 logit tolerance at tensor-core speed.
                                      hidden_size 128 or 256, batch % 32 == 0.
                                      Both tensor-core paths take any n_features (the layer-0 operands are stored with the
                                      feature extent zero-padded to a multiple of 8 inside the plan's workspaces).  Other
                                      batch sizes: append zero rows to x (and zero rows to d_logits) up to the next multiple -
                                      batch rows are independent; the Python mirror does exactly that.  Smaller hidden sizes:
                                      zero-pad the parameters to the next supported hidden size (padded units stay at state 0 and
                                      feed zero weights; BiGRU.plan_hidden / _Padding of the mirror).  Anything else returns
                                      BIGRU_ERR_UNSUPPORTED. */

#define BIGRU_LOSS_CE   0          /* torch.nn.CrossEntropyLoss (BASELINE.json configs) */
#define BIGRU_LOSS_BCE  1          /* torch.nn.BCEWithLogitsLoss(weight,pos_weight) notebook raw :1192 */
#define BIGRU_LOSS_MLSM 2          /* torch.nn.MultiLabelSoftMarginLoss  predict.py:94 */
/* bigru_loss_param only: */
#define BIGRU_LOSS_CE_WEIGHTED 3   /* torch.nn.CrossEntropyLoss(weight=w) */
#define BIGRU_LOSS_MSE         4   /* torch.nn.MSELoss */
#define BIGRU_LOSS_L1          5   /* torch.nn.L1Loss */
#define BIGRU_LOSS_SMOOTH_L1   6   /* torch.nn.SmoothL1Loss(beta = param) */
#define BIGRU_LOSS_HUBER       7   /* torch.nn.HuberLoss(delta = param) */

typedef struct bigru_plan bigru_plan;

const char* bigru_last_error(void);
int  bigru_version(void);
/* 0 when device `dev` exists and is an sm_90 (H100) device */
int  bigru_device_check(int dev);

/* --- plan: shapes, offsets, workspace sizes.  Replaces BiGRU.__init__ bookkeeping
 *     (biGRU_model.py:32-60).  Immutable after creation. */
int  bigru_plan_create(int B, int T, int F, int H, int L, int C, int bidirectional, int precision,
                       bigru_plan** out);
/* --- recurrent (variational) dropout, Gal & Ghahramani 2016 (DESIGN.md §4.8): the same plans with recurrent_p in [0, 1)
 *  (else BIGRU_ERR_ARG).  recurrent_p = 0 gives exactly the plan of bigru_plan_create / bigru_gru_plan_create.  On a plan with
 *  recurrent_p > 0, a training forward (training != 0: bigru_forward*, bigru_gru_forward) draws, for every layer l and
 *  direction d, a mask m[b][j] in {0, 1/(1-p)} per batch row and hidden unit, the same at every step, and runs each valid
 *  step as h_t = GRUCell(x_t, m * h_{t-1}) (h_{-1} = h0, or 0).  y_t = h_t and h_n are unmasked; a padded step applies no
 *  cell and no mask.  m[b][j] is 0 where bigru_uniform(seed, BIGRU_RD_STREAM + l, (b*D + d)*H + j) < p; input and
 *  inter-layer dropout use the streams l < 16, which never reach BIGRU_RD_STREAM.  The backward must get the forward's seed
 *  and training flag.  Inference (bigru_infer*, bigru_gru_infer) and training = 0 never mask.  The stash grows by the masks
 *  and the masked states (BIGRU_WS_RD_MASK, BIGRU_WS_RD_STATE). */
#define BIGRU_RD_STREAM 65536u
int  bigru_plan_create_rd(int B, int T, int F, int H, int L, int C, int bidirectional, int precision, float recurrent_p,
                          bigru_plan** out);
int  bigru_gru_plan_create_rd(int B, int T, int F, int H, int L, int bidirectional, int precision, float recurrent_p,
                              bigru_plan** out);
int  bigru_plan_destroy(bigru_plan* plan);
int64_t bigru_param_count(const bigru_plan* plan);
/* which: 0 w_ih, 1 w_hh, 2 b_ih, 3 b_hh for layer<L; layer==L: 0 lin_w, 2 lin_b (BIGRU_ERR_ARG on a plan without a head) */
int  bigru_param_offset(const bigru_plan* plan, int layer, int dir, int which,
                        int64_t* offset, int64_t* rows, int64_t* cols);
/* stash: activations kept from forward for backward; scratch: reusable temporary space */
int  bigru_workspace_bytes(const bigru_plan* plan, size_t* stash_bytes, size_t* scratch_bytes);

/* byte offset, inside the stash written by the last forward, of argmax_t of the max-pooled output (int32 [B][H],
 * biGRU_model.py:125).  The max-pool's gradient routing is discontinuous where two time steps tie to within rounding;
 * parity tests read the routing that was actually taken (tests/test_gpu_parity.py). */
int  bigru_stash_argmax_offset(const bigru_plan* plan, size_t* byte_offset);
/* byte offset, inside the same stash, of layer `layer`'s fp32 output Y[B][T][D*H] (the nn.GRU output of that layer, direction
 * d in columns [d*H, d*H+H)); lets tests compare every layer at every time step. */
int  bigru_stash_output_offset(const bigru_plan* plan, int layer, size_t* byte_offset);
/* Test support, like the two offsets above: where an intermediate of the tensor-core forward or backward lives, so that
 * tests can recompute each step and each GEMM from the kernels' own operands.  *in_scratch: 0 stash, 1 scratch;
 * *byte_offset: start of the region (of the hi plane for planes); *lo_byte_offset: the lo plane at BIGRU_PREC_BF16X3,
 * SIZE_MAX otherwise; *pitch: elements per row.  Planes are bf16 in the layout of their fp32 producer.  Rows are b*T + t.
 *   which                   buffer   layer      contents; valid after
 *   BIGRU_WS_GATES          stash    0..L-1     G [D][B*T][4H] fp32: r, z, n, W_hn h_{t-1} + b_hn; bigru_forward
 *   BIGRU_WS_Y_PLANES       stash    0..L-1     planes of Y [B*T][D*H]; bigru_forward
 *   BIGRU_WS_IN_PLANES      stash    0..L-1     planes of the layer's own input [B*T][rup(I_l, 8)], zero-padded columns;
 *                                               bigru_forward, layer 0 always, layers above only in training with dropout
 *   BIGRU_WS_DGI, _DGH      scratch  s          dgi, dgh [D][B*T][3H] fp32 of layer s, the backward stop (0 unless
 *                                               bigru_plan_set_backward_stop set it); bigru_backward (each layer reuses them)
 *   BIGRU_WS_DGI_PLANES,    scratch  s          their planes; dgi's n-gate rows hold dan, the dgh rows are zero at each
 *   BIGRU_WS_DGH_PLANES                         sequence's first step (t = 0 forward, t = T-1 reverse); bigru_backward.
 *                                               With lengths, these and the Y planes are zero at padded steps
 *   BIGRU_WS_DY             scratch  0, 1       upstream gradient of the layer's output [B*T][D*H]; bigru_backward.  The
 *                                               two ping-pong buffers: at a stop s > 0 they hold layers s-1 and s instead
 *   BIGRU_WS_DHC            scratch  s          dh_{-1} of layer s [D][B][H]; bigru_backward
 *   BIGRU_WS_DCAT           scratch  L (head)   d cat [B][3H] (last | max | mean); bigru_backward
 *   BIGRU_WS_RD_MASK        stash    0..L-1     recurrent-dropout masks m [D][B][H] fp32; training bigru_forward, plans with
 *                                               recurrent_p > 0 only
 *   BIGRU_WS_RD_STATE       stash    0..L-1     the masked state m * h_t [B*T][D*H] (0 at padded steps): planes at the
 *                                               tensor-core precisions, fp32 at BIGRU_PREC_FP32; as BIGRU_WS_RD_MASK
 * Planes at BIGRU_PREC_FP32: BIGRU_ERR_UNSUPPORTED.  Another layer or an unknown `which`: BIGRU_ERR_ARG. */
#define BIGRU_WS_GATES       0
#define BIGRU_WS_Y_PLANES    1
#define BIGRU_WS_IN_PLANES   2
#define BIGRU_WS_DGI         3
#define BIGRU_WS_DGH         4
#define BIGRU_WS_DGI_PLANES  5
#define BIGRU_WS_DGH_PLANES  6
#define BIGRU_WS_DY          7
#define BIGRU_WS_DHC         8
#define BIGRU_WS_DCAT        9
#define BIGRU_WS_RD_MASK    10
#define BIGRU_WS_RD_STATE   11
#define BIGRU_WS_COUNT      12
int  bigru_workspace_region(const bigru_plan* plan, int which, int layer, int* in_scratch, size_t* byte_offset,
                            size_t* lo_byte_offset, int64_t* pitch);

/* --- Backward stop (test support): every later backward call on the plan (bigru_backward*, bigru_gru_backward) runs the
 *  head and layers L-1 .. layer, then returns, so that the scratch regions above hold layer `layer`'s intermediates.
 *  d_grads is still zeroed first: the gradients of the layers below stay 0, and d_dx and their d_dh0 slices are not
 *  written.  Plans start at 0, the whole backward.  A null plan or a layer outside [0, L): BIGRU_ERR_ARG. */
int  bigru_plan_set_backward_stop(bigru_plan* plan, int layer);

/* --- Recurrence scan geometry of a tensor-core plan on the current device (test support).  *R: clusters of the scan the
 *  device holds at once.  scan 0, the forward (training instantiation): *n_split = clusters that take two 16-row batch
 *  tiles (the lowest cluster ids; always 0 at BIGRU_PREC_BF16).  scan 1, the backward: *n_split = batch tiles of the last
 *  round split into two 8-row clusters each (the highest cluster ids).  No result depends on them.  On a plan with
 *  recurrent_p > 0 both describe the recurrent-dropout scans, which that plan's training calls launch.
 *  BIGRU_PREC_FP32: BIGRU_ERR_UNSUPPORTED; another scan: BIGRU_ERR_ARG. */
int  bigru_scan_geometry(const bigru_plan* plan, int scan, int* R, int* n_split);

/* --- One tensor-core GEMM job (test support): the persistent wgmma GEMM every projection and gradient of the tensor-core
 *  plans runs, on the caller's fp32 operands, through the same host code as the plans' jobs.
 *      C[z][m][n] (+)= sum_k A[z][m][k] * B[z][n][k] (+ d_bias[z * z_bias + n]),   z < batch, m < M, n < N, k < K
 *  precision BIGRU_PREC_BF16 or BIGRU_PREC_BF16X3 (operands split into bf16 hi, and lo, as the plans split them; fp32
 *  accumulation).  mn_major 0: d_a [batch][M][K], d_b [batch][N][K], packed into K-major planes (as the head's operands);
 *  mn_major 1: d_a [batch][K][M], d_b [batch][K][N], MN-major planes (as the weight gradients' operands).  C element
 *  (z, m, n) is d_c[z * z_c + m * ldc + n]; beta != 0 adds to it.  d_bias nullable.  splits: split-K count, 0 = the plans'
 *  own rule for the shape.  *staged: 1 when the output tile went out through shared memory and bulk tensor stores, 0
 *  when it was stored element by element; the library decides it as for every plan job, from beta and the alignment of
 *  the output (C, or with splits > 1 the partials in d_workspace): base, ldc and z_c multiples of 16 bytes and N of 4 (a
 *  row ending inside a 16-byte chunk is stored element by element).  d_workspace:
 *  bigru_tc_gemm_workspace_bytes bytes, 16-byte aligned.  BIGRU_ERR_ARG, before any device work: an unknown precision or
 *  mn_major, M, N, K or batch < 1, a null operand, ldc < N, z_c < (M-1)*ldc + N when batch > 1, z_bias < 0, a split
 *  count that leaves a split empty, and a bias with more than one split (split-K has no bias). */
int  bigru_tc_gemm_workspace_bytes(int precision, int mn_major, int M, int N, int K, int batch, int splits, size_t* bytes);
int  bigru_tc_gemm(int precision, int mn_major, int M, int N, int K, int batch, const float* d_a, const float* d_b,
                   const float* d_bias, int64_t z_bias, float* d_c, int64_t ldc, int64_t z_c, int beta, int splits,
                   void* d_workspace, int* staged, void* stream);

/* --- BiGRU.forward (biGRU_model.py:63-138): dropout :87-94, nn.GRU :102, head :111-137.
 *  d_x[B,T,F]; d_h0 nullable [L*D,B,H] (the `hidden` argument); d_logits[B,C];
 *  d_hn nullable [L*D,B,H]; training!=0 applies dropout p (spatial!=0: per (b,f) channel over T,
 *  :87-92; inter-layer dropout when L>1, :55) with a counter-based generator keyed by `seed`. */
int  bigru_forward(const bigru_plan* plan, const float* d_params, const float* d_x, const float* d_h0,
                   float dropout_p, int spatial, int training, uint64_t seed,
                   void* d_stash, void* d_scratch, float* d_logits, float* d_hn, void* stream);

/* --- eval-mode BiGRU.forward (no dropout, nothing kept for a backward): logits of the plan's batch (evaluate_model,
 *  biGRU_model.py:227-286).  Same plans, precisions, shape rules and d_h0 rules as bigru_forward (d_h0 at BIGRU_PREC_BF16:
 *  BIGRU_ERR_UNSUPPORTED), and bit-identical logits: the same launch sequence and kernels, with the scans writing only what
 *  the next layer and the head read.  d_workspace: bigru_infer_workspace_bytes(plan) bytes; neither the stash nor the
 *  scratch of bigru_forward is used.  At configs[1] bf16x3 (B512 T128 F64 H256 L2) that is about 0.69 GB against
 *  1915 + 2329 MB of stash + scratch. */
int  bigru_infer_workspace_bytes(const bigru_plan* plan, size_t* bytes);
int  bigru_infer(const bigru_plan* plan, const float* d_params, const float* d_x, const float* d_h0,
                 void* d_workspace, float* d_logits, void* stream);

/* --- per-sequence lengths (torch.nn.utils.rnn.pack_padded_sequence semantics) for bigru_forward, bigru_infer and
 *  bigru_backward: the same arguments plus d_lengths, a DEVICE int32 [B] or NULL (every row T steps long; then each call is
 *  exactly its twin without lengths).  Row b's valid steps are t < d_lengths[b], with 1 <= d_lengths[b] <= T; its inputs at
 *  t >= d_lengths[b] are ignored (any finite values).  Every layer runs as nn.GRU on the packed sequence: layer outputs are
 *  0 at padded steps, the reverse direction starts from the zero state at t = len - 1, d_hn holds the state after each
 *  direction's last valid step; the head takes `last` at t = len - 1 (forward direction) and t = 0 (reverse), and max- and
 *  mean-pools over t < len.  The backward is the gradient of that function: d_dx is 0 at padded steps.  A backward must get
 *  the d_lengths of its forward.  The library does not read d_lengths on the host: the caller guarantees the range (the
 *  Python mirror checks it).  d_lengths together with d_h0 or d_dh0: BIGRU_ERR_UNSUPPORTED. */
int  bigru_forward_lengths(const bigru_plan* plan, const float* d_params, const float* d_x, const float* d_h0,
                           float dropout_p, int spatial, int training, uint64_t seed,
                           void* d_stash, void* d_scratch, float* d_logits, float* d_hn, const int32_t* d_lengths,
                           void* stream);
int  bigru_infer_lengths(const bigru_plan* plan, const float* d_params, const float* d_x, const float* d_h0,
                         void* d_workspace, float* d_logits, const int32_t* d_lengths, void* stream);
int  bigru_backward_lengths(const bigru_plan* plan, const float* d_params, const float* d_x, const float* d_h0,
                            float dropout_p, int spatial, int training, uint64_t seed,
                            const void* d_stash, void* d_scratch, const float* d_dlogits,
                            float* d_grads, float* d_dx, float* d_dh0, const int32_t* d_lengths, void* stream);

/* --- loss.backward() through the model (biGRU_model.py:204): every parameter gradient into
 *  d_grads (flat, overwritten), optional d_dx[B,T,F] and d_dh0[L*D,B,H].  d_x (required) is the
 *  input the forward read.  Must follow bigru_forward on the same plan/stash with the same dropout arguments. */
int  bigru_backward(const bigru_plan* plan, const float* d_params, const float* d_x, const float* d_h0,
                    float dropout_p, int spatial, int training, uint64_t seed,
                    const void* d_stash, void* d_scratch, const float* d_dlogits,
                    float* d_grads, float* d_dx, float* d_dh0, void* stream);

/* --- torch.nn.GRU on the same kernels: a plan without the pooling head (C = 0), for any head or model built on a GRU
 *  encoder (biGRU_model.py:102 `self.gru(input_seq, hidden)`).  Shapes and precisions follow bigru_plan_create.  Its
 *  parameter vector is the recurrent prefix of the flat order above (nn.GRU's own parameters, order and count; no lin_w,
 *  lin_b); bigru_param_offset(layer == L): BIGRU_ERR_ARG.  Workspace sizes come from bigru_workspace_bytes and
 *  bigru_infer_workspace_bytes of this plan.  The BiGRU entry points (bigru_forward*, bigru_infer*, bigru_backward*,
 *  bigru_stash_argmax_offset, BIGRU_WS_DCAT) refuse such a plan with BIGRU_ERR_ARG, and the bigru_gru_* entry points refuse a
 *  plan with a head the same way.  The top layer's output lives in the caller's d_y, not in the stash:
 *  bigru_stash_output_offset(L-1) and BIGRU_WS_DY of layer L-1 are BIGRU_ERR_ARG.  d_lengths, d_h0 / d_dh0 rules and
 *  BIGRU_ERR_UNSUPPORTED cases are those of the *_lengths entry points above. */
int  bigru_gru_plan_create(int B, int T, int F, int H, int L, int bidirectional, int precision, bigru_plan** out);
/*  Training forward: d_y[B][T][D*H] (required) gets the top layer's output (direction d in columns [d*H, d*H+H), 0 at padded
 *  steps), d_hn [L*D][B][H] (nullable) the final state of every layer and direction.  training != 0 with dropout_p > 0 drops
 *  each layer's output except the last's, elementwise, as nn.GRU(dropout=p) does; x is never dropped.  The masks come from
 *  the generator keyed by (seed, layer) that bigru_forward uses, so for layers above 0 they are BiGRU's inter-layer masks. */
int  bigru_gru_forward(const bigru_plan* plan, const float* d_params, const float* d_x, const float* d_h0,
                       float dropout_p, int training, uint64_t seed, void* d_stash, void* d_scratch, float* d_y,
                       float* d_hn, const int32_t* d_lengths, void* stream);
/*  Eval forward on bigru_infer_workspace_bytes(plan) bytes of d_workspace; d_y and d_hn bit-identical to bigru_gru_forward
 *  with training = 0 (the same launch sequence and kernels, as for bigru_infer). */
int  bigru_gru_infer(const bigru_plan* plan, const float* d_params, const float* d_x, const float* d_h0,
                     void* d_workspace, float* d_y, float* d_hn, const int32_t* d_lengths, void* stream);
/*  Backward of the last bigru_gru_forward on this plan and stash, with the same arguments and lengths.  d_y: that forward's
 *  output (read where the top layer's h_{t-1} is needed).  d_dy [B][T][D*H] (required): the gradient of d_y, ignored at
 *  padded steps.  d_dhn [L*D][B][H] (nullable: zero): the gradient of h_n; layer l's slice seeds that layer's dh carry.
 *  Outputs: d_grads (the plan's parameter vector, overwritten), d_dx [B][T][F] and d_dh0 [L*D][B][H] (both nullable). */
int  bigru_gru_backward(const bigru_plan* plan, const float* d_params, const float* d_x, const float* d_h0,
                        float dropout_p, int training, uint64_t seed, const void* d_stash, void* d_scratch,
                        const float* d_y, const float* d_dy, const float* d_dhn, float* d_grads, float* d_dx,
                        float* d_dh0, const int32_t* d_lengths, void* stream);

/* --- torch.nn.GRUCell: one step h' = GRUCell(x, h), for loops that advance a step at a time (a decoder over a GRU encoder,
 *  one step per new bar in a live path).  No plan: a cell keeps no per-shape state.  d_params is nn.GRUCell's vector
 *  w_ih[3H,I] w_hh[3H,H] b_ih[3H] b_hh[3H], the layer-0, direction-0 block of the flat order above (a GRU(I, H, 1)'s vector);
 *  d_x [B][I], d_h and d_hout [B][H] (d_hout must not overlap an input).  Every precision takes every shape 1 <= B <= 32768,
 *  1 <= I, H <= 65536 (beyond: BIGRU_ERR_UNSUPPORTED), d_h included at BIGRU_PREC_BF16; ragged edges are handled inside the
 *  kernels, nothing is padded.  Operands are split into bf16 (hi, and lo at BIGRU_PREC_BF16X3) where the kernels load them; state,
 *  gate math and outputs are fp32.  A row's bits depend neither on B, nor on the row's position, nor on d_stash.
 *  Workspaces (bytes, every precision): stash B*4H*4 (G [B][4H] = r, z, n, W_hn h + b_hn), scratch 2*B*3H*4 (dgi, dgh). */
int  bigru_cell_workspace_bytes(int B, int I, int H, int precision, size_t* stash_bytes, size_t* scratch_bytes);
/*  One launch.  d_h nullable: the zero state.  d_stash nullable: inference (nothing kept for a backward). */
int  bigru_cell_forward(int B, int I, int H, int precision, const float* d_params, const float* d_x, const float* d_h,
                        float* d_hout, void* d_stash, void* stream);
/*  Backward of a bigru_cell_forward with the same shapes, precision, d_params, d_x and d_h whose stash was kept.  d_dhout [B][H]:
 *  the gradient of d_hout.  d_grads (parameter vector) is overwritten, each element written once, in a fixed order (bitwise
 *  reproducible); d_dx [B][I] and d_dh [B][H] nullable.  Three launches, two when both are null. */
int  bigru_cell_backward(int B, int I, int H, int precision, const float* d_params, const float* d_x, const float* d_h,
                         const void* d_stash, const float* d_dhout, float* d_grads, float* d_dx, float* d_dh, void* d_scratch,
                         void* stream);

/* --- losses (biGRU_model.py:202 `self.loss_fn(pred, target)`), fused value + d(loss)/d(logits).
 *  kind CE: d_target int64[B]; BCE/MLSM: d_target float[B,C]; d_weight/d_pos_weight nullable [C]
 *  (BCE only).  Mean reduction over `denom` elements (B for CE, B*C otherwise; pass the GLOBAL
 *  count under data parallelism).  d_loss: one float, overwritten.  CE needs every target in [0, C): it does not
 *  implement nn.CrossEntropyLoss's ignore_index, and a row whose target lies outside [0, C) (ignore_index = -100
 *  included) is not read through but makes the loss and that row's dlogits NaN. */
int  bigru_loss(int kind, const float* d_logits, const void* d_target, const float* d_weight,
                const float* d_pos_weight, int B, int C, double denom, float* d_loss,
                float* d_dlogits, void* stream);
/*  bigru_loss_param: every kind above, with the scalar `param` of the kinds that have one (SmoothL1's beta >= 0,
 *  Huber's delta > 0; ignored otherwise).  Kinds 0-2 compute bitwise what bigru_loss computes (which calls this).
 *  CE_WEIGHTED: d_target int64[B] as CE, d_weight [C] required; loss = sum_b w[y_b] nll_b / (W * denom) with
 *  W = sum_b w[y_b] formed in the same launch in a fixed order, i.e. torch's weighted mean when denom = 1.  Under data
 *  parallelism pass denom = world size: the all-reduced sum is then the mean over ranks of each rank's weighted mean.
 *  W = 0 (every target weight zero) gives a NaN loss and NaN dlogits, as torch does.  Targets outside [0, C) as CE.
 *  MSE / L1 / SMOOTH_L1 / HUBER: d_target float[B,C], mean over denom (B*C, times the world size under data
 *  parallelism), d_weight / d_pos_weight ignored.  The gradient at the kinks is torch's: L1 gives 0 where x == y,
 *  SmoothL1 with beta = 0 is L1, and at |x - y| == beta (delta) both take the quadratic side's value. */
int  bigru_loss_param(int kind, const float* d_logits, const void* d_target, const float* d_weight,
                      const float* d_pos_weight, int B, int C, double denom, float param, float* d_loss,
                      float* d_dlogits, void* stream);

/* --- nn.utils.clip_grad_norm_ + optimizer.step() (biGRU_model.py:208-210, Adam, notebook raw :1194)
 *  bigru_sqnorm accumulates sum(g^2) into *d_out (caller zeroes it first); d_ws: BIGRU_SQNORM_WS floats of
 *  device scratch for the per-block partial sums, which are added in a fixed order (bit-reproducible).
 *  Adam's step count lives in device memory, so that the train step can be captured in a CUDA graph (SURVEY.md 8(f) N5):
 *  bigru_adam_tick: *d_step += 1, *d_sqnorm = 0 (one tiny launch, before bigru_sqnorm);
 *  bigru_clip_adam_step_dev: g *= grad_scale; coef = min(1, clip/(sqrt(*d_sqnorm)*grad_scale+1e-6));
 *  g *= coef; Adam(lr,b1,b2,eps) with bias correction for step *d_step (1-based). */
#define BIGRU_SQNORM_WS 528
int  bigru_sqnorm(const float* d_g, int64_t n, float* d_out, float* d_ws, void* stream);
int  bigru_adam_tick(int* d_step, float* d_sqnorm, void* stream);
int  bigru_clip_adam_step_dev(float* d_params, float* d_grads, float* d_m, float* d_v, int64_t n,
                              const float* d_sqnorm, float clip, float lr, float b1, float b2, float eps,
                              const int* d_step, float grad_scale, void* stream);

/* --- the same clip + update with its hyperparameters in device memory, one set per parameter group
 *  (torch.optim.Adam / AdamW param_groups), so that a captured CUDA graph of the step follows a learning-rate schedule.
 *  d_groups [n_groups] (1 <= n_groups <= BIGRU_ADAM_MAX_GROUPS); d_segments [n_segments] (>= 1): ranges of the flat
 *  vector sorted by offset and disjoint, each updated with the hyperparameters of its group.  An element outside every
 *  segment, or in a segment whose group is outside [0, n_groups), is left as it is (p, g, m and v).  Per element,
 *  after the clip of bigru_clip_adam_step_dev:
 *    weight_decay != 0 and decoupled (AdamW):  p *= 1 - lr * weight_decay   (formed in double), then Adam on g;
 *    weight_decay != 0, not decoupled (Adam):  Adam on g + weight_decay * p  (g itself keeps the clipped gradient);
 *  and the Adam update and bias corrections of bigru_clip_adam_step_dev.  bigru_clip_adam_step_dev is this update with
 *  one group (lr, b1, b2, eps, no weight decay) and one segment [0, n).  No atomics, each element written once. */
#define BIGRU_ADAM_MAX_GROUPS 64
typedef struct { float lr, beta1, beta2, eps, weight_decay, decoupled; } bigru_adam_group;  /* decoupled: 0 or 1 */
typedef struct { int64_t offset, count, group; } bigru_adam_segment;
int  bigru_clip_adam_groups_dev(float* d_params, float* d_grads, float* d_m, float* d_v, int64_t n,
                                const float* d_sqnorm, float clip, const bigru_adam_group* d_groups, int n_groups,
                                const bigru_adam_segment* d_segments, int n_segments, const int* d_step,
                                float grad_scale, void* stream);

/* --- MySQLBatchLoader collation (sql_pytorch_dataloader.py:239-245 + default_collate):
 *  out[b,t,f] = (s - xmin[f]) / (xmax[f] - xmin[f]), an IEEE float division, with s = src[start+b+t, f] and a NaN s
 *  (SQL NULL) read as 0, the IFNULL(field, 0) of the SQL path;  src is [N,F], start+B+T-1 <= N.
 *  xmin/xmax nullable together (then a plain gather, NaN still read as 0).  B = 0 writes nothing.
 *  targets: out[b,0,c] = y[start+b+T-1, c]. */
int  bigru_window_gather_norm(const float* d_src, const float* d_xmin, const float* d_xmax,
                              int64_t start, int64_t N, int B, int T, int F, float* d_out, void* stream);
int  bigru_window_targets(const float* d_y, int64_t start, int64_t N, int B, int T, int C,
                          float* d_out, void* stream);

/* --- SURVEY.md 8(f) N3, chunk statistics on the GPU: per-feature MIN / MAX over rows [row_lo, row_hi) of a
 *  table[N,F] (NaN = SQL NULL, ignored), i.e. the two aggregate queries of MySQLChunkLoader
 *  (sql_pytorch_dataloader.py:96-105).  A column with no non-NaN value in the range gets min = +inf, max = -inf
 *  (SQL would give NULL).  The min==max guard and order-book sharing stay on the host. */
int  bigru_chunk_minmax(const float* d_table, int64_t N, int F, int64_t row_lo, int64_t row_hi, float* d_min,
                        float* d_max, void* stream);

/* --- SURVEY.md 8(f) N4, the SQL window-function features of the reference (create_database.py:76-190) over the joined
 *  table's columns (device pointers, n rows, time order): per row, in the order of the reference's join statement
 *  (create_database.py:239-240): [upper_BB_dist, lower_BB_dist] (bb_period > 0; STD is the population std), vol_MA{p},
 *  price_MA{p}, delta_MA{p} (AVG over ROWS BETWEEN p-1 PRECEDING AND CURRENT ROW, shorter at the head of the table),
 *  [stoch] (15-row MIN / MAX of close; NaN = SQL NULL when max == min), ATR (15-row AVG(high - low)), price_change
 *  (close - LAG(close, 1); NaN on the first row) -> d_out[n][n_out]; and the four targets up1, up2, down1, down2
 *  (create_database.py:163-185: LEAD(close, 8 / 15) against close +- n1 / n2 * ATR, 0 where the lead is NULL)
 *  -> d_targets[n][4] (nullable), decided as the SQL decides them in double, ties included.  n1 and n2 are fp32: the
 *  reference's 1.5 and 3 are exact, other factors are rounded to fp32 first.  At most 8 periods per list.  Returns n_out through *n_out (pass d_out = NULL to query). */
int  bigru_window_features(const float* d_close, const float* d_high, const float* d_low, const float* d_volume,
                           const float* d_delta, int64_t n, const int* vol_periods, int n_vol, const int* price_periods,
                           int n_price, const int* delta_periods, int n_delta, int bb_period, float bb_std,
                           int stochastic, float n1, float n2, float* d_out, float* d_targets, int* n_out, void* stream);

/* --- SURVEY.md 8(f) N5, the live predictor's forward pass in one launch (predict.py:165-181): normalise the raw
 *  window(s) d_x[B,T,F] with d_xmin/d_xmax[F] (nullable: already normalised), eval-mode forward of the flat parameters
 *  (order above), d_logits[B,C] and d_probs[B,C] = sigmoid(logits) (nullable).  One CTA per window, activations in shared
 *  memory, fp32 exact math; for small live windows only: D*H <= 1024 and T*(max(F,D*H)+D*H)*4 bytes of shared memory
 *  (BIGRU_ERR_UNSUPPORTED beyond) - batches belong to bigru_forward. */
int  bigru_infer_window(const float* d_params, const float* d_x, const float* d_xmin, const float* d_xmax, int B, int T,
                        int F, int H, int L, int C, int bidirectional, float* d_logits, float* d_probs, void* stream);

/* --- train_model/evaluate_model metrics (biGRU_model.py:213-221): pred = sigmoid(logit) > 0.5 with the sigmoid
 *  evaluated in fp32 as torch.sigmoid does (false for positive logits below about 1e-7, where it rounds to 0.5);
 *  true = target > 0.5;
 *  d_counts[0] += #rows with all labels right; [1] += #label mismatches;
 *  [2+3c], [3+3c], [4+3c] += tp, fp, fn of class c.  int64 accumulators, caller zeroes. */
int  bigru_multilabel_counts(const float* d_logits, const float* d_target, int B, int C,
                             long long* d_counts, void* stream);

/* --- measurement hooks used by bench.py (no reference counterpart).
 *  bigru_launch_count: kernels launched by this library since load (gpu_launches).
 *  bigru_prof_enable(1): every subsequent launch is bracketed by CUDA events on its own stream;
 *  bigru_prof_report(cls): summed device time, launch count, algorithmic flops and bytes of one
 *  kernel class (names via bigru_prof_class_name) since the last enable.  Timing adds event records
 *  to the stream, so bench.py enables it only for a separate, untimed-for-throughput pass. */
long long   bigru_launch_count(void);
void        bigru_launch_count_add(long long n);   /* launches replayed from a captured CUDA graph (not seen by the macros) */
int         bigru_prof_enable(int on);
int         bigru_prof_classes(void);
const char* bigru_prof_class_name(int cls);
int         bigru_prof_report(int cls, double* ms, long long* launches, double* flops, double* bytes);

#ifdef __cplusplus
}
#endif
#endif
