/*
 * ta3n_b200.h -- C ABI of libta3n_sm90.so: the H100 (sm_90a) implementation of the
 * TA3N hot path (TRN-M relation aggregation + domain-attentive pooling + gradient-reversal
 * discriminators inside VideoModel.forward of cmhungsteve/TA3N).
 *
 * The reference has no FFI: its "operator interface" for this path is the set of Python
 * methods of models.py / TRNmodule.py that call ATen.  Each entry point below replaces one
 * of those methods (cited as file:line, paths relative to the reference root) and is what a
 * ctypes / pybind stub in the reference would bind (see INTEGRATION.md).
 *
 * Conventions
 *   - every tensor is fp32, row-major, contiguous unless a leading dimension is given;
 *     all pointers are DEVICE pointers unless the name ends in _host;
 *   - weights use the nn.Linear layout [out_features, in_features];
 *   - the library allocates nothing and never synchronises: the caller passes outputs,
 *     saved-for-backward buffers and a workspace (sizes from the *_workspace_bytes queries);
 *     every call enqueues work on `stream` (a cudaStream_t) of the current device and is
 *     CUDA-graph capturable;
 *   - return value: 0 on success, a TA3N_ERR_* code otherwise (never throws/aborts);
 *     ta3n_last_error() gives a thread-local message;
 *   - "rows" M is the number of videos (source rows first, then target rows: weights are
 *     shared between domains -- models.py:565-566 with share_params='Y' -- and no op on the
 *     path mixes rows, so both domains go through one launch).
 */
#ifndef TA3N_B200_H_
#define TA3N_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TA3N_ABI_VERSION 5

enum {
  TA3N_OK = 0,
  TA3N_ERR_INVALID = 1,   /* bad argument (null pointer, unsupported size)           */
  TA3N_ERR_WORKSPACE = 2, /* workspace too small                                      */
  TA3N_ERR_CUDA = 3,      /* a CUDA runtime / driver call failed                      */
  TA3N_ERR_UNSUPPORTED = 4
};

/* GEMM engines for the dense contractions. */
enum {
  TA3N_GEMM_FP32_SIMT = 0,   /* exact fp32 FFMA tiles (parity / debugging engine)     */
  TA3N_GEMM_TF32_TCGEN05 = 1,/* wgmma tf32, TMA-staged, register accumulators: fastest, forward ~3e-4      */
  TA3N_GEMM_TF32X3_TCGEN05 = 2 /* the default: the same engine with every FORWARD layer at fp32 grade (operands split
                                  in two tf32 pieces, three products per K step, K accumulated in chunks of 256), so that
                                  no ReLU unit changes state against the fp32 reference; backward GEMMs as engine 1  */
};

typedef void* ta3n_stream_t; /* cudaStream_t */

/* Relation table of RelationModuleMultiScale (TRNmodule.py:30-41, 66-71), host arrays:
 *   n_scales            = T-1 (scale i uses scale_size[i] = T-i frames)
 *   rel_count[i]        = relations evaluated for scale i (1 for i==0, else min(3, C(T,s)))
 *   frames              = concatenation over scales i, relations r, of scale_size[i] frame ids
 */
typedef struct {
  int num_frames;           /* T */
  int n_scales;             /* R = T-1 */
  const int* scale_size;    /* [n_scales] host */
  const int* rel_count;     /* [n_scales] host */
  const int* frames;        /* [sum_i rel_count[i]*scale_size[i]] host */
} ta3n_relation_table;

/* Dropout control.  keep==NULL and p>0 -> counter-based in-kernel RNG keyed by
 * (seed, *step_dev) (step_dev may be NULL); keep!=NULL -> caller-provided 0/1 keep mask
 * (uint8, same shape as the tensor it masks).  p<=0 -> no dropout.                       */
typedef struct {
  float p;
  const uint8_t* keep;
  uint64_t seed;
  const uint64_t* step_dev;
} ta3n_dropout;

/* ---- library state ---------------------------------------------------------------- */
int ta3n_abi_version(void);
const char* ta3n_last_error(void);
/* number of kernels this library has launched since load / last reset (all threads) */
uint64_t ta3n_launch_count(void);
void ta3n_reset_launch_count(void);
/* select the GEMM engine used by subsequent calls (process-wide). */
int ta3n_set_gemm_engine(int engine);
int ta3n_get_gemm_engine(void);
/* Optional device scratch (caller-owned, 256-byte aligned; NULL / 0 removes it) for the calling THREAD's forward
 * launches under the tf32x3 engine: with it the precise kernel balances its one-CTA-per-SM grid by splitting K
 * (deterministic partials + fixed-order reduce).  The forward entry points take no workspace argument, hence this
 * registration; the launches that use it are stream-ordered, so one buffer serves them all.  48 MB cover cfg5.      */
int ta3n_set_forward_scratch(void* scratch, size_t bytes);
/* Host-only (no CUDA call): the split-K factors that balancing would choose for one precise forward launch of
 * n_groups GEMMs C[M,N] = A[M,K] B[N,K]^T on `sms` SMs with scratch_bytes of forward scratch -> ksplit_out[n_groups];
 * makespan_out (optional, 2 doubles) = {unsplit, chosen} longest per-SM queue of the planner's model, in K-slab units. */
int ta3n_plan_forward_splits(int n_groups, const int* M, const int* N, const int* K, int sms, size_t scratch_bytes,
                             int* ksplit_out, double* makespan_out);
/* Per-call-site device timing (CUDA events on the launching stream, eager mode only; not for use
 * under graph capture).  ta3n_timing_report synchronises the recorded events, writes lines
 * "label count total_ms\n" to buf, clears the registry and returns the bytes needed.           */
void ta3n_timing_enable(int on);
size_t ta3n_timing_report(char* buf, size_t buf_bytes);

/* ---- shared frame layer: Dropout(ReLU(x W^T + b))  (models.py:565-575) ------------- */
/* x_src [rows_src, D], x_tgt [rows_tgt, D] (rows = videos*T); feat [rows_src+rows_tgt, F] */
int ta3n_shared_fc_fwd(const float* x_src, int rows_src, const float* x_tgt, int rows_tgt, int D,
                       const float* W, const float* b, int F, const ta3n_dropout* drop,
                       float* feat, ta3n_stream_t stream);
size_t ta3n_shared_fc_bwd_workspace_bytes(int rows, int D, int F);
/* dfeat [rows, F] is consumed (overwritten with d pre-activation). Inputs carry no grad
 * (SURVEY 3.3) so only dW [F, D], db [F] are produced.                                   */
int ta3n_shared_fc_bwd(const float* x_src, int rows_src, const float* x_tgt, int rows_tgt, int D,
                       int F, const float* feat, float* dfeat, const float* g_feat_ext, float p,
                       float* dW, float* db, void* workspace, size_t workspace_bytes,
                       ta3n_stream_t stream);

/* ---- GradReverse + two-layer domain discriminator ---------------------------------- */
/* models.py:456-462 (frame level), :464-470 (video level):
 *   logits = W2 relu(W1 GRL_beta(x) + b1) + b2,  x [rows, K], W1 [Kh, K], W2 [2, Kh]     */
int ta3n_disc_fwd(const float* x, int rows, int K, int Kh, const float* W1, const float* b1,
                  const float* W2, const float* b2, float* hidden, float* logits,
                  ta3n_stream_t stream);
size_t ta3n_disc_bwd_workspace_bytes(int rows, int K, int Kh);
/* dx += -beta * dgrad (accumulate!=0) or dx = -beta * dgrad;  dx may be NULL.            */
int ta3n_disc_bwd(const float* x, int rows, int K, int Kh, const float* W1, const float* W2,
                  const float* hidden, const float* g_logits, float beta, float* dx,
                  int accumulate, float* dW1, float* db1, float* dW2, float* db2,
                  void* workspace, size_t workspace_bytes, ta3n_stream_t stream);
/* stand-alone gradient reversal backward, models.py:27-29: out = -beta * g               */
int ta3n_grl_bwd(const float* g, float beta, float* out, size_t n, ta3n_stream_t stream);

/* ---- frame-level transferable attention (models.py:368-377, use_attn_frame) -------- */
/* w = 1 - H(softmax(logits)); out = (w + 1) * feat;  logits [rows,2], feat [rows,F]      */
int ta3n_frame_attn_fwd(const float* feat, const float* logits, int rows, int F, float* out,
                        ta3n_stream_t stream);
/* d_out [rows,F] is rewritten in place with d feat; g_logits [rows,2] += d w * dw/dlogits */
int ta3n_frame_attn_bwd(const float* feat, const float* logits, int rows, int F, float* d_out,
                        float* g_logits, ta3n_stream_t stream);

/* ---- average over the segments (frame_aggregation='avgpool', models.py:425-433) ---- */
/* x [M,T,F] -> out [M,F] = sum_t x / T (nn.AvgPool2d([T, 1]));  backward: g [M,F] -> dx [M,T,F] = g / T        */
int ta3n_segment_mean_fwd(const float* x, int M, int T, int F, float* out, ta3n_stream_t stream);
int ta3n_segment_mean_bwd(const float* g, int M, int T, int F, float* dx, ta3n_stream_t stream);

/* ---- multi-scale temporal relation module (TRNmodule.py:58-82) --------------------- */
/* x [M, T, F];  W_host[i] -> device [H, scale_size[i]*F];  b_host[i] -> device [H]
 * act [n_rel_total, M, H] : relu'd relation activations (saved for backward)
 * feat_rel [M, R, H]      : per-scale sums (the module output)
 * relu_input != 0 applies the leading nn.ReLU of fc_fusion (TRNmodule.py:49) to x; callers
 * that know x >= 0 (inside VideoModel: post-ReLU/dropout features) may pass 0.           */
int ta3n_trn_fwd(const float* x, int M, int F, int H, const ta3n_relation_table* tab,
                 const float* const* W_host, const float* const* b_host, int relu_input,
                 float* act, float* feat_rel, ta3n_stream_t stream);
size_t ta3n_trn_bwd_workspace_bytes(int M, int F, int H, const ta3n_relation_table* tab);
/* d_feat_rel [M,R,H] -> dW_host[i] [H, s_i F], db_host[i] [H], dx [M,T,F] (dx may be NULL);
 * accumulate_dx != 0: dx += ... (lets an independent branch, e.g. the frame discriminator, write dx first) */
int ta3n_trn_bwd(const float* x, int M, int F, int H, const ta3n_relation_table* tab,
                 const float* const* W_host, int relu_input, const float* act,
                 const float* d_feat_rel, float* const* dW_host, float* const* db_host, float* dx,
                 int accumulate_dx, void* workspace, size_t workspace_bytes, ta3n_stream_t stream);

/* ---- relation discriminators + domain attention + pooling -------------------------- */
/* models.py:472-488 (per-relation GRL + MLP), :351-357 (entropy attention), :379-388
 * (re-weighting), :651-652 (sum over relations).
 *   feat_rel [M,R,H]; W1_host[i] [H,H], b1_host[i] [H], W2_host[i] [2,H], b2_host[i] [2]
 *   hidden [R,M,H] (saved), pred_rel [M,R,2], attn [M,R], feat_video [M,H]
 * use_attn == 0 reproduces use_attn='none' (:647): plain sum, attn = feat_rel[:,:,0].    */
int ta3n_relattn_fwd(const float* feat_rel, int M, int R, int H, const float* const* W1_host,
                     const float* const* b1_host, const float* const* W2_host,
                     const float* const* b2_host, int use_attn, float* hidden, float* pred_rel,
                     float* attn, float* feat_video, ta3n_stream_t stream);
size_t ta3n_relattn_bwd_workspace_bytes(int M, int R, int H);
/* g_feat_video [M,H], g_pred_rel [M,R,2] (may be NULL), g_attn [M,R] (may be NULL)
 * -> d_feat_rel [M,R,H] and the discriminator gradients; beta = beta[0].
 * use_attn == 2: the weights in attn [M,R] were produced by ta3n_general_attn_fwd: G is scaled by (attn + 1) as for
 * TransAttn, but no gradient flows from the weights into pred_rel (g_attn is ignored; ta3n_general_attn_bwd owns it). */
int ta3n_relattn_bwd(const float* feat_rel, int M, int R, int H, const float* const* W1_host,
                     const float* const* W2_host, int use_attn, const float* hidden,
                     const float* pred_rel, const float* attn, const float* g_feat_video,
                     const float* g_pred_rel, const float* g_attn, float beta,
                     float* d_feat_rel, float* const* dW1_host, float* const* db1_host,
                     float* const* dW2_host, float* const* db2_host, void* workspace,
                     size_t workspace_bytes, ta3n_stream_t stream);

/* ---- 'general' attention over the relation features (use_attn='general') ----------- */
/* models.py:320-325 (attn_layer = Linear(H,H), Tanh, Linear(H,1)), :359-366 (softmax over the R relations),
 * :379-388 (re-weighting by attn + 1), :651 (sum).  Call after ta3n_relattn_fwd(use_attn = 0), which leaves the
 * plain sum in feat_video:
 *   hidden [M*R,H] <- tanh(feat_rel W1^T + b1) (saved);  attn [M,R] <- softmax_r(hidden w2 + b2);
 *   feat_video [M,H] += sum_r attn[:,r] feat_rel[:,r,:].      W1 [H,H], b1 [H], w2 [1,H], b2 [1]               */
int ta3n_general_attn_fwd(const float* feat_rel, int M, int R, int H, const float* W1, const float* b1,
                          const float* w2, const float* b2, float* hidden, float* attn, float* feat_video,
                          ta3n_stream_t stream);
size_t ta3n_general_attn_bwd_workspace_bytes(int M, int R, int H);
/* Call after ta3n_relattn_bwd(use_attn = 2), which has written d_feat_rel = (attn + 1) G + discriminator part:
 * g_feat_video = G [M,H], g_attn [M,R] (may be NULL) -> d_feat_rel [M,R,H] += gradient through the weights;
 * dW1 [H,H], db1 [H], dw2 [1,H], db2 [1] are written.                                                            */
int ta3n_general_attn_bwd(const float* feat_rel, int M, int R, int H, const float* W1, const float* w2,
                          const float* hidden, const float* attn, const float* g_feat_video, const float* g_attn,
                          float* d_feat_rel, float* dW1, float* db1, float* dw2, float* db2, void* workspace,
                          size_t workspace_bytes, ta3n_stream_t stream);

/* ---- video head: Dropout -> [GRL_mu] -> Linear(H -> C)  (models.py:679-687) -------- */
/* feat_video [M,H] -> dropped [M,H] (saved; equals feat_video when no dropout),
 * pred [M,C].                                                                            */
int ta3n_video_head_fwd(const float* feat_video, int M, int H, int C, const float* Wc,
                        const float* bc, const ta3n_dropout* drop, float* dropped, float* pred,
                        ta3n_stream_t stream);
size_t ta3n_video_head_bwd_workspace_bytes(int M, int H, int C);
/* g_pred [M,C] (may be NULL), d_dropped_extra [M,H] = gradient already accumulated on the
 * dropped features by the video discriminator (may be NULL), g_feat_video_ext [M,H] (may be
 * NULL).  grad_scale multiplies everything that flows through the optional GRL_mu
 * (reverse ? -mu : 1).  Produces d_feat_video [M,H], dWc [C,H], dbc [C].  d_feat_video may be
 * NULL: only the weight / bias gradient is computed (MCD's reverse pass with mu == 0).   */
int ta3n_video_head_bwd(const float* dropped, int M, int H, int C, const float* Wc,
                        const ta3n_dropout* drop, const float* g_pred,
                        const float* d_dropped_extra, const float* g_feat_video_ext,
                        float grad_scale, float* d_feat_video, float* dWc, float* dbc,
                        void* workspace, size_t workspace_bytes, ta3n_stream_t stream);

/* ---- forward batching (optional) ------------------------------------------------------ */
/* Between begin and flush (same host thread) ta3n_disc_fwd and ta3n_trn_fwd only register their GEMMs;
 * the flush issues them as ONE grouped launch followed by their light follow-up kernels.  Only calls
 * whose inputs are already final may be batched together (e.g. the frame discriminator and the TRN,
 * which both read the shared features when use_attn_frame == 'none').  The workspace arguments are reserved
 * (may be NULL / 0).                                                                                     */
int ta3n_fwd_batch_begin(void);
size_t ta3n_fwd_batch_workspace_bytes(void);
int ta3n_fwd_batch_flush(void* workspace, size_t workspace_bytes, ta3n_stream_t stream);

/* ---- deferred weight gradients (optional) ------------------------------------------- */
/* Between begin and flush (same host thread) the *_bwd entry points above launch only their
 * data-gradient chain; their weight-gradient GEMMs and bias column sums are collected and issued by
 * the flush as one grouped launch per GEMM engine plus one column-sum launch.  The caller must keep
 * every buffer those calls were given (workspaces included) alive and unmodified until the flush. */
int ta3n_wgrad_defer_begin(void);
size_t ta3n_wgrad_defer_workspace_bytes(void);
int ta3n_wgrad_defer_flush(void* workspace, size_t workspace_bytes, ta3n_stream_t stream);

/* ---- fused loss heads of the shipped training configuration ------------------------- */
/* main.py:446 (class CE on the Bs source rows), main.py:508-538 (domain CE per level, labels
 * 0 = source rows, 1 = target rows), main.py:559-562 + loss.py:15-25 (gamma * attentive entropy).
 * flags: 1 relation-level adv, 2 video-level adv, 4 frame-level adv, 8 attentive entropy.
 * Inputs are the (Bs+Bt)-row outputs of the path; labels [Bs] int64.  Writes the scalar loss and
 * d loss / d logits of every head (zeros for disabled levels).
 * valid_rows (device, optional): {real source rows, real target rows} when the batch is the
 * zero-padded last one of an epoch (main.py:354-372 pads, main.py:421-422 slices the padding off
 * before the loss): padded rows get zero loss / gradient, means run over the real rows only.   */
size_t ta3n_loss_workspace_bytes(int M);
int ta3n_loss_fwd_bwd(const float* pred_video, const long long* labels, const float* pred_rel,
                      const float* pred_dom_video, const float* pred_frame, int Bs, int Bt, int T,
                      int R, int C, float gamma, int flags, const int* valid_rows, float* loss,
                      float* g_pred_video,
                      float* g_pred_rel, float* g_pred_dom_video, float* g_pred_frame,
                      void* workspace, size_t workspace_bytes, ta3n_stream_t stream);
/* *counter += 1 on the stream (dropout step counter for CUDA-graph replays). */
int ta3n_counter_inc(uint64_t* counter, ta3n_stream_t stream);

/* ---- loss terms of ens_DA='MCD' (main.py:446-448, 548-556; loss.py:29-30) ------------------------------------- */
/* Both are one single-block launch whose rows are summed in a fixed order, so that graph replays give bit-identical
 * losses; both ADD to *loss.  rows == 0 is a no-op.  valid_rows (device, optional) is the {real source rows, real
 * target rows} pair of ta3n_loss_fwd_bwd: padded rows get zero gradient and the means run over the real rows.
 *
 * Class CE of the second classifier on the source rows (main.py:447-448):
 *   loss += mean over r < valid_rows[0] of CE(pred[r], labels[r]);  g_pred [rows,C] = its gradient.             */
int ta3n_ce_loss_fwd_bwd(const float* pred, const long long* labels, int rows, int C, const int* valid_rows,
                         float* loss, float* g_pred, ta3n_stream_t stream);
/* Classifier discrepancy of the reverse pass on the target rows (main.py:548-556):
 *   loss += -mean |softmax(pred1) - softmax(pred2)| over r < valid_rows[1] and the C classes
 * (0 when there is no real row); g_pred1 / g_pred2 [rows,C] = its gradients (sign(0) = 0, as torch).
 * g_move1 [rows,C] (optional, must not alias the outputs): gradient other loss terms already left on pred1 -- the
 * attentive entropy of main.py:559-562 reads the target logits of this pass; it is added to g_pred1 and then zeroed,
 * so that the buffer it lives in can carry the other pass's gradient.                                            */
int ta3n_mcd_loss_fwd_bwd(const float* pred1, const float* pred2, int rows, int C, const int* valid_rows, float* loss,
                          float* g_pred1, float* g_pred2, float* g_move1, ta3n_stream_t stream);
/* dst[i] += src[i] for n floats (both 16-byte aligned): sums the gradient buckets of two backward passes.          */
int ta3n_accumulate(float* dst, const float* src, long long n, ta3n_stream_t stream);

/* ---- device-resident input pipeline (main.py:343-372 from feature banks in device memory) ---------------------- */
/* One launch fills the input slot of a paired mini-batch for BOTH domains, for use as the first launch of a captured
 * training step.  Per domain: bank [n_rows, row_floats] fp32 (16-byte aligned; row_floats % 4 == 0), the epoch's row
 * list rows [n_epoch] int32 (bank row of every epoch position) and, source only, its label list labels [n_epoch]
 * int64; the slot x [batch, row_floats] (16-byte aligned) and, source only, y [batch] int64.
 * state [2] uint32: {iteration i, arrival counter (0 between launches)}.  The launch copies the rows of epoch
 * positions [i*batch, min((i+1)*batch, n_epoch)) into the slot, zero-fills the rest (main.py:359-364 pads with zero
 * dummies; padded labels are 0), writes valid_rows [2] = {real source rows, real target rows} (the pair
 * ta3n_loss_fwd_bwd and the step program read) and advances state[0] by one; the last CTA to finish advances it, so
 * there is no extra launch.  Offsets are 64-bit (banks above 2^31 floats are fine).  A bank row id outside
 * [0, n_rows) gives a NaN row.  Kernel label "gather_batch".                                                        */
int ta3n_gather_batch(const float* bank_s, long long n_rows_s, const int* rows_s, const long long* labels_s,
                      long long n_epoch_s, int batch_s, float* x_s, long long* y_s,
                      const float* bank_t, long long n_rows_t, const int* rows_t, long long n_epoch_t, int batch_t,
                      float* x_t, long long row_floats, int* valid_rows, unsigned int* state, ta3n_stream_t stream);
/* The same gather for ONE labelled domain in a fixed order (validation: main.py:178 uses shuffle=False; the row list
 * carries the num_dataload tiling): the rows of epoch positions [i*batch, min((i+1)*batch, n_epoch)) go to x
 * [batch, row_floats], their labels to y [batch], the rest is zero-filled with label 0, valid_rows [1] = the number of
 * real rows (what ta3n_eval_head reads), and state [2] advances as in ta3n_gather_batch.  Kernel label "gather_rows". */
int ta3n_gather_rows(const float* bank, long long n_rows, const int* rows, const long long* labels, long long n_epoch,
                     int batch, float* x, long long* y, long long row_floats, int* valid_rows, unsigned int* state,
                     ta3n_stream_t stream);

/* ---- validation head (main.py:707-730 validate(), test_models.py:115-193) ------------------------------------- */
/* Epoch accumulator in device memory (8-byte aligned; zero it to start an epoch).                                  */
typedef struct {
  double loss_sum;            /* sum over batches of n_b * loss_b (losses.update(loss.item(), n_b), main.py:728)      */
  long long n;                /* real rows seen                                                                      */
  long long correct[4];       /* real rows whose label ranks below k[i]                                              */
  int batch;                  /* launches folded in so far (the batch index of the next launch)                     */
  unsigned int arrive;        /* arrival counter of the launch, 0 between launches                                  */
} ta3n_eval_accum;

size_t ta3n_eval_workspace_bytes(int rows);
/* One launch per validation batch of `rows` rows, of which the first *valid_rows (device int) are real (the rest is
 * the zero padding main.py:690-693 adds and removeDummy drops, :710):
 *   logits [rows,C] = feat_video [rows,H] Wc^T + bc, in fp32 FFMA whatever GEMM engine is selected (Wc staged in
 *     shared memory when it fits, streamed through it otherwise);
 *   per real row r with label y = labels[r] (int64):  ce = logsumexp(z) - z_y (shifted by the max, summed in fp64);
 *     w_y = class_weight[y] (class_weight may be NULL: 1);  rank = #{j : z_j > z_y} + #{j < y : z_j == z_y}, i.e.
 *     TIES RANK BY CLASS INDEX (torch.topk leaves their order unspecified; this pins it);  correct@k = rank < k;
 *     top-1 = the lowest index among the maxima (so top-1 == y exactly when rank == 0);
 *   batch: loss_b = sum w_y ce / sum w_y over the real rows (CrossEntropyLoss(weight=...), main.py:205, 725), folded
 *     into *accum as loss_sum += n_b * loss_b, n += n_b, correct[i] += its count for k_host[i] (n_k <= 4, 1 <= k <= C);
 *     confusion [C,C] int64 (may be NULL) gets +1 at (y, top-1) per real row (test_models.py's cf);
 *   epoch buffers (may be NULL): scores [n_epoch,C] and attn_out [n_epoch,R] receive the real rows' logits and
 *     attention (row r of attn at attn + r*attn_ld, R floats) at row accum->batch * rows + r (dataset order when every
 *     earlier batch was full); rows past n_epoch are dropped.
 * A label outside [0, C), or a NaN among a row's logits, makes the batch loss NaN (as torch's criterion does for NaN)
 * and that row counts at no k and in no confusion cell; it still counts in n.  A row of -inf logits is ordered by the
 * rule above (every class ties: rank = y, top-1 = 0).  Per-CTA partials go to the workspace; the last
 * CTA to arrive sums them in CTA order, folds them into *accum, advances accum->batch and re-arms accum->arrive, so
 * reruns are bit-identical (no float atomics; the confusion counts are integer atomics).  Kernel label "eval_head". */
int ta3n_eval_head(const float* feat_video, int rows, int H, int C, const float* Wc, const float* bc,
                   const long long* labels, const float* class_weight, const int* valid_rows, int n_k,
                   const int* k_host, const float* attn, int R, long long attn_ld, float* logits,
                   ta3n_eval_accum* accum, long long* confusion, float* scores, float* attn_out, long long n_epoch,
                   void* workspace, size_t workspace_bytes, ta3n_stream_t stream);

/* ---- the training step as one step program (SURVEY 8a rows a1-a13 + 8f row n1) ----------------------------- */
/* main.py:418 (model forward, models.py:545-722 trn-m branch), main.py:446, 508-538, 559-562 (composed loss:
 * class CE + domain CE per adversarial level + gamma * attentive entropy, loss.py:15-25) and main.py:576
 * (backward to every parameter gradient) for one paired mini-batch, use_attn_frame == 'none'.
 *
 * Everything is described once by a ta3n_step_desc (device pointers unless noted).  ta3n_step_run_phased enqueues
 * one launch per dependency level: 8 grouped GEMM launches (engine as selected), 4 row kernels (frame rows; per
 * video: relation pooling, loss heads, relation backward) and 2 column-sum launches (14 launches; the round-1
 * sequence had 25).  It is CUDA-graph capturable.                                                                 */
typedef struct {
  int Bs, Bt;                 /* source / target videos of the mini-batch (M = Bs + Bt rows, source first)         */
  int T, D, F, H, C;          /* frames per video, input width, shared width (fc_dim), bottleneck (256), classes    */
  int use_attn;               /* 1: use_attn='TransAttn', 0: 'none' (models.py:646-648)                             */
  int loss_flags;             /* as ta3n_loss_fwd_bwd: 1 relation / 2 video / 4 frame adversarial CE, 8 attentive entropy */
  float gamma;                /* weight of the attentive entropy (main.py:561)                                      */
  float domain_weight[2];     /* criterion_domain weights (main.py:165-167); {1, 1} = unweighted                    */
  const float* class_weight;  /* [C] criterion weights (main.py:160-163, 204) or NULL                               */
  const float* beta_dev;      /* [3] {relation, video, frame} GRL coefficients in DEVICE memory, so that the per-step
                                 DANN schedule (main.py:350-352) replays inside a captured graph                     */
  const ta3n_relation_table* tab;
  /* inputs */
  const float* x_src;         /* [Bs, T, D] */
  const float* x_tgt;         /* [Bt, T, D] */
  const long long* labels;    /* [Bs] */
  const int* valid_rows;      /* {real source rows, real target rows} or NULL (see ta3n_loss_fwd_bwd)               */
  ta3n_dropout drop_i, drop_v;/* dropout of the shared layer / of the video features (p <= 0: none)                 */
  /* parameters and their gradients; *_host are HOST arrays of R = T-1 device pointers                               */
  const float *W_sh, *b_sh;                 /* fc_feature_shared_source   [F, D], [F]                                */
  const float *W1f, *b1f, *W2f, *b2f;       /* fc_feature_domain [F, F], fc_classifier_domain [2, F]                 */
  const float* const* W_trn_host;           /* TRN.fc_fusion_scales[i][1] [H, (T-i) F]                               */
  const float* const* b_trn_host;
  const float* const* W1r_host;             /* relation_domain_classifier_all[i][0] [H, H], [i][2] [2, H]            */
  const float* const* b1r_host;
  const float* const* W2r_host;
  const float* const* b2r_host;
  const float *Wc, *bc;                     /* fc_classifier_video_source [C, H]                                     */
  const float *W1v, *b1v, *W2v, *b2v;       /* fc_feature_domain_video [H, H], fc_classifier_domain_video [2, H]     */
  float *dW_sh, *db_sh, *dW1f, *db1f, *dW2f, *db2f;
  float* const* dW_trn_host;
  float* const* db_trn_host;
  float* const* dW1r_host;
  float* const* db1r_host;
  float* const* dW2r_host;
  float* const* db2r_host;
  float *dWc, *dbc, *dW1v, *db1v, *dW2v, *db2v;
  /* outputs / saved activations (caller-provided, M = Bs + Bt rows)                                                  */
  float* feat;                /* [M*T, F]   shared features (post ReLU / dropout)                                    */
  float* hid_f;               /* [M*T, F]   frame-discriminator hidden layer                                         */
  float* pred_frame;          /* [M*T, 2]                                                                            */
  float* act;                 /* [n_rel, M, H] relation activations                                                  */
  float* feat_rel;            /* [M, R, H]                                                                           */
  float* hid_r;               /* [R, M, H]  relation-discriminator hidden layers                                     */
  float* pred_rel;            /* [M, R, 2]                                                                           */
  float* attn;                /* [M, R]                                                                              */
  float* feat_video;          /* [M, H]                                                                              */
  float* dropped;             /* [M, H]                                                                              */
  float* pred_video;          /* [M, C]                                                                              */
  float* hid_v;               /* [M, H]                                                                              */
  float* pred_dom;            /* [M, 2]                                                                              */
  float* loss;                /* [1]                                                                                 */
  uint64_t* step_counter;     /* optional: += 1 at the END of the step (dropout RNG key of the next replay)          */
  void* workspace;            /* ta3n_step_workspace_bytes(desc) bytes of scratch                                    */
  size_t workspace_bytes;
} ta3n_step_desc;

/* Bytes of desc->workspace: the fixed scratch tensors plus the column sums' partials.  Pointers in desc only need to
 * be non-null; no CUDA call.  0 on an invalid descriptor (ta3n_last_error() says why).                              */
size_t ta3n_step_workspace_bytes(const ta3n_step_desc* desc);
int ta3n_step_run_phased(const ta3n_step_desc* desc, ta3n_stream_t stream);

/* ---- gradient all-reduce over NVLink / NVSwitch peer memory (SURVEY 8e; replaces nn.DataParallel's reduce, main.py:79) */
/* In-place MEAN over the `world` ranks of one node of n floats (n % 4 == 0) that live at the same offset of a symmetric,
 * peer-mapped allocation on every rank.  peer_bufs_host / peer_flags_host: HOST arrays of `world` device pointers -- this
 * process's mappings of every rank's buffer / flag array ([rank] = the local one); flag arrays hold
 * ta3n_allreduce_flag_bytes(world) bytes, zero-initialised once.  multicast_buf: the NVSwitch multicast mapping of the
 * buffer (the switch reduces in flight: multimem.ld_reduce / multimem.st) or NULL (peer loads / stores).  *seq_dev: a
 * device counter with the same value on every rank that has INCREASED since the previous call (the train step's step
 * counter).  One kernel, two-shot, deterministic, bit-identical results on all ranks, CUDA-graph capturable.        */
size_t ta3n_allreduce_flag_bytes(int world);
int ta3n_allreduce_mean(float* const* peer_bufs_host, float* multicast_buf, uint32_t* const* peer_flags_host,
                        const uint64_t* seq_dev, int rank, int world, long long n, ta3n_stream_t stream);

/* ---- optimizer step (SURVEY 8f n2) ---------------------------------------------------- */
/* main.py:578-581 clip_grad_norm_(parameters, max_norm) followed by main.py:83/583
 * torch.optim.SGD(lr, momentum, weight_decay, nesterov=True).step(), over FLAT fp32 buffers of n
 * elements (params, grads, momentum buffers in the same order; momentum zero-initialised):
 *     coef = min(1, max_norm / (||g||_2 + 1e-6))        (max_norm <= 0: no clipping, coef = 1)
 *     d = coef*g + weight_decay*p;  m = momentum*m + d;  p -= lr * (d + momentum*m)
 * lr is read from device memory (*lr_dev) so a per-step schedule (main.py:800-802) replays inside a
 * CUDA graph.  stats (optional, 2 floats) receives {||g||_2, coef}.  Two launches; deterministic.  */
size_t ta3n_sgd_workspace_bytes(void);
int ta3n_sgd_nesterov_step(float* params, const float* grads, float* momentum_buf, long long n,
                           const float* lr_dev, float momentum, float weight_decay, float max_norm,
                           void* workspace, size_t workspace_bytes, float* stats,
                           ta3n_stream_t stream);
/* The same with an optional per-element mask (n floats, device; 0 = leave parameter and momentum untouched): parameters
 * the configured losses give no gradient -- torch.optim.SGD skips parameters whose .grad is None (main.py:83), it does
 * not weight-decay them.  The mask must be constant over each aligned group of four elements.                         */
int ta3n_sgd_nesterov_step_masked(float* params, const float* grads, float* momentum_buf, long long n,
                                  const float* lr_dev, float momentum, float weight_decay, float max_norm,
                                  void* workspace, size_t workspace_bytes, float* stats, const float* active,
                                  ta3n_stream_t stream);

/* ---- self test of the tensor-core GEMM engine (used by tests; device buffers) ------ */
/* C[M,N] = A[M,K] * B[N,K]^T with the selected engine; A, B, C row-major fp32.           */
int ta3n_gemm_tn(const float* A, const float* B, float* C, int M, int N, int K,
                 ta3n_stream_t stream);
/* General form: a_kmajor ? A(m,k)=A[m*lda+k] : A(m,k)=A[k*lda+m];  b_kmajor ? B(k,n)=B[n*ldb+k] :
 * B(k,n)=B[k*ldb+n].  workspace (optional) enables deterministic split-K.                 */
int ta3n_gemm_ex(const float* A, int lda, int a_kmajor, const float* B, int ldb, int b_kmajor,
                 float* C, int ldc, int M, int N, int K, void* workspace, size_t workspace_bytes,
                 ta3n_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* TA3N_B200_H_ */
