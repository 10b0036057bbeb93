// ta3n_api.cu -- extern "C" entry points of libta3n_sm90.so (see include/ta3n_b200.h).
// Every function only builds launch tables on the host and enqueues kernels on the caller's
// stream: no allocation, no synchronisation, CUDA-graph capturable.
#include "common.cuh"
#include "seg_gemm.cuh"
#include "rowops.cuh"
#include "gemm_wgmma.cuh"
#include "optim.cuh"
#include "step_plan.cuh"
#include "allreduce.cuh"
#include "gather.cuh"
#include "eval.cuh"

#include <functional>

using namespace ta3n;

namespace {

struct RelLayout {
  int T, R, n_rel, n_slots;
  std::vector<int> scale_size, rel_count, rel_begin;   // per scale
  std::vector<int> rel_scale;                          // per relation q
  std::vector<int> slot_begin;                         // per relation q: offset into frames
  const int* frames;
};

int parse_table(const ta3n_relation_table* tab, RelLayout* L) {
  TA3N_REQUIRE(tab != nullptr, "relation table is null");
  TA3N_REQUIRE(tab->num_frames >= 2 && tab->n_scales >= 1 && tab->n_scales <= kMaxScales, "bad table sizes");
  TA3N_REQUIRE(tab->scale_size && tab->rel_count && tab->frames, "relation table arrays are null");
  L->T = tab->num_frames;
  L->R = tab->n_scales;
  L->frames = tab->frames;
  L->n_rel = 0;
  L->n_slots = 0;
  for (int i = 0; i < L->R; ++i) {
    const int s = tab->scale_size[i], n = tab->rel_count[i];
    TA3N_REQUIRE(s >= 1 && s <= L->T && n >= 1, "bad scale entry");
    L->scale_size.push_back(s);
    L->rel_count.push_back(n);
    L->rel_begin.push_back(L->n_rel);
    for (int r = 0; r < n; ++r) {
      L->rel_scale.push_back(i);
      L->slot_begin.push_back(L->n_slots);
      for (int j = 0; j < s; ++j) {
        const int t = tab->frames[L->n_slots + j];
        TA3N_REQUIRE(t >= 0 && t < L->T, "frame id out of range");
      }
      L->n_slots += s;
    }
    L->n_rel += n;
  }
  L->rel_begin.push_back(L->n_rel);
  TA3N_REQUIRE(L->n_rel <= kMaxRel, "too many relations");
  return TA3N_OK;
}

RelMap make_relmap(const RelLayout& L) {
  RelMap m;
  memset(&m, 0, sizeof(m));
  m.n_rel = L.n_rel;
  m.n_scales = L.R;
  for (int i = 0; i <= L.R; ++i) m.rel_begin[i] = L.rel_begin[i];
  for (int q = 0; q < L.n_rel; ++q) m.scale_of[q] = (unsigned char)L.rel_scale[q];
  return m;
}

void set_dropout_epilogue(Group& g, const DropArgs& d, const uint8_t* keep, int ldkeep, uint64_t rng_offset) {
  if (d.mode == 0) return;
  g.drop_scale = d.scale;
  g.drop_p = d.p;
  if (d.mode == 1) {
    g.flags |= EPI_DROP_MASK;
    g.keep = keep;
    g.ldkeep = ldkeep;
  } else {
    g.flags |= EPI_DROP_RNG;
    g.seed = d.seed;
    g.step_dev = d.step_dev;
    g.rng_offset = rng_offset;
  }
}

inline cudaStream_t S(ta3n_stream_t s) { return static_cast<cudaStream_t>(s); }

// Upper bound of the split-K partial buffers plan_splitk() may carve for `n_groups` outputs:
// sum_g ksplit_g * M_g * N_g <= (target_ctas + tiles) * tile_elems <= 2 * 296 * 128*128 floats
// (tile_elems of the tensor-core engine; the SIMT engine's 64x64 tiles need a quarter of that).
inline size_t splitk_bytes(int n_groups) {
  return (size_t)2 * 296 * 128 * 128 * sizeof(float) + (size_t)256 * (n_groups + 1) + 4096;
}

// ---- deferred weight-gradient work ------------------------------------------------------------------
// Between ta3n_wgrad_defer_begin() and ta3n_wgrad_defer_flush() the *_bwd entry points enqueue only
// their data-gradient chain; their weight-gradient GEMMs (all M-major x N-major) and bias column sums
// are collected here and issued by the flush as ONE grouped launch per engine + ONE column-sum launch.
// The buffers they read (workspaces, saved activations) must stay alive and unmodified until the flush.
struct DeferCtx {
  bool active = false;
  GemmPlan wgrad;
  ColsumPlan cs;
  void reset() {
    wgrad = GemmPlan();
    wgrad.a_kmaj = false;
    wgrad.b_kmaj = false;
    wgrad.label = "wgrad_all";
    cs = ColsumPlan();
  }
};
DeferCtx& defer_ctx() {
  static thread_local DeferCtx c;
  return c;
}

int submit_wgrad(GemmPlan& plan, cudaStream_t st, Arena* arena) {
  DeferCtx& d = defer_ctx();
  if (!d.active || plan.load_flags != 0) return run_gemm(plan, st, arena);
  for (const Group& src : plan.groups) {
    Group g = src;
    g.seg_begin = (int)d.wgrad.segs.size();
    for (int k = 0; k < src.seg_count; ++k) d.wgrad.segs.push_back(plan.segs[src.seg_begin + k]);
    d.wgrad.groups.push_back(g);
  }
  return TA3N_OK;
}

// Forward-side batching: independent K-major x K-major GEMMs (frame discriminator hidden layer and the TRN
// relation GEMMs both read the shared features) collected into one grouped launch; the light kernels that
// consume their outputs run right after it, in submission order.
struct FwdBatch {
  bool active = false;
  GemmPlan plan;
  std::vector<std::function<int(cudaStream_t)>> post;
  void reset() {
    plan = GemmPlan();
    plan.label = "fwd_batch";
    plan.precise = true;
    post.clear();
  }
};
FwdBatch& fwd_batch() {
  static thread_local FwdBatch b;
  return b;
}

int submit_fwd(GemmPlan& plan, cudaStream_t st, std::function<int(cudaStream_t)> post) {
  FwdBatch& b = fwd_batch();
  if (!b.active || plan.load_flags != 0 || !plan.a_kmaj || !plan.b_kmaj) {
    TA3N_TRY(run_gemm(plan, st));
    return post(st);
  }
  for (const Group& src : plan.groups) {
    Group g = src;
    g.seg_begin = (int)b.plan.segs.size();
    for (int k = 0; k < src.seg_count; ++k) b.plan.segs.push_back(plan.segs[src.seg_begin + k]);
    b.plan.groups.push_back(g);
  }
  b.post.push_back(std::move(post));
  return TA3N_OK;
}

int submit_colsum(ColsumPlan& cs, cudaStream_t st, Arena* arena) {
  DeferCtx& d = defer_ctx();
  if (!d.active) return cs.run(st, arena);
  for (auto& j : cs.jobs) d.cs.jobs.push_back(j);
  return TA3N_OK;
}

// workspace of the (weighted) column sums producing `out_elems` gradient values
inline size_t colsum_bytes(size_t out_elems) { return ColsumPlan::workspace_bytes(out_elems); }

}  // namespace

extern "C" {

int ta3n_fwd_batch_begin(void) {
  FwdBatch& b = fwd_batch();
  b.reset();
  b.active = true;
  return TA3N_OK;
}

size_t ta3n_fwd_batch_workspace_bytes(void) { return 0; }

int ta3n_fwd_batch_flush(void* workspace, size_t workspace_bytes, ta3n_stream_t stream) {
  FwdBatch& b = fwd_batch();
  if (!b.active) return fail(TA3N_ERR_INVALID, "ta3n_fwd_batch_flush without ta3n_fwd_batch_begin");
  b.active = false;
  (void)workspace;      // reserved: the forward batch is launched unsplit (more than half a wave of tiles)
  (void)workspace_bytes;
  int rc = run_gemm(b.plan, S(stream), nullptr);
  for (auto& f : b.post)
    if (rc == TA3N_OK) rc = f(S(stream));
  b.reset();
  return rc;
}

int ta3n_wgrad_defer_begin(void) {
  DeferCtx& d = defer_ctx();
  d.reset();
  d.active = true;
  return TA3N_OK;
}

size_t ta3n_wgrad_defer_workspace_bytes(void) { return splitk_bytes(64) + colsum_bytes((size_t)1 << 18); }

int ta3n_wgrad_defer_flush(void* workspace, size_t workspace_bytes, ta3n_stream_t stream) {
  DeferCtx& d = defer_ctx();
  if (!d.active) return fail(TA3N_ERR_INVALID, "ta3n_wgrad_defer_flush without ta3n_wgrad_defer_begin");
  d.active = false;
  Arena arena(workspace, workspace_bytes);
  int rc = d.cs.run(S(stream), &arena);   // first: its partials are small and must fit
  if (rc == TA3N_OK) rc = run_gemm(d.wgrad, S(stream), workspace ? &arena : nullptr);
  d.reset();
  return rc;
}

int ta3n_abi_version(void) { return TA3N_ABI_VERSION; }
const char* ta3n_last_error(void) { return last_error_buf(); }
uint64_t ta3n_launch_count(void) { return launch_counter().load(); }
void ta3n_reset_launch_count(void) { launch_counter().store(0); }
int ta3n_set_gemm_engine(int engine) {
  if (engine != TA3N_GEMM_FP32_SIMT && engine != TA3N_GEMM_TF32_TCGEN05 && engine != TA3N_GEMM_TF32X3_TCGEN05)
    return fail(TA3N_ERR_INVALID, "unknown GEMM engine %d", engine);
  gemm_engine().store(engine);
  return TA3N_OK;
}
int ta3n_get_gemm_engine(void) { return gemm_engine().load(); }

int ta3n_set_forward_scratch(void* scratch, size_t bytes) {
  TA3N_REQUIRE(scratch == nullptr || (reinterpret_cast<uintptr_t>(scratch) & 255u) == 0, "scratch must be 256-byte aligned");
  forward_scratch().ptr = bytes > 0 ? scratch : nullptr;
  forward_scratch().bytes = scratch ? bytes : 0;
  return TA3N_OK;
}

void ta3n_timing_enable(int on) { timing().enabled.store(on != 0); }

// Synchronises the recorded events, aggregates device time per call-site label and writes lines
// "label count total_ms\n" into buf.  Returns the number of bytes needed (excluding the NUL).
size_t ta3n_timing_report(char* buf, size_t buf_bytes) {
  TimingRegistry& t = timing();
  std::vector<TimingRegistry::Rec> recs;
  {
    std::lock_guard<std::mutex> g(t.mu);
    recs.swap(t.recs);
  }
  struct Agg {
    const char* label;
    int count;
    double ms;
  };
  std::vector<Agg> agg;
  for (auto& r : recs) {
    float ms = 0.f;
    if (cudaEventSynchronize(r.b) == cudaSuccess && cudaEventElapsedTime(&ms, r.a, r.b) == cudaSuccess) {
      bool found = false;
      for (auto& a : agg)
        if (strcmp(a.label, r.label) == 0) {
          a.count++;
          a.ms += ms;
          found = true;
          break;
        }
      if (!found) agg.push_back({r.label, 1, (double)ms});
    }
    cudaEventDestroy(r.a);
    cudaEventDestroy(r.b);
  }
  std::string out;
  char line[160];
  for (auto& a : agg) {
    snprintf(line, sizeof(line), "%s %d %.6f\n", a.label, a.count, a.ms);
    out += line;
  }
  if (buf && buf_bytes > 0) {
    size_t n = out.size() < buf_bytes - 1 ? out.size() : buf_bytes - 1;
    memcpy(buf, out.data(), n);
    buf[n] = 0;
  }
  return out.size();
}

// ------------------------------------------------------------------------------------------------
// shared frame layer                                                        models.py:565-575
// ------------------------------------------------------------------------------------------------
int ta3n_shared_fc_fwd(const float* x_src, int rows_src, const float* x_tgt, int rows_tgt, int D,
                       const float* W, const float* b, int F, const ta3n_dropout* drop, float* feat,
                       ta3n_stream_t stream) {
  TA3N_REQUIRE(rows_src >= 0 && rows_tgt >= 0 && D > 0 && F > 0, "bad sizes");
  TA3N_REQUIRE(W && b && feat, "null pointer");
  TA3N_REQUIRE((rows_src == 0 || x_src) && (rows_tgt == 0 || x_tgt), "null input");
  const DropArgs d = make_drop(drop);
  GemmPlan plan;
    plan.label = "shared_fc_fwd";
    plan.precise = true;
  const float* xs[2] = {x_src, x_tgt};
  const int rows[2] = {rows_src, rows_tgt};
  size_t row0 = 0;
  for (int dom = 0; dom < 2; ++dom) {
    if (rows[dom] > 0) {
      Group& g = plan.add_group(rows[dom], F, feat + row0 * F, F);
      g.flags = EPI_BIAS | EPI_RELU;
      g.bias = b;
      set_dropout_epilogue(g, d, d.keep ? d.keep + row0 * F : nullptr, F, row0 * F);
      plan.add_seg(xs[dom], D, W, D, D);
    }
    row0 += rows[dom];
  }
  return run_gemm(plan, S(stream));
}

size_t ta3n_shared_fc_bwd_workspace_bytes(int rows, int D, int F) {
  (void)rows; (void)D;
  return splitk_bytes(1) + colsum_bytes(F);
}

int ta3n_shared_fc_bwd(const float* x_src, int rows_src, const float* x_tgt, int rows_tgt, int D, int F,
                       const float* feat, float* dfeat, const float* g_feat_ext, float p, float* dW,
                       float* db, void* workspace, size_t workspace_bytes, ta3n_stream_t stream) {
  TA3N_REQUIRE(rows_src >= 0 && rows_tgt >= 0 && D > 0 && F > 0, "bad sizes");
  TA3N_REQUIRE(feat && dfeat && dW && db, "null pointer");
  TA3N_REQUIRE(p >= 0.f && p < 1.f, "dropout p must be in [0,1)");
  const int rows = rows_src + rows_tgt;
  if (rows == 0) {
    TA3N_CUDA(cudaMemsetAsync(dW, 0, sizeof(float) * F * D, S(stream)));
    TA3N_CUDA(cudaMemsetAsync(db, 0, sizeof(float) * F, S(stream)));
    return TA3N_OK;
  }
  const size_t total = (size_t)rows * F;
  pre_launch("dpre", S(stream));
  launch_dpre(feat, dfeat, g_feat_ext, 1.0f / (1.0f - p), total, S(stream));
  TA3N_TRY(after_launch());

  Arena arena(workspace, workspace_bytes);
  GemmPlan plan;
    plan.label = "shared_fc_wgrad";
  plan.a_kmaj = false;
  plan.b_kmaj = false;
  plan.add_group(F, D, dW, D);
  if (rows_src > 0) plan.add_seg(dfeat, F, x_src, D, rows_src);
  if (rows_tgt > 0) plan.add_seg(dfeat + (size_t)rows_src * F, F, x_tgt, D, rows_tgt);
  TA3N_TRY(submit_wgrad(plan, S(stream), &arena));

  ColsumPlan cs;
  cs.add(db, F, F);
  cs.seg(dfeat, rows);
  return submit_colsum(cs, S(stream), &arena);
}

// ------------------------------------------------------------------------------------------------
// GradReverse + two-layer discriminator                        models.py:456-470, 20-29
// ------------------------------------------------------------------------------------------------
int ta3n_disc_fwd(const float* x, int rows, int K, int Kh, const float* W1, const float* b1, const float* W2,
                  const float* b2, float* hidden, float* logits, ta3n_stream_t stream) {
  TA3N_REQUIRE(rows >= 0 && K > 0 && Kh > 0, "bad sizes");
  if (rows == 0) return TA3N_OK;
  TA3N_REQUIRE(x && W1 && b1 && W2 && b2 && hidden && logits, "null pointer");
  GemmPlan plan;
    plan.label = "disc_fwd";
    plan.precise = true;
  Group& g = plan.add_group(rows, Kh, hidden, Kh);
  g.flags = EPI_BIAS | EPI_RELU;
  g.bias = b1;
  plan.add_seg(x, K, W1, K, K);
  return submit_fwd(plan, S(stream), [=](cudaStream_t st) -> int {
    return launch_head_fwd(hidden, Kh, W2, b2, logits, 2, rows, Kh, 2, st);
  });
}

size_t ta3n_disc_bwd_workspace_bytes(int rows, int K, int Kh) {
  (void)K;
  return Arena::round((size_t)rows * Kh * sizeof(float)) + splitk_bytes(2) + colsum_bytes((size_t)3 * Kh + 2);
}

int ta3n_disc_bwd(const float* x, int rows, int K, int Kh, const float* W1, const float* W2,
                  const float* hidden, const float* g_logits, float beta, float* dx, int accumulate,
                  float* dW1, float* db1, float* dW2, float* db2, void* workspace, size_t workspace_bytes,
                  ta3n_stream_t stream) {
  TA3N_REQUIRE(rows >= 0 && K > 0 && Kh > 0, "bad sizes");
  TA3N_REQUIRE(dW1 && db1 && dW2 && db2, "null gradient pointer");
  cudaStream_t st = S(stream);
  if (rows == 0 || g_logits == nullptr) {
    TA3N_CUDA(cudaMemsetAsync(dW1, 0, sizeof(float) * Kh * K, st));
    TA3N_CUDA(cudaMemsetAsync(db1, 0, sizeof(float) * Kh, st));
    TA3N_CUDA(cudaMemsetAsync(dW2, 0, sizeof(float) * 2 * Kh, st));
    TA3N_CUDA(cudaMemsetAsync(db2, 0, sizeof(float) * 2, st));
    if (dx && !accumulate && rows > 0) TA3N_CUDA(cudaMemsetAsync(dx, 0, sizeof(float) * rows * K, st));
    return TA3N_OK;
  }
  TA3N_REQUIRE(x && W1 && W2 && hidden, "null pointer");
  Arena arena(workspace, workspace_bytes);
  float* dH = arena.floats((size_t)rows * Kh);
  if (!dH) return fail(TA3N_ERR_WORKSPACE, "ta3n_disc_bwd: workspace too small (%zu bytes)", workspace_bytes);

  // dH = (g_logits W2) * 1[hidden > 0]
  pre_launch("head_bwd_data", st);
  launch_head_bwd_data(g_logits, 2, W2, hidden, 1.0f, 0, dH, rows, Kh, st);
  TA3N_TRY(after_launch());

  {  // dW2 [2,Kh] = g_logits^T hidden (skinny: weighted column sum), db2, db1
    ColsumPlan cs;
    cs.add_weighted(dW2, Kh, 2, Kh, Kh, 2);
    cs.seg(hidden, rows, g_logits);
    cs.add(db2, 2, 2);
    cs.seg(g_logits, rows);
    cs.add(db1, Kh, Kh);
    cs.seg(dH, rows);
    TA3N_TRY(submit_colsum(cs, st, &arena));
  }
  {  // dW1 [Kh,K] = dH^T x
    GemmPlan plan;
    plan.label = "disc_wgrad";
    plan.a_kmaj = false;
    plan.b_kmaj = false;
    plan.add_group(Kh, K, dW1, K);
    plan.add_seg(dH, Kh, x, K, rows);
    TA3N_TRY(submit_wgrad(plan, st, &arena));
  }
  if (dx) {  // dx (+)= -beta * dH W1
    GemmPlan plan;
    plan.label = "disc_dgrad";
    plan.precise_dgrad = true;
    plan.a_kmaj = true;
    plan.b_kmaj = false;
    Group& g = plan.add_group(rows, K, dx, K);
    g.alpha = -beta;
    if (accumulate) g.flags |= EPI_ACCUM;
    plan.add_seg(dH, Kh, W1, K, Kh);
    TA3N_TRY(run_gemm(plan, st));
  }
  return TA3N_OK;
}

int ta3n_grl_bwd(const float* g, float beta, float* out, size_t n, ta3n_stream_t stream) {
  if (n == 0) return TA3N_OK;
  TA3N_REQUIRE(g && out, "null pointer");
  pre_launch("grl_bwd", S(stream));
  launch_kernel(grl_bwd_kernel, blocks_for(n, 256), 256, 0, S(stream), g, beta, out, n);
  return after_launch();
}

// ------------------------------------------------------------------------------------------------
// frame-level attention                                                    models.py:368-377
// ------------------------------------------------------------------------------------------------
int ta3n_frame_attn_fwd(const float* feat, const float* logits, int rows, int F, float* out,
                        ta3n_stream_t stream) {
  TA3N_REQUIRE(rows >= 0 && F > 0, "bad sizes");
  if (rows == 0) return TA3N_OK;
  TA3N_REQUIRE(feat && logits && out, "null pointer");
  pre_launch("frame_attn_fwd", S(stream));
  launch_kernel(frame_attn_fwd_kernel, blocks_for((size_t)rows * F, 256), 256, 0, S(stream), feat, logits, rows, F, out);
  return after_launch();
}

int ta3n_frame_attn_bwd(const float* feat, const float* logits, int rows, int F, float* d_out, float* g_logits,
                        ta3n_stream_t stream) {
  TA3N_REQUIRE(rows >= 0 && F > 0, "bad sizes");
  if (rows == 0) return TA3N_OK;
  TA3N_REQUIRE(feat && logits && d_out && g_logits, "null pointer");
  pre_launch("frame_attn_bwd", S(stream));
  launch_kernel(frame_attn_bwd_kernel, blocks_for((size_t)rows * 32, 256), 256, 0, S(stream), feat, logits, rows, F, d_out,
                                                                                   g_logits);
  return after_launch();
}

// ------------------------------------------------------------------------------------------------
// average over the segments (frame_aggregation='avgpool')                   models.py:425-433
// ------------------------------------------------------------------------------------------------
int ta3n_segment_mean_fwd(const float* x, int M, int T, int F, float* out, ta3n_stream_t stream) {
  TA3N_REQUIRE(M >= 0 && T > 0 && F > 0, "bad sizes");
  if (M == 0) return TA3N_OK;
  TA3N_REQUIRE(x && out, "null pointer");
  pre_launch("segment_mean_fwd", S(stream));
  launch_kernel(segment_mean_fwd_kernel, blocks_for((size_t)M * F, 256), 256, 0, S(stream), x, out, M, T, F);
  return after_launch();
}

int ta3n_segment_mean_bwd(const float* g, int M, int T, int F, float* dx, ta3n_stream_t stream) {
  TA3N_REQUIRE(M >= 0 && T > 0 && F > 0, "bad sizes");
  if (M == 0) return TA3N_OK;
  TA3N_REQUIRE(g && dx, "null pointer");
  pre_launch("segment_mean_bwd", S(stream));
  launch_kernel(segment_mean_bwd_kernel, blocks_for((size_t)M * T * F, 256), 256, 0, S(stream), g, dx, M, T, F);
  return after_launch();
}

// ------------------------------------------------------------------------------------------------
// multi-scale temporal relation module                                   TRNmodule.py:58-82
// ------------------------------------------------------------------------------------------------
int ta3n_trn_fwd(const float* x, int M, int F, int H, const ta3n_relation_table* tab,
                 const float* const* W_host, const float* const* b_host, int relu_input, float* act,
                 float* feat_rel, ta3n_stream_t stream) {
  RelLayout L;
  TA3N_TRY(parse_table(tab, &L));
  TA3N_REQUIRE(M >= 0 && F > 0 && H > 0, "bad sizes");
  if (M == 0) return TA3N_OK;
  TA3N_REQUIRE(x && W_host && b_host && act && feat_rel, "null pointer");
  const int ldx = L.T * F;
  GemmPlan plan;
    plan.label = "trn_fwd";
    plan.precise = true;
  plan.load_flags = relu_input ? LD_RELU_A : 0;
  for (int q = 0; q < L.n_rel; ++q) {
    const int i = L.rel_scale[q], s = L.scale_size[i];
    TA3N_REQUIRE(W_host[i] && b_host[i], "null weight pointer");
    Group& g = plan.add_group(M, H, act + (size_t)q * M * H, H);
    g.flags = EPI_BIAS | EPI_RELU;
    g.bias = b_host[i];
    for (int j = 0; j < s; ++j) {
      const int t = L.frames[L.slot_begin[q] + j];
      plan.add_seg(x + (size_t)t * F, ldx, W_host[i] + (size_t)j * F, s * F, F);
    }
  }
  const RelMap map = make_relmap(L);
  const int R = L.R;
  const size_t act_f4 = (size_t)M * L.n_rel * (H / 4);      // the largest float4 index the kernel forms
  return submit_fwd(plan, S(stream), [=](cudaStream_t st) -> int {
    pre_launch("relsum", st);
    if (H % 4 == 0 && aligned16(act) && aligned16(feat_rel) && act_f4 < (1ull << 31))
      launch_kernel(relsum_v4_kernel, blocks_for((size_t)M * R * (H / 4), 256), 256, 0, st,
                    reinterpret_cast<const float4*>(act), reinterpret_cast<float4*>(feat_rel), M, H / 4, map);
    else
      launch_kernel(relsum_kernel, blocks_for((size_t)M * R * H, 256), 256, 0, st, act, feat_rel, M, H, map);
    return after_launch();
  });
}

size_t ta3n_trn_bwd_workspace_bytes(int M, int F, int H, const ta3n_relation_table* tab) {
  RelLayout L;
  if (parse_table(tab, &L) != TA3N_OK) return 0;
  (void)F;
  return Arena::round((size_t)L.n_rel * M * H * sizeof(float)) + splitk_bytes(L.n_slots) +
         colsum_bytes((size_t)L.R * H);
}

int ta3n_trn_bwd(const float* x, int M, int F, int H, const ta3n_relation_table* tab,
                 const float* const* W_host, int relu_input, const float* act, const float* d_feat_rel,
                 float* const* dW_host, float* const* db_host, float* dx, int accumulate_dx, void* workspace,
                 size_t workspace_bytes, ta3n_stream_t stream) {
  RelLayout L;
  TA3N_TRY(parse_table(tab, &L));
  TA3N_REQUIRE(M >= 0 && F > 0 && H > 0, "bad sizes");
  TA3N_REQUIRE(dW_host && db_host, "null gradient tables");
  cudaStream_t st = S(stream);
  if (M == 0) {
    for (int i = 0; i < L.R; ++i) {
      TA3N_CUDA(cudaMemsetAsync(dW_host[i], 0, sizeof(float) * H * L.scale_size[i] * F, st));
      TA3N_CUDA(cudaMemsetAsync(db_host[i], 0, sizeof(float) * H, st));
    }
    return TA3N_OK;
  }
  TA3N_REQUIRE(x && W_host && act && d_feat_rel, "null pointer");
  const int ldx = L.T * F;
  const size_t plane = (size_t)M * H;
  Arena arena(workspace, workspace_bytes);
  float* dz = arena.floats(plane * L.n_rel);
  if (!dz) return fail(TA3N_ERR_WORKSPACE, "ta3n_trn_bwd: workspace too small (%zu bytes)", workspace_bytes);

  const RelMap map = make_relmap(L);
  pre_launch("dz", st);
  if (H % 4 == 0 && aligned16(act) && aligned16(d_feat_rel) && aligned16(dz) && plane * L.n_rel / 4 < (1ull << 31))
    launch_kernel(dz_v4_kernel, blocks_for(plane * L.n_rel / 4, 256), 256, 0, st, reinterpret_cast<const float4*>(act),
                  reinterpret_cast<const float4*>(d_feat_rel), reinterpret_cast<float4*>(dz), M, H / 4, map);
  else
    launch_kernel(dz_kernel, blocks_for(plane * L.n_rel, 256), 256, 0, st, act, d_feat_rel, dz, M, H, map);
  TA3N_TRY(after_launch());

  {  // wgrad: dW_i[:, jF:(j+1)F] = sum_r dz_{i,r}^T x[:, tau_{i,r}[j], :]
    GemmPlan plan;
    plan.label = "trn_wgrad";
    plan.a_kmaj = false;
    plan.b_kmaj = false;
    plan.load_flags = relu_input ? LD_RELU_B : 0;
    for (int i = 0; i < L.R; ++i) {
      const int s = L.scale_size[i];
      TA3N_REQUIRE(dW_host[i] && db_host[i], "null gradient pointer");
      for (int j = 0; j < s; ++j) {
        plan.add_group(H, F, dW_host[i] + (size_t)j * F, s * F);
        for (int q = L.rel_begin[i]; q < L.rel_begin[i + 1]; ++q) {
          const int t = L.frames[L.slot_begin[q] + j];
          plan.add_seg(dz + q * plane, H, x + (size_t)t * F, ldx, M);
        }
      }
    }
    TA3N_TRY(submit_wgrad(plan, st, &arena));
  }
  {  // db_i = sum_r colsum(dz_{i,r})
    ColsumPlan cs;
    for (int i = 0; i < L.R; ++i) {
      cs.add(db_host[i], H, H);
      for (int q = L.rel_begin[i]; q < L.rel_begin[i + 1]; ++q) cs.seg(dz + q * plane, M);
    }
    TA3N_TRY(submit_colsum(cs, st, &arena));
  }
  if (dx) {  // dgrad, deterministic per frame: dx[:, t, :] = sum_{(q,j): tau_q[j]=t} dz_q W_i[:, jF:(j+1)F]
    GemmPlan plan;
    plan.label = "trn_dgrad";
    plan.precise_dgrad = true;
    plan.a_kmaj = true;
    plan.b_kmaj = false;
    std::vector<int> untouched;
    for (int t = 0; t < L.T; ++t) {
      bool any = false;
      for (int q = 0; q < L.n_rel && !any; ++q)
        for (int j = 0; j < L.scale_size[L.rel_scale[q]]; ++j)
          if (L.frames[L.slot_begin[q] + j] == t) any = true;
      if (!any) {
        untouched.push_back(t);
        continue;
      }
      Group& g = plan.add_group(M, F, dx + (size_t)t * F, ldx);
      if (relu_input) {
        g.flags |= EPI_GATE;
        g.gate = x + (size_t)t * F;
        g.ldgate = ldx;
      }
      if (accumulate_dx) g.flags |= EPI_ACCUM;
      for (int q = 0; q < L.n_rel; ++q) {
        const int i = L.rel_scale[q], s = L.scale_size[i];
        for (int j = 0; j < s; ++j)
          if (L.frames[L.slot_begin[q] + j] == t) plan.add_seg(dz + q * plane, H, W_host[i] + (size_t)j * F, s * F, H);
      }
    }
    if (!accumulate_dx)
      for (int t : untouched)   // frames no relation reads get a zero gradient
        TA3N_CUDA(cudaMemset2DAsync(dx + (size_t)t * F, sizeof(float) * ldx, 0, sizeof(float) * F, M, st));
    TA3N_TRY(run_gemm(plan, st));
  }
  return TA3N_OK;
}

// ------------------------------------------------------------------------------------------------
// relation discriminators + attention + pooling      models.py:472-488, 351-357, 379-388, 651-652
// ------------------------------------------------------------------------------------------------
int ta3n_relattn_fwd(const float* feat_rel, int M, int R, int H, const float* const* W1_host,
                     const float* const* b1_host, const float* const* W2_host, const float* const* b2_host,
                     int use_attn, float* hidden, float* pred_rel, float* attn, float* feat_video,
                     ta3n_stream_t stream) {
  TA3N_REQUIRE(M >= 0 && R >= 1 && R <= kMaxScales && H > 0, "bad sizes");
  if (M == 0) return TA3N_OK;
  TA3N_REQUIRE(feat_rel && W1_host && b1_host && W2_host && b2_host && hidden && pred_rel && attn && feat_video,
               "null pointer");
  GemmPlan plan;
    plan.label = "relattn_fwd";
    plan.precise = true;
  PtrTable w2, b2;
  memset(&w2, 0, sizeof(w2));
  memset(&b2, 0, sizeof(b2));
  for (int i = 0; i < R; ++i) {
    TA3N_REQUIRE(W1_host[i] && b1_host[i] && W2_host[i] && b2_host[i], "null weight pointer");
    Group& g = plan.add_group(M, H, hidden + (size_t)i * M * H, H);
    g.flags = EPI_BIAS | EPI_RELU;
    g.bias = b1_host[i];
    plan.add_seg(feat_rel + (size_t)i * H, R * H, W1_host[i], H, H);
    w2.p[i] = W2_host[i];
    b2.p[i] = b2_host[i];
  }
  TA3N_TRY(run_gemm(plan, S(stream)));
  pre_launch("relattn_fwd", S(stream));
  const int rel_threads = 32 * (R < kRelWarps ? R : kRelWarps);
  launch_kernel(relattn_fwd_kernel, M, rel_threads, 0, S(stream), feat_rel, hidden, M, R, H, w2, b2, use_attn, pred_rel, attn,
                                                       feat_video);
  return after_launch();
}

size_t ta3n_relattn_bwd_workspace_bytes(int M, int R, int H) {
  return Arena::round((size_t)M * R * 2 * sizeof(float)) + Arena::round((size_t)R * M * H * sizeof(float)) +
         splitk_bytes(2 * R) + colsum_bytes((size_t)R * (3 * H + 2));
}

int ta3n_relattn_bwd(const float* feat_rel, int M, int R, int H, const float* const* W1_host,
                     const float* const* W2_host, int use_attn, const float* hidden, const float* pred_rel,
                     const float* attn, const float* g_feat_video, const float* g_pred_rel, const float* g_attn,
                     float beta, float* d_feat_rel, float* const* dW1_host, float* const* db1_host,
                     float* const* dW2_host, float* const* db2_host, void* workspace, size_t workspace_bytes,
                     ta3n_stream_t stream) {
  TA3N_REQUIRE(M >= 0 && R >= 1 && R <= kMaxScales && H > 0, "bad sizes");
  TA3N_REQUIRE(dW1_host && db1_host && dW2_host && db2_host, "null gradient tables");
  // use_attn: 0 = plain sum, 1 = TransAttn (weights derived from pred_rel; their gradient flows into the logits),
  //           2 = the weights in `attn` come from elsewhere ('general' attention): only the (w + 1) scaling of G here,
  //               the weights' own gradient is ta3n_general_attn_bwd's business (g_attn is ignored)
  TA3N_REQUIRE(use_attn >= 0 && use_attn <= 2, "use_attn must be 0, 1 or 2");
  cudaStream_t st = S(stream);
  if (M == 0) {
    for (int i = 0; i < R; ++i) {
      TA3N_CUDA(cudaMemsetAsync(dW1_host[i], 0, sizeof(float) * H * H, st));
      TA3N_CUDA(cudaMemsetAsync(db1_host[i], 0, sizeof(float) * H, st));
      TA3N_CUDA(cudaMemsetAsync(dW2_host[i], 0, sizeof(float) * 2 * H, st));
      TA3N_CUDA(cudaMemsetAsync(db2_host[i], 0, sizeof(float) * 2, st));
    }
    return TA3N_OK;
  }
  TA3N_REQUIRE(feat_rel && W1_host && W2_host && hidden && pred_rel && attn && g_feat_video && d_feat_rel,
               "null pointer");
  Arena arena(workspace, workspace_bytes);
  float* Pt = arena.floats((size_t)M * R * 2);
  float* dHid = arena.floats((size_t)R * M * H);
  if (!Pt || !dHid)
    return fail(TA3N_ERR_WORKSPACE, "ta3n_relattn_bwd: workspace too small (%zu bytes)", workspace_bytes);

  PtrTable w2;
  memset(&w2, 0, sizeof(w2));
  for (int i = 0; i < R; ++i) w2.p[i] = W2_host[i];
  pre_launch("relattn_bwd_pre", st);
  launch_kernel(relattn_bwd_pre_kernel, M, 32 * (R < kRelWarps ? R : kRelWarps), 0, st, 
      feat_rel, hidden, pred_rel, g_feat_video, g_pred_rel, g_attn, M, R, H, w2, use_attn == 1 ? 1 : 0, Pt, dHid);
  TA3N_TRY(after_launch());

  {  // weight gradients of both layers of every relation discriminator
    GemmPlan plan;
    plan.label = "relattn_wgrad";
    plan.a_kmaj = false;
    plan.b_kmaj = false;
    for (int i = 0; i < R; ++i) {
      plan.add_group(H, H, dW1_host[i], H);
      plan.add_seg(dHid + (size_t)i * M * H, H, feat_rel + (size_t)i * H, R * H, M);
    }
    TA3N_TRY(submit_wgrad(plan, st, &arena));
  }
  {
    ColsumPlan cs;
    for (int i = 0; i < R; ++i) {
      cs.add_weighted(dW2_host[i], H, 2, H, H, R * 2);           // dW2_i [2,H] = Pt_i^T hidden_i
      cs.seg(hidden + (size_t)i * M * H, M, Pt + (size_t)i * 2);
      cs.add(db2_host[i], 2, R * 2);
      cs.seg(Pt + (size_t)i * 2, M);
      cs.add(db1_host[i], H, H);
      cs.seg(dHid + (size_t)i * M * H, M);
    }
    TA3N_TRY(submit_colsum(cs, st, &arena));
  }
  {  // d_feat_rel[:, i, :] = (w_i + 1) G - beta * dHid_i W1_i
    GemmPlan plan;
    plan.label = "relattn_dgrad";
    plan.precise_dgrad = true;
    plan.a_kmaj = true;
    plan.b_kmaj = false;
    for (int i = 0; i < R; ++i) {
      Group& g = plan.add_group(M, H, d_feat_rel + (size_t)i * H, R * H);
      g.alpha = -beta;
      g.flags = EPI_ADDROW;
      g.add = g_feat_video;
      g.ldadd = H;
      if (use_attn) {
        g.rowscale = attn + i;
        g.rs_stride = R;
        g.rs_bias = 1.0f;
      }
      plan.add_seg(dHid + (size_t)i * M * H, H, W1_host[i], H, H);
    }
    TA3N_TRY(run_gemm(plan, st));
  }
  if (!use_attn && g_attn) {
    pre_launch("attn_placeholder_bwd", st);
    launch_kernel(attn_placeholder_bwd_kernel, blocks_for((size_t)M * R, 256), 256, 0, st, g_attn, d_feat_rel, M, R, H);
    TA3N_TRY(after_launch());
  }
  return TA3N_OK;
}

// ------------------------------------------------------------------------------------------------
// 'general' attention over the relation features          models.py:320-325, 359-366, 379-388, 651
// ------------------------------------------------------------------------------------------------
int ta3n_general_attn_fwd(const float* feat_rel, int M, int R, int H, const float* W1, const float* b1,
                          const float* w2, const float* b2, float* hidden, float* attn, float* feat_video,
                          ta3n_stream_t stream) {
  TA3N_REQUIRE(M >= 0 && R >= 1 && R <= kMaxScales && H > 0, "bad sizes");
  if (M == 0) return TA3N_OK;
  TA3N_REQUIRE(feat_rel && W1 && b1 && w2 && b2 && hidden && attn && feat_video, "null pointer");
  {  // hidden [M*R, H] = feat_rel W1^T + b1   (tanh is applied by the row kernel)
    GemmPlan plan;
    plan.label = "general_attn_fwd";
    plan.precise = true;
    Group& g = plan.add_group(M * R, H, hidden, H);
    g.flags = EPI_BIAS;
    g.bias = b1;
    plan.add_seg(feat_rel, H, W1, H, H);
    TA3N_TRY(run_gemm(plan, S(stream)));
  }
  pre_launch("general_attn_rows", S(stream));
  launch_kernel(general_attn_fwd_kernel, M, 32 * (R < kRelWarps ? R : kRelWarps), 0, S(stream), feat_rel, hidden, M, R,
                H, w2, b2, attn, feat_video);
  return after_launch();
}

size_t ta3n_general_attn_bwd_workspace_bytes(int M, int R, int H) {
  return Arena::round((size_t)M * R * H * sizeof(float)) + Arena::round((size_t)M * R * sizeof(float)) +
         splitk_bytes(1) + colsum_bytes((size_t)2 * H + 1);
}

int ta3n_general_attn_bwd(const float* feat_rel, int M, int R, int H, const float* W1, const float* w2,
                          const float* hidden, const float* attn, const float* g_feat_video, const float* g_attn,
                          float* d_feat_rel, float* dW1, float* db1, float* dw2, float* db2, void* workspace,
                          size_t workspace_bytes, ta3n_stream_t stream) {
  TA3N_REQUIRE(M >= 0 && R >= 1 && R <= kMaxScales && H > 0, "bad sizes");
  TA3N_REQUIRE(dW1 && db1 && dw2 && db2, "null gradient pointer");
  cudaStream_t st = S(stream);
  if (M == 0) {
    TA3N_CUDA(cudaMemsetAsync(dW1, 0, sizeof(float) * H * H, st));
    TA3N_CUDA(cudaMemsetAsync(db1, 0, sizeof(float) * H, st));
    TA3N_CUDA(cudaMemsetAsync(dw2, 0, sizeof(float) * H, st));
    TA3N_CUDA(cudaMemsetAsync(db2, 0, sizeof(float), st));
    return TA3N_OK;
  }
  TA3N_REQUIRE(feat_rel && W1 && w2 && hidden && attn && g_feat_video && d_feat_rel, "null pointer");
  Arena arena(workspace, workspace_bytes);
  float* d_pre = arena.floats((size_t)M * R * H);
  float* d_s = arena.floats((size_t)M * R);
  if (!d_pre || !d_s)
    return fail(TA3N_ERR_WORKSPACE, "ta3n_general_attn_bwd: workspace too small (%zu bytes)", workspace_bytes);
  pre_launch("general_attn_bwd_rows", st);
  launch_kernel(general_attn_bwd_kernel, M, 32 * (R < kRelWarps ? R : kRelWarps), 0, st, feat_rel, hidden, attn,
                g_feat_video, g_attn, M, R, H, w2, d_s, d_pre);
  TA3N_TRY(after_launch());
  {  // dW1 [H,H] = d_pre^T feat_rel
    GemmPlan plan;
    plan.label = "general_attn_wgrad";
    plan.a_kmaj = false;
    plan.b_kmaj = false;
    plan.add_group(H, H, dW1, H);
    plan.add_seg(d_pre, H, feat_rel, H, M * R);
    TA3N_TRY(submit_wgrad(plan, st, &arena));
  }
  {  // dw2 [1,H] = d_s^T hidden, db2 = sum d_s, db1 = column sums of d_pre
    ColsumPlan cs;
    cs.add_weighted(dw2, H, 1, H, H, 1);
    cs.seg(hidden, M * R, d_s);
    cs.add(db2, 1, 1);
    cs.seg(d_s, M * R);
    cs.add(db1, H, H);
    cs.seg(d_pre, M * R);
    TA3N_TRY(submit_colsum(cs, st, &arena));
  }
  {  // d_feat_rel += d_pre W1
    GemmPlan plan;
    plan.label = "general_attn_dgrad";
    plan.precise_dgrad = true;
    plan.a_kmaj = true;
    plan.b_kmaj = false;
    Group& g = plan.add_group(M * R, H, d_feat_rel, H);
    g.flags = EPI_ACCUM;
    plan.add_seg(d_pre, H, W1, H, H);
    TA3N_TRY(run_gemm(plan, st));
  }
  return TA3N_OK;
}

// ------------------------------------------------------------------------------------------------
// video head                                                                models.py:679-687
// ------------------------------------------------------------------------------------------------
int ta3n_video_head_fwd(const float* feat_video, int M, int H, int C, const float* Wc, const float* bc,
                        const ta3n_dropout* drop, float* dropped, float* pred, ta3n_stream_t stream) {
  TA3N_REQUIRE(M >= 0 && H > 0 && C > 0, "bad sizes");
  if (M == 0) return TA3N_OK;
  TA3N_REQUIRE(feat_video && Wc && bc && dropped && pred, "null pointer");
  const DropArgs d = make_drop(drop);
  // one kernel: Dropout (writes `dropped`, needed by the video discriminator and by backward) + Linear(H -> C)
  TA3N_REQUIRE(feat_video != dropped, "dropped must not alias feat_video");
  return launch_head_fwd(feat_video, H, Wc, bc, pred, C, M, H, C, S(stream), &d, dropped);
}

size_t ta3n_video_head_bwd_workspace_bytes(int M, int H, int C) {
  (void)M;
  return splitk_bytes(1) + colsum_bytes((size_t)C * (H + 1));
}

int ta3n_video_head_bwd(const float* dropped, int M, int H, int C, const float* Wc, const ta3n_dropout* drop,
                        const float* g_pred, const float* d_dropped_extra, const float* g_feat_video_ext,
                        float grad_scale, float* d_feat_video, float* dWc, float* dbc, void* workspace,
                        size_t workspace_bytes, ta3n_stream_t stream) {
  TA3N_REQUIRE(M >= 0 && H > 0 && C > 0, "bad sizes");
  TA3N_REQUIRE(dWc && dbc, "null gradient pointer");
  cudaStream_t st = S(stream);
  if (M == 0 || g_pred == nullptr) {
    TA3N_CUDA(cudaMemsetAsync(dWc, 0, sizeof(float) * C * H, st));
    TA3N_CUDA(cudaMemsetAsync(dbc, 0, sizeof(float) * C, st));
  }
  if (M == 0) return TA3N_OK;
  TA3N_REQUIRE(dropped && Wc, "null pointer");
  if (d_feat_video) {
    const DropArgs d = make_drop(drop);
    pre_launch("video_head_bwd", st);
    launch_kernel(video_head_bwd_kernel, blocks_for((size_t)M * H, 256), 256, 0, st, g_pred, C, Wc, d_dropped_extra,
                  g_feat_video_ext, grad_scale, d, d_feat_video, M, H);
    TA3N_TRY(after_launch());
  }
  if (g_pred) {
    Arena arena(workspace, workspace_bytes);
    if (C <= 32) {   // dWc [C,H] = g_pred^T dropped: skinny -> weighted column sum
      ColsumPlan cs;
      cs.add_weighted(dWc, H, C, H, H, C);
      cs.seg(dropped, M, g_pred);
      cs.add(dbc, C, C);
      cs.seg(g_pred, M);
      TA3N_TRY(submit_colsum(cs, st, &arena));
    } else {
      GemmPlan plan;
      plan.label = "video_head_wgrad";
      plan.a_kmaj = false;
      plan.b_kmaj = false;
      plan.add_group(C, H, dWc, H);
      plan.add_seg(g_pred, C, dropped, H, M);
      TA3N_TRY(submit_wgrad(plan, st, &arena));
      ColsumPlan cs;
      cs.add(dbc, C, C);
      cs.seg(g_pred, M);
      TA3N_TRY(submit_colsum(cs, st, &arena));
    }
  }
  return TA3N_OK;
}

// ------------------------------------------------------------------------------------------------
// fused loss heads (main.py:446, 508-538, 559-562; loss.py:15-25)
// ------------------------------------------------------------------------------------------------
size_t ta3n_loss_workspace_bytes(int M) { return Arena::round((size_t)M * sizeof(float)) + 256; }

int ta3n_loss_fwd_bwd(const float* pred_video, const long long* labels, const float* pred_rel,
                      const float* pred_dom_video, const float* pred_frame, int Bs, int Bt, int T, int R, int C,
                      float gamma, int flags, const int* valid_rows, float* loss, float* g_pred_video,
                      float* g_pred_rel, float* g_pred_dom_video, float* g_pred_frame, void* workspace,
                      size_t workspace_bytes, ta3n_stream_t stream) {
  TA3N_REQUIRE(Bs >= 1 && Bt >= 0 && T >= 1 && R >= 1 && C >= 1, "bad sizes");
  TA3N_REQUIRE(pred_video && labels && pred_rel && pred_dom_video && pred_frame && loss, "null input");
  TA3N_REQUIRE(g_pred_video && g_pred_rel && g_pred_dom_video && g_pred_frame, "null gradient output");
  const int M = Bs + Bt;
  Arena arena(workspace, workspace_bytes);
  float* row_loss = arena.floats(M);
  if (!row_loss) return fail(TA3N_ERR_WORKSPACE, "ta3n_loss_fwd_bwd: workspace too small (%zu bytes)", workspace_bytes);
  pre_launch("loss_heads", S(stream));
  launch_kernel(loss_heads_kernel, blocks_for((size_t)M * 32, 256), 256, 0, S(stream), 
      pred_video, labels, pred_rel, pred_dom_video, pred_frame, Bs, M, T, R, C, gamma, flags, valid_rows,
      g_pred_video, g_pred_rel, g_pred_dom_video, g_pred_frame, row_loss);
  TA3N_TRY(after_launch());
  pre_launch("loss_reduce", S(stream));
  launch_kernel(loss_reduce_kernel, 1, 1024, 0, S(stream), row_loss, M, loss);
  return after_launch();
}

int ta3n_counter_inc(uint64_t* counter, ta3n_stream_t stream) {
  TA3N_REQUIRE(counter != nullptr, "null counter");
  pre_launch("counter_inc", S(stream));
  launch_kernel(counter_inc_kernel, 1, 1, 0, S(stream), reinterpret_cast<unsigned long long*>(counter));
  return after_launch();
}

// ------------------------------------------------------------------------------------------------
// ens_DA='MCD' loss terms (main.py:446-448, 548-556; loss.py:29-30)
// ------------------------------------------------------------------------------------------------
int ta3n_ce_loss_fwd_bwd(const float* pred, const long long* labels, int rows, int C, const int* valid_rows,
                         float* loss, float* g_pred, ta3n_stream_t stream) {
  TA3N_REQUIRE(rows >= 0 && C >= 1, "bad sizes");
  if (rows == 0) return TA3N_OK;
  TA3N_REQUIRE(pred && labels && loss && g_pred, "null pointer");
  pre_launch("ce_loss", S(stream));
  launch_kernel(ce_loss_kernel, 1, kMcdThreads, 0, S(stream), pred, labels, rows, C, valid_rows, loss, g_pred);
  return after_launch();
}

int ta3n_mcd_loss_fwd_bwd(const float* pred1, const float* pred2, int rows, int C, const int* valid_rows, float* loss,
                          float* g_pred1, float* g_pred2, float* g_move1, ta3n_stream_t stream) {
  TA3N_REQUIRE(rows >= 0 && C >= 1, "bad sizes");
  if (rows == 0) return TA3N_OK;
  TA3N_REQUIRE(pred1 && pred2 && loss && g_pred1 && g_pred2, "null pointer");
  TA3N_REQUIRE(g_pred1 != g_pred2 && g_move1 != g_pred1 && g_move1 != g_pred2, "gradient buffers must not alias");
  pre_launch("mcd_loss", S(stream));
  launch_kernel(mcd_loss_kernel, 1, kMcdThreads, 0, S(stream), pred1, pred2, rows, C, valid_rows, loss, g_pred1,
                g_pred2, g_move1);
  return after_launch();
}

int ta3n_accumulate(float* dst, const float* src, long long n, ta3n_stream_t stream) {
  TA3N_REQUIRE(n >= 0, "bad size");
  if (n == 0) return TA3N_OK;
  TA3N_REQUIRE(dst && src, "null pointer");
  TA3N_REQUIRE(aligned16(dst) && aligned16(src), "buffers must be 16-byte aligned");
  pre_launch("accumulate", S(stream));
  launch_kernel(accumulate_kernel, blocks_for((size_t)(n + 3) / 4, 256), 256, 0, S(stream), dst, src, (size_t)n);
  return after_launch();
}

// ------------------------------------------------------------------------------------------------
// device-resident input pipeline (include/ta3n_b200.h: ta3n_gather_batch)
// ------------------------------------------------------------------------------------------------
int ta3n_gather_batch(const float* bank_s, long long n_rows_s, const int* rows_s, const long long* labels_s,
                      long long n_epoch_s, int batch_s, float* x_s, long long* y_s,
                      const float* bank_t, long long n_rows_t, const int* rows_t, long long n_epoch_t, int batch_t,
                      float* x_t, long long row_floats, int* valid_rows, unsigned int* state, ta3n_stream_t stream) {
  TA3N_REQUIRE(batch_s >= 1 && batch_t >= 1 && batch_s + batch_t <= 65535, "batch sizes must be >= 1, together <= 65535");
  TA3N_REQUIRE(row_floats >= 4 && row_floats % 4 == 0, "row_floats must be a positive multiple of 4 (16-byte rows)");
  TA3N_REQUIRE(n_epoch_s >= 1 && n_epoch_t >= 1, "empty epoch");
  TA3N_REQUIRE(n_rows_s >= 1 && n_rows_t >= 1 && n_rows_s <= INT32_MAX && n_rows_t <= INT32_MAX,
               "bank rows must be in [1, 2^31) (row lists are int32)");
  TA3N_REQUIRE(n_rows_s <= INT64_MAX / row_floats && n_rows_t <= INT64_MAX / row_floats, "bank too large");
  TA3N_REQUIRE(bank_s && rows_s && labels_s && x_s && y_s, "null source pointer");
  TA3N_REQUIRE(bank_t && rows_t && x_t, "null target pointer");
  TA3N_REQUIRE(valid_rows && state, "null valid_rows / state");
  TA3N_REQUIRE(aligned16(bank_s) && aligned16(bank_t) && aligned16(x_s) && aligned16(x_t),
               "banks and slots must be 16-byte aligned");
  GatherDomain s{reinterpret_cast<const float4*>(bank_s), n_rows_s, rows_s, labels_s, n_epoch_s,
                 reinterpret_cast<float4*>(x_s), y_s, batch_s};
  GatherDomain t{reinterpret_cast<const float4*>(bank_t), n_rows_t, rows_t, nullptr, n_epoch_t,
                 reinterpret_cast<float4*>(x_t), nullptr, batch_t};
  const long long row_f4 = row_floats / 4;
  const dim3 grid((unsigned)((row_f4 + kGatherChunk - 1) / kGatherChunk), (unsigned)(batch_s + batch_t));
  TA3N_REQUIRE(grid.x <= 65535u, "rows too long");
  pre_launch("gather_batch", S(stream));
  launch_kernel(gather_batch_kernel, grid, kGatherThreads, 0, S(stream), s, t, row_f4, valid_rows, state);
  return after_launch();
}

int ta3n_gather_rows(const float* bank, long long n_rows, const int* rows, const long long* labels, long long n_epoch,
                     int batch, float* x, long long* y, long long row_floats, int* valid_rows, unsigned int* state,
                     ta3n_stream_t stream) {
  TA3N_REQUIRE(batch >= 1 && batch <= 65535, "batch must be in [1, 65535]");
  TA3N_REQUIRE(row_floats >= 4 && row_floats % 4 == 0, "row_floats must be a positive multiple of 4 (16-byte rows)");
  TA3N_REQUIRE(n_epoch >= 1, "empty epoch");
  TA3N_REQUIRE(n_rows >= 1 && n_rows <= INT32_MAX, "bank rows must be in [1, 2^31) (row lists are int32)");
  TA3N_REQUIRE(n_rows <= INT64_MAX / row_floats, "bank too large");
  TA3N_REQUIRE(bank && rows && labels && x && y, "null pointer");
  TA3N_REQUIRE(valid_rows && state, "null valid_rows / state");
  TA3N_REQUIRE(aligned16(bank) && aligned16(x), "bank and slot must be 16-byte aligned");
  GatherDomain s{reinterpret_cast<const float4*>(bank), n_rows, rows, labels, n_epoch, reinterpret_cast<float4*>(x),
                 y, batch};
  GatherDomain none{nullptr, 0, nullptr, nullptr, 0, nullptr, nullptr, 0};     // batch 0: no slot row, no count
  const long long row_f4 = row_floats / 4;
  const dim3 grid((unsigned)((row_f4 + kGatherChunk - 1) / kGatherChunk), (unsigned)batch);
  TA3N_REQUIRE(grid.x <= 65535u, "rows too long");
  pre_launch("gather_rows", S(stream));
  launch_kernel(gather_batch_kernel, grid, kGatherThreads, 0, S(stream), s, none, row_f4, valid_rows, state);
  return after_launch();
}

// ------------------------------------------------------------------------------------------------
// validation head (include/ta3n_b200.h: ta3n_eval_head)
// ------------------------------------------------------------------------------------------------
static int eval_grid(int rows) { return (rows + kEvalRows - 1) / kEvalRows; }

size_t ta3n_eval_workspace_bytes(int rows) {
  return rows < 1 ? 0 : Arena::round((size_t)eval_grid(rows) * sizeof(EvalPartial));
}

int ta3n_eval_head(const float* feat_video, int rows, int H, int C, const float* Wc, const float* bc,
                   const long long* labels, const float* class_weight, const int* valid_rows, int n_k,
                   const int* k_host, const float* attn, int R, long long attn_ld, float* logits,
                   ta3n_eval_accum* accum, long long* confusion, float* scores, float* attn_out, long long n_epoch,
                   void* workspace, size_t workspace_bytes, ta3n_stream_t stream) {
  TA3N_REQUIRE(rows >= 1 && H >= 1 && C >= 1, "rows, H and C must be >= 1");
  TA3N_REQUIRE(n_k >= 1 && n_k <= kEvalMaxK && k_host, "between 1 and 4 top-k values");
  for (int i = 0; i < n_k; ++i)
    if (k_host[i] < 1 || k_host[i] > C)
      return fail(TA3N_ERR_INVALID, "ta3n_eval_head: top-k value %d is outside [1, C=%d]", k_host[i], C);
  TA3N_REQUIRE(feat_video && Wc && bc && labels && valid_rows && logits && accum, "null pointer");
  TA3N_REQUIRE(reinterpret_cast<uintptr_t>(accum) % 8 == 0 && reinterpret_cast<uintptr_t>(confusion) % 8 == 0,
               "accum and confusion must be 8-byte aligned");
  TA3N_REQUIRE(!(scores || attn_out) || n_epoch >= 1, "epoch buffers need n_epoch >= 1");
  TA3N_REQUIRE(!attn_out || (attn && R >= 1 && attn_ld >= R), "attn_out needs attn [rows, R] with attn_ld >= R");
  const int grid = eval_grid(rows);
  const size_t need = ta3n_eval_workspace_bytes(rows);
  TA3N_REQUIRE(workspace && reinterpret_cast<uintptr_t>(workspace) % 16 == 0, "null or misaligned workspace");
  if (workspace_bytes < need)
    return fail(TA3N_ERR_WORKSPACE, "ta3n_eval_head: workspace too small (%zu < %zu bytes)", workspace_bytes, need);
  const size_t x_bytes = (size_t)kEvalRows * H * sizeof(float), w_row = (size_t)(H + 1) * sizeof(float);
  if (x_bytes + w_row > kEvalSmemBudget)
    return fail(TA3N_ERR_UNSUPPORTED, "ta3n_eval_head: H=%d is too wide for the shared-memory staging", H);
  EvalArgs a;
  a.feat = feat_video, a.Wc = Wc, a.bc = bc, a.labels = labels, a.class_weight = class_weight;
  a.valid_rows = valid_rows, a.attn = attn, a.logits = logits, a.accum = accum, a.confusion = confusion;
  a.scores = scores, a.attn_out = attn_out, a.n_epoch = n_epoch, a.attn_ld = attn_ld;
  a.rows = rows, a.H = H, a.C = C, a.R = R, a.n_k = n_k;
  a.c_tile = (int)std::min<size_t>((size_t)C, (kEvalSmemBudget - x_bytes) / w_row);
  for (int i = 0; i < kEvalMaxK; ++i) a.k[i] = i < n_k ? k_host[i] : 0;
  const size_t smem = x_bytes + (size_t)a.c_tile * w_row;
  {
    std::lock_guard<std::mutex> lock(device_mu());
    DeviceInfo* d = device_info();
    if (!d) return fail(TA3N_ERR_CUDA, "cudaGetDevice failed");
    if (!d->eval_configured) {
      TA3N_CUDA(cudaFuncSetAttribute(eval_head_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)kEvalSmemBudget));
      d->eval_configured = true;
    }
  }
  pre_launch("eval_head", S(stream));
  launch_kernel(eval_head_kernel, grid, kEvalThreads, smem, S(stream), a,
                reinterpret_cast<EvalPartial*>(workspace));
  return after_launch();
}

// ------------------------------------------------------------------------------------------------
// the training step (include/ta3n_b200.h: ta3n_step_*)
// ------------------------------------------------------------------------------------------------
size_t ta3n_step_workspace_bytes(const ta3n_step_desc* desc) {
  StepProgram P;
  if (build_step_program(desc, &P, /*dry=*/true) != TA3N_OK) return 0;
  // the column-sum partials follow the fixed scratch: carved by the same walk as in ta3n_step_run_phased, from an
  // arena that only hands out addresses (nothing is dereferenced)
  Arena partials(reinterpret_cast<void*>(uintptr_t(1) << 20), size_t(1) << 46);
  if (step_colsum_batches(P, &partials, [](const WColsumTable&, bool) { return TA3N_OK; }) != TA3N_OK) return 0;
  return P.scratch_bytes + partials.used;
}

int ta3n_step_run_phased(const ta3n_step_desc* desc, ta3n_stream_t stream) {
  StepProgram P;
  TA3N_TRY(build_step_program(desc, &P));
  cudaStream_t st = S(stream);
  const int n_row = (P.M + kRowVideos - 1) / kRowVideos;
  auto rows = [&](const char* label, int kind) {
    pre_launch(label, st);
    launch_kernel(video_row_kernel, n_row, kRowThreads, 0, st, P.tail, kind);
    return after_launch();
  };
  TA3N_TRY(run_gemm(P.g1, st));
  TA3N_TRY(run_gemm(P.g2, st));
  pre_launch("step_frame_rows", st);
  launch_kernel(frame_row_kernel, (P.MT + kRowFrames - 1) / kRowFrames, kRowThreads, 0, st, P.tail);
  TA3N_TRY(after_launch());
  TA3N_TRY(run_gemm(P.g3, st));
  TA3N_TRY(rows("step_relpool", ROW_RELPOOL));
  TA3N_TRY(run_gemm(P.g4a, st));
  TA3N_TRY(rows("step_heads", ROW_HEADS));
  TA3N_TRY(run_gemm(P.g4b, st));
  TA3N_TRY(rows("step_relbwd", ROW_RELBWD));
  TA3N_TRY(run_gemm(P.g5, st));
  TA3N_TRY(run_gemm(P.g6, st));
  TA3N_TRY(run_gemm(P.g7, st));
  // column sums: parts, then the fixed-order reduction (whose last launch also advances the dropout step counter)
  Arena arena(static_cast<char*>(desc->workspace) + P.scratch_bytes, desc->workspace_bytes - P.scratch_bytes);
  return step_colsum_batches(P, &arena, [&](const WColsumTable& tab, bool last) {
    int max_cb = 1, max_split = 1;
    for (int k = 0; k < tab.n_jobs; ++k) {
      max_cb = std::max(max_cb, (tab.job[k].N + 127) / 128);
      max_split = std::max(max_split, tab.job[k].nsplit);
    }
    pre_launch("step_colsum", st);
    launch_kernel(step_colsum_part_kernel, dim3(max_cb, tab.n_jobs, max_split), kRowThreads, 0, st, tab);
    TA3N_TRY(after_launch());
    pre_launch("step_colsum_reduce", st);
    launch_kernel(step_colsum_reduce_kernel, tab.n_jobs, kRowThreads, 0, st, tab,
                  reinterpret_cast<unsigned long long*>(last ? desc->step_counter : nullptr));
    return after_launch();
  });
}

// Host-only: the split-K factors the balanced planner (gemm_wgmma.cuh: plan_splitk_balanced) would choose for a
// precise forward launch of n_groups GEMMs C[M,N] += A[M,K] B[N,K]^T on `sms` SMs with `scratch_bytes` of forward
// scratch; ksplit_out[n_groups] receives them, makespan_out[2] = {unsplit, chosen} makespan of the LPT model in K-slab
// units.  No CUDA call: the planner's policy is testable on a machine without a GPU.
int ta3n_plan_forward_splits(int n_groups, const int* M, const int* N, const int* K, int sms, size_t scratch_bytes,
                             int* ksplit_out, double* makespan_out) {
  if (n_groups <= 0 || !M || !N || !K || !ksplit_out || sms <= 0)
    return fail(TA3N_ERR_INVALID, "ta3n_plan_forward_splits: bad arguments");
  GemmPlan plan;
  for (int i = 0; i < n_groups; ++i) {
    if (M[i] <= 0 || N[i] <= 0 || K[i] <= 0)
      return fail(TA3N_ERR_INVALID, "ta3n_plan_forward_splits: group %d has M=%d N=%d K=%d", i, M[i], N[i], K[i]);
    plan.add_group(M[i], N[i], nullptr, N[i]);
    plan.add_seg(nullptr, K[i], nullptr, K[i], K[i]);
  }
  std::vector<int> ones(n_groups, 1);
  const double before = x3_makespan(plan, ones, sms);
  // the arena only hands out addresses here (nothing is dereferenced); any non-null base will do
  Arena scratch(reinterpret_cast<void*>(uintptr_t(256)), scratch_bytes);
  plan_splitk_balanced(plan, &scratch, sms);
  std::vector<int> ks(n_groups);
  for (int i = 0; i < n_groups; ++i) ks[i] = ksplit_out[i] = plan.groups[i].ksplit;
  if (makespan_out) {
    makespan_out[0] = before;
    makespan_out[1] = x3_makespan(plan, ks, sms);
  }
  return TA3N_OK;
}

// ------------------------------------------------------------------------------------------------
// gradient all-reduce over peer / multicast memory (csrc/allreduce.cuh)
// ------------------------------------------------------------------------------------------------
size_t ta3n_allreduce_flag_bytes(int world) { return (size_t)2 * kArBlocks * (world > 0 ? world : 1) * sizeof(unsigned); }

int ta3n_allreduce_mean(float* const* peer_bufs_host, float* multicast_buf, uint32_t* const* peer_flags_host,
                        const uint64_t* seq_dev, int rank, int world, long long n, ta3n_stream_t stream) {
  TA3N_REQUIRE(peer_bufs_host && peer_flags_host && seq_dev, "null argument");
  TA3N_REQUIRE(world >= 1 && world <= kArMaxWorld && rank >= 0 && rank < world, "bad rank / world size");
  TA3N_REQUIRE(n > 0 && n % 4 == 0, "element count must be a positive multiple of 4");
  ArPeers P;
  memset(&P, 0, sizeof(P));
  for (int p = 0; p < world; ++p) {
    TA3N_REQUIRE(peer_bufs_host[p] && peer_flags_host[p], "null peer pointer");
    TA3N_REQUIRE((reinterpret_cast<uintptr_t>(peer_bufs_host[p]) & 15u) == 0, "buffers must be 16-byte aligned");
    P.buf[p] = peer_bufs_host[p];
    P.flags[p] = reinterpret_cast<unsigned*>(peer_flags_host[p]);
  }
  TA3N_REQUIRE((reinterpret_cast<uintptr_t>(multicast_buf) & 15u) == 0, "multicast mapping must be 16-byte aligned");
  pre_launch("allreduce_mean", S(stream));
  // CTAs of the kernel (each one is a participant of the two flag barriers): TA3N_AR_BLOCKS overrides the default
  static const int env_blocks = []() {
    const char* e = getenv("TA3N_AR_BLOCKS");
    return e ? atoi(e) : 0;
  }();
  // from three ranks on 64 CTAs: fewer barrier participants, still enough loads in flight; two ranks use the peer
  // path and want all 128 (chosen on an 8-GPU NVSwitch box of the previous generation; TA3N_AR_BLOCKS overrides)
  int blocks = env_blocks > 0 ? env_blocks : (world > 2 ? 64 : kArBlocks);
  blocks = std::max(1, std::min(blocks, kArBlocks));
  launch_kernel(allreduce_mean_kernel, blocks, kArThreads, 0, S(stream), P, multicast_buf,
                reinterpret_cast<const unsigned long long*>(seq_dev), rank, world, (size_t)(n / 4), 1.0f / (float)world);
  return after_launch();
}

// ---- optimizer step: clip_grad_norm_ + SGD-Nesterov over flat buffers (main.py:83, 578-583) ----
size_t ta3n_sgd_workspace_bytes(void) { return Arena::round(kSqnormBlocks * sizeof(float)); }

int ta3n_sgd_nesterov_step_masked(float* params, const float* grads, float* momentum_buf, long long n, const float* lr_dev,
                                  float momentum, float weight_decay, float max_norm, void* workspace,
                                  size_t workspace_bytes, float* stats, const float* active, ta3n_stream_t stream) {
  TA3N_REQUIRE(params && grads && momentum_buf && lr_dev && n > 0, "bad arguments");
  TA3N_REQUIRE(((reinterpret_cast<uintptr_t>(params) | reinterpret_cast<uintptr_t>(grads) |
                 reinterpret_cast<uintptr_t>(momentum_buf)) & 15) == 0, "flat buffers must be 16-byte aligned");
  TA3N_REQUIRE(momentum >= 0.f && weight_decay >= 0.f, "negative momentum / weight decay");
  TA3N_REQUIRE(active == nullptr || (reinterpret_cast<uintptr_t>(active) & 15) == 0, "active mask must be 16-byte aligned");
  float* partial = nullptr;
  if (max_norm > 0.f) {
    TA3N_REQUIRE(workspace != nullptr && workspace_bytes >= ta3n_sgd_workspace_bytes(), "workspace too small");
    partial = static_cast<float*>(workspace);
    pre_launch("sqnorm", S(stream));
    launch_kernel(sqnorm_partial_kernel, kSqnormBlocks, kOptThreads, 0, S(stream), grads, n, partial);
    TA3N_TRY(after_launch());
  }
  long long n4 = (n + 3) / 4;
  int blocks = static_cast<int>(std::min<long long>((n4 + kOptThreads - 1) / kOptThreads, 132 * 8));
  pre_launch("sgd_nesterov", S(stream));
  launch_kernel(sgd_nesterov_kernel, blocks, kOptThreads, 0, S(stream), params, grads, momentum_buf, n, lr_dev,
                momentum, weight_decay, max_norm, static_cast<const float*>(partial), kSqnormBlocks, stats, active);
  return after_launch();
}

int ta3n_sgd_nesterov_step(float* params, const float* grads, float* momentum_buf, long long n, const float* lr_dev,
                           float momentum, float weight_decay, float max_norm, void* workspace,
                           size_t workspace_bytes, float* stats, ta3n_stream_t stream) {
  return ta3n_sgd_nesterov_step_masked(params, grads, momentum_buf, n, lr_dev, momentum, weight_decay, max_norm, workspace,
                                       workspace_bytes, stats, nullptr, stream);
}

// ------------------------------------------------------------------------------------------------
int ta3n_gemm_tn(const float* A, const float* B, float* C, int M, int N, int K, ta3n_stream_t stream) {
  TA3N_REQUIRE(A && B && C && M > 0 && N > 0 && K > 0, "bad arguments");
  GemmPlan plan;
    plan.label = "gemm_tn";
    plan.precise = true;
  plan.add_group(M, N, C, N);
  plan.add_seg(A, K, B, K, K);
  return run_gemm(plan, S(stream));
}


int ta3n_gemm_ex(const float* A, int lda, int a_kmajor, const float* B, int ldb, int b_kmajor, float* C, int ldc,
                 int M, int N, int K, void* workspace, size_t workspace_bytes, ta3n_stream_t stream) {
  TA3N_REQUIRE(A && B && C && M > 0 && N > 0 && K > 0, "bad arguments");
  Arena arena(workspace, workspace_bytes);
  GemmPlan plan;
  plan.label = "gemm_ex";
  plan.a_kmaj = a_kmajor != 0;
  plan.b_kmaj = b_kmajor != 0;
  plan.add_group(M, N, C, ldc);
  plan.add_seg(A, lda, B, ldb, K);
  return run_gemm(plan, S(stream), workspace ? &arena : nullptr);
}

}  // extern "C"
