// train_stats.cuh -- the training meters (C ABI ta3n_train_stats_accumulate): the per-term losses and the top-k
// accuracy main.py's train() keeps in AverageMeters (main.py:446-571), recomputed from the logits the loss kernels
// read and folded into a device-resident epoch accumulator, so a training epoch needs a readback per log line only.
// Same fold as the validation head (eval.cuh): per-CTA partials, summed in CTA order by the last CTA to arrive.
#pragma once

#include "common.cuh"
#include "eval.cuh"

namespace ta3n {

constexpr int kStatsThreads = 256;
constexpr int kStatsRows = kStatsThreads / 32;    // one warp per video row

enum : int { STATS_REL = 1, STATS_VIDEO = 2, STATS_FRAME = 4, STATS_ENT = 8 };

struct TrainStatsArgs {
  const float* pred_video;      // [M, C]; target rows: the logits the attentive entropy reads
  const long long* labels;      // [Bs]
  const long long* labels_t;    // [Bt] or nullptr (use_target='Sv': the class CE and top-k cover the target rows too)
  double* prec_sum;             // [n_k] with labels_t: sum over steps of the top-k percent * vs, else nullptr
  const float* pred_rel;        // [M, R, 2]
  const float* pred_dom;        // [M, 2]
  const float* pred_frame;      // [M * T, 2]
  const float* pred2_s;         // [Bs, C] or nullptr (MCD: second classifier, pass 1)
  const float* pred2_t;         // [Bt, C] or nullptr (MCD: second classifier, pass 2)
  const float* loss;            // [1] the step's loss
  const int* valid_rows;        // [2] or nullptr
  const float* class_weight;    // [C] or nullptr
  ta3n_train_stats* accum;
  float dw[2];                  // domain weights {source, target}
  int Bs, Bt, T, R, C, flags, n_k;
  int k[kEvalMaxK];
};

// Sums of one CTA (or of the whole step), in this order.
enum : int { P_CWCE, P_CW, P_C2WCE, P_ENT, P_DIS, P_RWCE, P_RW, P_VWCE, P_VW, P_FWCE, P_FW, P_N };

struct TrainStatsPartial {
  double s[P_N];
  long long n_src;
  long long correct[kEvalMaxK];
};

// Softmax statistics of one logit row held by a warp (lane j takes classes j, j + 32, ...): max, log-sum-exp
// (shifted by the max, fp32 as the loss kernels compute them) and the NaN count.
struct RowStats {
  float mx, lse;
  int nan;
};
__device__ __forceinline__ RowStats row_stats(const float* z, int C, int lane) {
  RowStats r;
  float m = -INFINITY;
  int nan = 0;
  for (int j = lane; j < C; j += 32) {
    m = fmaxf(m, z[j]);                             // fmaxf skips NaN; the sum below still turns NaN
    nan += isnan(z[j]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  float se = 0.f;
  for (int j = lane; j < C; j += 32) se += expf(z[j] - m);
  r.mx = m;
  r.lse = logf(warp_sum(se));
  r.nan = warp_sum_i(nan);
  return r;
}

// -log softmax(z)_d of a two-logit domain row
__device__ __forceinline__ float domain_ce(const float* p, int d) {
  const Attn2 a = attn_from_logits(p[0], p[1]);
  return d ? -a.lq1 : -a.lq0;
}

// grid = ceil(M / kStatsRows), block = kStatsThreads.  Warp w of CTA b takes video row b * kStatsRows + w.
__global__ void __launch_bounds__(kStatsThreads)
train_stats_kernel(const __grid_constant__ TrainStatsArgs a, TrainStatsPartial* __restrict__ partials) {
  __shared__ double s_row[kStatsRows][P_N];
  __shared__ int s_rank[kStatsRows], s_src[kStatsRows];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int M = a.Bs + a.Bt;
  const int m = blockIdx.x * kStatsRows + warp;
  pdl_wait();
  const int vs = a.valid_rows ? max(0, min(a.valid_rows[0], a.Bs)) : a.Bs;
  const int vt = a.valid_rows ? max(0, min(a.valid_rows[1], a.Bt)) : a.Bt;
  const bool mcd = a.pred2_s != nullptr;

  double t[P_N];
#pragma unroll
  for (int i = 0; i < P_N; ++i) t[i] = 0.0;
  int rank = 0x7fffffff, src = 0;
  const int d = m >= a.Bs ? 1 : 0;
  const bool real = m < M && (d ? m - a.Bs < vt : m < vs);
  if (real) {
    const float* z = a.pred_video + (size_t)m * a.C;
    const RowStats rs = row_stats(z, a.C, lane);
    if (!d || a.labels_t) {
      // class CE (criterion, main.py:446) and the rank of the label (accuracy, main.py:565-567); under Sv the target
      // rows with their labels too (main.py:442-444)
      const long long y = d ? a.labels_t[m - a.Bs] : a.labels[m];
      const bool in_range = y >= 0 && y < a.C;
      const float zy = in_range ? z[y] : 0.f;
      int gt = 0, tie_before = 0;
      for (int j = lane; j < a.C; j += 32) {
        const float v = z[j];
        gt += v > zy;
        tie_before += (j < y) && (v == zy);
      }
      gt = warp_sum_i(gt);
      tie_before = warp_sum_i(tie_before);
      const double w = !in_range ? 1.0 : (a.class_weight ? (double)a.class_weight[y] : 1.0);
      t[P_CWCE] = in_range ? w * (double)(rs.mx + rs.lse - zy) : (double)NAN;
      t[P_CW] = w;
      if (mcd && !d) {                              // main.py:447-448: the same criterion on the second classifier
        const float* z2 = a.pred2_s + (size_t)m * a.C;
        const RowStats r2 = row_stats(z2, a.C, lane);
        t[P_C2WCE] = in_range ? w * (double)(r2.mx + r2.lse - z2[y]) : (double)NAN;
      }
      rank = (in_range && rs.nan == 0) ? gt + tie_before : 0x7fffffff;
      src = 1;
    }
    if (a.flags & STATS_ENT) {
      // loss.py:15-25 on cat(out_source, out_target) and pred_domain_all[1] (the video level): one row's product
      float hc = 0.f;
      for (int j = lane; j < a.C; j += 32) {
        const float lq = z[j] - rs.mx - rs.lse;
        hc -= expf(lq) * lq;
      }
      hc = warp_sum(hc);
      const Attn2 dv = attn_from_logits(a.pred_dom[(size_t)m * 2], a.pred_dom[(size_t)m * 2 + 1]);
      t[P_ENT] = (double)((1.f + dv.ent) * hc);
    }
    if (mcd && d) {
      // loss.py:29-30: sum over the classes of |softmax(out_t) - softmax(out_t_2)| of one target row
      const float* z2 = a.pred2_t + (size_t)(m - a.Bs) * a.C;
      const RowStats r2 = row_stats(z2, a.C, lane);
      float sabs = 0.f;
      for (int j = lane; j < a.C; j += 32)
        sabs += fabsf(expf(z[j] - rs.mx - rs.lse) - expf(z2[j] - r2.mx - r2.lse));
      t[P_DIS] = (double)warp_sum(sabs);
    }
    // domain CE per level (main.py:508-537): label 0 for source rows, 1 for target rows, weight dw[label]
    const double wd = (double)a.dw[d];
    if (a.flags & STATS_VIDEO) {
      t[P_VWCE] = wd * (double)domain_ce(a.pred_dom + (size_t)m * 2, d);
      t[P_VW] = wd;
    }
    if (a.flags & STATS_REL) {
      double s = 0.0;
      for (int i = lane; i < a.R; i += 32) s += (double)domain_ce(a.pred_rel + ((size_t)m * a.R + i) * 2, d);
      t[P_RWCE] = wd * warp_sum_d(s);
      t[P_RW] = wd * a.R;
    }
    if (a.flags & STATS_FRAME) {
      double s = 0.0;
      for (int i = lane; i < a.T; i += 32) s += (double)domain_ce(a.pred_frame + ((size_t)m * a.T + i) * 2, d);
      t[P_FWCE] = wd * warp_sum_d(s);
      t[P_FW] = wd * a.T;
    }
  }
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < P_N; ++i) s_row[warp][i] = t[i];
    s_rank[warp] = rank;
    s_src[warp] = src;
  }
  __syncthreads();

  // The folds run one sum per thread (thread j < P_N: sum j; then the row count and the k counts), each in a fixed
  // order -- rows within the CTA, then CTAs -- so the result is the same bit pattern on every run.  With every sum
  // folded by one thread the launch took 29 us at cfg2 (64 CTAs) instead of 17 (library CUDA events, L2 flushed).
  const int j = threadIdx.x;
  TrainStatsPartial* mine = partials + blockIdx.x;
  if (j < P_N) {
    double v = 0.0;
#pragma unroll
    for (int r = 0; r < kStatsRows; ++r) v += s_row[r][j];
    mine->s[j] = v;
  } else if (j == P_N) {
    long long n = 0;
#pragma unroll
    for (int r = 0; r < kStatsRows; ++r) n += s_src[r];
    mine->n_src = n;
  } else if (j < P_N + 1 + kEvalMaxK) {
    const int q = j - P_N - 1;
    long long n = 0;
    if (q < a.n_k)
#pragma unroll
      for (int r = 0; r < kStatsRows; ++r) n += s_src[r] && s_rank[r] < a.k[q];
    mine->correct[q] = n;
  }
  __threadfence();                                  // every writer's partial precedes the arrival below
  __syncthreads();
  __shared__ bool s_last;
  if (threadIdx.x == 0) s_last = atomicAdd(&a.accum->arrive, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  __shared__ double s_tot[P_N];
  __shared__ long long s_cnt[1 + kEvalMaxK];
  if (j < P_N) {
    double v = 0.0;
#pragma unroll 8
    for (unsigned b = 0; b < gridDim.x; ++b) v += __ldcg(&partials[b].s[j]);     // CTA order
    s_tot[j] = v;
  } else if (j < P_N + 1 + kEvalMaxK) {
    long long n = 0;
    const int q = j - P_N - 1;
#pragma unroll 8
    for (unsigned b = 0; b < gridDim.x; ++b) n += q < 0 ? __ldcg(&partials[b].n_src) : __ldcg(&partials[b].correct[q]);
    s_cnt[j - P_N] = n;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  TrainStatsPartial tot;
#pragma unroll
  for (int i = 0; i < P_N; ++i) tot.s[i] = s_tot[i];
  tot.n_src = s_cnt[0];
#pragma unroll
  for (int q = 0; q < kEvalMaxK; ++q) tot.correct[q] = s_cnt[1 + q];

  ta3n_train_stats* acc = a.accum;
  const long long n_all = (long long)vs + vt;
  // AverageMeter.update(val, n): a meter given n = 0 takes the val and keeps its sum (the reference's val can be the
  // mean of an empty tensor, NaN, which would poison the sum)
  auto update = [&](int i, double val, long long n) {
    acc->val[i] = val;
    if (n > 0) {
      acc->sum[i] += val * (double)n;
      acc->count[i] += n;
    }
  };
  update(0, (double)a.loss[0], 1);                                          // losses.update(loss.item())   :569
  double lc = tot.s[P_CWCE] / tot.s[P_CW];                                  // losses_c                     :446-450
  if (mcd) lc += tot.s[P_C2WCE] / tot.s[P_CW];
  update(1, lc, vs);
  if (a.flags & (STATS_REL | STATS_VIDEO | STATS_FRAME)) {                  // losses_a                     :508-537
    double la = 0.0;
    if (a.flags & STATS_REL) la += tot.s[P_RWCE] / tot.s[P_RW];
    if (a.flags & STATS_VIDEO) la += tot.s[P_VWCE] / tot.s[P_VW];
    if (a.flags & STATS_FRAME) la += tot.s[P_FWCE] / tot.s[P_FW];
    const long long n = (a.flags & STATS_FRAME) ? n_all * a.T : (a.flags & STATS_VIDEO) ? n_all : n_all * a.R;
    update(2, la, n);
  }
  if (a.flags & STATS_ENT) update(3, tot.s[P_ENT] / (double)n_all, vt);    // losses_e                     :559-561
  if (mcd) update(4, vt > 0 ? -tot.s[P_DIS] / ((double)vt * a.C) : 0.0, vt);   // losses_s                 :554-555
  for (int q = 0; q < a.n_k; ++q) {                                         // top1 / top5                  :565-571
    acc->correct[q] += tot.correct[q];
    acc->correct_step[q] = tot.correct[q];
    // Sv: accuracy() over the vs + vt labelled rows, folded with n = vs
    if (a.prec_sum && tot.n_src > 0) a.prec_sum[q] += 100.0 * (double)tot.correct[q] / (double)tot.n_src * (double)vs;
  }
  acc->rows += tot.n_src;
  acc->rows_step = tot.n_src;
  acc->steps += 1;
  __threadfence();
  acc->arrive = 0;
}

}  // namespace ta3n
