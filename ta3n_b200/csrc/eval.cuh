// eval.cuh -- the validation head (C ABI ta3n_eval_head): classifier logits, the validation criterion, top-k
// correctness and the confusion counts of one batch, folded into a device-resident epoch accumulator in the same
// launch.  It replaces the video head + CrossEntropyLoss + accuracy() + .item() of main.py:718-730, so a validation
// epoch is a series of graph replays with one readback at the end.
#pragma once

#include "common.cuh"

namespace ta3n {

constexpr int kEvalThreads = 256;
constexpr int kEvalRows = kEvalThreads / 32;      // rows per CTA: one warp per row for the metrics
constexpr int kEvalMaxK = 4;
constexpr size_t kEvalSmemBudget = 96 * 1024;     // feature rows + one weight tile

struct EvalArgs {
  const float* feat;            // [rows, H]
  const float* Wc;              // [C, H]
  const float* bc;              // [C]
  const long long* labels;      // [rows]
  const float* class_weight;    // [C] or nullptr
  const int* valid_rows;        // [1]
  const float* attn;            // row r at attn + r * attn_ld, R floats; or nullptr
  float* logits;                // [rows, C]
  ta3n_eval_accum* accum;
  long long* confusion;         // [C, C] or nullptr
  float* scores;                // [n_epoch, C] or nullptr
  float* attn_out;              // [n_epoch, R] or nullptr
  long long n_epoch;
  long long attn_ld;
  int rows, H, C, R, n_k, c_tile;
  int k[kEvalMaxK];
};

// Per-CTA partial of one batch, written to the workspace and summed in CTA order by the last CTA to arrive.
struct EvalPartial {
  double wce;                   // sum of w_y * ce over the CTA's real rows, in row order
  double w;                     // sum of w_y
  long long n;                  // real rows
  long long correct[kEvalMaxK];
};

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ int warp_sum_i(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// grid = ceil(rows / kEvalRows), block = kEvalThreads, dynamic smem = (kEvalRows * H + c_tile * (H + 1)) floats.
// Logits: each (row, class) pair is one thread's sequential fp32 FFMA chain over H, from the CTA's feature rows and a
// tile of c_tile classifier rows in shared memory (padded by one float per row: conflict-free column reads).  C <=
// c_tile stages the whole classifier once; otherwise it streams through the tile.
__global__ void __launch_bounds__(kEvalThreads)
eval_head_kernel(const __grid_constant__ EvalArgs a, EvalPartial* __restrict__ partials) {
  extern __shared__ float smem[];
  float* sX = smem;                                   // [kEvalRows, H]
  float* sW = smem + (size_t)kEvalRows * a.H;         // [c_tile, H + 1]
  __shared__ int s_valid, s_batch;
  __shared__ double s_wce[kEvalRows], s_w[kEvalRows];
  __shared__ int s_rank[kEvalRows], s_real[kEvalRows];
  const int row0 = blockIdx.x * kEvalRows;
  const int nrow = min(kEvalRows, a.rows - row0);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  pdl_wait();
  if (threadIdx.x == 0) {
    s_valid = min(max(*a.valid_rows, 0), a.rows);
    s_batch = a.accum->batch;
  }
  for (int i = threadIdx.x; i < nrow * a.H; i += kEvalThreads) sX[i] = a.feat[(size_t)row0 * a.H + i];

  const int ldw = a.H + 1;
  for (int c0 = 0; c0 < a.C; c0 += a.c_tile) {
    const int nc = min(a.c_tile, a.C - c0);
    __syncthreads();                                  // previous tile consumed (first pass: sX staged)
    for (int i = threadIdx.x; i < nc * a.H; i += kEvalThreads) {
      const int j = i / a.H, h = i - j * a.H;
      sW[j * ldw + h] = a.Wc[(size_t)(c0 + j) * a.H + h];
    }
    __syncthreads();
    for (int p = threadIdx.x; p < nrow * nc; p += kEvalThreads) {
      const int r = p / nc, j = p - r * nc;
      const float* x = sX + (size_t)r * a.H;
      const float* w = sW + (size_t)j * ldw;
      float acc = 0.f;
      for (int h = 0; h < a.H; ++h) acc = fmaf(x[h], w[h], acc);
      a.logits[(size_t)(row0 + r) * a.C + c0 + j] = acc + a.bc[c0 + j];
    }
  }
  __syncthreads();                                    // the CTA's logits are written (block-visible)

  // metrics: warp `warp` takes row row0 + warp
  if (warp < nrow) {
    const int r = row0 + warp;
    const float* z = a.logits + (size_t)r * a.C;
    const long long y = a.labels[r];
    const bool real = r < s_valid;
    const bool in_range = y >= 0 && y < a.C;
    const float zy = in_range ? z[y] : 0.f;
    float m = -INFINITY;
    int gt = 0, tie_before = 0, nan = 0;
    // top-1: (value, index) of the first maximum.  Lane `lane` always sees class `lane` first when C > lane, so its
    // index is set from the first element on, whatever the values (-inf included); lanes with no class keep
    // index C and lose every merge.
    float best = -INFINITY;
    int best_j = a.C;
    for (int j = lane; j < a.C; j += 32) {
      const float v = z[j];
      m = fmaxf(m, v);                                 // fmaxf skips NaN; a NaN logit still makes the sum below NaN
      nan += isnan(v);
      gt += v > zy;
      tie_before += (j < y) && (v == zy);
      if (best_j == a.C || v > best) { best = v; best_j = j; }   // ascending j per lane: the first maximum is kept
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
      const float ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oj = __shfl_xor_sync(0xffffffffu, best_j, o);
      if (oj < a.C && (best_j == a.C || ob > best || (ob == best && oj < best_j))) { best = ob; best_j = oj; }
    }
    gt = warp_sum_i(gt);
    tie_before = warp_sum_i(tie_before);
    nan = warp_sum_i(nan);
    double s = 0.0;
    for (int j = lane; j < a.C; j += 32) s += exp((double)z[j] - (double)m);
    s = warp_sum_d(s);
    if (lane == 0) {
      // ce = logsumexp(z) - z_y, shifted by the max; a label outside [0, C) gives NaN (torch raises), and so does
      // a NaN logit (as in torch).  A row with a NaN logit or a label outside [0, C) is a hit at no k and counts in
      // no confusion cell: its order is undefined.
      const bool ranked = in_range && nan == 0;
      const double ce = in_range ? (double)m + log(s) - (double)zy : (double)NAN;
      const double w = !in_range ? 1.0 : (a.class_weight ? (double)a.class_weight[y] : 1.0);
      s_wce[warp] = real ? w * ce : 0.0;
      s_w[warp] = real ? w : 0.0;
      s_rank[warp] = ranked ? gt + tie_before : 0x7fffffff;
      s_real[warp] = real;
      if (real && ranked && a.confusion && best_j >= 0 && best_j < a.C)
        atomicAdd(reinterpret_cast<unsigned long long*>(a.confusion) + y * a.C + best_j, 1ull);
    }
    // epoch buffers: real rows land at row batch * rows + r (dataset order)
    const long long dst = (long long)s_batch * a.rows + r;
    if (real && dst < a.n_epoch) {
      if (a.scores)
        for (int j = lane; j < a.C; j += 32) a.scores[dst * a.C + j] = z[j];
      if (a.attn_out)
        for (int j = lane; j < a.R; j += 32) a.attn_out[dst * a.R + j] = a.attn[r * a.attn_ld + j];
    }
  }
  __syncthreads();

  __shared__ EvalPartial s_part[kEvalThreads];
  __shared__ bool s_last;
  if (threadIdx.x == 0) {
    EvalPartial part;
    part.wce = 0.0;
    part.w = 0.0;
    part.n = 0;
    for (int i = 0; i < kEvalMaxK; ++i) part.correct[i] = 0;
    for (int i = 0; i < nrow; ++i) {                  // row order: deterministic
      part.wce += s_wce[i];
      part.w += s_w[i];
      part.n += s_real[i];
      for (int q = 0; q < a.n_k; ++q) part.correct[q] += s_real[i] && s_rank[i] < a.k[q];
    }
    partials[blockIdx.x] = part;
    __threadfence();                                  // partial and this CTA's read of accum->batch precede arrival
    s_last = atomicAdd(&a.accum->arrive, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (s_last) {
    __threadfence();
    EvalPartial tot;
    tot.wce = 0.0;
    tot.w = 0.0;
    tot.n = 0;
    for (int i = 0; i < kEvalMaxK; ++i) tot.correct[i] = 0;
    // the partials are loaded by the whole CTA (L2, one load per thread in flight), then summed in CTA order
    for (unsigned c0 = 0; c0 < gridDim.x; c0 += kEvalThreads) {
      const unsigned b = c0 + threadIdx.x;
      if (b < gridDim.x) {
        const EvalPartial* p = partials + b;
        s_part[threadIdx.x].wce = __ldcg(&p->wce);
        s_part[threadIdx.x].w = __ldcg(&p->w);
        s_part[threadIdx.x].n = __ldcg(&p->n);
        for (int q = 0; q < kEvalMaxK; ++q) s_part[threadIdx.x].correct[q] = __ldcg(&p->correct[q]);
      }
      __syncthreads();
      if (threadIdx.x == 0) {
        const unsigned nb = min((unsigned)kEvalThreads, gridDim.x - c0);
        for (unsigned i = 0; i < nb; ++i) {        // CTA order: deterministic
          tot.wce += s_part[i].wce;
          tot.w += s_part[i].w;
          tot.n += s_part[i].n;
          for (int q = 0; q < a.n_k; ++q) tot.correct[q] += s_part[i].correct[q];
        }
      }
      __syncthreads();
    }
    if (threadIdx.x == 0) {
      ta3n_eval_accum* acc = a.accum;
      if (tot.n > 0) {
        acc->loss_sum += (double)tot.n * (tot.wce / tot.w);     // losses.update(loss.item(), n_b), main.py:728
        acc->n += tot.n;
        for (int q = 0; q < a.n_k; ++q) acc->correct[q] += tot.correct[q];
      }
      acc->batch = s_batch + 1;
      __threadfence();
      acc->arrive = 0;
    }
  }
}

}  // namespace ta3n
