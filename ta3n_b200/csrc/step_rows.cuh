// step_rows.cuh -- the row ("SIMT") tasks of the step program: everything of the path that is not a dense
// contraction, written as device functions over a group of 256 threads, and the kernels that launch them
// (ta3n_step_run_phased).
//
//   frame_task   : per frame row -- frame head models.py:461, its domain loss and gradient main.py:513-538, data
//                  gradient down to the hidden layer of the frame discriminator.
//   relpool_task : per video -- relation heads models.py:479, entropy attention :351-357, attentive pooling
//                  :379-388 + :651-652, dropout :679-680.
//   heads_task   : per video -- classifier :681-687 and video-domain head :469-470, all video / relation level loss
//                  terms and gradients (main.py:446, 508-538, 559-562; loss.py:15-25), first backward step of both heads.
//   relbwd_task  : per video -- attention gradient, gradient of the relation heads down to their hidden layer.
//   The two 256 x 256 layers of the video discriminator between them (forward and data gradient) are tensor-core
//   tiles of the step.  Together these replace ten launches of the per-op sequence (relattn_fwd, head_fwd x3, two
//   launches of the video discriminator, loss_heads, loss_reduce, head_bwd_data, video_head_bwd, relattn_bwd_pre).
//   colsum_task : one (job, column block, row split) of the deterministic weighted column sums (bias gradients and
//                 the skinny head weight gradients), and the fixed-order reduction of its row splits.
#pragma once

#include "rowops.cuh"

namespace ta3n {

constexpr int kRowThreads = 256;          // threads of a row task (8 warps)
constexpr int kRowVideos = 8;             // videos per video-level row task: one warp per video
constexpr int kRowFrames = 32;            // frame rows per frame-level row task: four per warp
constexpr int kTailMaxT = 32, kTailMaxC = 128;

__device__ __forceinline__ void row_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

struct TailArgs {
  int M, Bs, T, R, H, F, C, n_rel;
  int use_attn, loss_flags;
  float gamma;
  float dom_w0, dom_w1;              // weight of criterion_domain (main.py:165-167)
  const float* class_weight;         // [C] weight of criterion (main.py:160-163) or nullptr
  const float* beta_dev;             // [3] relation, video, frame GRL coefficients (device: main.py:350-352)
  const long long* labels;
  const int* valid_rows;
  RelMap map;
  // forward inputs
  const float* hid_f;                // [M*T, F]
  const float* act;                  // [n_rel, M, H]
  const float* hid_r;                // [R, M, H]
  // weights
  const float* W2f;
  const float* b2f;
  PtrTable W2r, b2r;
  const float* Wc;
  const float* bc;
  const float* W2v;
  const float* b2v;
  DropArgs drop_v;
  // forward outputs
  float* pred_frame;                 // [M*T, 2]
  float* feat_rel;                   // [M, R, H]
  float* pred_rel;                   // [M, R, 2]
  float* attn;                       // [M, R]
  float* feat_video;                 // [M, H]
  float* dropped;                    // [M, H]
  float* pred_video;                 // [M, C]
  const float* hid_v;                // [M, H]   (video-discriminator hidden layer: a GEMM of the step)
  float* pred_dom;                   // [M, 2]
  float* row_loss;                   // [M]      video- and relation-level loss terms of the row
  float* frame_loss;                 // [M*T]    frame-level domain loss terms
  // backward outputs (operands of the dgrad / wgrad GEMMs and of the column sums)
  float* g_video;                    // [M, C]
  float* g_dom;                      // [M, 2]
  float* g_frame;                    // [M*T, 2]
  float* g_rel;                      // [M, R, 2]  d loss / d pred_rel of the relation-level domain loss alone
  float* Pt;                         // [M, R, 2]  ... plus the attention path (what the relation heads receive)
  float* dHv;                        // [M, H]
  float* Gc;                         // [M, H]     classifier part of d loss / d dropped: g_video Wc
  const float* G;                    // [M, H]     d loss / d feat_video (completed by the video-discriminator dgrad GEMM)
  float* dHid;                       // [R, M, H]
  float* dHf;                        // [M*T, F]
};

// The argument blocks of the row tasks live in file-scope shared memory, and the tasks are compiled out of line
// and read them through a reference to that known __shared__ object: every field access stays an LDS that global
// stores cannot alias.  Passed as `const TailArgs&` the block became generic loads repeated after every store.
__shared__ TailArgs g_tail;
__shared__ WColsumJob g_job;

// normalisers of the (weighted) means shared by the loss tasks: CrossEntropyLoss(weight=w) divides by the sum of the
// weights of the rows it sees (main.py:160-167, 204-206); padding rows of a short last batch are excluded
// (main.py:354-372, 421-422)
struct LossNorm {
  int vs, vt;                        // real source / target videos
  float n_dom;                       // sum of the domain weights over the real videos (per level: times rows per video)
  float n_all;                       // real videos (attentive entropy: plain mean)
};
__device__ __forceinline__ LossNorm loss_norm(const TailArgs& a) {
  LossNorm n;
  const int vs_in = a.valid_rows ? a.valid_rows[0] : a.Bs;
  const int vt_in = a.valid_rows ? a.valid_rows[1] : a.M - a.Bs;
  n.vs = min(vs_in, a.Bs);
  n.vt = min(vt_in, a.M - a.Bs);
  n.n_dom = fmaxf(a.dom_w0 * (float)n.vs + a.dom_w1 * (float)n.vt, 1e-30f);
  n.n_all = (float)max(n.vs + n.vt, 1);
  return n;
}

// ---- frame task: rows [r0, r0 + nr) of the M*T frame rows, one warp per row (4 rows per warp) ------------------
// frame logits (models.py:461), frame-level domain loss + its gradient (main.py:513-538), data gradient of the head
// through the ReLU of the hidden layer: dHf = (g_frame W2f) * 1[hid_f > 0].  Depends on hid_f alone, so the whole frame
// branch runs beside the video-level chain.
template <int FV>      // F <= 128 * FV
__device__ __noinline__ void frame_task_t(const int r0, const int nr, const int tid) {
  const TailArgs& a = g_tail;
  const int lane = tid & 31, warp = tid >> 5;
  const int T = a.T, F = a.F, Bs = a.Bs;
  const float* __restrict__ W2f = a.W2f;
  const LossNorm ln = loss_norm(a);
  const float b0 = __ldg(a.b2f), b1 = __ldg(a.b2f + 1);
  constexpr int RW = kRowFrames / 8;                        // rows per warp, all in flight at once
  float4 h[RW][FV];
#pragma unroll
  for (int j = 0; j < RW; ++j) {
    const int it = min(warp + 8 * j, nr - 1);               // clamped: every element is loaded (no branches)
#pragma unroll
    for (int kk = 0; kk < FV; ++kk) {
      const int k = min(lane * 4 + 128 * kk, F - 4);
      h[j][kk] = __ldcg(reinterpret_cast<const float4*>(a.hid_f + ((size_t)r0 + it) * F + k));
      if (lane * 4 + 128 * kk >= F) h[j][kk] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
  float4 w0[FV], w1[FV];
#pragma unroll
  for (int kk = 0; kk < FV; ++kk) {
    const int k = min(lane * 4 + 128 * kk, F - 4);
    w0[kk] = __ldg(reinterpret_cast<const float4*>(W2f + k));
    w1[kk] = __ldg(reinterpret_cast<const float4*>(W2f + F + k));
    if (lane * 4 + 128 * kk >= F) w0[kk] = w1[kk] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  float s0[RW], s1[RW];
#pragma unroll
  for (int j = 0; j < RW; ++j) {
    float x0 = 0.f, x1 = 0.f;
#pragma unroll
    for (int kk = 0; kk < FV; ++kk) {
      x0 = fmaf(h[j][kk].x, w0[kk].x, fmaf(h[j][kk].y, w0[kk].y, fmaf(h[j][kk].z, w0[kk].z, fmaf(h[j][kk].w, w0[kk].w, x0))));
      x1 = fmaf(h[j][kk].x, w1[kk].x, fmaf(h[j][kk].y, w1[kk].y, fmaf(h[j][kk].z, w1[kk].z, fmaf(h[j][kk].w, w1[kk].w, x1))));
    }
    s0[j] = x0;
    s1[j] = x1;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
    for (int j = 0; j < RW; ++j) {
      s0[j] += __shfl_xor_sync(0xffffffffu, s0[j], o);
      s1[j] += __shfl_xor_sync(0xffffffffu, s1[j], o);
    }
  }
#pragma unroll
  for (int j = 0; j < RW; ++j) {
    const int it = warp + 8 * j;
    const bool live = it < nr;
    const size_t row = (size_t)r0 + (live ? it : 0);
    const float p0 = s0[j] + b0, p1 = s1[j] + b1;
    const int m = (int)(row / T);
    const int dom = m >= Bs ? 1 : 0;
    const bool real = dom ? (m - Bs < ln.vt) : (m < ln.vs);
    float g0 = 0.f, g1 = 0.f, l = 0.f;
    if (real && (a.loss_flags & LOSS_ADV_FRAME)) {
      const float wd = dom ? a.dom_w1 : a.dom_w0;
      const Attn2 x = attn_from_logits(p0, p1);
      const float inv = wd / (ln.n_dom * (float)T);
      l = -(dom ? x.lq1 : x.lq0) * inv;
      g0 = (x.q0 - (dom ? 0.f : 1.f)) * inv;
      g1 = (x.q1 - (dom ? 1.f : 0.f)) * inv;
    }
    if (lane == 0 && live) {
      a.pred_frame[row * 2] = p0;
      a.pred_frame[row * 2 + 1] = p1;
      a.g_frame[row * 2] = g0;
      a.g_frame[row * 2 + 1] = g1;
      a.frame_loss[row] = l;
    }
    float* __restrict__ dh = a.dHf + row * F;
#pragma unroll
    for (int kk = 0; kk < FV; ++kk) {
      const int k = lane * 4 + 128 * kk;
      if (k < F && live) {
        float4 d;
        d.x = h[j][kk].x > 0.f ? fmaf(g0, w0[kk].x, g1 * w1[kk].x) : 0.f;
        d.y = h[j][kk].y > 0.f ? fmaf(g0, w0[kk].y, g1 * w1[kk].y) : 0.f;
        d.z = h[j][kk].z > 0.f ? fmaf(g0, w0[kk].z, g1 * w1[kk].z) : 0.f;
        d.w = h[j][kk].w > 0.f ? fmaf(g0, w0[kk].w, g1 * w1[kk].w) : 0.f;
        *reinterpret_cast<float4*>(dh + k) = d;
      }
    }
  }
}
// any F % 4 == 0, one row at a time (F > 512: fc_dim = 2048 runs)
__device__ __noinline__ void frame_task_any(const int r0, const int nr, const int tid) {
  const TailArgs& a = g_tail;
  const int lane = tid & 31, warp = tid >> 5;
  const int T = a.T, F = a.F, Bs = a.Bs;
  const float* __restrict__ W2f = a.W2f;
  const LossNorm ln = loss_norm(a);
  const float b0 = __ldg(a.b2f), b1 = __ldg(a.b2f + 1);
  for (int it = warp; it < nr; it += 8) {
    const size_t row = (size_t)r0 + it;
    const float* __restrict__ hr = a.hid_f + row * F;
    float* __restrict__ dh = a.dHf + row * F;
    float s0 = 0.f, s1 = 0.f;
    for (int k = lane * 4; k < F; k += 128) {
      const float4 h = __ldcg(reinterpret_cast<const float4*>(hr + k));
      const float4 w0 = __ldg(reinterpret_cast<const float4*>(W2f + k));
      const float4 w1 = __ldg(reinterpret_cast<const float4*>(W2f + F + k));
      s0 = fmaf(h.x, w0.x, fmaf(h.y, w0.y, fmaf(h.z, w0.z, fmaf(h.w, w0.w, s0))));
      s1 = fmaf(h.x, w1.x, fmaf(h.y, w1.y, fmaf(h.z, w1.z, fmaf(h.w, w1.w, s1))));
    }
    s0 = warp_sum(s0) + b0;
    s1 = warp_sum(s1) + b1;
    const int m = (int)(row / T);
    const int dom = m >= Bs ? 1 : 0;
    const bool real = dom ? (m - Bs < ln.vt) : (m < ln.vs);
    float g0 = 0.f, g1 = 0.f, l = 0.f;
    if (real && (a.loss_flags & LOSS_ADV_FRAME)) {
      const float wd = dom ? a.dom_w1 : a.dom_w0;
      const Attn2 x = attn_from_logits(s0, s1);
      const float inv = wd / (ln.n_dom * (float)T);
      l = -(dom ? x.lq1 : x.lq0) * inv;
      g0 = (x.q0 - (dom ? 0.f : 1.f)) * inv;
      g1 = (x.q1 - (dom ? 1.f : 0.f)) * inv;
    }
    if (lane == 0) {
      a.pred_frame[row * 2] = s0;
      a.pred_frame[row * 2 + 1] = s1;
      a.g_frame[row * 2] = g0;
      a.g_frame[row * 2 + 1] = g1;
      a.frame_loss[row] = l;
    }
    for (int k = lane * 4; k < F; k += 128) {
      const float4 h = __ldcg(reinterpret_cast<const float4*>(hr + k));
      const float4 w0 = __ldg(reinterpret_cast<const float4*>(W2f + k));
      const float4 w1 = __ldg(reinterpret_cast<const float4*>(W2f + F + k));
      float4 d;
      d.x = h.x > 0.f ? fmaf(g0, w0.x, g1 * w1.x) : 0.f;
      d.y = h.y > 0.f ? fmaf(g0, w0.y, g1 * w1.y) : 0.f;
      d.z = h.z > 0.f ? fmaf(g0, w0.z, g1 * w1.z) : 0.f;
      d.w = h.w > 0.f ? fmaf(g0, w0.w, g1 * w1.w) : 0.f;
      *reinterpret_cast<float4*>(dh + k) = d;
    }
  }
}
// the path has F = 512: all four rows of a warp in flight; wider layers take the row-at-a-time form
__device__ __forceinline__ void frame_task(const int r0, const int nr, const int tid) {
  if (g_tail.F <= 512)
    frame_task_t<4>(r0, nr, tid);
  else
    frame_task_any(r0, nr, tid);
}

// The video-level row tasks give every video to ONE warp: lane l holds the feature elements 4l .. 4l+3 of each
// 128-wide chunk of a length-H row (HV = H / 128 chunks), so the tasks need no shared memory and no block barrier.
template <int HV>
struct RowVec {
  float4 c[HV];
};
template <int HV>
__device__ __forceinline__ RowVec<HV> row_load_cg(const float* p, int lane) {
  RowVec<HV> r;
#pragma unroll
  for (int kk = 0; kk < HV; ++kk) r.c[kk] = __ldcg(reinterpret_cast<const float4*>(p + lane * 4 + 128 * kk));
  return r;
}
template <int HV>
__device__ __forceinline__ RowVec<HV> row_load_ro(const float* p, int lane) {
  RowVec<HV> r;
#pragma unroll
  for (int kk = 0; kk < HV; ++kk) r.c[kk] = __ldg(reinterpret_cast<const float4*>(p + lane * 4 + 128 * kk));
  return r;
}
template <int HV>
__device__ __forceinline__ void row_store(float* p, int lane, const RowVec<HV>& r) {
#pragma unroll
  for (int kk = 0; kk < HV; ++kk) *reinterpret_cast<float4*>(p + lane * 4 + 128 * kk) = r.c[kk];
}
template <int HV>
__device__ __forceinline__ float row_dot(const RowVec<HV>& a, const RowVec<HV>& b) {
  float s = 0.f;
#pragma unroll
  for (int kk = 0; kk < HV; ++kk)
    s = fmaf(a.c[kk].x, b.c[kk].x, fmaf(a.c[kk].y, b.c[kk].y, fmaf(a.c[kk].z, b.c[kk].z, fmaf(a.c[kk].w, b.c[kk].w, s))));
  return warp_sum(s);
}

// ---- relpool task: videos [v0, v0 + nv): relation sums, relation logits, entropy attention, attentive pooling,
// dropout of the pooled feature              TRNmodule.py:79, models.py:479, 351-357, 379-388, 651-652, 679-680 ----
template <int HV>
__device__ __noinline__ void relpool_task_t(const int v0, const int nv, const int tid) {
  const TailArgs& a = g_tail;
  const int lane = tid & 31, warp = tid >> 5;
  const int M = a.M, R = a.R, H = a.H;
  const size_t plane = (size_t)M * H;
  for (int v = warp; v < nv; v += 8) {
    const int m = v0 + v;
    // relation logits from the discriminators' hidden layer -> attention weights; lane i keeps w_i + 1 of scale i.
    // Four scales per round: their hidden rows are requested together (the task is a chain of L2 round trips otherwise)
    float wp1 = 1.0f;
    for (int i0 = 0; i0 < R; i0 += 4) {
      RowVec<HV> h[4];
#pragma unroll
      for (int j = 0; j < 4; ++j)                  // clamped index: every register of the array is written (no branches)
        h[j] = row_load_cg<HV>(a.hid_r + ((size_t)min(i0 + j, R - 1) * M + m) * H, lane);
      float s0[4], s1[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        s0[j] = s1[j] = 0.f;
        {
          const float* w = a.W2r.p[min(i0 + j, R - 1)];
          const RowVec<HV> x0 = row_load_ro<HV>(w, lane), x1 = row_load_ro<HV>(w + H, lane);
#pragma unroll
          for (int kk = 0; kk < HV; ++kk) {
            s0[j] = fmaf(h[j].c[kk].x, x0.c[kk].x, fmaf(h[j].c[kk].y, x0.c[kk].y, fmaf(h[j].c[kk].z, x0.c[kk].z, fmaf(h[j].c[kk].w, x0.c[kk].w, s0[j]))));
            s1[j] = fmaf(h[j].c[kk].x, x1.c[kk].x, fmaf(h[j].c[kk].y, x1.c[kk].y, fmaf(h[j].c[kk].z, x1.c[kk].z, fmaf(h[j].c[kk].w, x1.c[kk].w, s1[j]))));
          }
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          s0[j] += __shfl_xor_sync(0xffffffffu, s0[j], o);
          s1[j] += __shfl_xor_sync(0xffffffffu, s1[j], o);
        }
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const bool live = i0 + j < R;
        const int i = min(i0 + j, R - 1);
        const float p0 = s0[j] + __ldg(a.b2r.p[i]), p1 = s1[j] + __ldg(a.b2r.p[i] + 1);
        const float wi = a.use_attn ? attn_from_logits(p0, p1).w : 0.f;
        const size_t o = (size_t)m * R + i;
        if (lane == 0 && live) {
          a.pred_rel[o * 2] = p0;
          a.pred_rel[o * 2 + 1] = p1;
          if (a.use_attn) a.attn[o] = wi;
        }
        if (live && (i & 31) == lane) wp1 = wi + 1.0f;    // R <= 32
      }
    }
    RowVec<HV> y;
#pragma unroll
    for (int kk = 0; kk < HV; ++kk) y.c[kk] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int i0 = 0; i0 < R; i0 += 2) {           // two scales (up to six relation rows) in flight
      RowVec<HV> x[2][3];
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int i = min(i0 + j, R - 1);
        const int qb = a.map.rel_begin[i], qn = a.map.rel_begin[i + 1] - qb;
#pragma unroll
        for (int r = 0; r < 3; ++r)               // clamped relation: the duplicate load is cheaper than a branch
          x[j][r] = row_load_cg<HV>(a.act + (qb + min(r, qn - 1)) * plane + (size_t)m * H, lane);
      }
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int i = i0 + j;
        if (i < R) {
        const int qn = a.map.rel_begin[i + 1] - a.map.rel_begin[i];
        RowVec<HV> f = x[j][0];
#pragma unroll
        for (int r = 1; r < 3; ++r)
          if (r < qn) {
#pragma unroll
            for (int kk = 0; kk < HV; ++kk) {
              f.c[kk].x += x[j][r].c[kk].x;
              f.c[kk].y += x[j][r].c[kk].y;
              f.c[kk].z += x[j][r].c[kk].z;
              f.c[kk].w += x[j][r].c[kk].w;
            }
          }
        row_store<HV>(a.feat_rel + ((size_t)m * R + i) * H, lane, f);
        const float wi = __shfl_sync(0xffffffffu, wp1, i & 31);
#pragma unroll
        for (int kk = 0; kk < HV; ++kk) {
          y.c[kk].x = fmaf(wi, f.c[kk].x, y.c[kk].x);
          y.c[kk].y = fmaf(wi, f.c[kk].y, y.c[kk].y);
          y.c[kk].z = fmaf(wi, f.c[kk].z, y.c[kk].z);
          y.c[kk].w = fmaf(wi, f.c[kk].w, y.c[kk].w);
        }
        if (!a.use_attn) {                        // models.py:647 placeholder output: feat_rel[:, :, 0]
          const float first = __shfl_sync(0xffffffffu, f.c[0].x, 0);
          if (lane == 0) a.attn[(size_t)m * R + i] = first;
        }
        }
      }
    }
    row_store<HV>(a.feat_video + (size_t)m * H, lane, y);
#pragma unroll
    for (int kk = 0; kk < HV; ++kk) {
      const size_t ge = (size_t)m * H + lane * 4 + 128 * kk;      // a multiple of 4: one hash for the quad
      if (a.drop_v.mode == 2) {
        const uint64_t hsh = rng_hash4(a.drop_v.seed, a.drop_v.step_dev ? *a.drop_v.step_dev : 0ull, ge >> 2);
        const uint32_t thr = rng_threshold(a.drop_v.p);
        y.c[kk].x = rng_keep_bits(hsh, 0, thr) ? y.c[kk].x * a.drop_v.scale : 0.f;
        y.c[kk].y = rng_keep_bits(hsh, 1, thr) ? y.c[kk].y * a.drop_v.scale : 0.f;
        y.c[kk].z = rng_keep_bits(hsh, 2, thr) ? y.c[kk].z * a.drop_v.scale : 0.f;
        y.c[kk].w = rng_keep_bits(hsh, 3, thr) ? y.c[kk].w * a.drop_v.scale : 0.f;
      } else {
        y.c[kk].x *= drop_factor(a.drop_v, ge);
        y.c[kk].y *= drop_factor(a.drop_v, ge + 1);
        y.c[kk].z *= drop_factor(a.drop_v, ge + 2);
        y.c[kk].w *= drop_factor(a.drop_v, ge + 3);
      }
    }
    row_store<HV>(a.dropped + (size_t)m * H, lane, y);
  }
}

// ---- heads task: class logits, video-domain logits, every video- and relation-level loss term and its gradient,
// then the first backward step of both video heads: dHv = (g_dom W2v) * 1[hid_v > 0], Gc = g_video Wc
//                              models.py:681-687, 469-470; main.py:446, 508-538, 559-562; loss.py:15-25 ----
template <int HV>
__device__ __noinline__ void heads_task_t(const int v0, const int nv, const int tid) {
  const TailArgs& a = g_tail;
  const int lane = tid & 31, warp = tid >> 5;
  const int R = a.R, H = a.H, C = a.C, Bs = a.Bs;
  const LossNorm ln = loss_norm(a);
  float n_cls = (float)max(ln.vs, 1);
  if (a.class_weight) {                                     // main.py:160-163, 204: sum_m w[y_m] over the real source rows
    float s = 0.f;
    for (int m = lane; m < ln.vs; m += 32) s += __ldg(a.class_weight + (int)a.labels[m]);
    n_cls = fmaxf(warp_sum(s), 1e-30f);
  }
  constexpr int CV = kTailMaxC / 32;                        // class logits per lane: c = lane + 32 j
  for (int v = warp; v < nv; v += 8) {
    const int m = v0 + v;
    const int dom = m >= Bs ? 1 : 0;
    const bool real = dom ? (m - Bs < ln.vt) : (m < ln.vs);
    const RowVec<HV> d = row_load_cg<HV>(a.dropped + (size_t)m * H, lane);
    const RowVec<HV> hv = row_load_cg<HV>(a.hid_v + (size_t)m * H, lane);
    const int y_lab = (m < Bs) ? (int)a.labels[m] : -1;    // requested early: off the critical chain below
    float pv[CV];
#pragma unroll
    for (int j = 0; j < CV; ++j) pv[j] = -INFINITY;
    for (int c0 = 0; c0 < C; c0 += 4) {                     // four classes per round: their reductions interleave
      float part[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        part[j] = 0.f;
        if (c0 + j < C) {
          const RowVec<HV> w = row_load_ro<HV>(a.Wc + (size_t)(c0 + j) * H, lane);
#pragma unroll
          for (int kk = 0; kk < HV; ++kk)
            part[j] = fmaf(d.c[kk].x, w.c[kk].x, fmaf(d.c[kk].y, w.c[kk].y, fmaf(d.c[kk].z, w.c[kk].z, fmaf(d.c[kk].w, w.c[kk].w, part[j]))));
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
        for (int j = 0; j < 4; ++j) part[j] += __shfl_xor_sync(0xffffffffu, part[j], o);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int c = c0 + j;
        if (c < C && (c & 31) == lane) {
          const float sres = part[j] + __ldg(a.bc + c);
#pragma unroll
          for (int jj = 0; jj < CV; ++jj)
            if (jj == (c >> 5)) pv[jj] = sres;
        }
      }
    }
    const RowVec<HV> w2v0 = row_load_ro<HV>(a.W2v, lane), w2v1 = row_load_ro<HV>(a.W2v + H, lane);
    const float pd0 = row_dot<HV>(hv, w2v0) + __ldg(a.b2v);
    const float pd1 = row_dot<HV>(hv, w2v1) + __ldg(a.b2v + 1);
#pragma unroll
    for (int j = 0; j < CV; ++j)
      if (lane + 32 * j < C) a.pred_video[(size_t)m * C + lane + 32 * j] = pv[j];
    if (lane == 0) {
      a.pred_dom[(size_t)m * 2] = pd0;
      a.pred_dom[(size_t)m * 2 + 1] = pd1;
    }
    // ---- loss heads ----
    float gv[CV];
    float g0 = 0.f, g1 = 0.f, loss = 0.f;
#pragma unroll
    for (int j = 0; j < CV; ++j) gv[j] = 0.f;
    float gr0 = 0.f, gr1 = 0.f;                             // lane i: gradient of relation i's logits (R <= 32)
    if (real) {
      const float wd = dom ? a.dom_w1 : a.dom_w0;
      float mx = -INFINITY;
#pragma unroll
      for (int j = 0; j < CV; ++j) mx = fmaxf(mx, pv[j]);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      float se = 0.f;
#pragma unroll
      for (int j = 0; j < CV; ++j)
        if (lane + 32 * j < C) se += expf(pv[j] - mx);
      se = warp_sum(se);
      const float lse = logf(se);
      float hc = 0.f;                                       // entropy of the class prediction
#pragma unroll
      for (int j = 0; j < CV; ++j)
        if (lane + 32 * j < C) {
          const float lq = pv[j] - mx - lse;
          hc -= expf(lq) * lq;
        }
      hc = warp_sum(hc);
      const Attn2 dv = attn_from_logits(pd0, pd1);
      const bool att = (a.loss_flags & LOSS_ATT_ENT) != 0;
      const float att_scale = att ? a.gamma / ln.n_all : 0.f;
      const int y = y_lab;
      const float wy = (m < Bs) ? (a.class_weight ? __ldg(a.class_weight + y) : 1.f) : 0.f;
#pragma unroll
      for (int j = 0; j < CV; ++j) {
        const int c = lane + 32 * j;
        if (c < C) {
          const float lq = pv[j] - mx - lse;
          const float q = expf(lq);
          float gq = 0.f;
          if (m < Bs) gq = wy * (q - (c == y ? 1.f : 0.f)) / n_cls;
          gq += att_scale * (1.f + dv.ent) * (-q * (lq + hc));
          gv[j] = gq;
          if (m < Bs && c == y) loss += -wy * lq / n_cls;
        }
      }
      loss = warp_sum(loss);                                // exactly one lane held the CE term
      loss += att_scale * (1.f + dv.ent) * hc;
      if (a.loss_flags & LOSS_ADV_VIDEO) {
        loss += -wd * (dom ? dv.lq1 : dv.lq0) / ln.n_dom;
        g0 = wd * (dv.q0 - (dom ? 0.f : 1.f)) / ln.n_dom;
        g1 = wd * (dv.q1 - (dom ? 1.f : 0.f)) / ln.n_dom;
      }
      g0 += att_scale * hc * (-dv.q0 * (dv.lq0 + dv.ent));
      g1 += att_scale * hc * (-dv.q1 * (dv.lq1 + dv.ent));
      float extra = 0.f;
      if ((a.loss_flags & LOSS_ADV_REL) && lane < R) {
        const float p0 = __ldcg(a.pred_rel + ((size_t)m * R + lane) * 2), p1 = __ldcg(a.pred_rel + ((size_t)m * R + lane) * 2 + 1);
        const Attn2 x = attn_from_logits(p0, p1);
        const float inv = wd / (ln.n_dom * (float)R);
        extra = -(dom ? x.lq1 : x.lq0) * inv;
        gr0 = (x.q0 - (dom ? 0.f : 1.f)) * inv;
        gr1 = (x.q1 - (dom ? 1.f : 0.f)) * inv;
      }
      loss += warp_sum(extra);
    }
#pragma unroll
    for (int j = 0; j < CV; ++j)
      if (lane + 32 * j < C) a.g_video[(size_t)m * C + lane + 32 * j] = gv[j];
    if (lane < R) {
      a.g_rel[((size_t)m * R + lane) * 2] = gr0;
      a.g_rel[((size_t)m * R + lane) * 2 + 1] = gr1;
    }
    if (lane == 0) {
      a.g_dom[(size_t)m * 2] = g0;
      a.g_dom[(size_t)m * 2 + 1] = g1;
      a.row_loss[m] = loss;
    }
    // ---- dHv = (g_dom W2v) * 1[hid_v > 0]                                                  (head_bwd_data) ----
    RowVec<HV> o;
#pragma unroll
    for (int kk = 0; kk < HV; ++kk) {
      o.c[kk].x = hv.c[kk].x > 0.f ? fmaf(g0, w2v0.c[kk].x, g1 * w2v1.c[kk].x) : 0.f;
      o.c[kk].y = hv.c[kk].y > 0.f ? fmaf(g0, w2v0.c[kk].y, g1 * w2v1.c[kk].y) : 0.f;
      o.c[kk].z = hv.c[kk].z > 0.f ? fmaf(g0, w2v0.c[kk].z, g1 * w2v1.c[kk].z) : 0.f;
      o.c[kk].w = hv.c[kk].w > 0.f ? fmaf(g0, w2v0.c[kk].w, g1 * w2v1.c[kk].w) : 0.f;
    }
    row_store<HV>(a.dHv + (size_t)m * H, lane, o);
    // ---- Gc = g_video Wc: the classifier's share of d loss / d dropped                   (video_head_bwd) ----
#pragma unroll
    for (int kk = 0; kk < HV; ++kk) o.c[kk] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int c = 0; c < C; ++c) {
      float g = 0.f;
#pragma unroll
      for (int j = 0; j < CV; ++j)
        if (j == (c >> 5)) g = gv[j];
      g = __shfl_sync(0xffffffffu, g, c & 31);
      const RowVec<HV> w = row_load_ro<HV>(a.Wc + (size_t)c * H, lane);
#pragma unroll
      for (int kk = 0; kk < HV; ++kk) {
        o.c[kk].x = fmaf(g, w.c[kk].x, o.c[kk].x);
        o.c[kk].y = fmaf(g, w.c[kk].y, o.c[kk].y);
        o.c[kk].z = fmaf(g, w.c[kk].z, o.c[kk].z);
        o.c[kk].w = fmaf(g, w.c[kk].w, o.c[kk].w);
      }
    }
    row_store<HV>(a.Gc + (size_t)m * H, lane, o);
  }
}

// ---- relbwd task: the attention gradient (attention weights are NOT detached, SURVEY 3.3), the gradient the
// relation heads receive, and their data gradient through the hidden ReLU: dHid_i = (Pt_i W2r_i) * 1[hid_r_i > 0]
//                                                                     backward of models.py:379-388, 479 ----
template <int HV>
__device__ __noinline__ void relbwd_task_t(const int v0, const int nv, const int tid) {
  const TailArgs& a = g_tail;
  const int lane = tid & 31, warp = tid >> 5;
  const int M = a.M, R = a.R, H = a.H;
  for (int v = warp; v < nv; v += 8) {
    const int m = v0 + v;
    const RowVec<HV> G = row_load_cg<HV>(a.G + (size_t)m * H, lane);
    for (int i0 = 0; i0 < R; i0 += 2) {             // two scales in flight: every load of the pair before the first use
      RowVec<HV> fr[2], h[2];
      float gr0[2], gr1[2], pr0[2], pr1[2];
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int i = min(i0 + j, R - 1);           // clamped: every register of the arrays is written
        const size_t o = (size_t)m * R + i;
        gr0[j] = __ldcg(a.g_rel + o * 2);
        gr1[j] = __ldcg(a.g_rel + o * 2 + 1);
        pr0[j] = __ldcg(a.pred_rel + o * 2);
        pr1[j] = __ldcg(a.pred_rel + o * 2 + 1);
        fr[j] = row_load_cg<HV>(a.feat_rel + o * H, lane);
        h[j] = row_load_cg<HV>(a.hid_r + ((size_t)i * M + m) * H, lane);
      }
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int i = i0 + j;
        if (i < R) {
        const size_t o = (size_t)m * R + i;
        float pt0 = gr0[j], pt1 = gr1[j];
        if (a.use_attn) {
          const float dw = row_dot<HV>(G, fr[j]);
          const Attn2 x = attn_from_logits(pr0[j], pr1[j]);
          pt0 += dw * x.q0 * (x.lq0 + x.ent);
          pt1 += dw * x.q1 * (x.lq1 + x.ent);
        }
        if (lane == 0) {
          a.Pt[o * 2] = pt0;
          a.Pt[o * 2 + 1] = pt1;
        }
        const float* w = a.W2r.p[i];
        const RowVec<HV> x0 = row_load_ro<HV>(w, lane), x1 = row_load_ro<HV>(w + H, lane);
        RowVec<HV> d;
#pragma unroll
        for (int kk = 0; kk < HV; ++kk) {
          d.c[kk].x = h[j].c[kk].x > 0.f ? fmaf(pt0, x0.c[kk].x, pt1 * x1.c[kk].x) : 0.f;
          d.c[kk].y = h[j].c[kk].y > 0.f ? fmaf(pt0, x0.c[kk].y, pt1 * x1.c[kk].y) : 0.f;
          d.c[kk].z = h[j].c[kk].z > 0.f ? fmaf(pt0, x0.c[kk].z, pt1 * x1.c[kk].z) : 0.f;
          d.c[kk].w = h[j].c[kk].w > 0.f ? fmaf(pt0, x0.c[kk].w, pt1 * x1.c[kk].w) : 0.f;
        }
        row_store<HV>(a.dHid + ((size_t)i * M + m) * H, lane, d);
        }
      }
    }
  }
}

// H = 128 * HV with HV in {1, 2} (checked by build_step_program): the path has H = 256 (models.py:223)
enum : int { ROW_RELPOOL = 0, ROW_HEADS = 1, ROW_RELBWD = 2 };
__device__ __forceinline__ void video_row_task(const int kind, const int v0, const int nv, const int tid) {
#define TA3N_ROW_DISPATCH(HVV)                                \
  if (kind == ROW_RELPOOL) relpool_task_t<HVV>(v0, nv, tid);  \
  else if (kind == ROW_HEADS) heads_task_t<HVV>(v0, nv, tid); \
  else relbwd_task_t<HVV>(v0, nv, tid);
  if (g_tail.H == 256) {
    TA3N_ROW_DISPATCH(2)
  } else {
    TA3N_ROW_DISPATCH(1)
  }
#undef TA3N_ROW_DISPATCH
}

// ---- column sums as tasks --------------------------------------------------------------------------------
// Same arithmetic and the same fixed summation order as wcolsum_stage1/2 (rowops.cuh); the block / split indices
// arrive as arguments instead of blockIdx.  part: (job, column block cb, row split) -> partial[split]; the job's
// reduce task then sums its splits in order.  tid in [0, 256) = (lane, warp) = (threadIdx.x, threadIdx.y) there.
template <int KMAX, bool VEC>
__device__ __forceinline__ void colsum_part_body(const WColsumJob& j, float4 (*red)[33], const int cb, const int split,
                                                 const int k0, const int lane, const int warp) {
  const int n = cb * 128 + lane * 4;
  const int nsplit = j.nsplit;
  float4 acc[KMAX];
#pragma unroll
  for (int k = 0; k < KMAX; ++k) acc[k] = f4_zero();
  auto ldx = [&](const float* X, int r) -> float4 {
    const float* q = X + (size_t)r * j.ld + n;
    if (VEC) return __ldcg(reinterpret_cast<const float4*>(q));
    float4 v = f4_zero();
    if (n < j.N) v.x = __ldcg(q);
    if (n + 1 < j.N) v.y = __ldcg(q + 1);
    if (n + 2 < j.N) v.z = __ldcg(q + 2);
    if (n + 3 < j.N) v.w = __ldcg(q + 3);
    return v;
  };
  if (n < j.N) {
    for (int sg = 0; sg < j.nseg; ++sg) {
      const float* X = j.X[sg];
      const float* P = j.P[sg];
      const int rows = j.rows[sg];
      const int per = (rows + nsplit - 1) / nsplit;
      const int r1 = min(rows, (split + 1) * per);
      int r = split * per + warp;
      for (; r + 24 < r1; r += 32) {
        const float4 x0 = ldx(X, r), x1 = ldx(X, r + 8), x2 = ldx(X, r + 16), x3 = ldx(X, r + 24);
        if (P == nullptr) {
          acc[0].x += (x0.x + x1.x) + (x2.x + x3.x);
          acc[0].y += (x0.y + x1.y) + (x2.y + x3.y);
          acc[0].z += (x0.z + x1.z) + (x2.z + x3.z);
          acc[0].w += (x0.w + x1.w) + (x2.w + x3.w);
        } else {
#pragma unroll
          for (int k = 0; k < KMAX; ++k)
            if (k0 + k < j.N2) {
              f4_fma(acc[k], __ldcg(P + (size_t)r * j.ldp + k0 + k), x0);
              f4_fma(acc[k], __ldcg(P + (size_t)(r + 8) * j.ldp + k0 + k), x1);
              f4_fma(acc[k], __ldcg(P + (size_t)(r + 16) * j.ldp + k0 + k), x2);
              f4_fma(acc[k], __ldcg(P + (size_t)(r + 24) * j.ldp + k0 + k), x3);
            }
        }
      }
      for (; r < r1; r += 8) {
        const float4 x = ldx(X, r);
        if (P == nullptr) {
          acc[0].x += x.x;
          acc[0].y += x.y;
          acc[0].z += x.z;
          acc[0].w += x.w;
        } else {
#pragma unroll
          for (int k = 0; k < KMAX; ++k)
            if (k0 + k < j.N2) f4_fma(acc[k], __ldcg(P + (size_t)r * j.ldp + k0 + k), x);
        }
      }
    }
  }
#pragma unroll
  for (int k = 0; k < KMAX; ++k) {
    if (k0 + k >= j.N2) break;
    red[warp][lane] = acc[k];
    row_sync();
    if (warp == 0 && n < j.N) {
      float4 t = f4_zero();
#pragma unroll
      for (int y = 0; y < 8; ++y) {
        const float4 v = red[y][lane];
        t.x += v.x;
        t.y += v.y;
        t.z += v.z;
        t.w += v.w;
      }
      float* o = j.partial + ((size_t)split * j.N2 + k0 + k) * j.N + n;
      if (VEC) {
        *reinterpret_cast<float4*>(o) = t;
      } else {
        o[0] = t.x;
        if (n + 1 < j.N) o[1] = t.y;
        if (n + 2 < j.N) o[2] = t.z;
        if (n + 3 < j.N) o[3] = t.w;
      }
    }
    row_sync();
  }
}

__device__ __noinline__ void colsum_part_task(float* __restrict__ sm, const int cb, const int split, const int tid) {
  const WColsumJob& j = g_job;      // file-scope shared memory: LDS, never aliased by the global stores
  float4(*red)[33] = reinterpret_cast<float4(*)[33]>(sm);
  const int lane = tid & 31, warp = tid >> 5;
  if (cb * 128 >= j.N || split >= j.nsplit) return;
  if (j.vec4) {
    if (j.N2 <= 1) {
      colsum_part_body<1, true>(j, red, cb, split, 0, lane, warp);
    } else if (j.N2 <= 2) {
      colsum_part_body<2, true>(j, red, cb, split, 0, lane, warp);
    } else {
      for (int k0 = 0; k0 < j.N2; k0 += 4) colsum_part_body<4, true>(j, red, cb, split, k0, lane, warp);
    }
  } else {
    if (j.N2 <= 1) {
      colsum_part_body<1, false>(j, red, cb, split, 0, lane, warp);
    } else if (j.N2 <= 2) {
      colsum_part_body<2, false>(j, red, cb, split, 0, lane, warp);
    } else {
      for (int k0 = 0; k0 < j.N2; k0 += 4) colsum_part_body<4, false>(j, red, cb, split, k0, lane, warp);
    }
  }
}

// out[k, n] = sum_split partial[split, k, n] in split order (the whole job: N2*N outputs, 256 threads)
__device__ __noinline__ void colsum_reduce_task(const int tid) {
  const WColsumJob& j = g_job;
  const int total = j.N2 * j.N;
  const int nsplit = j.nsplit;
  for (int e = tid; e < total; e += kRowThreads) {
    const float* p = j.partial + e;
    float s = 0.f;
    int sp = 0;
    for (; sp + 8 <= nsplit; sp += 8) {
      float v[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] = __ldcg(p + (size_t)(sp + i) * total);
      s += ((v[0] + v[1]) + (v[2] + v[3])) + ((v[4] + v[5]) + (v[6] + v[7]));
    }
    for (; sp < nsplit; ++sp) s += __ldcg(p + (size_t)sp * total);
    j.out[(size_t)(e / j.N) * j.ldo + (e % j.N)] = s;
  }
}

// ---- stand-alone row kernels of the phased executor --------------------------------------------------------
__global__ void __launch_bounds__(kRowThreads) frame_row_kernel(const __grid_constant__ TailArgs a) {
  for (int i = threadIdx.x; i < (int)(sizeof(TailArgs) / sizeof(int)); i += kRowThreads)
    reinterpret_cast<int*>(&g_tail)[i] = reinterpret_cast<const int*>(&a)[i];
  __syncthreads();
  pdl_wait();
  const int r0 = blockIdx.x * kRowFrames;
  const int nr = min(kRowFrames, a.M * a.T - r0);
  if (nr > 0) frame_task(r0, nr, threadIdx.x);
}

__global__ void __launch_bounds__(kRowThreads) video_row_kernel(const __grid_constant__ TailArgs a, const int kind) {
  for (int i = threadIdx.x; i < (int)(sizeof(TailArgs) / sizeof(int)); i += kRowThreads)
    reinterpret_cast<int*>(&g_tail)[i] = reinterpret_cast<const int*>(&a)[i];
  __syncthreads();
  pdl_wait();
  const int v0 = blockIdx.x * kRowVideos;
  const int nv = min(kRowVideos, a.M - v0);
  if (nv > 0) video_row_task(kind, v0, nv, threadIdx.x);
}

// column sums of the phased executor: the same task functions, (job, column block, row split) from the block index
__global__ void __launch_bounds__(kRowThreads) step_colsum_part_kernel(const __grid_constant__ WColsumTable tab) {
  __shared__ __align__(16) float red_sm[8 * 33 * 4];
  pdl_wait();
  for (int i = threadIdx.x; i < (int)(sizeof(WColsumJob) / sizeof(int)); i += kRowThreads)
    reinterpret_cast<int*>(&g_job)[i] = reinterpret_cast<const int*>(&tab.job[blockIdx.y])[i];
  __syncthreads();
  colsum_part_task(red_sm, blockIdx.x, blockIdx.z, threadIdx.x);
}

__global__ void __launch_bounds__(kRowThreads)
step_colsum_reduce_kernel(const __grid_constant__ WColsumTable tab, unsigned long long* step_counter) {
  pdl_wait();
  for (int i = threadIdx.x; i < (int)(sizeof(WColsumJob) / sizeof(int)); i += kRowThreads)
    reinterpret_cast<int*>(&g_job)[i] = reinterpret_cast<const int*>(&tab.job[blockIdx.x])[i];
  __syncthreads();
  colsum_reduce_task(threadIdx.x);
  if (step_counter && blockIdx.x == 0 && threadIdx.x == 0) step_counter[0] += 1ull;   // last launch of the step
}

}  // namespace ta3n
