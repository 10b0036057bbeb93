// rowops.cuh -- the light (HBM-bound) kernels of the path: small heads, entropy attention and
// pooling, ReLU/dropout masks, bias-gradient column sums.  All fp32, coalesced along the
// feature dimension; warp-per-row where a row reduction is needed.
#pragma once

#include "common.cuh"

namespace ta3n {

constexpr int kMaxScales = 32;   // R = T-1 <= 32
constexpr int kMaxRel = 96;      // relations evaluated (1 + 3*(R-1)) <= 96

struct PtrTable {
  const float* p[kMaxScales];
};
struct MutPtrTable {
  float* p[kMaxScales];
};
struct RelMap {
  int n_rel;
  int n_scales;
  int rel_begin[kMaxScales + 1];   // relations of scale i are [rel_begin[i], rel_begin[i+1])
  unsigned char scale_of[kMaxRel];
};

inline unsigned blocks_for(size_t n, int threads) {
  size_t b = (n + threads - 1) / threads;
  if (b > 132u * 32u) b = 132u * 32u;   // grid-stride beyond 32 CTAs per SM
  if (b == 0) b = 1;
  return (unsigned)b;
}

// ---- feat_rel[m,i,:] = sum_r act[q(i,r)][m,:]                              TRNmodule.py:79 ----
__global__ void __launch_bounds__(256) relsum_kernel(const float* __restrict__ act, float* __restrict__ feat_rel,
                                                     int M, int H, const __grid_constant__ RelMap map) {
  pdl_wait();
  const int R = map.n_scales;
  const size_t total = (size_t)M * R * H;
  const size_t plane = (size_t)M * H;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const int h = (int)(e % H);
    const size_t mi = e / H;
    const int i = (int)(mi % R);
    const size_t m = mi / R;
    float s = 0.f;
    for (int q = map.rel_begin[i]; q < map.rel_begin[i + 1]; ++q) s += act[q * plane + m * H + h];
    feat_rel[e] = s;
  }
}

// ---- dZ[q][m,h] = d_feat_rel[m,i(q),h] * 1[act[q][m,h] > 0] ------------------------------------
__global__ void __launch_bounds__(256) dz_kernel(const float* __restrict__ act, const float* __restrict__ d_feat_rel,
                                                 float* __restrict__ dz, int M, int H,
                                                 const __grid_constant__ RelMap map) {
  pdl_wait();
  const int R = map.n_scales;
  const size_t plane = (size_t)M * H;
  const size_t total = plane * map.n_rel;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const int q = (int)(e / plane);
    const size_t mh = e % plane;
    const size_t m = mh / H;
    const int h = (int)(mh % H);
    const int i = map.scale_of[q];
    dz[e] = act[e] > 0.f ? d_feat_rel[(m * R + i) * H + h] : 0.f;
  }
}

// ---- 16-byte variants of the two kernels above (H % 4 == 0, 16 B aligned buffers, < 2^31 float4s): one thread
// per 4 consecutive h shares the index arithmetic (32-bit), and the relation tables are read from shared
// memory -- run-time indexed kernel parameters are ~300-cycle generic loads on the critical path.
inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

__global__ void __launch_bounds__(256) relsum_v4_kernel(const float4* __restrict__ act, float4* __restrict__ feat_rel,
                                                        int M, int H4, const __grid_constant__ RelMap map) {
  __shared__ int rb[kMaxScales + 1];
  const int R = map.n_scales;
  if (threadIdx.x <= R) rb[threadIdx.x] = map.rel_begin[threadIdx.x];
  __syncthreads();
  pdl_wait();
  const unsigned total = (unsigned)M * R * H4, plane = (unsigned)M * H4;
  for (unsigned e = blockIdx.x * blockDim.x + threadIdx.x; e < total; e += gridDim.x * blockDim.x) {
    const unsigned mi = e / H4, h = e - mi * H4;
    const unsigned m = mi / R, i = mi - m * R;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int q = rb[i]; q < rb[i + 1]; ++q) {
      const float4 a = act[q * plane + m * H4 + h];
      s.x += a.x;
      s.y += a.y;
      s.z += a.z;
      s.w += a.w;
    }
    feat_rel[e] = s;
  }
}

__global__ void __launch_bounds__(256) dz_v4_kernel(const float4* __restrict__ act, const float4* __restrict__ d_feat_rel,
                                                    float4* __restrict__ dz, int M, int H4,
                                                    const __grid_constant__ RelMap map) {
  __shared__ unsigned char so[kMaxRel];
  for (int q = threadIdx.x; q < map.n_rel; q += blockDim.x) so[q] = map.scale_of[q];
  __syncthreads();
  pdl_wait();
  const unsigned R = map.n_scales;
  const unsigned plane = (unsigned)M * H4, total = plane * map.n_rel;
  for (unsigned e = blockIdx.x * blockDim.x + threadIdx.x; e < total; e += gridDim.x * blockDim.x) {
    const unsigned q = e / plane, mh = e - q * plane;
    const unsigned m = mh / H4, h = mh - m * H4;
    const float4 a = act[e];
    const float4 g = d_feat_rel[(m * R + so[q]) * H4 + h];
    dz[e] = make_float4(a.x > 0.f ? g.x : 0.f, a.y > 0.f ? g.y : 0.f, a.z > 0.f ? g.z : 0.f, a.w > 0.f ? g.w : 0.f);
  }
}

// ---- dropout helpers -----------------------------------------------------------------------------
struct DropArgs {
  float p, scale;
  const uint8_t* keep;
  uint64_t seed;
  const uint64_t* step_dev;
  int mode;   // 0 none, 1 mask, 2 rng
};
inline DropArgs make_drop(const ta3n_dropout* d) {
  DropArgs a;
  memset(&a, 0, sizeof(a));
  a.scale = 1.0f;
  if (d && d->p > 0.0f) {
    a.p = d->p;
    a.scale = 1.0f / (1.0f - d->p);
    a.keep = d->keep;
    a.seed = d->seed;
    a.step_dev = d->step_dev;
    a.mode = d->keep ? 1 : 2;
  }
  return a;
}
__device__ __forceinline__ float drop_factor(const DropArgs& a, size_t e) {
  if (a.mode == 0) return 1.0f;
  bool k = (a.mode == 1) ? (a.keep[e] != 0) : rng_keep(a.seed, a.step_dev ? *a.step_dev : 0ull, e, a.p);
  return k ? a.scale : 0.0f;
}

// ---- small head: out[row, n] = <x[row,:], W[n,:]> + b[n], n < N2 (warp per row) -----------------
// W (N2 x K, a few KB) is staged in shared memory by the whole block with all loads in flight at once; a
// warp then keeps its row of x in registers and produces the N2 logits from on-chip data only.  (The first
// version re-read W through L1 inside the n loop: N2 dependent round trips per row.)
constexpr int kHeadMaxK = 1024;   // x row held in registers: K/32 values per lane
__global__ void __launch_bounds__(128) head_fwd_kernel(const float* __restrict__ x, int ldx,
                                                       const float* __restrict__ W, const float* __restrict__ b,
                                                       float* __restrict__ out, int ldo, int rows, int K, int N2,
                                                       int w_in_smem, const DropArgs drop, float* __restrict__ x_out) {
  pdl_wait();
  extern __shared__ float head_ws[];
  const int lane = threadIdx.x & 31;
  const int warps_per_block = blockDim.x >> 5;
  if (w_in_smem) {
    for (int i = threadIdx.x; i < N2 * K; i += blockDim.x) head_ws[i] = __ldg(W + i);
    __syncthreads();
  }
  const float* Wp = w_in_smem ? head_ws : W;
  for (int row = blockIdx.x * warps_per_block + (threadIdx.x >> 5); row < rows; row += gridDim.x * warps_per_block) {
    const float* xr = x + (size_t)row * ldx;
    if (K <= kHeadMaxK) {
      float xv[kHeadMaxK / 32];
#pragma unroll
      for (int i = 0; i < kHeadMaxK / 32; ++i) xv[i] = (lane + 32 * i < K) ? xr[lane + 32 * i] : 0.f;
      if (x_out) {   // fused Dropout in front of the head (models.py:679-680): x_out = x * keep / (1-p)
#pragma unroll
        for (int i = 0; i < kHeadMaxK / 32; ++i)
          if (lane + 32 * i < K) {
            const size_t e = (size_t)row * K + lane + 32 * i;
            xv[i] *= drop_factor(drop, e);
            x_out[e] = xv[i];
          }
      }
      // Logits in chunks of 32: lane n ends up holding logit n0 + n, the bias is read once per chunk, not per
      // logit (a dependent L2 round trip inside the loop was the longest part of the C-logit head)
      for (int n0 = 0; n0 < N2; n0 += 32) {
        const int nn = min(32, N2 - n0);
        float res = (b && lane < nn) ? b[n0 + lane] : 0.f;
        for (int n = 0; n < nn; ++n) {
          const float* wr = Wp + (size_t)(n0 + n) * K;
          float s = 0.f;
#pragma unroll
          for (int i = 0; i < kHeadMaxK / 32; ++i)
            if (lane + 32 * i < K) s = fmaf(xv[i], wr[lane + 32 * i], s);
          s = warp_sum(s);
          if (lane == n) res += s;
        }
        if (lane < nn) out[(size_t)row * ldo + n0 + lane] = res;
      }
    } else {   // very wide rows (fc_dim >= 2048): stream x from L1/L2
      if (x_out) {
        for (int k = lane; k < K; k += 32) x_out[(size_t)row * K + k] = xr[k] * drop_factor(drop, (size_t)row * K + k);
        __syncwarp();
        xr = x_out + (size_t)row * K;
      }
      for (int n = 0; n < N2; ++n) {
        const float* wr = Wp + (size_t)n * K;
        float s = 0.f;
        for (int k = lane; k < K; k += 32) s = fmaf(xr[k], wr[k], s);
        s = warp_sum(s);
        if (lane == 0) out[(size_t)row * ldo + n] = s + (b ? b[n] : 0.f);
      }
    }
  }
}

inline int launch_head_fwd(const float* x, int ldx, const float* W, const float* b, float* out, int ldo, int rows,
                           int K, int N2, cudaStream_t st, const DropArgs* drop = nullptr, float* x_out = nullptr) {
  DropArgs d;
  memset(&d, 0, sizeof(d));
  d.scale = 1.0f;
  if (drop) d = *drop;
  const size_t wbytes = (size_t)N2 * K * sizeof(float);
  const int in_smem = wbytes <= 48 * 1024 ? 1 : 0;
  size_t blocks = ((size_t)rows + 3) / 4;
  if (blocks > 132 * 8) blocks = 132 * 8;
  if (blocks == 0) blocks = 1;
  pre_launch("head_fwd", st);
  launch_kernel(head_fwd_kernel, (unsigned)blocks, 128, in_smem ? wbytes : 0, st, x, ldx, W, b, out, ldo, rows, K, N2, in_smem, d, x_out);
  return after_launch();
}

// ---- out[row,k] = alpha * (sum_n g[row,n] W[n,k]) * 1[gate[row,k] > 0]  (+ out if accumulate) ----
__global__ void __launch_bounds__(256) head_bwd_data_kernel(const float* __restrict__ g, int N2,
                                                            const float* __restrict__ W,
                                                            const float* __restrict__ gate, float alpha,
                                                            int accumulate, float* __restrict__ out, int rows, int K) {
  pdl_wait();
  const size_t total = (size_t)rows * K;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const size_t row = e / K;
    const int k = (int)(e % K);
    float s = 0.f;
    for (int n = 0; n < N2; ++n) s = fmaf(g[row * N2 + n], __ldg(W + (size_t)n * K + k), s);
    s *= alpha;
    if (gate && !(gate[e] > 0.f)) s = 0.f;
    out[e] = accumulate ? out[e] + s : s;
  }
}

// 16-byte variant (K % 4 == 0, aligned buffers, rows*K/4 < 2^31, N2 <= 32)
__global__ void __launch_bounds__(256) head_bwd_data_v4_kernel(const float* __restrict__ g, int N2,
                                                               const float4* __restrict__ W,
                                                               const float4* __restrict__ gate, float alpha,
                                                               int accumulate, float4* __restrict__ out, int rows,
                                                               int K4) {
  pdl_wait();
  const unsigned total = (unsigned)rows * K4;
  for (unsigned e = blockIdx.x * blockDim.x + threadIdx.x; e < total; e += gridDim.x * blockDim.x) {
    const unsigned row = e / K4, k = e - row * K4;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int n = 0; n < N2; ++n) {
      const float gv = g[row * N2 + n];
      const float4 w = __ldg(W + (size_t)n * K4 + k);
      s.x = fmaf(gv, w.x, s.x);
      s.y = fmaf(gv, w.y, s.y);
      s.z = fmaf(gv, w.z, s.z);
      s.w = fmaf(gv, w.w, s.w);
    }
    s.x *= alpha;
    s.y *= alpha;
    s.z *= alpha;
    s.w *= alpha;
    if (gate) {
      const float4 t = gate[e];
      if (!(t.x > 0.f)) s.x = 0.f;
      if (!(t.y > 0.f)) s.y = 0.f;
      if (!(t.z > 0.f)) s.z = 0.f;
      if (!(t.w > 0.f)) s.w = 0.f;
    }
    if (accumulate) {
      const float4 o = out[e];
      s.x += o.x;
      s.y += o.y;
      s.z += o.z;
      s.w += o.w;
    }
    out[e] = s;
  }
}

inline void launch_head_bwd_data(const float* g, int N2, const float* W, const float* gate, float alpha, int accumulate,
                                 float* out, int rows, int K, cudaStream_t st) {
  const size_t total = (size_t)rows * K;
  if (K % 4 == 0 && aligned16(W) && aligned16(out) && (!gate || aligned16(gate)) && total / 4 < (1ull << 31)) {
    launch_kernel(head_bwd_data_v4_kernel, blocks_for(total / 4, 256), 256, 0, st, g, N2,
                  reinterpret_cast<const float4*>(W), reinterpret_cast<const float4*>(gate), alpha, accumulate,
                  reinterpret_cast<float4*>(out), rows, K / 4);
  } else {
    launch_kernel(head_bwd_data_kernel, blocks_for(total, 256), 256, 0, st, g, N2, W, gate, alpha, accumulate, out,
                  rows, K);
  }
}

// ---- relation heads + entropy attention + attentive pooling (block per video, warp per relation) ---
// models.py:479 (second Linear of each relation discriminator), :351-357, :379-388, :651-652
constexpr int kRelWarps = 8;
__global__ void __launch_bounds__(kRelWarps * 32)
relattn_fwd_kernel(const float* __restrict__ feat_rel, const float* __restrict__ hidden, int M, int R, int H,
                   const __grid_constant__ PtrTable W2, const __grid_constant__ PtrTable b2, int use_attn,
                   float* __restrict__ pred_rel, float* __restrict__ attn, float* __restrict__ feat_video) {
  pdl_wait();
  __shared__ float wsh[kMaxScales];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
  const int m = blockIdx.x;
  for (int i = warp; i < R; i += nwarp) {
    const float* hr = hidden + ((size_t)i * M + m) * H;
    const float* w0 = W2.p[i];
    const float* w1 = w0 + H;
    float s0 = 0.f, s1 = 0.f;
    for (int h = lane; h < H; h += 32) {
      const float hv = hr[h];
      s0 = fmaf(hv, __ldg(w0 + h), s0);
      s1 = fmaf(hv, __ldg(w1 + h), s1);
    }
    s0 = warp_sum(s0) + b2.p[i][0];
    s1 = warp_sum(s1) + b2.p[i][1];
    const float w = use_attn ? attn_from_logits(s0, s1).w : 0.f;   // 'none': plain sum, (w + 1) == 1
    if (lane == 0) {
      pred_rel[((size_t)m * R + i) * 2 + 0] = s0;
      pred_rel[((size_t)m * R + i) * 2 + 1] = s1;
      attn[(size_t)m * R + i] = use_attn ? w : feat_rel[((size_t)m * R + i) * H];   // :647 placeholder
      wsh[i] = w + 1.0f;
    }
  }
  __syncthreads();
  for (int h = threadIdx.x; h < H; h += blockDim.x) {
    float y = 0.f;
    for (int i = 0; i < R; ++i) y = fmaf(wsh[i], feat_rel[((size_t)m * R + i) * H + h], y);
    feat_video[(size_t)m * H + h] = y;
  }
}

// ---- backward of the above up to the hidden layer (block per video, warp per relation) ----------
//   dw_i   = <G[m], feat_rel[m,i]> + g_attn[m,i]
//   Pt_ik  = g_pred[m,i,k] + dw_i * q_ik (log q_ik + E_i)
//   dHid_i = (Pt_i0 W2_i[0,:] + Pt_i1 W2_i[1,:]) * 1[hidden_i > 0]
__global__ void __launch_bounds__(kRelWarps * 32)
relattn_bwd_pre_kernel(const float* __restrict__ feat_rel, const float* __restrict__ hidden,
                       const float* __restrict__ pred_rel, const float* __restrict__ G,
                       const float* __restrict__ g_pred, const float* __restrict__ g_attn, int M, int R, int H,
                       const __grid_constant__ PtrTable W2, int use_attn, float* __restrict__ Pt,
                       float* __restrict__ d_hidden) {
  pdl_wait();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
  const int m = blockIdx.x;
  for (int i = warp; i < R; i += nwarp) {
    float pt0 = g_pred ? g_pred[((size_t)m * R + i) * 2 + 0] : 0.f;
    float pt1 = g_pred ? g_pred[((size_t)m * R + i) * 2 + 1] : 0.f;
    if (use_attn) {
      const float* fr = feat_rel + ((size_t)m * R + i) * H;
      const float* gr = G + (size_t)m * H;
      float dw = 0.f;
      for (int h = lane; h < H; h += 32) dw = fmaf(gr[h], fr[h], dw);
      dw = warp_sum(dw);
      if (g_attn) dw += g_attn[(size_t)m * R + i];
      const Attn2 a = attn_from_logits(pred_rel[((size_t)m * R + i) * 2 + 0], pred_rel[((size_t)m * R + i) * 2 + 1]);
      pt0 += dw * a.q0 * (a.lq0 + a.ent);
      pt1 += dw * a.q1 * (a.lq1 + a.ent);
    }
    if (lane == 0) {
      Pt[((size_t)m * R + i) * 2 + 0] = pt0;
      Pt[((size_t)m * R + i) * 2 + 1] = pt1;
    }
    const float* w0 = W2.p[i];
    const float* w1 = w0 + H;
    const float* hr = hidden + ((size_t)i * M + m) * H;
    float* dh = d_hidden + ((size_t)i * M + m) * H;
    for (int h = lane; h < H; h += 32)
      dh[h] = hr[h] > 0.f ? fmaf(pt0, __ldg(w0 + h), pt1 * __ldg(w1 + h)) : 0.f;
  }
}

// d_feat_rel[m,i,0] += g_attn[m,i]   (use_attn='none' placeholder output, models.py:647)
__global__ void attn_placeholder_bwd_kernel(const float* __restrict__ g_attn, float* __restrict__ d_feat_rel,
                                            int M, int R, int H) {
  pdl_wait();
  const int total = M * R;
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < total; e += gridDim.x * blockDim.x)
    d_feat_rel[(size_t)e * H] += g_attn[e];
}

// ---- 'general' attention over the relation features              models.py:320-325, 359-366, 379-388 ----
// attn_layer = Linear(H,H) -> Tanh -> Linear(H,1); the first Linear (+ bias) has been applied by a GEMM and sits in
// `hidden` [M*R, H] (row m*R + r).  Block per video, warp per relation:
//   hidden <- tanh(hidden);  s_r = <w2, hidden_r> + b2;  a = softmax_r(s);  attn[m,:] = a
//   feat_video[m,:] += sum_r a_r feat_rel[m,r,:]          (it already holds the plain sum: (a_r + 1) in total)
__global__ void __launch_bounds__(kRelWarps * 32)
general_attn_fwd_kernel(const float* __restrict__ feat_rel, float* __restrict__ hidden, int M, int R, int H,
                        const float* __restrict__ w2, const float* __restrict__ b2, float* __restrict__ attn,
                        float* __restrict__ feat_video) {
  pdl_wait();
  __shared__ float ssh[kMaxScales];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
  const int m = blockIdx.x;
  for (int r = warp; r < R; r += nwarp) {
    float* hr = hidden + ((size_t)m * R + r) * H;
    float s = 0.f;
    for (int h = lane; h < H; h += 32) {
      const float t = tanhf(hr[h]);
      hr[h] = t;
      s = fmaf(t, __ldg(w2 + h), s);
    }
    s = warp_sum(s) + __ldg(b2);
    if (lane == 0) ssh[r] = s;
  }
  __syncthreads();
  float mx = ssh[0];
  for (int r = 1; r < R; ++r) mx = fmaxf(mx, ssh[r]);
  float den = 0.f;
  for (int r = 0; r < R; ++r) den += expf(ssh[r] - mx);
  const float inv = 1.0f / den;
  if ((int)threadIdx.x < R) attn[(size_t)m * R + threadIdx.x] = expf(ssh[threadIdx.x] - mx) * inv;
  for (int h = threadIdx.x; h < H; h += blockDim.x) {
    float y = feat_video[(size_t)m * H + h];
    for (int r = 0; r < R; ++r) y = fmaf(expf(ssh[r] - mx) * inv, feat_rel[((size_t)m * R + r) * H + h], y);
    feat_video[(size_t)m * H + h] = y;
  }
}

// backward of the above up to the pre-activation of the first Linear (block per video, warp per relation):
//   da_r = <G[m], feat_rel[m,r]> + g_attn[m,r];  ds_r = a_r (da_r - sum_q a_q da_q)
//   d_pre[m,r,:] = ds_r * w2 * (1 - hidden[m,r,:]^2);  d_s[m,r] = ds_r
__global__ void __launch_bounds__(kRelWarps * 32)
general_attn_bwd_kernel(const float* __restrict__ feat_rel, const float* __restrict__ hidden,
                        const float* __restrict__ attn, const float* __restrict__ G, const float* __restrict__ g_attn,
                        int M, int R, int H, const float* __restrict__ w2, float* __restrict__ d_s,
                        float* __restrict__ d_pre) {
  pdl_wait();
  __shared__ float da[kMaxScales];
  __shared__ float ds[kMaxScales];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
  const int m = blockIdx.x;
  for (int r = warp; r < R; r += nwarp) {
    const float* fr = feat_rel + ((size_t)m * R + r) * H;
    const float* gr = G + (size_t)m * H;
    float dot = 0.f;
    for (int h = lane; h < H; h += 32) dot = fmaf(gr[h], fr[h], dot);
    dot = warp_sum(dot);
    if (g_attn) dot += g_attn[(size_t)m * R + r];
    if (lane == 0) da[r] = dot;
  }
  __syncthreads();
  if ((int)threadIdx.x < R) {
    float mean = 0.f;
    for (int q = 0; q < R; ++q) mean = fmaf(attn[(size_t)m * R + q], da[q], mean);
    const float v = attn[(size_t)m * R + threadIdx.x] * (da[threadIdx.x] - mean);
    ds[threadIdx.x] = v;
    d_s[(size_t)m * R + threadIdx.x] = v;
  }
  __syncthreads();
  for (int r = warp; r < R; r += nwarp) {
    const float* hr = hidden + ((size_t)m * R + r) * H;
    float* dp = d_pre + ((size_t)m * R + r) * H;
    const float v = ds[r];
    for (int h = lane; h < H; h += 32) {
      const float t = hr[h];
      dp[h] = v * __ldg(w2 + h) * (1.0f - t * t);
    }
  }
}

// ---- average over the segments (frame_aggregation='avgpool')        models.py:425-433 (AvgPool2d([T, 1])) ----
// out[m, f] = (sum_t x[m, t, f]) / T ; consecutive threads take consecutive f: coalesced, each x element read once.
__global__ void __launch_bounds__(256) segment_mean_fwd_kernel(const float* __restrict__ x, float* __restrict__ out,
                                                               int M, int T, int F) {
  pdl_wait();
  const size_t total = (size_t)M * F;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const size_t m = e / F, f = e % F;
    const float* p = x + m * T * F + f;
    float s = 0.f;
    for (int t = 0; t < T; ++t) s += p[(size_t)t * F];
    out[e] = s / (float)T;
  }
}
// dx[m, t, f] = g[m, f] / T
__global__ void __launch_bounds__(256) segment_mean_bwd_kernel(const float* __restrict__ g, float* __restrict__ dx,
                                                               int M, int T, int F) {
  pdl_wait();
  const size_t total = (size_t)M * T * F;
  const size_t tf = (size_t)T * F;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const size_t m = e / tf, f = e % F;
    dx[e] = g[m * F + f] / (float)T;
  }
}

// ---- frame-level attention                                         models.py:368-377 ----------
__global__ void __launch_bounds__(256) frame_attn_fwd_kernel(const float* __restrict__ feat,
                                                             const float* __restrict__ logits, int rows, int F,
                                                             float* __restrict__ out) {
  pdl_wait();
  const size_t total = (size_t)rows * F;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const size_t row = e / F;
    const float w = attn_from_logits(logits[row * 2], logits[row * 2 + 1]).w;
    out[e] = (w + 1.0f) * feat[e];
  }
}

// warp per row: dw = <d_out, feat>; d_out *= (w+1); g_logits += dw * dw/dlogits
__global__ void __launch_bounds__(256) frame_attn_bwd_kernel(const float* __restrict__ feat,
                                                             const float* __restrict__ logits, int rows, int F,
                                                             float* __restrict__ d_out, float* __restrict__ g_logits) {
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const int warps_per_block = blockDim.x >> 5;
  for (int row = blockIdx.x * warps_per_block + (threadIdx.x >> 5); row < rows; row += gridDim.x * warps_per_block) {
    const float* fr = feat + (size_t)row * F;
    float* dr = d_out + (size_t)row * F;
    const Attn2 a = attn_from_logits(logits[(size_t)row * 2], logits[(size_t)row * 2 + 1]);
    float dw = 0.f;
    for (int k = lane; k < F; k += 32) dw = fmaf(dr[k], fr[k], dw);
    dw = warp_sum(dw);
    const float sc = a.w + 1.0f;
    for (int k = lane; k < F; k += 32) dr[k] *= sc;
    if (lane == 0) {
      g_logits[(size_t)row * 2 + 0] += dw * a.q0 * (a.lq0 + a.ent);
      g_logits[(size_t)row * 2 + 1] += dw * a.q1 * (a.lq1 + a.ent);
    }
  }
}

// d_feat_video = ((g_pred Wc) + extra) * grad_scale * keep/(1-p) + g_ext
__global__ void __launch_bounds__(256)
video_head_bwd_kernel(const float* __restrict__ g_pred, int C, const float* __restrict__ Wc,
                      const float* __restrict__ extra, const float* __restrict__ g_ext, float grad_scale,
                      const DropArgs a, float* __restrict__ out, int M, int H) {
  pdl_wait();
  const size_t total = (size_t)M * H;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const size_t m = e / H;
    const int h = (int)(e % H);
    float s = extra ? extra[e] : 0.f;
    if (g_pred)
      for (int c = 0; c < C; ++c) s = fmaf(g_pred[m * C + c], __ldg(Wc + (size_t)c * H + h), s);
    s *= grad_scale * drop_factor(a, e);
    if (g_ext) s += g_ext[e];
    out[e] = s;
  }
}

// d_pre = (d_feat + g_ext) * 1[feat > 0] * scale   (ReLU + dropout backward; feat>0 <=> kept & pre>0)
__global__ void __launch_bounds__(256) dpre_kernel(const float* __restrict__ feat, float* __restrict__ d_feat,
                                                   const float* __restrict__ g_ext, float scale, size_t total) {
  pdl_wait();
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    float g = d_feat[e] + (g_ext ? g_ext[e] : 0.f);
    d_feat[e] = feat[e] > 0.f ? g * scale : 0.f;
  }
}

__global__ void __launch_bounds__(256) dpre_v4_kernel(const float4* __restrict__ feat, float4* __restrict__ d_feat,
                                                      const float4* __restrict__ g_ext, float scale, unsigned total4) {
  pdl_wait();
  for (unsigned e = blockIdx.x * blockDim.x + threadIdx.x; e < total4; e += gridDim.x * blockDim.x) {
    float4 g = d_feat[e];
    if (g_ext) {
      const float4 x = g_ext[e];
      g.x += x.x;
      g.y += x.y;
      g.z += x.z;
      g.w += x.w;
    }
    const float4 f = feat[e];
    d_feat[e] = make_float4(f.x > 0.f ? g.x * scale : 0.f, f.y > 0.f ? g.y * scale : 0.f,
                            f.z > 0.f ? g.z * scale : 0.f, f.w > 0.f ? g.w * scale : 0.f);
  }
}

inline void launch_dpre(const float* feat, float* d_feat, const float* g_ext, float scale, size_t total, cudaStream_t st) {
  if (total % 4 == 0 && aligned16(feat) && aligned16(d_feat) && (!g_ext || aligned16(g_ext)) && total / 4 < (1ull << 31)) {
    launch_kernel(dpre_v4_kernel, blocks_for(total / 4, 256), 256, 0, st, reinterpret_cast<const float4*>(feat),
                  reinterpret_cast<float4*>(d_feat), reinterpret_cast<const float4*>(g_ext), scale,
                  (unsigned)(total / 4));
  } else {
    launch_kernel(dpre_kernel, blocks_for(total, 256), 256, 0, st, feat, d_feat, g_ext, scale, total);
  }
}

__global__ void __launch_bounds__(256) grl_bwd_kernel(const float* __restrict__ g, float beta, float* __restrict__ out,
                                                      size_t n) {
  pdl_wait();
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (size_t)gridDim.x * blockDim.x)
    out[e] = -beta * g[e];
}

// ---- fused loss heads of the shipped configuration (SURVEY 8f row n1) ----------------------------
//   main.py:446      CE(out_source, label)                         mean over Bs
//   main.py:508-538  CE(cat(pred_S, pred_T), cat(0s, 1s)) per level mean over the level's rows
//   main.py:559-562  gamma * mean_m (1 + H(softmax(dom_video_m))) * H(softmax(out_m))   (loss.py:15-25)
// One warp per video: writes d loss / d logits for every head and the video's loss contribution.
enum : int { LOSS_ADV_REL = 1, LOSS_ADV_VIDEO = 2, LOSS_ADV_FRAME = 4, LOSS_ATT_ENT = 8 };

__global__ void __launch_bounds__(256)
loss_heads_kernel(const float* __restrict__ pred_video, const long long* __restrict__ labels,
                  const long long* __restrict__ labels_t, const float* __restrict__ pred_rel, const float* __restrict__ pred_dom,
                  const float* __restrict__ pred_frame, int Bs, int M, int T, int R, int C, float gamma, int flags,
                  const int* __restrict__ valid_rows, float* __restrict__ g_video, float* __restrict__ g_rel,
                  float* __restrict__ g_dom, float* __restrict__ g_frame, float* __restrict__ row_loss) {
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const int warps_per_block = blockDim.x >> 5;
  // valid_rows = {real source rows, real target rows} of a zero-padded last mini-batch (main.py:354-372 pads,
  // main.py:421-422 "ignore dummy tensors" slices the padding off again before any loss): padded rows get zero
  // loss and zero gradient, and every mean runs over the real rows only.
  const int vs = valid_rows ? min(valid_rows[0], Bs) : Bs;
  const int vt = valid_rows ? min(valid_rows[1], M - Bs) : M - Bs;
  const float n_src = (float)max(vs, 1), n_all = (float)max(vs + vt, 1);
  // labels_t (use_target='Sv', main.py:442-446): the class CE also covers the target rows, its mean over vs + vt
  const bool sv = labels_t != nullptr;
  const float n_cls = sv ? n_all : n_src;
  for (int m = blockIdx.x * warps_per_block + (threadIdx.x >> 5); m < M; m += gridDim.x * warps_per_block) {
    const int dom = m >= Bs ? 1 : 0;
    if (dom ? (m - Bs >= vt) : (m >= vs)) {   // padding row
      for (int c = lane; c < C; c += 32) g_video[(size_t)m * C + c] = 0.f;
      for (int i = lane; i < 2 * R; i += 32) g_rel[(size_t)m * R * 2 + i] = 0.f;
      for (int t = lane; t < 2 * T; t += 32) g_frame[(size_t)m * T * 2 + t] = 0.f;
      if (lane < 2) g_dom[(size_t)m * 2 + lane] = 0.f;
      if (lane == 0) row_loss[m] = 0.f;
      continue;
    }
    float loss = 0.f;
    // class logits: softmax statistics over C
    const float* pv = pred_video + (size_t)m * C;
    float mx = -INFINITY;
    for (int c = lane; c < C; c += 32) mx = fmaxf(mx, pv[c]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float se = 0.f;
    for (int c = lane; c < C; c += 32) se += expf(pv[c] - mx);
    se = warp_sum(se);
    const float lse = logf(se);
    float hc = 0.f;   // entropy of the class prediction
    for (int c = lane; c < C; c += 32) {
      const float lq = pv[c] - mx - lse;
      hc -= expf(lq) * lq;
    }
    hc = warp_sum(hc);
    // video-level domain logits
    const Attn2 dv = attn_from_logits(pred_dom[(size_t)m * 2], pred_dom[(size_t)m * 2 + 1]);
    const bool att = (flags & LOSS_ATT_ENT) != 0;
    const float att_scale = att ? gamma / n_all : 0.f;
    const bool labelled = m < Bs || sv;
    const long long y = (m < Bs) ? labels[m] : (sv ? labels_t[m - Bs] : -1);
    for (int c = lane; c < C; c += 32) {
      const float lq = pv[c] - mx - lse;
      const float q = expf(lq);
      float gq = 0.f;
      if (labelled) gq = (q - (c == (int)y ? 1.f : 0.f)) / n_cls;
      gq += att_scale * (1.f + dv.ent) * (-q * (lq + hc));
      g_video[(size_t)m * C + c] = gq;
      if (labelled && c == (int)y && lane == (c & 31)) loss += -lq / n_cls;
    }
    loss = warp_sum(loss);   // exactly one lane held the CE term
    if (lane == 0) {
      float l = loss + att_scale * (1.f + dv.ent) * hc;
      float g0 = 0.f, g1 = 0.f;
      if (flags & LOSS_ADV_VIDEO) {
        l += -(dom ? dv.lq1 : dv.lq0) / n_all;
        g0 = (dv.q0 - (dom ? 0.f : 1.f)) / n_all;
        g1 = (dv.q1 - (dom ? 1.f : 0.f)) / n_all;
      }
      g0 += att_scale * hc * (-dv.q0 * (dv.lq0 + dv.ent));
      g1 += att_scale * hc * (-dv.q1 * (dv.lq1 + dv.ent));
      g_dom[(size_t)m * 2] = g0;
      g_dom[(size_t)m * 2 + 1] = g1;
      loss = l;
    }
    // relation-level and frame-level domain logits: one lane per (relation | frame)
    float extra = 0.f;
    for (int i = lane; i < R; i += 32) {
      const size_t o = ((size_t)m * R + i) * 2;
      float g0 = 0.f, g1 = 0.f;
      if (flags & LOSS_ADV_REL) {
        const Attn2 a = attn_from_logits(pred_rel[o], pred_rel[o + 1]);
        const float inv = 1.f / (n_all * (float)R);
        extra += -(dom ? a.lq1 : a.lq0) * inv;
        g0 = (a.q0 - (dom ? 0.f : 1.f)) * inv;
        g1 = (a.q1 - (dom ? 1.f : 0.f)) * inv;
      }
      g_rel[o] = g0;
      g_rel[o + 1] = g1;
    }
    for (int t = lane; t < T; t += 32) {
      const size_t o = ((size_t)m * T + t) * 2;
      float g0 = 0.f, g1 = 0.f;
      if (flags & LOSS_ADV_FRAME) {
        const Attn2 a = attn_from_logits(pred_frame[o], pred_frame[o + 1]);
        const float inv = 1.f / (n_all * (float)T);
        extra += -(dom ? a.lq1 : a.lq0) * inv;
        g0 = (a.q0 - (dom ? 0.f : 1.f)) * inv;
        g1 = (a.q1 - (dom ? 1.f : 0.f)) * inv;
      }
      g_frame[o] = g0;
      g_frame[o + 1] = g1;
    }
    extra = warp_sum(extra);
    if (lane == 0) row_loss[m] = loss + extra;
  }
}

// deterministic sum of row_loss[0..M) -> out[0]  (single block, fixed tree)
__global__ void __launch_bounds__(1024) loss_reduce_kernel(const float* __restrict__ row_loss, int M,
                                                           float* __restrict__ out) {
  pdl_wait();
  __shared__ float red[32];
  float s = 0.f;
  for (int i = threadIdx.x; i < M; i += blockDim.x) s += row_loss[i];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    t = warp_sum(t);
    if (threadIdx.x == 0) out[0] = t;
  }
}

// The counter advances at the START of a step: the video head's backward re-derives its dropout mask from the
// same counter value the forward used (rowops: video_head_bwd_kernel), so it must not move in between.
__global__ void counter_inc_kernel(unsigned long long* ctr) {
  pdl_wait(); ctr[0] += 1ull; }

// ---- loss terms of ens_DA='MCD' (main.py:446-448, 548-556; loss.py:29-30) ---------------------------
// One block: warp w takes rows w, w + 8, ...; every row's term is added to its warp's running sum in row order and
// the eight warp sums are added in warp order, so the scalar is the same bit pattern on every replay.
constexpr int kMcdThreads = 256;

__device__ __forceinline__ float row_max(const float* p, int C, int lane) {
  float mx = -INFINITY;
  for (int c = lane; c < C; c += 32) mx = fmaxf(mx, p[c]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  return mx;
}

__device__ __forceinline__ void block_add_scalar(float warp_total, float scale, float* out) {
  __shared__ float red[kMcdThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) red[warp] = warp_total;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < kMcdThreads / 32; ++w) t += red[w];
    out[0] += t * scale;
  }
}

// loss += mean over the real rows r < valid_rows[0] of CE(pred[r], labels[r]);  g_pred = its gradient (0 on padding)
__global__ void __launch_bounds__(kMcdThreads)
ce_loss_kernel(const float* __restrict__ pred, const long long* __restrict__ labels, int rows, int C,
               const int* __restrict__ valid_rows, float* __restrict__ loss, float* __restrict__ g_pred) {
  pdl_wait();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int vs = valid_rows ? max(0, min(valid_rows[0], rows)) : rows;
  const float inv = 1.f / (float)max(vs, 1);
  float acc = 0.f;   // lane 0: this warp's sum of -log q_y
  for (int r = warp; r < rows; r += kMcdThreads / 32) {
    float* g = g_pred + (size_t)r * C;
    if (r >= vs) {
      for (int c = lane; c < C; c += 32) g[c] = 0.f;
      continue;
    }
    const float* p = pred + (size_t)r * C;
    const float mx = row_max(p, C, lane);
    float se = 0.f;
    for (int c = lane; c < C; c += 32) se += expf(p[c] - mx);
    const float lse = logf(warp_sum(se));
    const int y = (int)labels[r];
    float ly = 0.f;
    for (int c = lane; c < C; c += 32) {
      const float lq = p[c] - mx - lse;
      g[c] = (expf(lq) - (c == y ? 1.f : 0.f)) * inv;
      if (c == y) ly = lq;
    }
    ly = warp_sum(ly);   // exactly one lane held log q_y
    if (lane == 0) acc -= ly;
  }
  block_add_scalar(acc, inv, loss);
}

// Discrepancy of the two classifiers on the real rows r < valid_rows[1] (main.py:548-556):
//   loss += -1/(n C) sum_r sum_c |s1_rc - s2_rc|,  s = softmax over C
//   u_c = dloss/ds1_c = -sign(s1_c - s2_c) / (n C)   (sign(0) = 0, as torch's abs backward)
//   g1_j = s1_j (u_j - sum_c s1_c u_c),  g2_j = s2_j (-u_j + sum_c s2_c u_c)
// g_move1 (optional): gradient other loss terms left on pred1; it is added to g1 and cleared.
__global__ void __launch_bounds__(kMcdThreads)
mcd_loss_kernel(const float* __restrict__ p1, const float* __restrict__ p2, int rows, int C,
                const int* __restrict__ valid_rows, float* __restrict__ loss, float* __restrict__ g1,
                float* __restrict__ g2, float* __restrict__ g_move1) {
  pdl_wait();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int vt = valid_rows ? max(0, min(valid_rows[1], rows)) : rows;
  const float inv = 1.f / ((float)max(vt, 1) * (float)C);
  float acc = 0.f;   // lane 0: this warp's sum of |s1 - s2|
  for (int r = warp; r < rows; r += kMcdThreads / 32) {
    const size_t o = (size_t)r * C;
    if (r >= vt) {
      for (int c = lane; c < C; c += 32) {
        g1[o + c] = g_move1 ? g_move1[o + c] : 0.f;
        g2[o + c] = 0.f;
        if (g_move1) g_move1[o + c] = 0.f;
      }
      continue;
    }
    const float m1 = row_max(p1 + o, C, lane), m2 = row_max(p2 + o, C, lane);
    float e1 = 0.f, e2 = 0.f;
    for (int c = lane; c < C; c += 32) {
      e1 += expf(p1[o + c] - m1);
      e2 += expf(p2[o + c] - m2);
    }
    const float l1 = logf(warp_sum(e1)), l2 = logf(warp_sum(e2));
    float sabs = 0.f, su1 = 0.f, su2 = 0.f;
    for (int c = lane; c < C; c += 32) {
      const float s1 = expf(p1[o + c] - m1 - l1), s2 = expf(p2[o + c] - m2 - l2);
      const float d = s1 - s2;
      const float u = d > 0.f ? -inv : (d < 0.f ? inv : 0.f);
      sabs += fabsf(d);
      su1 += s1 * u;
      su2 += s2 * u;
    }
    sabs = warp_sum(sabs);
    su1 = warp_sum(su1);
    su2 = warp_sum(su2);
    for (int c = lane; c < C; c += 32) {
      const float s1 = expf(p1[o + c] - m1 - l1), s2 = expf(p2[o + c] - m2 - l2);
      const float d = s1 - s2;
      const float u = d > 0.f ? -inv : (d < 0.f ? inv : 0.f);
      float a = s1 * (u - su1);
      if (g_move1) {
        a += g_move1[o + c];
        g_move1[o + c] = 0.f;
      }
      g1[o + c] = a;
      g2[o + c] = s2 * (su2 - u);
    }
    if (lane == 0) acc += sabs;
  }
  block_add_scalar(acc, -inv, loss);
}

constexpr int kEntThreads = 1024;

// Entropy of the target predictions, --add_loss_DA target_entropy (main.py:541-545, loss.py:8-12), on the real rows
// r < valid_rows[1]:
//   term = 1/n sum_r H_r,  H_r = -sum_c q_rc log q_rc,  q = softmax over C;  loss += gamma * term
//   g_pred[r] += gamma/n * (-q_rc (log q_rc + H_r))   (padded rows untouched)
// Warp w of 32 takes rows w, w + 32, ... (a row costs a few dependent warp reductions, so the block is as wide as it
// gets); the row entropies are summed in fp64, per warp in row order and then the warps in order, so the term is the
// same bit pattern on every replay.  n == 0 adds nothing.
// meter (optional, 3 doubles): {sum += term * n, last = term, count += n} -- the losses_e meter of main.py:544.
__global__ void __launch_bounds__(kEntThreads)
target_entropy_kernel(const float* __restrict__ pred, int rows, int C, float gamma, const int* __restrict__ valid_rows,
                      float* __restrict__ loss, float* __restrict__ g_pred, double* __restrict__ meter) {
  pdl_wait();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int vt = valid_rows ? max(0, min(valid_rows[1], rows)) : rows;
  const float scale = gamma / (float)max(vt, 1);
  double acc = 0.0;   // lane 0: this warp's sum of H_r
  for (int r = warp; r < vt; r += kEntThreads / 32) {
    const float* p = pred + (size_t)r * C;
    float* g = g_pred + (size_t)r * C;
    const float mx = row_max(p, C, lane);
    float se = 0.f;
    for (int c = lane; c < C; c += 32) se += expf(p[c] - mx);
    const float lse = logf(warp_sum(se));
    float h = 0.f;
    for (int c = lane; c < C; c += 32) {
      const float lq = p[c] - mx - lse;
      h -= expf(lq) * lq;
    }
    h = warp_sum(h);
    for (int c = lane; c < C; c += 32) {
      const float lq = p[c] - mx - lse;
      g[c] += scale * (-expf(lq) * (lq + h));
    }
    if (lane == 0) acc += (double)h;
  }
  __shared__ double red[kEntThreads / 32];
  if (lane == 0) red[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < kEntThreads / 32; ++w) t += red[w];
    const double term = vt > 0 ? t / (double)vt : 0.0;
    if (vt > 0) loss[0] += (float)((double)gamma * term);
    if (meter) {
      meter[0] += term * (double)vt;
      meter[1] = term;
      meter[2] += (double)vt;
    }
  }
}

// dst += src (n floats)
__global__ void __launch_bounds__(256) accumulate_kernel(float* __restrict__ dst, const float* __restrict__ src,
                                                         size_t n) {
  pdl_wait();
  const size_t n4 = n / 4;
  float4* d4 = reinterpret_cast<float4*>(dst);
  const float4* s4 = reinterpret_cast<const float4*>(src);
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < n4; e += (size_t)gridDim.x * blockDim.x) {
    float4 a = d4[e];
    const float4 b = s4[e];
    a.x += b.x;
    a.y += b.y;
    a.z += b.z;
    a.w += b.w;
    d4[e] = a;
  }
  for (size_t e = 4 * n4 + (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (size_t)gridDim.x * blockDim.x)
    dst[e] += src[e];
}

// ---- deterministic (weighted) column sums: bias gradients and the skinny head weight gradients ----
//   out[k*ldo + n] = sum_seg sum_r  P_seg[r*ldp + k] * X_seg[r*ld + n]      k < N2 <= 32, n < N
// P == nullptr -> N2 = 1 with unit weights (a plain column sum = a bias gradient).  The N2 x N outputs of
// the two-logit / C-logit heads (dW2 [2,H], dWc [C,H]) are tall-skinny reductions over the rows; as GEMM
// tiles they would be 98 % padding.  Two stages (row splits -> fixed-order sum) keep it deterministic.
// A block covers 128 columns x one row split: each thread owns 4 consecutive columns (one 16 B load per row,
// a warp reads 512 contiguous bytes) and keeps 4 rows in flight; the 8 warps of the block take rows r, r+1, ..
// The number of row splits is per job (tall inputs get more), so every block has 2-3 iterations of work.
struct WColsumJob {
  const float* X[4];
  const float* P[4];
  int rows[4];
  int nseg;
  int ld, ldp;
  int N, N2;
  int ldo;
  int nsplit;       // row splits of this job (<= kWColsumMaxSplits)
  int vec4;         // 1: N % 4 == 0, ld % 4 == 0 and every X 16-byte aligned -> float4 path
  float* out;
  float* partial;   // [nsplit, N2, N]
};
constexpr int kMaxWColsumJobs = 40;
constexpr int kWColsumMaxSplits = 32;
struct WColsumTable {
  int n_jobs;
  WColsumJob job[kMaxWColsumJobs];
};

__device__ __forceinline__ float4 f4_zero() { return make_float4(0.f, 0.f, 0.f, 0.f); }
__device__ __forceinline__ void f4_fma(float4& a, float p, const float4& x) {
  a.x = fmaf(p, x.x, a.x);
  a.y = fmaf(p, x.y, a.y);
  a.z = fmaf(p, x.z, a.z);
  a.w = fmaf(p, x.w, a.w);
}

// stage 1: grid (ceil(maxN/128), n_jobs, max splits), block (32, 8)
// One pass handles the weight columns k0 .. k0+KMAX-1 (KMAX <= 4 keeps the kernel at ~64 registers; the C-logit
// classifier head takes ceil(C/4) passes over its small, L2-resident input).
template <int KMAX, bool VEC>
__device__ __forceinline__ void wcolsum_body(const WColsumJob& j, float4 (*red)[33], const int k0) {
  const int n = blockIdx.x * 128 + threadIdx.x * 4;
  const int split = blockIdx.z, nsplit = j.nsplit;
  float4 acc[KMAX];
#pragma unroll
  for (int k = 0; k < KMAX; ++k) acc[k] = f4_zero();
  auto ldx = [&](const float* X, int r) -> float4 {
    const float* q = X + (size_t)r * j.ld + n;
    if (VEC) return *reinterpret_cast<const float4*>(q);
    float4 v = f4_zero();
    if (n < j.N) v.x = q[0];
    if (n + 1 < j.N) v.y = q[1];
    if (n + 2 < j.N) v.z = q[2];
    if (n + 3 < j.N) v.w = q[3];
    return v;
  };
  if (n < j.N) {
    for (int sg = 0; sg < j.nseg; ++sg) {
      const float* X = j.X[sg];
      const float* P = j.P[sg];
      const int rows = j.rows[sg];
      const int per = (rows + nsplit - 1) / nsplit;
      const int r1 = min(rows, (split + 1) * per);
      int r = split * per + threadIdx.y;
      // four independent rows in flight per thread (the loads, not the adds, bound this kernel)
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
              f4_fma(acc[k], __ldg(P + (size_t)r * j.ldp + k0 + k), x0);
              f4_fma(acc[k], __ldg(P + (size_t)(r + 8) * j.ldp + k0 + k), x1);
              f4_fma(acc[k], __ldg(P + (size_t)(r + 16) * j.ldp + k0 + k), x2);
              f4_fma(acc[k], __ldg(P + (size_t)(r + 24) * j.ldp + k0 + k), x3);
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
            if (k0 + k < j.N2) f4_fma(acc[k], __ldg(P + (size_t)r * j.ldp + k0 + k), x);
        }
      }
    }
  }
#pragma unroll
  for (int k = 0; k < KMAX; ++k) {
    if (k0 + k >= j.N2) break;
    red[threadIdx.y][threadIdx.x] = acc[k];
    __syncthreads();
    if (threadIdx.y == 0 && n < j.N) {
      float4 t = f4_zero();
#pragma unroll
      for (int y = 0; y < 8; ++y) {
        const float4 v = red[y][threadIdx.x];
        t.x += v.x;
        t.y += v.y;
        t.z += v.z;
        t.w += v.w;
      }
      float* o = j.partial + ((size_t)split * j.N2 + k0 + k) * j.N + n;
      if (VEC) {
        *reinterpret_cast<float4*>(o) = t;      // partial rows are 16 B aligned when N % 4 == 0
      } else {
        o[0] = t.x;
        if (n + 1 < j.N) o[1] = t.y;
        if (n + 2 < j.N) o[2] = t.z;
        if (n + 3 < j.N) o[3] = t.w;
      }
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(256) wcolsum_stage1_kernel(const __grid_constant__ WColsumTable tab) {
  pdl_wait();
  __shared__ float4 red[8][33];
  __shared__ WColsumJob j;   // staged: run-time indexed kernel parameters are slow generic loads
  {
    const int* src = reinterpret_cast<const int*>(&tab.job[blockIdx.y]);
    int* dst = reinterpret_cast<int*>(&j);
    const int t = threadIdx.y * 32 + threadIdx.x;
    if (t < (int)(sizeof(WColsumJob) / sizeof(int))) dst[t] = src[t];
    __syncthreads();
  }
  if (blockIdx.x * 128 >= j.N || (int)blockIdx.z >= j.nsplit) return;
  if (j.vec4) {
    if (j.N2 <= 1) {
      wcolsum_body<1, true>(j, red, 0);
    } else if (j.N2 <= 2) {
      wcolsum_body<2, true>(j, red, 0);
    } else {
      for (int k0 = 0; k0 < j.N2; k0 += 4) wcolsum_body<4, true>(j, red, k0);
    }
  } else {
    if (j.N2 <= 1) {
      wcolsum_body<1, false>(j, red, 0);
    } else if (j.N2 <= 2) {
      wcolsum_body<2, false>(j, red, 0);
    } else {
      for (int k0 = 0; k0 < j.N2; k0 += 4) wcolsum_body<4, false>(j, red, k0);
    }
  }
}

// stage 2: out[k, n] = sum_split partial[split, k, n]; grid (blocks, n_jobs), one thread per output, eight
// splits in flight per thread in a fixed order (one dependent load per split was 10 us at 32 splits; a warp per
// output with a shuffle tree was slower still: 9600 mostly idle blocks each staging its job).
__global__ void __launch_bounds__(256) wcolsum_stage2_kernel(const __grid_constant__ WColsumTable tab) {
  pdl_wait();
  __shared__ WColsumJob j;
  {
    const int* src = reinterpret_cast<const int*>(&tab.job[blockIdx.y]);
    int* dst = reinterpret_cast<int*>(&j);
    if (threadIdx.x < (int)(sizeof(WColsumJob) / sizeof(int))) dst[threadIdx.x] = src[threadIdx.x];
    __syncthreads();
  }
  const int total = j.N2 * j.N;
  const int nsplit = j.nsplit;
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < total; e += gridDim.x * blockDim.x) {
    const float* p = j.partial + e;
    float s = 0.f;
    int sp = 0;
    for (; sp + 8 <= nsplit; sp += 8) {
      float v[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] = p[(size_t)(sp + i) * total];
      s += ((v[0] + v[1]) + (v[2] + v[3])) + ((v[4] + v[5]) + (v[6] + v[7]));
    }
    for (; sp < nsplit; ++sp) s += p[(size_t)sp * total];
    j.out[(size_t)(e / j.N) * j.ldo + (e % j.N)] = s;
  }
}

struct ColsumPlan {
  std::vector<WColsumJob> jobs;
  // plain column sum of X (N columns, leading dimension ld) -> out[N]
  WColsumJob& add(float* out, int N, int ld) {
    WColsumJob j;
    memset(&j, 0, sizeof(j));
    j.out = out;
    j.N = N;
    j.ld = ld;
    j.N2 = 1;
    j.ldo = N;
    jobs.push_back(j);
    return jobs.back();
  }
  // weighted: out[k*ldo + n] = sum_r P[r*ldp + k] X[r*ld + n]
  WColsumJob& add_weighted(float* out, int ldo, int N2, int N, int ld, int ldp) {
    WColsumJob& j = add(out, N, ld);
    j.N2 = N2;
    j.ldo = ldo;
    j.ldp = ldp;
    return j;
  }
  void seg(const float* X, int rows, const float* P = nullptr) {
    WColsumJob& j = jobs.back();
    if (rows <= 0) return;
    j.X[j.nseg] = X;
    j.P[j.nseg] = P;
    j.rows[j.nseg] = rows;
    j.nseg++;
  }
  static size_t workspace_bytes(size_t total_out_elems) {
    return Arena::round(total_out_elems * kWColsumMaxSplits * sizeof(float)) + 256 * (size_t)kMaxWColsumJobs;
  }
  // Needs arena space for the stage-1 partials (row splits x outputs).
  int run(cudaStream_t stream, Arena* arena) {
    size_t i = 0;
    while (i < jobs.size()) {
      WColsumTable tab;
      tab.n_jobs = 0;
      int maxN = 0, maxOut = 0, maxSplit = 1;
      while (i < jobs.size() && tab.n_jobs < kMaxWColsumJobs) {
        WColsumJob j = jobs[i];
        if (j.nseg == 0) {   // nothing to sum: the gradient is zero
          for (int k = 0; k < j.N2; ++k)
            TA3N_CUDA(cudaMemsetAsync(j.out + (size_t)k * j.ldo, 0, sizeof(float) * j.N, stream));
          ++i;
          continue;
        }
        // row splits: ~64 rows of the tallest segment per block (8 rows per thread), 4 ... 32
        int tall = 0;
        bool vec = (j.N % 4 == 0) && (j.ld % 4 == 0);
        for (int q = 0; q < j.nseg; ++q) {
          if (j.rows[q] > tall) tall = j.rows[q];
          if (reinterpret_cast<uintptr_t>(j.X[q]) & 15u) vec = false;
        }
        j.nsplit = std::min(kWColsumMaxSplits, std::max(4, (tall * j.nseg + 63) / 64));
        j.vec4 = vec ? 1 : 0;
        j.partial = arena ? arena->floats((size_t)j.nsplit * j.N2 * j.N) : nullptr;
        if (!j.partial) return fail(TA3N_ERR_WORKSPACE, "column-sum workspace too small");
        if (j.nsplit > maxSplit) maxSplit = j.nsplit;
        tab.job[tab.n_jobs++] = j;
        if (j.N > maxN) maxN = j.N;
        if (j.N * j.N2 > maxOut) maxOut = j.N * j.N2;
        ++i;
      }
      if (tab.n_jobs == 0) continue;
      dim3 grid((maxN + 127) / 128, tab.n_jobs, maxSplit), block(32, 8);
      pre_launch("wcolsum", stream);
      launch_kernel(wcolsum_stage1_kernel, grid, block, 0, stream, tab);
      TA3N_TRY(after_launch());
      dim3 grid2((maxOut + 255) / 256, tab.n_jobs);
      pre_launch("wcolsum_reduce", stream);
      launch_kernel(wcolsum_stage2_kernel, grid2, 256, 0, stream, tab);
      TA3N_TRY(after_launch());
    }
    return TA3N_OK;
  }
};

}  // namespace ta3n
