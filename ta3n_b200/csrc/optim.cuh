// Optimizer step of the training iteration (SURVEY 8f row n2): what the reference does right after
// loss.backward() (main.py:576-583):
//     total_norm = clip_grad_norm_(model.parameters(), args.clip_gradient)       main.py:578-581
//     optimizer.step()    # torch.optim.SGD(lr, momentum, weight_decay, nesterov=True)   main.py:83, 583
// over the flat fp32 gradient bucket the backward wrote (and NCCL averaged).  Two launches, HBM-bound:
//   1. sqnorm_partial_kernel: one fixed-order partial sum of squares per block          (reads g once)
//   2. sgd_nesterov_kernel:   every block folds the partials in the same order (so all blocks agree on the
//      clip coefficient bit for bit), then  g' = coef*g;  d = g' + wd*p;  m = mu*m + d;  p -= lr*(d + mu*m)
//      (reads p, g, m; writes p, m: 20 B per parameter).
// lr lives in device memory so a per-step schedule (main.py:800-802, DANN) replays inside a CUDA graph.
// With --optimizer Adam (main.py:84-86: torch.optim.Adam(lr, weight_decay)) launch 2 is adam_step_kernel instead: the
// same clip coefficient, then torch's single-tensor Adam update (reads p, g, m, v; writes p, m, v: 28 B per parameter).
#pragma once
#include "common.cuh"

namespace ta3n {

constexpr int kSqnormBlocks = 296;     // 2+ per SM on a 132-SM part; also the number of partials
constexpr int kOptThreads = 256;

__device__ __forceinline__ float block_sum_256(float s, float* red) {
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  float t = 0.f;
  if (threadIdx.x < 32) {
    t = threadIdx.x < (kOptThreads >> 5) ? red[threadIdx.x] : 0.f;
    t = warp_sum(t);
  }
  return t;     // valid in thread 0
}

__global__ void __launch_bounds__(kOptThreads) sqnorm_partial_kernel(const float* __restrict__ g, long long n,
                                                                     float* __restrict__ partial) {
  pdl_wait();
  __shared__ float red[32];
  const long long n4 = n >> 2;
  const float4* g4 = reinterpret_cast<const float4*>(g);
  float s0 = 0.f, s1 = 0.f;
  const long long stride = static_cast<long long>(gridDim.x) * kOptThreads;
  long long i = static_cast<long long>(blockIdx.x) * kOptThreads + threadIdx.x;
  for (; i + stride < n4; i += 2 * stride) {       // two independent loads in flight per thread
    float4 a = g4[i], b = g4[i + stride];
    s0 += a.x * a.x + a.y * a.y + a.z * a.z + a.w * a.w;
    s1 += b.x * b.x + b.y * b.y + b.z * b.z + b.w * b.w;
  }
  if (i < n4) {
    float4 a = g4[i];
    s0 += a.x * a.x + a.y * a.y + a.z * a.z + a.w * a.w;
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {  // tail (n not a multiple of 4)
    float v = g[(n4 << 2) + threadIdx.x];
    s1 += v * v;
  }
  float t = block_sum_256(s0 + s1, red);
  if (threadIdx.x == 0) partial[blockIdx.x] = t;
}

// The clip coefficient of clip_grad_norm_ from the sqnorm partials, called by every thread of a block.  Every block
// folds the partials in the same fixed order (thread t sums partial[t], partial[t+256], ...; then the fixed tree), so
// all blocks agree on the coefficient bit for bit.  Block 0 writes stats[0] = total gradient norm, stats[1] = coef.
__device__ __forceinline__ float clip_coef_fold(const float* __restrict__ partial, int n_partial, float max_norm,
                                                float* __restrict__ stats, float* red, float* coef_s) {
  float s = 0.f;
  for (int i = threadIdx.x; i < n_partial; i += kOptThreads) s += partial[i];
  float t = block_sum_256(s, red);
  if (threadIdx.x == 0) {
    float norm = sqrtf(t);
    float c = max_norm / (norm + 1e-6f);          // torch.nn.utils.clip_grad_norm_
    *coef_s = c < 1.f ? c : 1.f;
    if (blockIdx.x == 0 && stats != nullptr) { stats[0] = norm; stats[1] = *coef_s; }
  }
  __syncthreads();
  return *coef_s;
}

// stats[0] = total gradient norm, stats[1] = clip coefficient applied (1 when not clipping)
__global__ void __launch_bounds__(kOptThreads) sgd_nesterov_kernel(
    float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, long long n,
    const float* __restrict__ lr_dev, float mu, float wd, float max_norm, const float* __restrict__ partial,
    int n_partial, float* __restrict__ stats, const float* __restrict__ active) {
  pdl_wait();
  __shared__ float red[32];
  __shared__ float coef_s;
  float coef = 1.f;
  if (max_norm > 0.f) coef = clip_coef_fold(partial, n_partial, max_norm, stats, red, &coef_s);
  const float lr = lr_dev[0];
  const long long n4 = n >> 2;
  float4* p4 = reinterpret_cast<float4*>(p);
  float4* m4 = reinterpret_cast<float4*>(m);
  const float4* g4 = reinterpret_cast<const float4*>(g);
  const long long stride = static_cast<long long>(gridDim.x) * kOptThreads;
#define TA3N_SGD_ELEM(P, G, M)              \
  {                                         \
    float d = fmaf(wd, (P), coef * (G));    \
    float mm = fmaf(mu, (M), d);            \
    (M) = mm;                               \
    (P) = (P) - lr * fmaf(mu, mm, d);       \
  }
  // `active` (optional, one float per element, 0 = skip): parameters the configured losses give no gradient --
  // torch.optim.SGD leaves a parameter whose .grad is None untouched (no weight decay, no momentum), main.py:83
  for (long long i = static_cast<long long>(blockIdx.x) * kOptThreads + threadIdx.x; i < n4; i += stride) {
    if (active != nullptr && reinterpret_cast<const float4*>(active)[i].x == 0.f) continue;      // slots are 64-float aligned
    float4 pv = p4[i], gv = g4[i], mv = m4[i];
    TA3N_SGD_ELEM(pv.x, gv.x, mv.x)
    TA3N_SGD_ELEM(pv.y, gv.y, mv.y)
    TA3N_SGD_ELEM(pv.z, gv.z, mv.z)
    TA3N_SGD_ELEM(pv.w, gv.w, mv.w)
    p4[i] = pv;
    m4[i] = mv;
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3) && (active == nullptr || active[(n4 << 2) + threadIdx.x] != 0.f)) {
    long long i = (n4 << 2) + threadIdx.x;
    float pv = p[i], gv = g[i], mv = m[i];
    TA3N_SGD_ELEM(pv, gv, mv)
    p[i] = pv;
    m[i] = mv;
  }
#undef TA3N_SGD_ELEM
}

// torch.optim.Adam(lr, betas, eps, weight_decay, amsgrad=False).step() after the clip coefficient, in the order of
// torch's single-tensor path (torch/optim/adam.py), per element:
//     g' = coef*g + wd*p;   m += (1-b1)*(g' - m)   (lerp_, weight < 0.5);   v = b2*v + (1-b2)*g'^2
//     p += -step_size * m / (sqrt(v)/bc2_sqrt + eps)
// with bc1 = 1 - b1^t, bc2_sqrt = sqrt(1 - b2^t), step_size = lr/bc1 computed in fp64 (b1, b2 are the Python floats
// torch uses) and rounded to fp32 once, as torch does when it hands Python floats to fp32 tensor ops.  t = *step_dev + 1:
// every block reads the count before it arrives at arrival[0] (0 between launches); the last block to arrive -- when
// none can still be reading it -- stores t and re-arms the counter, so the count advances once per launch and a
// replayed graph applies the right bias correction without a launch of its own.
__global__ void __launch_bounds__(kOptThreads) adam_step_kernel(
    float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v, long long n,
    const float* __restrict__ lr_dev, unsigned long long* __restrict__ step_dev, double beta1, double beta2, float eps,
    float wd, float max_norm, const float* __restrict__ partial, int n_partial, unsigned int* __restrict__ arrival,
    float* __restrict__ stats, const float* __restrict__ active) {
  pdl_wait();
  __shared__ float red[32];
  __shared__ float coef_s;
  __shared__ float scal_s[2];     // step_size, bc2_sqrt
  float coef = 1.f;
  if (max_norm > 0.f) coef = clip_coef_fold(partial, n_partial, max_norm, stats, red, &coef_s);
  if (threadIdx.x == 0) {
    const unsigned long long t = step_dev[0] + 1ull;
    const double td = static_cast<double>(t);
    const double bc1 = 1.0 - pow(beta1, td);
    const double bc2 = 1.0 - pow(beta2, td);
    scal_s[0] = static_cast<float>(static_cast<double>(lr_dev[0]) / bc1);
    scal_s[1] = static_cast<float>(sqrt(bc2));
    __threadfence();               // this block's read of *step_dev is ordered before its arrival
    if (atomicAdd(arrival, 1u) == gridDim.x - 1) {
      step_dev[0] = t;
      arrival[0] = 0u;
    }
  }
  __syncthreads();
  const float neg_step = -scal_s[0], bc2s = scal_s[1];
  const float omb1 = static_cast<float>(1.0 - beta1), b2 = static_cast<float>(beta2),
              omb2 = static_cast<float>(1.0 - beta2);
  const long long n4 = n >> 2;
  float4* p4 = reinterpret_cast<float4*>(p);
  float4* m4 = reinterpret_cast<float4*>(m);
  float4* v4 = reinterpret_cast<float4*>(v);
  const float4* g4 = reinterpret_cast<const float4*>(g);
  const long long stride = static_cast<long long>(gridDim.x) * kOptThreads;
#define TA3N_ADAM_ELEM(P, G, M, V)                                \
  {                                                               \
    float d = fmaf(wd, (P), coef * (G));                          \
    (M) = fmaf(omb1, d - (M), (M));                               \
    (V) = fmaf(omb2, d * d, b2 * (V));                            \
    (P) = fmaf(neg_step, (M) / (sqrtf(V) / bc2s + eps), (P));     \
  }
  // `active` as for SGD: torch.optim.Adam leaves a parameter whose .grad is None untouched (no state, no decay)
  for (long long i = static_cast<long long>(blockIdx.x) * kOptThreads + threadIdx.x; i < n4; i += stride) {
    if (active != nullptr && reinterpret_cast<const float4*>(active)[i].x == 0.f) continue;      // slots are 64-float aligned
    float4 pv = p4[i], gv = g4[i], mv = m4[i], vv = v4[i];
    TA3N_ADAM_ELEM(pv.x, gv.x, mv.x, vv.x)
    TA3N_ADAM_ELEM(pv.y, gv.y, mv.y, vv.y)
    TA3N_ADAM_ELEM(pv.z, gv.z, mv.z, vv.z)
    TA3N_ADAM_ELEM(pv.w, gv.w, mv.w, vv.w)
    p4[i] = pv;
    m4[i] = mv;
    v4[i] = vv;
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3) && (active == nullptr || active[(n4 << 2) + threadIdx.x] != 0.f)) {
    long long i = (n4 << 2) + threadIdx.x;
    float pv = p[i], gv = g[i], mv = m[i], vv = v[i];
    TA3N_ADAM_ELEM(pv, gv, mv, vv)
    p[i] = pv;
    m[i] = mv;
    v[i] = vv;
  }
#undef TA3N_ADAM_ELEM
}

}  // namespace ta3n
