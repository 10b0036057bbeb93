// gather.cuh -- the device-resident input pipeline: ONE launch assembles the paired mini-batch of an iteration from
// two feature banks in device memory (C ABI ta3n_gather_batch).  It is the first launch of a captured step, so a
// whole epoch is a series of graph replays with no host gather, no host-to-device copy and no host synchronisation.
#pragma once

#include "common.cuh"

namespace ta3n {

struct GatherDomain {
  const float4* bank;         // [n_rows, row_f4]
  long long n_rows;
  const int* rows;            // [n_epoch] bank row of every position of the epoch
  const long long* labels;    // [n_epoch] or nullptr (target domain)
  long long n_epoch;
  float4* dst;                // [batch, row_f4]
  long long* dst_labels;      // [batch] or nullptr
  int batch;
};

constexpr int kGatherThreads = 256;
constexpr int kGatherUnroll = 4;                                  // 16-byte loads in flight per thread
constexpr int kGatherChunk = kGatherThreads * kGatherUnroll;      // float4s per CTA: 16 KB of one row

// Streaming load: the bank is read once per epoch, so it neither allocates in L1 nor displaces the slot (which the
// shared layer's GEMM reads right after) from L2.
__device__ __forceinline__ uint64_t l2_evict_first_policy() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}

__device__ __forceinline__ float4 ld_stream_f4(const float4* p, uint64_t pol) {
  float4 v;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.f32 {%0, %1, %2, %3}, [%4], %5;"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(p), "l"(pol));
  return v;
}

// grid = (ceil(row_f4 / kGatherChunk), Bs + Bt): blockIdx.y is the slot row (source rows first), blockIdx.x a 16 KB
// chunk of it.  state[0] is the iteration i, state[1] an arrival counter that is 0 between launches.  Slot row k of
// a domain takes epoch position i*batch + k; past the end of the epoch it is zero-filled (main.py:359-364 pads with
// zero dummies).  Every CTA reads state[0] once before it arrives; the last CTA to arrive -- when no CTA can still be
// reading it -- advances the iteration and re-arms the counter, so the index moves once per launch without a launch
// of its own.  A bank row id outside [0, n_rows) (a broken row list) yields a NaN row instead of a stray read.
__global__ void __launch_bounds__(kGatherThreads)
gather_batch_kernel(const __grid_constant__ GatherDomain src, const __grid_constant__ GatherDomain tgt,
                    long long row_f4, int* __restrict__ valid_rows, unsigned int* __restrict__ state) {
  __shared__ long long s_row;      // bank row of this slot row, -1 = padding, -2 = invalid id
  __shared__ unsigned int s_it;
  pdl_wait();
  const bool is_src = blockIdx.y < (unsigned)src.batch;
  const GatherDomain& d = is_src ? src : tgt;
  const int k = is_src ? (int)blockIdx.y : (int)blockIdx.y - src.batch;
  if (threadIdx.x == 0) {
    const unsigned int it = state[0];
    const long long pos = (long long)it * d.batch + k;
    long long row = -1;
    if (pos < d.n_epoch) {
      row = d.rows[pos];
      if (row < 0 || row >= d.n_rows) row = -2;
    }
    s_row = row;
    s_it = it;
    if (blockIdx.x == 0 && d.dst_labels) d.dst_labels[k] = pos < d.n_epoch ? d.labels[pos] : 0ll;
    if (blockIdx.x == 0 && blockIdx.y == 0) {
      const long long ns = src.n_epoch - (long long)it * src.batch, nt = tgt.n_epoch - (long long)it * tgt.batch;
      valid_rows[0] = (int)max(0ll, min(ns, (long long)src.batch));
      valid_rows[1] = (int)max(0ll, min(nt, (long long)tgt.batch));
    }
  }
  __syncthreads();
  const long long row = s_row;
  const float4* in = row >= 0 ? d.bank + row * row_f4 : nullptr;
  float4* out = d.dst + (long long)k * row_f4;
  const float fill = row == -2 ? __int_as_float(0x7fc00000) : 0.f;
  const long long c0 = (long long)blockIdx.x * kGatherChunk + threadIdx.x;
  const uint64_t pol = l2_evict_first_policy();
  float4 v[kGatherUnroll];
#pragma unroll
  for (int u = 0; u < kGatherUnroll; ++u) {
    const long long c = c0 + u * kGatherThreads;
    v[u] = make_float4(fill, fill, fill, fill);
    if (in && c < row_f4) v[u] = ld_stream_f4(in + c, pol);
  }
#pragma unroll
  for (int u = 0; u < kGatherUnroll; ++u) {
    const long long c = c0 + u * kGatherThreads;
    if (c < row_f4) out[c] = v[u];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();               // this CTA's read of state[0] is ordered before its arrival
    const unsigned int n_cta = gridDim.x * gridDim.y;
    if (atomicAdd(&state[1], 1u) == n_cta - 1) {
      state[0] = s_it + 1;
      state[1] = 0;
    }
  }
}

}  // namespace ta3n
