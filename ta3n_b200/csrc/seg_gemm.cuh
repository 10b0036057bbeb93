// seg_gemm.cuh -- "segmented grouped GEMM": the one contraction primitive behind every dense
// layer of the path.
//
//   C_g[m, n] = epilogue( sum_{seg in group g} sum_{k < len_seg} A_seg(m, k) * B_seg(k, n) )
//
// A group is one output matrix; its K dimension is a concatenation of segments, each with its
// own A / B base pointer.  That one abstraction expresses, without materialising any gather:
//   * TRN forward   (TRNmodule.py:60,75-77): segment j = frame tau[j] of x, columns jF..(j+1)F of W
//   * TRN dgrad     : segment = every (relation, slot) that touched frame t
//   * TRN wgrad     : segment = every relation r of scale i (reduction over videos)
//   * source/target inputs living in two separate tensors (shared FC forward and wgrad)
// Operand layouts (template parameters):
//   A_KMAJ: A(m,k) = A[m*lda + k]   (activations, forward/dgrad)   else A(m,k) = A[k*lda + m] (wgrad)
//   B_KMAJ: B(k,n) = B[n*ldb + k]   (nn.Linear weight, forward)    else B(k,n) = B[k*ldb + n]
//
// This file holds the table types, the epilogue, the exact-fp32 SIMT engine and the split-K
// reducer.  The tensor-core engine (gemm_wgmma.cuh) consumes the same tables.
#pragma once

#include <vector>

#include "common.cuh"

namespace ta3n {

#ifndef TA3N_MAX_GROUPS
#define TA3N_MAX_GROUPS 48
#endif
#ifndef TA3N_MAX_SEGS
#define TA3N_MAX_SEGS 128
#endif
constexpr int kMaxGroups = TA3N_MAX_GROUPS;
constexpr int kMaxSegs = TA3N_MAX_SEGS;

enum : int {
  EPI_BIAS = 1,        // v += bias[n]
  EPI_RELU = 2,        // v = max(v, 0)
  EPI_DROP_MASK = 4,   // v = keep[m,n] ? v * drop_scale : 0
  EPI_DROP_RNG = 8,    // same with the counter-based RNG
  EPI_ADDROW = 16,     // v += (rowscale ? rowscale[m*rs_stride] + rs_bias : 1) * add[m*ldadd + n]
  EPI_GATE = 32,       // v = gate[m*ldgate + n] > 0 ? v : 0
  EPI_ACCUM = 64,      // v += C[m,n]
  EPI_DPRE = 128,      // LAST: v = gate[m*ldgate + n] > 0 ? v * drop_scale : 0   (ReLU + dropout backward of the shared
                       //       layer folded into the data-gradient GEMM that completes d_feat; rowops dpre_kernel)
  EPI_DROP_LATE = 512, // modifier of EPI_DROP_MASK / EPI_DROP_RNG: the dropout factor is applied AFTER the row add
                       //       (data gradient through dropout: G = (Gc - beta * acc) * keep / (1 - p); models.py:679-680)
  EPI_MULTI = 256      // additionally store v * 1[multi_gate[q][m*ldmulti + n] > 0] to multi_out[q], q < n_multi
                       //       (d_feat_rel -> the dZ planes of every relation of the scale; rowops dz_kernel)
};
enum : int { LD_RELU_A = 1, LD_RELU_B = 2 };

struct Seg {
  const float* A;
  const float* B;
  int len;
  int lda, ldb;   // leading dimensions of this segment's operands
  int pad_;
};

struct Group {
  int seg_begin, seg_count;
  int M, N;
  int ldc;
  int tile_begin;   // first linear tile of this group in the launch
  int tiles_m, tiles_n;
  int ksplit;       // >= 1; when > 1 raw partial sums go to `partial`
  int flags;
  float alpha;
  float drop_scale, drop_p;
  float rs_bias;
  int ldkeep, ldadd, rs_stride, ldgate;
  int fix_slot;     // >= 0: split-K partials are folded in by the LAST split of each tile inside the GEMM kernel
  int pad2_;        //       (arrival counters fix_flags[fix_slot + tile]); -1: separate reduce kernel
  float* C;
  float* partial;   // [ksplit, M, N] when ksplit > 1
  const float* bias;
  const uint8_t* keep;
  const float* add;
  const float* rowscale;
  const float* gate;
  const uint64_t* step_dev;
  uint64_t seed;
  uint64_t rng_offset;  // added to the element index m*N+n (keeps source/target streams apart)
  const float* alpha_dev;       // optional: alpha *= *alpha_dev (device-resident GRL coefficient, main.py:350-352)
  float* multi_out[3];          // EPI_MULTI
  const float* multi_gate[3];
  int n_multi, ldmulti;
};

struct GemmTable {
  int n_groups;
  int total_tiles;
  int load_flags;
  int pad_;
  Group g[kMaxGroups];
  Seg s[kMaxSegs];
};
static_assert(sizeof(GemmTable) < 16000, "kernel parameter space is 32 KB");

inline Group make_group() {
  Group g;
  memset(&g, 0, sizeof(g));
  g.alpha = 1.0f;
  g.ksplit = 1;
  g.fix_slot = -1;
  return g;
}

// ---- epilogue (shared by the SIMT engine, the split-K reducer and the tensor-core engine) --------
// F >= 0: flag set known at compile time (dead branches -- notably the 64-bit RNG mixing -- vanish);
// F < 0 : generic, flags read at run time.  The kernels dispatch the common sets to the specialised
// instantiations: evaluated per output element, the generic form costs ~100 issued instructions even when
// every feature is off, which was 80 % of the run time of a small GEMM tile.
template <int F>
__device__ __forceinline__ float epilogue_t(const Group& g, int m, int n, float acc) {
  const int f = (F >= 0) ? F : g.flags;
  float v = (g.alpha_dev ? g.alpha * __ldg(g.alpha_dev) : g.alpha) * acc;
  if (f & EPI_BIAS) v += g.bias[n];
  if (f & EPI_RELU) v = fmaxf(v, 0.0f);
  float dropf = 1.0f;
  if (f & EPI_DROP_MASK) dropf = g.keep[(size_t)m * g.ldkeep + n] ? g.drop_scale : 0.0f;
  if (f & EPI_DROP_RNG) {
    uint64_t step = g.step_dev ? *g.step_dev : 0ull;
    dropf = rng_keep(g.seed, step, g.rng_offset + (uint64_t)m * (uint64_t)g.N + (uint64_t)n, g.drop_p) ? g.drop_scale : 0.0f;
  }
  if ((f & (EPI_DROP_MASK | EPI_DROP_RNG)) && !(f & EPI_DROP_LATE)) v = dropf != 0.0f ? v * dropf : 0.0f;
  if (f & EPI_ADDROW) {
    float rs = g.rowscale ? g.rowscale[(size_t)m * g.rs_stride] + g.rs_bias : 1.0f;
    v += rs * g.add[(size_t)m * g.ldadd + n];
  }
  if ((f & (EPI_DROP_MASK | EPI_DROP_RNG)) && (f & EPI_DROP_LATE)) v = dropf != 0.0f ? v * dropf : 0.0f;
  if (f & EPI_GATE) v = g.gate[(size_t)m * g.ldgate + n] > 0.0f ? v : 0.0f;
  if (f & EPI_ACCUM) v += g.C[(size_t)m * g.ldc + n];
  if (f & EPI_DPRE) v = g.gate[(size_t)m * g.ldgate + n] > 0.0f ? v * g.drop_scale : 0.0f;
  if (f & EPI_MULTI) {
#pragma unroll
    for (int q = 0; q < 3; ++q)      // constant indices: the Group copy stays in registers
      if (q < g.n_multi)
        g.multi_out[q][(size_t)m * g.ldmulti + n] = g.multi_gate[q][(size_t)m * g.ldmulti + n] > 0.0f ? v : 0.0f;
  }
  return v;
}

__device__ __forceinline__ float apply_epilogue(const Group& g, int m, int n, float acc) {
  return epilogue_t<-1>(g, m, n, acc);
}

// Call `body(tag)` with tag = std::integral_constant<int, F> for the flag set of `flags`.
#define TA3N_EPI_DISPATCH(flags, ...)                                              \
  switch (flags) {                                                                  \
    case 0: { constexpr int EPI_F = 0; __VA_ARGS__; } break;                               \
    case (EPI_BIAS | EPI_RELU): { constexpr int EPI_F = EPI_BIAS | EPI_RELU; __VA_ARGS__; } break; \
    case (EPI_BIAS | EPI_RELU | EPI_DROP_RNG): { constexpr int EPI_F = EPI_BIAS | EPI_RELU | EPI_DROP_RNG; __VA_ARGS__; } break; \
    case EPI_ADDROW: { constexpr int EPI_F = EPI_ADDROW; __VA_ARGS__; } break;              \
    case EPI_ACCUM: { constexpr int EPI_F = EPI_ACCUM; __VA_ARGS__; } break;                \
    case (EPI_ACCUM | EPI_DPRE): { constexpr int EPI_F = EPI_ACCUM | EPI_DPRE; __VA_ARGS__; } break; \
    case (EPI_ADDROW | EPI_DROP_RNG | EPI_DROP_LATE): { constexpr int EPI_F = EPI_ADDROW | EPI_DROP_RNG | EPI_DROP_LATE; __VA_ARGS__; } break; \
    case (EPI_ADDROW | EPI_MULTI): { constexpr int EPI_F = EPI_ADDROW | EPI_MULTI; __VA_ARGS__; } break; \
    default: { constexpr int EPI_F = -1; __VA_ARGS__; } break;                              \
  }

// ---- per-CTA tile context ------------------------------------------------------------------------
// The launch tables live in kernel-parameter space; indexing them with run-time indices makes every
// field access a ~300-cycle generic load.  Each CTA therefore copies ITS group and the lengths /
// operand bases of that group's segments into shared memory once (one parallel round of loads) and
// works from there.
struct SegLite {
  const float* A;
  const float* B;
  int len, lda, ldb;
  unsigned short amap, bmap;   // tensor-map slots (tensor-core engine only)
};
constexpr int kCtxMaxSegs = kMaxSegs;

struct TileCtx {
  Group g;
  SegLite seg[kCtxMaxSegs];
  int gi;
};

// Find the group owning `tile` (groups are sorted by tile_begin) with one parallel probe per warp,
// then stage it.  Must be called by all threads of the CTA; ends with __syncthreads().
__device__ __forceinline__ void load_tile_ctx(const GemmTable& tab, int tile, TileCtx* ctx,
                                              const unsigned char* amap, const unsigned char* bmap) {
  if (threadIdx.x < 32) {
    int best = 0;
    for (int i = threadIdx.x; i < tab.n_groups; i += 32)
      if (tile >= tab.g[i].tile_begin) best = max(best, i);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
    if (threadIdx.x == 0) ctx->gi = best;
  }
  __syncthreads();
  const int gi = ctx->gi;
  const int* src = reinterpret_cast<const int*>(&tab.g[gi]);
  int* dst = reinterpret_cast<int*>(&ctx->g);
  for (int i = threadIdx.x; i < (int)(sizeof(Group) / sizeof(int)); i += blockDim.x) dst[i] = src[i];
  const int sb = tab.g[gi].seg_begin, sc = tab.g[gi].seg_count;
  for (int i = threadIdx.x; i < sc; i += blockDim.x) {
    const Seg& s = tab.s[sb + i];
    SegLite l;
    l.A = s.A;
    l.B = s.B;
    l.len = s.len;
    l.lda = s.lda;
    l.ldb = s.ldb;
    l.amap = amap ? amap[sb + i] : 0;
    l.bmap = bmap ? bmap[sb + i] : 0;
    ctx->seg[i] = l;
  }
  __syncthreads();
}

// =============================================================================================
// exact-fp32 SIMT engine: 64x64x16 tiles, 256 threads, 4x4 register micro-tile, double-buffered
// =============================================================================================
constexpr int SG_BM = 64, SG_BN = 64, SG_BK = 16, SG_THREADS = 256, SG_PAD = 4;

// load 4 consecutive floats p[0..3]; element i is valid iff i < nvalid; zero fill otherwise
__device__ __forceinline__ float4 ld4_guard(const float* p, int nvalid, bool relu) {
  float4 r = make_float4(0.f, 0.f, 0.f, 0.f);
  if (nvalid >= 4 && ((reinterpret_cast<uintptr_t>(p) & 15u) == 0)) {
    r = __ldg(reinterpret_cast<const float4*>(p));
  } else {
    if (nvalid > 0) r.x = __ldg(p);
    if (nvalid > 1) r.y = __ldg(p + 1);
    if (nvalid > 2) r.z = __ldg(p + 2);
    if (nvalid > 3) r.w = __ldg(p + 3);
  }
  if (relu) {
    r.x = fmaxf(r.x, 0.f);
    r.y = fmaxf(r.y, 0.f);
    r.z = fmaxf(r.z, 0.f);
    r.w = fmaxf(r.w, 0.f);
  }
  return r;
}

// Fetch this thread's float4 of an operand tile.
//   KMAJ : tile rows = "outer" index (m or n), 16 k per row  -> thread (row = tid/4, kq = tid%4*4)
//   !KMAJ: tile rows = k, 64 outer per row                    -> thread (krow = tid/16, oq = tid%16*4)
template <bool KMAJ>
__device__ __forceinline__ float4 fetch_operand(const float* base, int ld, int outer0, int outer_lim,
                                                int k0, int klen, int tid, bool relu) {
  if (KMAJ) {
    int row = tid >> 2, kq = (tid & 3) * 4;
    int o = outer0 + row;
    int nv = (o < outer_lim) ? min(4, klen - (k0 + kq)) : 0;
    if (nv <= 0) return make_float4(0.f, 0.f, 0.f, 0.f);
    return ld4_guard(base + (size_t)o * ld + k0 + kq, nv, relu);
  } else {
    int krow = tid >> 4, oq = (tid & 15) * 4;
    int k = k0 + krow;
    int nv = (k < klen) ? min(4, outer_lim - (outer0 + oq)) : 0;
    if (nv <= 0) return make_float4(0.f, 0.f, 0.f, 0.f);
    return ld4_guard(base + (size_t)k * ld + outer0 + oq, nv, relu);
  }
}

template <bool KMAJ>
__device__ __forceinline__ void stash_operand(float (*S)[SG_BM + SG_PAD], float4 r, int tid) {
  if (KMAJ) {
    int row = tid >> 2, kq = (tid & 3) * 4;
    S[kq + 0][row] = r.x;
    S[kq + 1][row] = r.y;
    S[kq + 2][row] = r.z;
    S[kq + 3][row] = r.w;
  } else {
    int krow = tid >> 4, oq = (tid & 15) * 4;
    *reinterpret_cast<float4*>(&S[krow][oq]) = r;
  }
}

template <bool A_KMAJ, bool B_KMAJ>
__global__ void __launch_bounds__(SG_THREADS)
seg_gemm_simt_kernel(const __grid_constant__ GemmTable tab) {
  __shared__ __align__(16) float As[2][SG_BK][SG_BM + SG_PAD];
  __shared__ __align__(16) float Bs[2][SG_BK][SG_BN + SG_PAD];

  __shared__ TileCtx ctx;
  const int tid = threadIdx.x;
  const int tile = blockIdx.x;
  load_tile_ctx(tab, tile, &ctx, nullptr, nullptr);
  pdl_wait();   // parameters staged; operands of the previous kernel are read from here on
  const Group& g = ctx.g;
  int local = tile - g.tile_begin;
  const int per_split = g.tiles_m * g.tiles_n;
  const int split = local / per_split;
  local -= split * per_split;
  const int m0 = (local / g.tiles_n) * SG_BM;
  const int n0 = (local % g.tiles_n) * SG_BN;

  // chunk range of this split over the concatenated K of all segments
  int total_chunks = 0;
  for (int s = 0; s < g.seg_count; ++s) total_chunks += (ctx.seg[s].len + SG_BK - 1) / SG_BK;
  const int cps = (total_chunks + g.ksplit - 1) / g.ksplit;
  const int c_begin = split * cps;
  const int c_end = min(total_chunks, c_begin + cps);

  const bool reluA = (tab.load_flags & LD_RELU_A) != 0;
  const bool reluB = (tab.load_flags & LD_RELU_B) != 0;

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  // position the chunk iterator on c_begin
  int seg = 0, k0 = 0;
  {
    int skip = c_begin;
    while (seg < g.seg_count) {
      int nch = (ctx.seg[seg].len + SG_BK - 1) / SG_BK;
      if (skip < nch) {
        k0 = skip * SG_BK;
        break;
      }
      skip -= nch;
      ++seg;
    }
  }

  const int n_iter = c_end - c_begin;
  if (n_iter > 0) {
    float4 ra, rb;
    {
      const SegLite& sg = ctx.seg[seg];
      ra = fetch_operand<A_KMAJ>(sg.A, sg.lda, m0, g.M, k0, sg.len, tid, reluA);
      rb = fetch_operand<B_KMAJ>(sg.B, sg.ldb, n0, g.N, k0, sg.len, tid, reluB);
    }
    stash_operand<A_KMAJ>(As[0], ra, tid);
    stash_operand<B_KMAJ>(Bs[0], rb, tid);
    __syncthreads();

    const int ty = tid >> 4, tx = tid & 15;
    int cur = 0;
    for (int it = 0; it < n_iter; ++it) {
      const bool has_next = (it + 1 < n_iter);
      if (has_next) {
        k0 += SG_BK;
        if (k0 >= ctx.seg[seg].len) {
          ++seg;
          k0 = 0;
        }
        const SegLite& sg = ctx.seg[seg];
        ra = fetch_operand<A_KMAJ>(sg.A, sg.lda, m0, g.M, k0, sg.len, tid, reluA);
        rb = fetch_operand<B_KMAJ>(sg.B, sg.ldb, n0, g.N, k0, sg.len, tid, reluB);
      }
#pragma unroll
      for (int kk = 0; kk < SG_BK; ++kk) {
        float4 a = *reinterpret_cast<const float4*>(&As[cur][kk][ty * 4]);
        float4 b = *reinterpret_cast<const float4*>(&Bs[cur][kk][tx * 4]);
        const float av[4] = {a.x, a.y, a.z, a.w};
        const float bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
      }
      if (has_next) {
        stash_operand<A_KMAJ>(As[cur ^ 1], ra, tid);
        stash_operand<B_KMAJ>(Bs[cur ^ 1], rb, tid);
        __syncthreads();
        cur ^= 1;
      }
    }
  }

  const int ty = tid >> 4, tx = tid & 15;
  const Group e = ctx.g;   // register copy: no reloads behind the global stores
  if (e.ksplit > 1) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int m = m0 + ty * 4 + i;
      if (m >= e.M) continue;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int n = n0 + tx * 4 + j;
        if (n < e.N) e.partial[((size_t)split * e.M + m) * e.N + n] = acc[i][j];
      }
    }
  } else {
    TA3N_EPI_DISPATCH(e.flags, {
      _Pragma("unroll") for (int i = 0; i < 4; ++i) {
        const int m = m0 + ty * 4 + i;
        if (m >= e.M) continue;
        _Pragma("unroll") for (int j = 0; j < 4; ++j) {
          const int n = n0 + tx * 4 + j;
          if (n < e.N) e.C[(size_t)m * e.ldc + n] = epilogue_t<EPI_F>(e, m, n, acc[i][j]);
        }
      }
    })
  }
}

// deterministic split-K reduction + epilogue: one thread per output element of every group
__global__ void __launch_bounds__(256) splitk_reduce_kernel(const __grid_constant__ GemmTable tab) {
  pdl_wait();
  // blockIdx.y = group, blockIdx.x strides over the elements
  __shared__ Group g;
  {
    const int* src = reinterpret_cast<const int*>(&tab.g[blockIdx.y]);
    int* dst = reinterpret_cast<int*>(&g);
    for (int i = threadIdx.x; i < (int)(sizeof(Group) / sizeof(int)); i += blockDim.x) dst[i] = src[i];
    __syncthreads();
  }
  if (g.ksplit <= 1 || g.fix_slot >= 0) return;
  const size_t total = (size_t)g.M * g.N;
  const Group gr = g;
  TA3N_EPI_DISPATCH(gr.flags, {
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
      float s = 0.f;
      for (int k = 0; k < gr.ksplit; ++k) s += gr.partial[(size_t)k * total + e];
      const int m = (int)(e / gr.N), n = (int)(e % gr.N);
      gr.C[(size_t)m * gr.ldc + n] = epilogue_t<EPI_F>(gr, m, n, s);
    }
  })
}

inline unsigned splitk_reduce_blocks(const GemmTable& tab) {
  size_t mx = 0;
  for (int i = 0; i < tab.n_groups; ++i)
    if (tab.g[i].ksplit > 1 && tab.g[i].fix_slot < 0 && (size_t)tab.g[i].M * tab.g[i].N > mx)
      mx = (size_t)tab.g[i].M * tab.g[i].N;
  size_t b = (mx + 255) / 256;
  if (b > 512) b = 512;
  return (unsigned)(b ? b : 1);
}

// The same reduction, four consecutive columns per thread (N % 4 == 0, aligned C / partial / bias: the forward layers):
// 16 B loads of every partial in flight together, one pass of the epilogue per quad, blocks only for split groups
// (blockIdx.y indexes `split_groups`).
struct SplitGroups {
  int n;
  unsigned char idx[kMaxGroups];
};
__global__ void __launch_bounds__(256) splitk_reduce_v4_kernel(const __grid_constant__ GemmTable tab,
                                                               const __grid_constant__ SplitGroups sg) {
  pdl_wait();
  __shared__ Group g;
  {
    const int* src = reinterpret_cast<const int*>(&tab.g[sg.idx[blockIdx.y]]);
    int* dst = reinterpret_cast<int*>(&g);
    for (int i = threadIdx.x; i < (int)(sizeof(Group) / sizeof(int)); i += blockDim.x) dst[i] = src[i];
    __syncthreads();
  }
  const size_t total4 = (size_t)g.M * g.N / 4;
  const int N4 = g.N / 4;
  const Group gr = g;
  const float4* part = reinterpret_cast<const float4*>(gr.partial);
  TA3N_EPI_DISPATCH(gr.flags, {
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total4; e += (size_t)gridDim.x * blockDim.x) {
      float4 p[8];
#pragma unroll
      for (int k = 0; k < 8; ++k)
        if (k < gr.ksplit) p[k] = __ldcg(part + (size_t)k * total4 + e);
      float4 s = p[0];
#pragma unroll
      for (int k = 1; k < 8; ++k)
        if (k < gr.ksplit) {
          s.x += p[k].x;
          s.y += p[k].y;
          s.z += p[k].z;
          s.w += p[k].w;
        }
      const int m = (int)(e / N4), n = (int)(e % N4) * 4;
      float4 o;
      o.x = epilogue_t<EPI_F>(gr, m, n, s.x);
      o.y = epilogue_t<EPI_F>(gr, m, n + 1, s.y);
      o.z = epilogue_t<EPI_F>(gr, m, n + 2, s.z);
      o.w = epilogue_t<EPI_F>(gr, m, n + 3, s.w);
      *reinterpret_cast<float4*>(gr.C + (size_t)m * gr.ldc + n) = o;
    }
  })
}

// =============================================================================================
// host side: table builder + launcher
// =============================================================================================
struct GemmPlan {
  std::vector<Group> groups;
  std::vector<Seg> segs;     // group.seg_begin indexes into this vector
  bool a_kmaj = true, b_kmaj = true;
  int load_flags = 0;
  bool precise = false;             // a forward layer: the x3 engine runs it at fp32 grade (gemm_wgmma.cuh)
  bool precise_dgrad = false;       // a data-gradient GEMM (feeds further GEMMs): x3 engine, fp32 grade as well
  const char* label = "seg_gemm";   // call-site name used by the timing registry

  // add a group; its segments must be pushed right after with add_seg
  Group& add_group(int M, int N, float* C, int ldc) {
    Group g = make_group();
    g.M = M;
    g.N = N;
    g.C = C;
    g.ldc = ldc;
    g.seg_begin = (int)segs.size();
    g.seg_count = 0;
    groups.push_back(g);
    return groups.back();
  }
  void add_seg(const float* A, int lda, const float* B, int ldb, int len) {
    Seg s;
    s.A = A;
    s.B = B;
    s.len = len;
    s.lda = lda;
    s.ldb = ldb;
    s.pad_ = 0;
    segs.push_back(s);
    groups.back().seg_count++;
  }
  size_t k_total(const Group& g) const {
    size_t k = 0;
    for (int i = 0; i < g.seg_count; ++i) k += segs[g.seg_begin + i].len;
    return k;
  }
};

// Choose a split-K factor for reduction-heavy, tile-poor problems (wgrads) and carve the partial
// buffers out of `arena` (which may be null -> no split-K).  bm/bn/bk: tile shape of the engine.
inline void plan_splitk(GemmPlan& plan, Arena* arena, int bm, int bn, int bk, int min_chunks,
                        int target_ctas = 132) {
  if (!arena) return;
  long tiles = 0;
  for (auto& g : plan.groups) tiles += (long)((g.M + bm - 1) / bm) * ((g.N + bn - 1) / bn);
  // At least half a wave already: partials + the reduce pass cost more than they buy (measured: splitting only
  // the long-K outliers of the merged weight-gradient launch made the step 17 % slower).
  if (tiles <= 0 || 2 * tiles > target_ctas) return;
  for (auto& g : plan.groups) {
    long chunks = 0;
    for (int i = 0; i < g.seg_count; ++i) chunks += (plan.segs[g.seg_begin + i].len + bk - 1) / bk;
    int want = (int)(target_ctas / tiles);
    int maxsplit = (int)(chunks / min_chunks);
    int ks = want < maxsplit ? want : maxsplit;
    if (ks > 8) ks = 8;
    if (ks < 2) continue;
    float* p = arena->floats((size_t)ks * g.M * g.N);
    if (!p) continue;  // not enough workspace: stay unsplit (still correct)
    g.ksplit = ks;
    g.partial = p;
  }
}

inline int launch_simt(const GemmPlan& plan, cudaStream_t stream) {
  size_t gi = 0;
  while (gi < plan.groups.size()) {
    GemmTable tab;
    memset(&tab, 0, sizeof(int) * 4);
    tab.load_flags = plan.load_flags;
    int ng = 0, ns = 0, tiles = 0;
    bool any_split = false;
    while (gi < plan.groups.size() && ng < kMaxGroups) {
      const Group& src = plan.groups[gi];
      if (src.seg_count > kMaxSegs)
        return fail(TA3N_ERR_UNSUPPORTED, "seg_gemm: a group has %d segments (max %d)", src.seg_count, kMaxSegs);
      if (ns + src.seg_count > kMaxSegs) break;
      Group g = src;
      for (int i = 0; i < src.seg_count; ++i) tab.s[ns + i] = plan.segs[src.seg_begin + i];
      g.seg_begin = ns;
      ns += src.seg_count;
      g.tiles_m = (g.M + SG_BM - 1) / SG_BM;
      g.tiles_n = (g.N + SG_BN - 1) / SG_BN;
      g.tile_begin = tiles;
      tiles += g.tiles_m * g.tiles_n * g.ksplit;
      any_split |= g.ksplit > 1;
      tab.g[ng++] = g;
      ++gi;
    }
    tab.n_groups = ng;
    tab.total_tiles = tiles;
    if (tiles > 0) {
      pre_launch(plan.label, stream);
      if (plan.a_kmaj && plan.b_kmaj)
        launch_kernel(seg_gemm_simt_kernel<true, true>, tiles, SG_THREADS, 0, stream, tab);
      else if (plan.a_kmaj && !plan.b_kmaj)
        launch_kernel(seg_gemm_simt_kernel<true, false>, tiles, SG_THREADS, 0, stream, tab);
      else if (!plan.a_kmaj && !plan.b_kmaj)
        launch_kernel(seg_gemm_simt_kernel<false, false>, tiles, SG_THREADS, 0, stream, tab);
      else
        launch_kernel(seg_gemm_simt_kernel<false, true>, tiles, SG_THREADS, 0, stream, tab);
      TA3N_TRY(after_launch());
      if (any_split) {
        dim3 grid(splitk_reduce_blocks(tab), ng);
        pre_launch("splitk_reduce", stream);
        launch_kernel(splitk_reduce_kernel, grid, 256, 0, stream, tab);
        TA3N_TRY(after_launch());
      }
    }
  }
  return TA3N_OK;
}

}  // namespace ta3n
