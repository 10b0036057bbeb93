// gemm_wgmma.cuh -- Hopper (sm_90a) tensor-core engine for the segmented grouped GEMM.
//
// Both kernels compute 128 x 128 output tiles with 384 threads in three warpgroups:
//   warps 0..7  : two consumer warpgroups -- wgmma.mma_async m64n128k8 tf32 with A from registers and B from shared
//                 memory, fp32 accumulators in registers (each warpgroup owns 64 rows of the tile), then the fused
//                 epilogue straight from the accumulator fragments
//   warp 8      : TMA producer -- cp.async.bulk.tensor into a ring of 128B-swizzled stages (mbarrier handshake)
//   warps 9..11 : B preparation -- write a K-major copy of each landed B tile beside it when B is MN-major (and, in
//                 the precise kernel, the tf32 lo part of B), then arrive on the stage's ready barrier
// setmaxnreg gives the producer warpgroup 40 registers per thread and the consumers 232 (64 / 216 in the plain kernel
// with MN-major B, whose B warps keep two transpose blocks in flight).
// Operands stay fp32 in HBM: the tf32 MMA reads the fp32 bit patterns (10-bit mantissa, fp32 range), so there is no
// conversion pass and no second copy of any tensor in global memory.
// The "gather" of TRN frame tuples, the source/target split and the per-frame dgrad are all
// expressed as TMA coordinates / tensor maps per K-segment: nothing is materialised.
//
// Operand layouts in a stage:
//   K-major  (A(m,k)=A[m*ld+k]) : one TMA box {32 k, 128 rows}, SWIZZLE_128B; descriptor SW128, SBO = 1024 B,
//                                 +32 B per K=8 step.  Read by the tensor core as loaded.
//   MN-major (A(m,k)=A[k*ld+m]) : four TMA boxes {32 m, 32 k}, SWIZZLE_128B (16 B chunk index ^= k & 7).  wgmma reads
//                                 shared-memory tf32 operands K-major only, so MN-major B is transposed by warps
//                                 9..11; A, fed from registers, is read in whichever layout it landed.
//
// The plain kernel (seg_gemm_tc_kernel, "tf32") runs one tile per CTA with one accumulator over its whole K range;
// its TFLOAT32 tensor maps make the TMA unit round each operand to tf32.  The precise kernel (seg_gemm_tc_x3_kernel,
// "tf32x3") splits both operands into hi + lo tf32 pieces (the consumers split their A fragments in registers) and
// issues three products per K step; its CTAs are persistent (one wave, a static task list per CTA) and the producer
// warps run ahead into the next task.
#pragma once

#include <cuda.h>
#include <stdlib.h>

#include <algorithm>
#include <cmath>
#include <functional>
#include <map>
#include <tuple>

#include "seg_gemm.cuh"

namespace ta3n {

constexpr int TC_BM = 128, TC_BN = 128, TC_BK = 32;
constexpr int TC_THREADS = 384;        // warps 0..7: two consumer warpgroups; warp 8: TMA producer; 9..11: B preparation
constexpr int TC_CONSUMER_WARPS = 8;
constexpr int TC_B_WARPS = 3;
constexpr int TC_B_THREADS = 32 * TC_B_WARPS;
// one CTA per SM: 65536 / 384 threads, rounded down to the allocation unit of 8, is 168 registers per thread at launch
constexpr int TC_PRODUCER_REGS = 40, TC_CONSUMER_REGS = 232;
static_assert(128 * TC_PRODUCER_REGS + 256 * TC_CONSUMER_REGS <= TC_THREADS * 168,
              "setmaxnreg budget exceeds the registers of one CTA");
// The plain kernel with MN-major B: the B warps keep two blocks of the transpose in flight (tc_transpose_b, 32
// registers of data), and its consumers (64 accumulators, two slabs of A fragments) need fewer than the precise
// kernel's, which hold 64 running sums and hi / lo fragments besides.
constexpr int TC_XPOSE_PRODUCER_REGS = 64, TC_XPOSE_CONSUMER_REGS = 216;
static_assert(128 * TC_XPOSE_PRODUCER_REGS + 256 * TC_XPOSE_CONSUMER_REGS <= TC_THREADS * 168,
              "setmaxnreg budget exceeds the registers of one CTA");
constexpr int TC_A_BYTES = TC_BM * TC_BK * 4;   // 16 KB
constexpr int TC_B_BYTES = TC_BN * TC_BK * 4;   // 16 KB
constexpr int TC_STAGE_BYTES = TC_A_BYTES + TC_B_BYTES;
// 4 stages (one CTA per SM; 129 KB of ring, or 193 KB when the precise kernel keeps its lo tile of B beside each
// stage): the grids of this workload are within a wave, so a CTA is alone on its SM and bound by TMA latency -- the
// bytes in flight per CTA matter more than a second resident CTA.
constexpr int TC_STAGES = 4;
// With MN-major B the plain kernel keeps two rings: the raw stages [A | B as loaded] (32 KB) and the K-major copies of
// B (16 KB).  A raw stage is free again once the consumers hold its A fragments in registers and the B warps have
// transposed its B, long before the MMAs that read the copy retire: TMA runs up to TC_RAW_STAGES slabs ahead, the B
// warps up to TC_KB_STAGES ahead of the MMAs.  5 x 32 + 3 x 16 = 208 KB (+ the slack and the ~4.3 KB of static
// tables: 227 KB is the opt-in limit).
constexpr int TC_RAW_STAGES = 5, TC_KB_STAGES = 3;
constexpr int kTcMaxStages = 8;
static_assert(TC_STAGES <= kTcMaxStages && TC_RAW_STAGES <= kTcMaxStages && TC_KB_STAGES <= kTcMaxStages,
              "ring deeper than its barrier arrays");
__host__ __device__ constexpr int tc_raw_stages(bool b_kmaj) { return b_kmaj ? TC_STAGES : TC_RAW_STAGES; }
constexpr int tc_smem_bytes(bool b_kmaj) {       // + alignment slack
  return tc_raw_stages(b_kmaj) * TC_STAGE_BYTES + (b_kmaj ? 0 : TC_KB_STAGES * TC_B_BYTES) + 1024;
}
#ifndef TA3N_MAX_MAPS
#define TA3N_MAX_MAPS 64
#endif
constexpr int kMaxMaps = TA3N_MAX_MAPS;

struct alignas(64) TcMaps {
  CUtensorMap m[kMaxMaps];
};
struct TcSegMaps {
  unsigned char a[kMaxSegs];
  unsigned char b[kMaxSegs];
};

// ---- PTX wrappers ---------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  uint32_t done;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(addr), "r"(parity)
        : "memory");
  } while (!done);
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1,
                                            int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
// L2 prefetch of a tile (no shared-memory destination, no barrier): warms the line ahead of the real load
__device__ __forceinline__ void tma_prefetch_2d(const CUtensorMap* map, int c0, int c1) {
  asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global.tile [%0, {%1, %2}];" ::"l"(map), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_prefetch_3d(const CUtensorMap* map, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.prefetch.tensor.3d.L2.global.tile [%0, {%1, %2, %3}];" ::"l"(map), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}

__device__ __forceinline__ void sts4(uint32_t saddr, const float4 v) {
  asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(saddr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ float4 lds4(uint32_t saddr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(saddr) : "memory");
  return v;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}

// wgmma shared-memory matrix descriptor of a K-major, 128B-swizzled tf32 tile (8-row atoms of 1024 B):
//   [0,14) start>>4 | [16,30) LBO>>4 (unused by swizzled K-major layouts: 1) | [32,46) SBO>>4 = 1024 B between
//   8-row groups | [62,64) layout: 1 = SWIZZLE_128B.  One K=8 step of tf32 is 32 B further along the row.
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t tile_base, int kstep) {
  const uint32_t a = tile_base + (uint32_t)kstep * 32u;
  return (uint64_t)((a >> 4) & 0x3FFF) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}

// d[64 x 128] += A[64 x 8] * B[128 x 8]^T (tf32 in, fp32 accumulate), issued by a whole warpgroup.  Fragment of
// thread (warp w of the warpgroup, lane l): d[4j + 2h + e] = row 16w + l/4 + 8h, column 8j + 2(l%4) + e.
__device__ __forceinline__ void wgmma_tf32(float (&d)[64], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(1)
      : "memory");
}
// The same product with A from registers: fragment of thread (warp w of the warpgroup, lane l) a[j] = A(row
// 16w + l/4 + 8(j&1), column l%4 + 4(j>>1)).  The registers must not be written until a wgmma.wait_group has
// retired the MMA.
__device__ __forceinline__ void wgmma_tf32_rs(float (&d)[64], const uint32_t a0, const uint32_t a1, const uint32_t a2,
                                              const uint32_t a3, uint64_t bdesc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %69, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %68, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "l"(bdesc), "r"(1)
      : "memory");
}
// pins a register value at this point of the instruction stream (before a wgmma.fence that must cover its write)
__device__ __forceinline__ void reg_fence(uint32_t& r) { asm volatile("" : "+r"(r)::"memory"); }
__device__ __forceinline__ float lds1(uint32_t saddr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(saddr) : "memory");
  return v;
}
// warpgroup register budget (every thread of the warpgroup executes it)
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

// ---- operand tiles as the tensor core reads them ---------------------------------------------------------
// byte offset of the 16 B chunk holding k = 4kq .. 4kq+3 of row m in a K-major SW128 tile
__device__ __forceinline__ uint32_t kmaj_chunk(int m, int kq) { return (uint32_t)(m * 128 + ((kq ^ (m & 7)) << 4)); }
// byte offset of the 16 B chunk holding m = 4mq .. 4mq+3 of k-row k in an MN-major tile (four SW128 boxes of 32 m)
__device__ __forceinline__ uint32_t mnmaj_chunk(int k, int mq) {
  return (uint32_t)((mq >> 3) * 4096 + k * 128 + (((mq & 7) ^ (k & 7)) << 4));
}
__device__ __forceinline__ float tf32_hi(float a) { return __uint_as_float(__float_as_uint(a) & 0xFFFFE000u); }
__device__ __forceinline__ float f4_at(const float4& v, int i) { return i == 0 ? v.x : i == 1 ? v.y : i == 2 ? v.z : v.w; }

// One 4 x 4 block (m = 4mq.., k = 4kq..) of an MN-major operand tile, block t of 256: read by tc_prep_load, written
// K-major (transposed) by tc_prep_store.  A 16 B access is served per quarter warp (8 consecutive blocks), so both
// are conflict-free when those 8 blocks hit 8 different 16 B chunks of the 128 B bank row:
//   load  chunk (mq & 7) ^ (k & 7), k = 4 kq + i:  bits (mq0, mq1, mq2 ^ kq0)
//   store chunk  kq ^ (m & 7),      m = 4 mq + i:  bits (kq0, kq1, kq2 ^ mq0)
// t0 -> mq0, t1 -> mq1 and kq1, t2 -> kq0 make both sets distinct over t0..t2; t7 gives kq1 its own bit
// (kq1 = t1 ^ t7), so the map is a bijection of the 256 blocks.
__device__ __forceinline__ void tc_prep_blk(const int t, int* mq, int* kq) {
  *mq = (t & 3) | (((t >> 3) & 7) << 2);
  *kq = ((t >> 2) & 1) | ((((t >> 1) ^ (t >> 7)) & 1) << 1) | (((t >> 6) & 1) << 2);
}
// Row i of block t sits at (tile + off) ^ (i << 4), + 128 i, in either tile: off keeps the SW128 chunk of row 0 in
// bits 4..6 and bits 7..8 clear, and tiles are 1024-B aligned.  One offset per block and tile (not four) stays live.
//   MN-major: mnmaj_chunk(4 kq + i, mq) = (mq >> 3) 4096 + 512 kq + 128 i + (((mq & 7) ^ 4 (kq & 1) ^ i) << 4)
//   K-major:  kmaj_chunk(4 mq + i, kq)  = 512 mq + 128 i + ((kq ^ 4 (mq & 1) ^ i) << 4)
__device__ __forceinline__ void tc_prep_load(const uint32_t base, const int t, float4 (&r)[4]) {
  int mq, kq;
  tc_prep_blk(t, &mq, &kq);
  const uint32_t p = base + (uint32_t)((mq >> 3) * 4096 + 512 * kq + (((mq & 7) ^ (4 * (kq & 1))) << 4));
#pragma unroll
  for (int i = 0; i < 4; ++i) r[i] = lds4((p ^ (i << 4)) + 128u * i);
}
__device__ __forceinline__ void tc_prep_store(const uint32_t base, const int t, const float4 (&r)[4]) {
  int mq, kq;
  tc_prep_blk(t, &mq, &kq);
  const uint32_t p = base + (uint32_t)(512 * mq + ((kq ^ (4 * (mq & 1))) << 4));
#pragma unroll
  for (int i = 0; i < 4; ++i)
    sts4((p ^ (i << 4)) + 128u * i, make_float4(f4_at(r[0], i), f4_at(r[1], i), f4_at(r[2], i), f4_at(r[3], i)));
}
// B preparation warps (thread t of 96): the MN-major B tile at b_mn, transposed into the K-major SW128 tile at b_k.
// Thread t moves blocks t, t + 96 and (t < 64) t + 192.  Under the MMAs' operand reads a shared-memory load takes
// hundreds of cycles; with TWO_IN_FLIGHT the loads of two blocks are in flight together and the third block's are
// issued before the second block is stored: two load round trips per tile instead of three, for 32 registers of data
// (the plain kernel; the precise kernel's split warps have 40 registers and move one block at a time).
static_assert(2 * TC_B_THREADS < 256 && 256 <= 3 * TC_B_THREADS, "tc_transpose_b moves two or three blocks per thread");
template <bool TWO_IN_FLIGHT>
__device__ __forceinline__ void tc_transpose_b(const uint32_t b_mn, const uint32_t b_k, const int t) {
  if (!TWO_IN_FLIGHT) {
#pragma unroll 1
    for (int blk = t; blk < 256; blk += TC_B_THREADS) {
      float4 r[4];
      tc_prep_load(b_mn, blk, r);
      tc_prep_store(b_k, blk, r);
    }
    return;
  }
  const bool third = t + 2 * TC_B_THREADS < 256;
  float4 r[4], q[4];
  tc_prep_load(b_mn, t, r);
  tc_prep_load(b_mn, t + TC_B_THREADS, q);
  tc_prep_store(b_k, t, r);
  if (third) tc_prep_load(b_mn, t + 2 * TC_B_THREADS, r);
  tc_prep_store(b_k, t + TC_B_THREADS, q);
  if (third) tc_prep_store(b_k, t + 2 * TC_B_THREADS, r);
}

// Per-thread part of the A fragment addresses of rows m = r0 (and r0 + 8, MN-major), column k = tq: the word offset
// in the landed tile, whose bits 4..6 are the SW128 chunk index.  Stage bases are 1024-B aligned, so tc_load_a reaches
// every other column by an XOR on those bits plus a constant, with no per-column offsets kept in registers.
template <bool A_KMAJ>
__device__ __forceinline__ uint32_t tc_a_thread_off(const int m, const int tq) {
  return A_KMAJ ? kmaj_chunk(m, 0) + 4u * tq : mnmaj_chunk(tq, m >> 2) + 4u * (m & 3);
}

// Consumer thread: the A fragment words of one slab (4 k-steps x 4 words, see wgmma_tf32_rs) from the landed A tile,
// in either layout.  K-major loads are conflict-free (the SW128 chunk index differs per row), MN-major ones 2-way.
//   K-major  (m, k = 8 ks + 4 half + tq): (a_base + off0) ^ ((2 ks + half) << 4), + 1024 for row r0 + 8 (same m & 7)
//   MN-major (m, k = 8 ks + 4 half + tq): (a_base + off_m) ^ (half << 6), + 128 (4 half + 8 ks) k-rows
template <bool A_KMAJ>
__device__ __forceinline__ void tc_load_a(const uint32_t a_base, const uint32_t off0, const uint32_t off1,
                                          uint32_t (&a)[16]) {
  const uint32_t p0 = a_base + off0, p1 = a_base + off1;
#pragma unroll
  for (int ks = 0; ks < TC_BK / 8; ++ks)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const uint32_t row = j & 1, half = j >> 1;
      const uint32_t addr = A_KMAJ ? (p0 ^ ((2u * ks + half) << 4)) + 1024u * row
                                   : ((row ? p1 : p0) ^ (half << 6)) + 512u * half + 1024u * ks;
      a[4 * ks + j] = __float_as_uint(lds1(addr));
    }
}

#ifdef TA3N_TC_TIMELINE
// Stage timeline of the plain kernel (tools/tc_stage_timeline.py; off in the product build): clock64 stamps of the
// first kTlSlabs slabs of every CTA, by event, and each CTA's globaltimer and clock64 at its start and end (the SM
// clock while it ran).  The producer stamps TMA issue; B warp 9 lane 0 the landed stage and the transpose; consumer
// thread 0 the rest.
constexpr int kTlCtas = 132, kTlSlabs = 64, kTlEvents = 9;
enum : int {
  TL_TMA_ISSUE,      // producer: the stage is free, TMA issued
  TL_FULL,           // B warps: the raw stage has landed
  TL_XPOSE_START,    // B warps: K-major slot free, transpose starts
  TL_XPOSE_END,      // B warps: transposed and fenced, ready arrived
  TL_CONS_START,     // consumers: slab entered
  TL_READY,          // consumers: A landed and B ready
  TL_RELEASED,       // consumers: MMAs issued, raw stage (MN-major B) released
  TL_RETIRED,        // consumers: the slab's MMAs retired
  TL_FENCE,          // B warps: transpose stores issued, proxy fence next
};
__device__ unsigned long long g_tc_tl[kTlCtas][kTlSlabs][kTlEvents];
__device__ unsigned long long g_tc_tl_clk[kTlCtas][4];   // globaltimer, clock64 at start; globaltimer, clock64 at end
__device__ __forceinline__ unsigned long long tl_globaltimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void tl_stamp(const uint32_t slab, const int ev) {
  if (blockIdx.x < kTlCtas && slab < (uint32_t)kTlSlabs) g_tc_tl[blockIdx.x][slab][ev] = clock64();
}
__device__ __forceinline__ void tl_clock(const int at_end) {
  if (blockIdx.x < kTlCtas) {
    g_tc_tl_clk[blockIdx.x][2 * at_end] = tl_globaltimer();
    g_tc_tl_clk[blockIdx.x][2 * at_end + 1] = clock64();
  }
}
#define TA3N_TL(cond, slab, ev) \
  do {                          \
    if (cond) tl_stamp((uint32_t)(slab), (ev)); \
  } while (0)
#else
#define TA3N_TL(cond, slab, ev) ((void)0)
#endif

// ---- one output tile, by warp role ---------------------------------------------------------------------
// The operand ring barriers are initialised once per CTA.  The precise kernel's producer runs ahead over its task
// list (it fills the ring with the slabs of task t+1 while the consumer warps still finish task t), so it passes its
// running slab count to tc_produce.
struct TcShared {
  uint64_t full_bar[kTcMaxStages];      // TMA landed
  uint64_t empty_bar[kTcMaxStages];     // every reader of the stage is done with it
};

// `readers`: warps that arrive on a stage's empty barrier (the consumer warps, + the B warps when they read the raw
// stage and the consumers release it before their MMAs retire)
template <int STAGES>
__device__ __forceinline__ void tc_pipe_init(TcShared* sh, const int readers = TC_CONSUMER_WARPS) {
  for (int s = 0; s < STAGES; ++s) {
    mbar_init(&sh->full_bar[s], 1);
    mbar_init(&sh->empty_bar[s], readers);
  }
  fence_barrier_init();
}

// TMA producer (ONE thread): the n_iter K slabs [c_begin, c_begin + n_iter) of tile (m0, n0) into the ring.
// `slabs` = slabs this CTA has pushed so far (advanced by the caller).
template <int STAGES, int STAGE_BYTES = TC_STAGE_BYTES>
__device__ __forceinline__ void tc_produce(const TileCtx& ctx, const CUtensorMap* __restrict__ maps, const bool a_kmaj,
                                           const bool b_kmaj, const int pad_flags, const int m0, const int n0,
                                           const int c_begin, const int n_iter, uint8_t* smem, TcShared* sh,
                                           const uint32_t slabs) {
  const Group& g = ctx.g;
  int seg = 0, k0 = 0;
  {
    int skip = c_begin;
    while (seg < g.seg_count) {
      const int nch = (ctx.seg[seg].len + TC_BK - 1) / TC_BK;
      if (skip < nch) {
        k0 = skip * TC_BK;
        break;
      }
      skip -= nch;
      ++seg;
    }
  }
  for (int it = 0; it < n_iter; ++it) {
    const uint32_t gl = slabs + (uint32_t)it;
    const int stage = (int)(gl % STAGES);
    const uint32_t phase = (gl / STAGES) & 1u;
    mbar_wait(&sh->empty_bar[stage], phase ^ 1u);
    TA3N_TL(true, gl, TL_TMA_ISSUE);
    mbar_expect_tx(&sh->full_bar[stage], TC_STAGE_BYTES);
    uint8_t* sA = smem + stage * STAGE_BYTES;
    uint8_t* sB = sA + TC_A_BYTES;
    const CUtensorMap* ma = &maps[ctx.seg[seg].amap];
    const CUtensorMap* mb = &maps[ctx.seg[seg].bmap];
    // MN-major tiles are four [32 k-rows][32 floats] slabs, one per group of 32 m (or n).  When the operand's
    // MN extent is a multiple of 32 a rank-3 tensor map {32 floats, k rows, groups of 32} fetches all four with
    // ONE instruction (the lone producer thread is issue-bound: ~50 cycles per TMA, 8 per chunk otherwise).
    if (a_kmaj) {
      tma_load_2d(sA, ma, &sh->full_bar[stage], k0, m0);
    } else if (pad_flags & 1) {
      tma_load_3d(sA, ma, &sh->full_bar[stage], 0, k0, m0 >> 5);
    } else {
#pragma unroll
      for (int q = 0; q < TC_BM / 32; ++q) tma_load_2d(sA + q * 4096, ma, &sh->full_bar[stage], m0 + 32 * q, k0);
    }
    if (b_kmaj) {
      tma_load_2d(sB, mb, &sh->full_bar[stage], k0, n0);
    } else if (pad_flags & 2) {
      tma_load_3d(sB, mb, &sh->full_bar[stage], 0, k0, n0 >> 5);
    } else {
#pragma unroll
      for (int q = 0; q < TC_BN / 32; ++q) tma_load_2d(sB + q * 4096, mb, &sh->full_bar[stage], n0 + 32 * q, k0);
    }
    k0 += TC_BK;
    if (k0 >= ctx.seg[seg].len) {
      ++seg;
      k0 = 0;
    }
  }
}

// chunk range [c_begin, c_begin + n_iter) of split `split` of the group staged in ctx
__device__ __forceinline__ void tc_chunk_range(const TileCtx& ctx, int split, int* c_begin, int* n_iter) {
  const Group& g = ctx.g;
  int total_chunks = 0;
  for (int s = 0; s < g.seg_count; ++s) total_chunks += (ctx.seg[s].len + TC_BK - 1) / TC_BK;
  const int cps = (total_chunks + g.ksplit - 1) / g.ksplit;
  *c_begin = split * cps;
  *n_iter = max(0, min(total_chunks, *c_begin + cps) - *c_begin);
}

// linear tile number -> (split, m0, n0) within the group staged in ctx
__device__ __forceinline__ void tc_decode(const TileCtx& ctx, const int tile, int* split, int* m0, int* n0) {
  const Group& g = ctx.g;
  int local = tile - g.tile_begin;
  const int per_split = g.tiles_m * g.tiles_n;
  *split = local / per_split;
  local -= *split * per_split;
  *m0 = (local / g.tiles_n) * TC_BM;
  *n0 = (local % g.tiles_n) * TC_BN;
}

// ---- epilogue straight from the accumulator fragment (consumer thread) ------------------------------------------
// Thread (warp w, lane l) holds rows r0 = 64 (w / 4) + 16 (w % 4) + l / 4 and r0 + 8 of the tile, columns
// 8j + 2(l % 4) + {0, 1} (see wgmma_tf32): v[4j + 2h + e] = (row r0 + 8h, column c0 + 8j + e), c0 = 2(l % 4).  A warp
// store instruction then covers 8 rows x 32 B, whole sectors.
__device__ __forceinline__ void frag_st2(float* p, const float x0, const float x1, const bool vec, const bool two) {
  if (vec) {
    *reinterpret_cast<float2*>(p) = make_float2(x0, x1);
  } else {
    p[0] = x0;
    if (two) p[1] = x1;
  }
}

// The fused epilogue of the fragment -> C.  The forward flag sets (bias, ReLU, RNG dropout) work from register copies
// of the group fields and draw one rng_hash4 per 4-column group; every other set applies epilogue_t per element.
template <int F>
__device__ __forceinline__ void frag_epilogue(const Group& g, const int m0, const int n0, const float (&v)[64]) {
  constexpr bool kFwd = F >= 0 && (F & ~(EPI_BIAS | EPI_RELU | EPI_DROP_RNG)) == 0;
  const int M = g.M, N = g.N, ldc = g.ldc;
  float* const C = g.C;
  const bool vec = (N % 2) == 0 && (ldc % 2) == 0 && (reinterpret_cast<uintptr_t>(C) & 7u) == 0;
  const float alpha = kFwd ? (g.alpha_dev ? g.alpha * __ldg(g.alpha_dev) : g.alpha) : 0.f;
  const float* const bias = g.bias;
  const uint64_t seed = g.seed, roff = g.rng_offset;
  const uint64_t step = (kFwd && (F & EPI_DROP_RNG) && g.step_dev) ? *g.step_dev : 0ull;
  const float dscale = g.drop_scale, dp = g.drop_p;
  const uint32_t thr = rng_threshold(dp);
  float b0[16], b1[16];                 // bias of the thread's columns, loaded before the first store
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int n = n0 + 8 * j;
    b0[j] = kFwd && (F & EPI_BIAS) && n < N ? bias[n] : 0.f;
    b1[j] = kFwd && (F & EPI_BIAS) && n + 1 < N ? bias[n + 1] : 0.f;
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = m0 + 8 * h;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int n = n0 + 8 * j;
      if (n >= N) continue;
      const bool two = n + 1 < N;
      float x0 = v[4 * j + 2 * h], x1 = v[4 * j + 2 * h + 1];
      if (kFwd) {
        x0 *= alpha;
        x1 *= alpha;
        if (F & EPI_BIAS) {
          x0 += b0[j];
          x1 += b1[j];
        }
        if (F & EPI_RELU) {
          x0 = fmaxf(x0, 0.0f);
          x1 = fmaxf(x1, 0.0f);
        }
        if (F & EPI_DROP_RNG) {
          const uint64_t e = roff + (uint64_t)m * (uint64_t)N + (uint64_t)n;
          bool k0, k1;
          if ((e & 1ull) == 0) {        // the pair lies in one 4-column group of the RNG stream
            const uint64_t hsh = rng_hash4(seed, step, e >> 2);
            k0 = rng_keep_bits(hsh, (int)(e & 3ull), thr);
            k1 = rng_keep_bits(hsh, (int)(e & 3ull) + 1, thr);
          } else {
            k0 = rng_keep(seed, step, e, dp);
            k1 = rng_keep(seed, step, e + 1, dp);
          }
          const float f0 = k0 ? dscale : 0.0f, f1 = k1 ? dscale : 0.0f;
          x0 = f0 != 0.0f ? x0 * f0 : 0.0f;
          x1 = f1 != 0.0f ? x1 * f1 : 0.0f;
        }
      } else {
        x0 = epilogue_t<F>(g, m, n, x0);
        if (two) x1 = epilogue_t<F>(g, m, n + 1, x1);
      }
      frag_st2(C + (size_t)m * ldc + n, x0, x1, vec, two);
    }
  }
}

// The finished tile (all 256 consumer threads; tile origin tm0, tn0).  Unsplit: epilogue -> C.  Split: raw partial
// -> partial[split] (the separate fixed-order reduce pass applies the epilogue).
__device__ __forceinline__ void frag_finish(const Group& g, const int split, const int tm0, const int tn0,
                                            const float (&v)[64]) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m0 = tm0 + (warp >> 2) * 64 + (warp & 3) * 16 + (lane >> 2), n0 = tn0 + 2 * (lane & 3);
  if (g.ksplit > 1) {
    const int M = g.M, N = g.N;
    float* const part = g.partial + (size_t)split * M * N;
    const bool vec = (N % 2) == 0;          // partial planes are 256-B aligned
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int m = m0 + 8 * h, n = n0 + 8 * j;
        if (m < M && n < N) frag_st2(part + (size_t)m * N + n, v[4 * j + 2 * h], v[4 * j + 2 * h + 1], vec, n + 1 < N);
      }
    return;
  }
  TA3N_EPI_DISPATCH(g.flags, { frag_epilogue<EPI_F>(g, m0, n0, v); })
}

// ---- the plain kernel ("tf32"): one tile per CTA ---------------------------------------------------------------
// Warp 8 lane 0 issues the TMA loads; for MN-major B, warps 9..11 write the K-major copy of each landed B tile into
// a ring of its own (TC_KB_STAGES) and mark it ready.  The consumers load their A fragments from the landed A tile
// (either layout) and issue one product per K step with B from shared memory: they do nothing else in the K loop.
// Per slab and CTA, shared memory moves 32 KB of TMA fill, 16 KB of A fragment loads and 32 KB of B operand reads
// (each warpgroup reads all of B), + 32 KB for the transpose of MN-major B.
//
// Ring hand-offs.  K-major B: one ring of TC_STAGES [A | B] stages, released by the consumers once the stage's MMAs
// have retired.  MN-major B: the raw stage (full_bar / empty_bar, TC_RAW_STAGES) is released by the 8 consumer warps
// once its A fragments are in registers (after the MMAs that read them are issued) and by the 3 B warps after its
// transpose; the K-major copy (kready_bar / kempty_bar, TC_KB_STAGES) is released by the consumers once the MMAs
// that read it have retired.

// Consumer warpgroups: slab `it` of the tile, A fragments in `a` (not the set of the group still in flight).  Leaves
// this slab's group in flight and releases what the previous slab's MMAs read: its stage (K-major B) or its K-major
// copy of B (MN-major B; the raw stage of this slab is released as soon as its MMAs are issued).
template <bool A_KMAJ, bool B_KMAJ>
__device__ __forceinline__ void tc_consume_slab(const uint32_t it, uint8_t* smem, TcShared* sh, uint64_t* kready_bar,
                                                uint64_t* kempty_bar, const uint32_t off0, const uint32_t off1,
                                                uint32_t (&a)[16], float (&d)[64], int& prev) {
  constexpr int kRaw = tc_raw_stages(B_KMAJ);
  const int stage = (int)(it % kRaw);
  const uint32_t parity = (it / kRaw) & 1u;
  const int kst = (int)(it % TC_KB_STAGES);
  TA3N_TL(threadIdx.x == 0, it, TL_CONS_START);
  mbar_wait(&sh->full_bar[stage], parity);          // A landed (read below with ordinary loads)
  if (!B_KMAJ) mbar_wait(&kready_bar[kst], (it / TC_KB_STAGES) & 1u);   // K-major copy of B written
  TA3N_TL(threadIdx.x == 0, it, TL_READY);
  const uint32_t a_base = smem_u32(smem + stage * TC_STAGE_BYTES);
  const uint32_t b_base = B_KMAJ ? a_base + TC_A_BYTES
                                 : smem_u32(smem + TC_RAW_STAGES * TC_STAGE_BYTES + kst * TC_B_BYTES);
  tc_load_a<A_KMAJ>(a_base, off0, off1, a);
#pragma unroll
  for (int j = 0; j < 16; ++j) reg_fence(a[j]);
  wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < TC_BK / 8; ++ks) {
    const int f = 4 * ks;
    wgmma_tf32_rs(d, a[f], a[f + 1], a[f + 2], a[f + 3], wgmma_desc(b_base, ks));
  }
  wgmma_commit();
  if (!B_KMAJ) {                                    // the MMAs took the A registers: the raw stage is read
    __syncwarp();
    if ((threadIdx.x & 31) == 0) mbar_arrive(&sh->empty_bar[stage]);
    TA3N_TL(threadIdx.x == 0, it, TL_RELEASED);
  }
  wgmma_wait<1>();                                  // the previous slab's MMAs are done: release what they read
  if (prev >= 0) {
    TA3N_TL(threadIdx.x == 0, it - 1, TL_RETIRED);
    __syncwarp();
    if ((threadIdx.x & 31) == 0) mbar_arrive(B_KMAJ ? &sh->empty_bar[prev] : &kempty_bar[prev]);
  }
  prev = B_KMAJ ? stage : kst;
}

template <bool A_KMAJ, bool B_KMAJ>
__global__ void __launch_bounds__(TC_THREADS, 1)
seg_gemm_tc_kernel(const __grid_constant__ GemmTable tab, const __grid_constant__ TcMaps maps,
                   const __grid_constant__ TcSegMaps segmaps, const int first_wave) {
  constexpr int kRaw = tc_raw_stages(B_KMAJ);
  extern __shared__ uint8_t tc_smem_raw[];
  __shared__ __align__(8) TcShared sh;
  __shared__ __align__(8) uint64_t kready_bar[TC_KB_STAGES];    // B transposed (one arrival per B warp)
  __shared__ __align__(8) uint64_t kempty_bar[TC_KB_STAGES];    // the MMAs that read the copy retired (consumer warps)
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(tc_smem_raw) + 1023) & ~uintptr_t(1023));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#ifdef TA3N_TC_TIMELINE
  if (threadIdx.x == 0) tl_clock(0);
#endif

  // ---- tile decode (same scheme as the SIMT engine, 128x128 tiles); group + segments staged in smem ----
  __shared__ TileCtx ctx;
  // Groups arrive sorted by K (longest first).  CTAs beyond the first wave (one per SM) take tiles from the END
  // of the list, so the SM that received the longest tile gets the shortest one next.
  int tile = blockIdx.x;
  if (tile >= first_wave) tile = tab.total_tiles - 1 - (tile - first_wave);
  load_tile_ctx(tab, tile, &ctx, segmaps.a, segmaps.b);
  int split, m0, n0, c_begin, n_iter;
  tc_decode(ctx, tile, &split, &m0, &n0);
  tc_chunk_range(ctx, split, &c_begin, &n_iter);

  if (warp == TC_CONSUMER_WARPS && lane == 0) {
    for (int s = 0; s < TC_KB_STAGES; ++s) {
      mbar_init(&kready_bar[s], TC_B_WARPS);
      mbar_init(&kempty_bar[s], TC_CONSUMER_WARPS);
    }
    tc_pipe_init<kRaw>(&sh, TC_CONSUMER_WARPS + (B_KMAJ ? 0 : TC_B_WARPS));
  }
  __syncthreads();
  // Everything above touched only kernel parameters and shared memory: it overlaps the previous kernel of the
  // stream.  From here on operands produced by that kernel are read.
  pdl_wait();

  if (warp >= TC_CONSUMER_WARPS) {
    setmaxnreg_dec<B_KMAJ ? TC_PRODUCER_REGS : TC_XPOSE_PRODUCER_REGS>();
    if (warp == TC_CONSUMER_WARPS) {
      if (lane == 0 && n_iter > 0)
        tc_produce<kRaw, TC_STAGE_BYTES>(ctx, maps.m, A_KMAJ, B_KMAJ, tab.pad_, m0, n0, c_begin, n_iter, smem, &sh, 0u);
    } else if (!B_KMAJ) {
      const int t = threadIdx.x - 32 * (TC_CONSUMER_WARPS + 1);
      const uint32_t kring = smem_u32(smem + TC_RAW_STAGES * TC_STAGE_BYTES);
      for (int it = 0; it < n_iter; ++it) {
        const int stage = it % TC_RAW_STAGES, kst = it % TC_KB_STAGES;
        mbar_wait(&sh.full_bar[stage], (uint32_t)(it / TC_RAW_STAGES) & 1u);
        TA3N_TL(t == 0, it, TL_FULL);
        mbar_wait(&kempty_bar[kst], ((uint32_t)(it / TC_KB_STAGES) & 1u) ^ 1u);
        TA3N_TL(t == 0, it, TL_XPOSE_START);
        tc_transpose_b<true>(smem_u32(smem + stage * TC_STAGE_BYTES) + TC_A_BYTES, kring + kst * TC_B_BYTES, t);
        TA3N_TL(t == 0, it, TL_FENCE);
        fence_proxy_async();            // generic-proxy writes -> the tensor core's reads
        __syncwarp();
        if (lane == 0) {
          mbar_arrive(&kready_bar[kst]);
          mbar_arrive(&sh.empty_bar[stage]);
        }
        TA3N_TL(t == 0, it, TL_XPOSE_END);
      }
    }
  } else {
    setmaxnreg_inc<B_KMAJ ? TC_CONSUMER_REGS : TC_XPOSE_CONSUMER_REGS>();
    const int r0 = (warp >> 2) * 64 + (warp & 3) * 16 + (lane >> 2);      // fragment rows r0, r0 + 8
    const uint32_t off0 = tc_a_thread_off<A_KMAJ>(r0, lane & 3), off1 = tc_a_thread_off<A_KMAJ>(r0 + 8, lane & 3);
    float d[64];
#pragma unroll
    for (int j = 0; j < 64; ++j) d[j] = 0.f;
    uint32_t a[2][16];                  // A fragments of the even / odd slabs
    int prev = -1;                      // stage (or K-major slot) whose MMAs may still be in flight
    // The odd last slab is peeled off the loop: with the pair's second slab conditional inside it, the back edge would
    // let one register set be rewritten while its own group is in flight, and ptxas would serialize every MMA (C7513).
    int it = 0;
    for (; it + 1 < n_iter; it += 2) {
      tc_consume_slab<A_KMAJ, B_KMAJ>((uint32_t)it, smem, &sh, kready_bar, kempty_bar, off0, off1, a[0], d, prev);
      tc_consume_slab<A_KMAJ, B_KMAJ>((uint32_t)(it + 1), smem, &sh, kready_bar, kempty_bar, off0, off1, a[1], d, prev);
    }
    if (it < n_iter)
      tc_consume_slab<A_KMAJ, B_KMAJ>((uint32_t)it, smem, &sh, kready_bar, kempty_bar, off0, off1, a[0], d, prev);
    wgmma_wait<0>();
    if (prev >= 0) {
      TA3N_TL(threadIdx.x == 0, n_iter - 1, TL_RETIRED);
      __syncwarp();
      if (lane == 0) mbar_arrive(B_KMAJ ? &sh.empty_bar[prev] : &kempty_bar[prev]);
    }
    frag_finish(ctx.g, split, m0, n0, d);
  }
#ifdef TA3N_TC_TIMELINE
  if (threadIdx.x == 0) tl_clock(1);
#endif
}

// ---- the precise forward kernel ("tf32x3"): fp32-grade products from the tensor cores -------------------------
// A tf32 MMA keeps 10 mantissa bits of each operand: every forward GEMM is accurate to ~3e-4, and ~1.3e-4 of the
// ReLU units behind them (pre-activation within that error of zero) come out with the wrong on/off state.  Each flip
// moves a gradient entry by O(1), which is where the 1-2 % gradient deviation of the plain tf32 engine comes from
// (tools/parity_report.py; with the pattern pinned the same gradients agree to 4e-4).  The forward layers therefore
// run here with the operands split in two tf32 pieces (a = hi + lo, hi = a with the low 13 mantissa bits cleared,
// lo = a - hi, exact):     a b ~= hi_a hi_b + lo_a hi_b + hi_a lo_b      (three MMAs per K step)
// Two more things are needed for fp32 grade (tools/x3_probe.py):
//   * K is accumulated in CHUNKS of 256 inside the tensor core and the chunks are added in fp32 registers: over the
//     full K = 2048 the tensor core's own accumulation limits the result to ~5e-6 whatever the operands; chunked, the
//     error of an fp32 FFMA loop;
//   * the tensor maps deliver the RAW fp32 words (no TMA rounding), so that hi + lo = a exactly.
// Roles (384 threads): warp 8 lane 0 issues the TMA loads of the raw words; warps 9..11 write the lo tile of each
// landed B tile beside it (the raw tile serves as hi), transposing MN-major B on the way, and mark the stage ready;
// the two consumer warpgroups load their A fragments from the raw stage into registers, split them there, and issue
// the three products with B from shared memory.  The consumer warps do nothing else in the K loop; they fold every
// finished chunk into 64 running sums.  setmaxnreg moves registers from the producer warpgroup to the consumers,
// which hold 64 accumulators, 64 sums and two slabs of A fragments (hi and lo).
constexpr int X3_STAGES = 4;
constexpr int X3_STAGE_BYTES = TC_STAGE_BYTES + TC_B_BYTES;   // [A raw | B raw (= B hi) | B lo]
constexpr int X3_CHUNK = 8;                                   // slabs (256 K columns) per tensor-core accumulation
static_assert(X3_CHUNK % 2 == 0, "the A fragment register sets alternate by slab within a chunk");
constexpr int x3_smem_bytes() { return X3_STAGES * X3_STAGE_BYTES + 1024; }

// Static schedule of a launch: CTA b runs the tasks (linear tile numbers, split included) task[off[b] .. off[b+1]),
// longest first, as assigned by the LPT model of the split planner (x3_makespan).  A launch with more tasks than the
// list holds runs them strided instead (task = blockIdx.x + i * gridDim.x).
constexpr int kX3MaxCtas = 144;
constexpr int kX3MaxTasks = 1024;
struct X3Sched {
  int listed;                                   // 1: the lists below; 0: strided
  unsigned short off[kX3MaxCtas + 1];
  unsigned short task[kX3MaxTasks];
};
static_assert(sizeof(GemmTable) + sizeof(TcMaps) + sizeof(TcSegMaps) + sizeof(X3Sched) + 256 <= 32764,
              "kernel parameters of the precise kernel exceed the 32 KB limit");

// One task as the roles read it: the group and segments (TileCtx), and where the task sits in it.  Two slots: the
// producer warp stages task k + 1 while the consumers still run the epilogue of task k.
struct X3Slot {
  TileCtx ctx;
  int split, m0, n0, c_begin, n_iter;
};
// readers that release a slot: the 8 consumer warps (after the epilogue) and the 3 split warps
constexpr int X3_SLOT_READERS = TC_CONSUMER_WARPS + 3;

__device__ __forceinline__ int x3_task(const X3Sched& sched, const int k) {
  return sched.listed ? (int)sched.task[sched.off[blockIdx.x] + k] : (int)(blockIdx.x + k * gridDim.x);
}

// Stage task `tile` into slot `sl` (one whole warp; parameter space and shared memory only).
__device__ __forceinline__ void x3_stage(const GemmTable& tab, const TcSegMaps& sm, const int tile, X3Slot* sl) {
  const int lane = threadIdx.x & 31;
  int best = 0;
  for (int i = lane; i < tab.n_groups; i += 32)
    if (tile >= tab.g[i].tile_begin) best = max(best, i);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
  const int* src = reinterpret_cast<const int*>(&tab.g[best]);
  int* dst = reinterpret_cast<int*>(&sl->ctx.g);
  for (int i = lane; i < (int)(sizeof(Group) / sizeof(int)); i += 32) dst[i] = src[i];
  const int sb = tab.g[best].seg_begin, sc = tab.g[best].seg_count;
  for (int i = lane; i < sc; i += 32) {
    const Seg& s = tab.s[sb + i];
    SegLite l;
    l.A = s.A;
    l.B = s.B;
    l.len = s.len;
    l.lda = s.lda;
    l.ldb = s.ldb;
    l.amap = sm.a[sb + i];
    l.bmap = sm.b[sb + i];
    sl->ctx.seg[i] = l;
  }
  __syncwarp();
  if (lane == 0) {
    sl->ctx.gi = best;
    tc_decode(sl->ctx, tile, &sl->split, &sl->m0, &sl->n0);
    tc_chunk_range(sl->ctx, sl->split, &sl->c_begin, &sl->n_iter);
  }
  __syncwarp();
}

// the 96 split threads only
__device__ __forceinline__ void x3_split_sync() { asm volatile("bar.sync 2, 96;" ::: "memory"); }

// Split warps (thread t of 96): lo = b - hi of the B tile of a landed stage, K-major SW128 at b_lo.  The hi tile is
// the raw K-major tile at b_raw itself: the tensor core reads an fp32 word as tf32 by ignoring its low 13 mantissa
// bits, which is hi exactly, so only lo is written.  MN-major B is first transposed into the lo tile and then written
// back K-major at b_raw on the way.
template <bool B_KMAJ>
__device__ __forceinline__ void x3_split_b(const uint32_t b_raw, const uint32_t b_lo, const int t) {
  uint32_t src = b_raw;
  if (!B_KMAJ) {
    tc_transpose_b<false>(b_raw, b_lo, t);
    x3_split_sync();                  // every read of the raw tile before the K-major writes over it
    src = b_lo;
  }
#pragma unroll 2
  for (int c = t; c < TC_B_BYTES / 16; c += TC_B_THREADS) {
    const float4 v = lds4(src + 16u * c);
    if (!B_KMAJ) sts4(b_raw + 16u * c, v);
    sts4(b_lo + 16u * c, make_float4(v.x - tf32_hi(v.x), v.y - tf32_hi(v.y), v.z - tf32_hi(v.z), v.w - tf32_hi(v.w)));
  }
}

// Consumer thread: the A fragments of one slab from the raw stage, split into hi and lo.
template <bool A_KMAJ>
__device__ __forceinline__ void x3_load_a(const uint32_t a_raw, const uint32_t off0, const uint32_t off1,
                                          uint32_t (&hi)[16], uint32_t (&lo)[16]) {
  uint32_t raw[16];
  tc_load_a<A_KMAJ>(a_raw, off0, off1, raw);
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const float a = __uint_as_float(raw[j]), h = tf32_hi(a);
    hi[j] = __float_as_uint(h);
    lo[j] = __float_as_uint(a - h);
  }
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    reg_fence(hi[j]);
    reg_fence(lo[j]);
  }
}

// Consumer warpgroups: slab `gl` of the CTA (running count over its tasks).  The fragments (hi, lo) must not belong to
// the group still in flight: the caller alternates two register sets.  Leaves this slab's group in flight and releases
// the previous stage.
template <bool A_KMAJ>
__device__ __forceinline__ void x3_consume_slab(const uint32_t gl, uint8_t* smem, TcShared* sh, uint64_t* ready_bar,
                                                const uint32_t off0, const uint32_t off1, uint32_t (&hi)[16],
                                                uint32_t (&lo)[16], float (&d)[64], int& prev) {
  const int stage = (int)(gl % X3_STAGES);
  const uint32_t parity = (gl / X3_STAGES) & 1u;
  mbar_wait(&sh->full_bar[stage], parity);          // raw A landed (read below with ordinary loads)
  mbar_wait(&ready_bar[stage], parity);             // B lo (and transposed MN-major B) written
  const uint32_t a_raw = smem_u32(smem + stage * X3_STAGE_BYTES);
  const uint32_t b_hi = a_raw + TC_A_BYTES, b_lo = b_hi + TC_B_BYTES;
  x3_load_a<A_KMAJ>(a_raw, off0, off1, hi, lo);
  wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < TC_BK / 8; ++ks) {          // small terms first
    const int f = 4 * ks;
    wgmma_tf32_rs(d, lo[f], lo[f + 1], lo[f + 2], lo[f + 3], wgmma_desc(b_hi, ks));
    wgmma_tf32_rs(d, hi[f], hi[f + 1], hi[f + 2], hi[f + 3], wgmma_desc(b_lo, ks));
    wgmma_tf32_rs(d, hi[f], hi[f + 1], hi[f + 2], hi[f + 3], wgmma_desc(b_hi, ks));
  }
  wgmma_commit();
  wgmma_wait<1>();                                  // the previous slab's MMAs are done: release its stage
  if (prev >= 0) {
    __syncwarp();
    if ((threadIdx.x & 31) == 0) mbar_arrive(&sh->empty_bar[prev]);
  }
  prev = stage;
}

template <bool A_KMAJ, bool B_KMAJ>
__global__ void __launch_bounds__(TC_THREADS, 1)
seg_gemm_tc_x3_kernel(const __grid_constant__ GemmTable tab, const __grid_constant__ TcMaps maps,
                      const __grid_constant__ TcSegMaps segmaps, const __grid_constant__ X3Sched sched) {
  extern __shared__ uint8_t tc_smem_raw[];
  __shared__ __align__(8) TcShared sh;
  __shared__ __align__(8) uint64_t ready_bar[X3_STAGES];     // B split done (one arrival per split warp)
  __shared__ __align__(8) uint64_t slot_full[2], slot_empty[2];
  __shared__ X3Slot slots[2];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(tc_smem_raw) + 1023) & ~uintptr_t(1023));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // every CTA has at least one task (the grid is no larger than the task count)
  const int n_tasks = sched.listed ? sched.off[blockIdx.x + 1] - sched.off[blockIdx.x]
                                   : (tab.total_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;

  if (warp == TC_CONSUMER_WARPS) {
    if (lane == 0) {
      for (int s = 0; s < X3_STAGES; ++s) mbar_init(&ready_bar[s], TC_B_WARPS);
      for (int s = 0; s < 2; ++s) {
        mbar_init(&slot_full[s], 1);
        mbar_init(&slot_empty[s], X3_SLOT_READERS);
      }
      tc_pipe_init<X3_STAGES>(&sh);
    }
    __syncwarp();
    x3_stage(tab, segmaps, x3_task(sched, 0), &slots[0]);
    if (lane == 0) mbar_arrive(&slot_full[0]);
  }
  __syncthreads();
  // Everything above touched only kernel parameters and shared memory: it overlaps the previous kernel of the
  // stream.  From here on operands produced by that kernel are read.
  pdl_wait();

  if (warp >= TC_CONSUMER_WARPS) {
    setmaxnreg_dec<TC_PRODUCER_REGS>();
    uint32_t slabs = 0;                 // slabs of the CTA so far: ring stage and parity
    if (warp == TC_CONSUMER_WARPS) {
      for (int k = 0; k < n_tasks; ++k) {
        const int s = k & 1;
        if (k > 0) {                    // stage task k once the epilogue of task k - 2 has left the slot
          mbar_wait(&slot_empty[s], ((uint32_t)(k >> 1) & 1u) ^ 1u);
          x3_stage(tab, segmaps, x3_task(sched, k), &slots[s]);
          if (lane == 0) mbar_arrive(&slot_full[s]);
        }
        const X3Slot& sl = slots[s];
        if (lane == 0 && sl.n_iter > 0)
          tc_produce<X3_STAGES, X3_STAGE_BYTES>(sl.ctx, maps.m, A_KMAJ, B_KMAJ, tab.pad_, sl.m0, sl.n0, sl.c_begin,
                                                sl.n_iter, smem, &sh, slabs);
        __syncwarp();
        slabs += (uint32_t)sl.n_iter;
      }
    } else {
      const int t = threadIdx.x - 32 * (TC_CONSUMER_WARPS + 1);
      for (int k = 0; k < n_tasks; ++k) {
        const int s = k & 1;
        mbar_wait(&slot_full[s], (uint32_t)(k >> 1) & 1u);
        const int n_iter = slots[s].n_iter;
        __syncwarp();
        if (lane == 0) mbar_arrive(&slot_empty[s]);
        for (int it = 0; it < n_iter; ++it) {
          const uint32_t gl = slabs + (uint32_t)it;
          const int stage = (int)(gl % X3_STAGES);
          mbar_wait(&sh.full_bar[stage], (gl / X3_STAGES) & 1u);
          const uint32_t b_raw = smem_u32(smem + stage * X3_STAGE_BYTES) + TC_A_BYTES;
          x3_split_b<B_KMAJ>(b_raw, b_raw + TC_B_BYTES, t);
          fence_proxy_async();          // generic-proxy writes -> the tensor core's reads
          __syncwarp();
          if (lane == 0) mbar_arrive(&ready_bar[stage]);
        }
        slabs += (uint32_t)n_iter;
      }
    }
  } else {
    setmaxnreg_inc<TC_CONSUMER_REGS>();
    const int r0 = (warp >> 2) * 64 + (warp & 3) * 16 + (lane >> 2);      // fragment rows r0, r0 + 8
    const uint32_t off0 = tc_a_thread_off<A_KMAJ>(r0, lane & 3), off1 = tc_a_thread_off<A_KMAJ>(r0 + 8, lane & 3);
    uint32_t slabs = 0;
    for (int k = 0; k < n_tasks; ++k) {
      const int s = k & 1;
      mbar_wait(&slot_full[s], (uint32_t)(k >> 1) & 1u);
      const int n_iter = slots[s].n_iter;
      float d[64], sum[64];
#pragma unroll
      for (int j = 0; j < 64; ++j) d[j] = sum[j] = 0.f;
      uint32_t hi[2][16], lo[2][16];    // A fragments of the even / odd slabs of a chunk
      // One group of MMAs stays in flight while the next slab's fragments are loaded; at the end of a chunk every MMA
      // must have finished before the fold reads the accumulator.
      int prev = -1;                    // stage whose MMAs may still be in flight
      for (int c0 = 0; c0 < n_iter; c0 += X3_CHUNK) {
        const int c1 = min(n_iter, c0 + X3_CHUNK);
        for (int it = c0; it < c1; it += 2) {
          x3_consume_slab<A_KMAJ>(slabs + (uint32_t)it, smem, &sh, ready_bar, off0, off1, hi[0], lo[0], d, prev);
          if (it + 1 < c1)
            x3_consume_slab<A_KMAJ>(slabs + (uint32_t)(it + 1), smem, &sh, ready_bar, off0, off1, hi[1], lo[1], d, prev);
        }
        wgmma_wait<0>();                // chunk complete: fold it into the fp32 sums
        __syncwarp();
        if (lane == 0) mbar_arrive(&sh.empty_bar[prev]);
        prev = -1;
#pragma unroll
        for (int j = 0; j < 64; ++j) {
          sum[j] += d[j];
          d[j] = 0.f;
        }
      }
      slabs += (uint32_t)n_iter;
      frag_finish(slots[s].ctx.g, slots[s].split, slots[s].m0, slots[s].n0, sum);
      __syncwarp();
      if (lane == 0) mbar_arrive(&slot_empty[s]);
    }
  }
}

// ---- host side ----------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline PFN_encodeTiled encode_fn() {
  static PFN_encodeTiled fn = []() -> PFN_encodeTiled {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess) return nullptr;
    if (q != cudaDriverEntryPointSuccess) return nullptr;
    return reinterpret_cast<PFN_encodeTiled>(p);
  }();
  return fn;
}

// Per-device facts and one-time kernel configuration.  cudaFuncSetAttribute is per DEVICE (a process may drive
// several GPUs, e.g. one host thread per replica as nn.DataParallel does -- main.py:79), so the bookkeeping is
// keyed by device ordinal and guarded by a mutex.
struct DeviceInfo {
  int sm_count = 0;
  bool configured[4] = {false, false, false, false};        // seg_gemm_tc_kernel, per operand layout
  bool x3_configured[4] = {false, false, false, false};      // seg_gemm_tc_x3_kernel, per operand layout
  bool eval_configured = false;                              // eval_head_kernel (eval.cuh)
};
inline std::mutex& device_mu() {
  static std::mutex mu;
  return mu;
}
inline DeviceInfo* device_info() {      // call with device_mu() held
  static std::map<int, DeviceInfo> devs;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return nullptr;
  DeviceInfo& d = devs[dev];
  if (d.sm_count == 0) {
    if (cudaDeviceGetAttribute(&d.sm_count, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || d.sm_count <= 0)
      d.sm_count = 132;
  }
  return &d;
}
inline int device_sm_count() {
  std::lock_guard<std::mutex> lock(device_mu());
  DeviceInfo* d = device_info();
  return d ? d->sm_count : 132;
}

struct MapKey {
  const void* ptr;
  long inner, outer, ld;
  int box_inner, box_outer;
  int rank3;    // 1: MN-major operand as {32 floats, outer rows, inner/32 groups}, box {32, box_outer, 4}
  int raw;      // 1: FLOAT32 (the raw words, precise kernel); 0: TFLOAT32 (TMA rounds to tf32)
  bool operator<(const MapKey& o) const {
    return std::tie(ptr, inner, outer, ld, box_inner, box_outer, rank3, raw) <
           std::tie(o.ptr, o.inner, o.outer, o.ld, o.box_inner, o.box_outer, o.rank3, o.raw);
  }
};

// fp32 2-D row-major tensor [outer, inner] with row pitch ld floats; 128B swizzle; OOB reads give zeros
inline int encode_map(const MapKey& k, CUtensorMap* out) {
  static thread_local std::map<MapKey, CUtensorMap> cache;
  auto it = cache.find(k);
  if (it != cache.end()) {
    *out = it->second;
    return TA3N_OK;
  }
  PFN_encodeTiled fn = encode_fn();
  if (!fn) return fail(TA3N_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  // a DRIVER call: the calling thread needs a current context.  A replica thread of nn.DataParallel (main.py:79) has
  // only selected its device through the runtime so far -- bind the primary context, once per thread: cudaFree is
  // illegal while a stream is being captured, and a miss can happen inside a CUDA graph capture (after the clear
  // below, keys its warm-up encoded are gone)
  static thread_local bool context_bound = false;
  if (!context_bound) {
    cudaFree(nullptr);
    context_bound = true;
  }
  cuuint64_t dims[3] = {(cuuint64_t)k.inner, (cuuint64_t)k.outer, 1};
  cuuint64_t strides[2] = {(cuuint64_t)k.ld * sizeof(float), 128};
  cuuint32_t box[3] = {(cuuint32_t)k.box_inner, (cuuint32_t)k.box_outer, 4};
  cuuint32_t estr[3] = {1, 1, 1};
  if (k.rank3) {
    dims[0] = 32;
    dims[2] = (cuuint64_t)(k.inner / 32);
  }
  // TFLOAT32: the TMA unit rounds fp32 -> tf32 (round to nearest) while filling shared memory, so the
  // tensor core never sees the truncation bias (-2^-11 relative per operand) it would apply to raw fp32
  // bit patterns (a -7e-4 bias per GEMM with FLOAT32 maps).
  CUresult r = fn(out, k.raw ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_TFLOAT32, k.rank3 ? 3 : 2,
                  const_cast<void*>(k.ptr), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(TA3N_ERR_CUDA, "cuTensorMapEncodeTiled failed with %d", (int)r);
  if (cache.size() > 4096) cache.clear();
  cache[k] = *out;
  return TA3N_OK;
}

inline bool tc_operand_ok(const float* p, int ld) {
  return p != nullptr && (reinterpret_cast<uintptr_t>(p) & 15u) == 0 && (ld % 4) == 0 && ld > 0;
}

// tensor-map keys of one segment of a group (launch_tc deduplicates them within a launch)
inline void tc_seg_keys(const Seg& s, const Group& g, bool a_kmaj, bool b_kmaj, bool a3d, bool b3d, MapKey* ka,
                        MapKey* kb, bool raw = false) {
  const int rw = raw ? 1 : 0;
  *ka = a_kmaj ? MapKey{s.A, s.len, g.M, s.lda, TC_BK, TC_BM, 0, rw} : MapKey{s.A, g.M, s.len, s.lda, 32, TC_BK, a3d ? 1 : 0, rw};
  *kb = b_kmaj ? MapKey{s.B, s.len, g.N, s.ldb, TC_BK, TC_BN, 0, rw} : MapKey{s.B, g.N, s.len, s.ldb, 32, TC_BK, b3d ? 1 : 0, rw};
}

// Is this group worth / able to run on the tensor-core engine?
inline bool tc_group_ok(const GemmPlan& plan, const Group& g) {
  if (plan.load_flags != 0) return false;                    // ReLU-on-load needs a register pass
  if ((long)g.M * g.N < 64L * 64L) return false;             // tiny heads stay on the SIMT engine
  if (g.seg_count > kMaxSegs) return false;
  std::map<MapKey, int> maps;
  for (int i = 0; i < g.seg_count; ++i) {
    const Seg& s = plan.segs[g.seg_begin + i];
    if (!tc_operand_ok(s.A, s.lda) || !tc_operand_ok(s.B, s.ldb) || s.len <= 0) return false;
    // the rank-3 and raw flags are the same for every segment of a launch: they do not change the count
    MapKey ka, kb;
    tc_seg_keys(s, g, plan.a_kmaj, plan.b_kmaj, false, false, &ka, &kb);
    maps[ka] = maps[kb] = 0;
  }
  // the maps of one launch sit in its kernel parameters: a group that needs more of them than one launch holds
  // (the data gradient of a frame of a long clip: one A and one B map per relation slot reading it) runs on the SIMT
  // engine
  return (int)maps.size() <= kMaxMaps;
}

template <bool A_KMAJ, bool B_KMAJ>
inline int tc_launch_one(const GemmTable& tab, const TcMaps& maps, const TcSegMaps& sm, cudaStream_t stream,
                         const char* label) {
  constexpr int slot = (A_KMAJ ? 0 : 1) + (B_KMAJ ? 0 : 2);
  int first_wave = 132;
  {
    std::lock_guard<std::mutex> lock(device_mu());
    DeviceInfo* d = device_info();
    if (!d) return fail(TA3N_ERR_CUDA, "cudaGetDevice failed");
    if (!d->configured[slot]) {
      TA3N_CUDA(cudaFuncSetAttribute(seg_gemm_tc_kernel<A_KMAJ, B_KMAJ>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     tc_smem_bytes(B_KMAJ)));
      d->configured[slot] = true;
    }
    first_wave = d->sm_count;
  }
  pre_launch(label, stream);
  launch_kernel(seg_gemm_tc_kernel<A_KMAJ, B_KMAJ>, tab.total_tiles, TC_THREADS, tc_smem_bytes(B_KMAJ), stream, tab,
                maps, sm, first_wave);
  return after_launch();
}

// the precise kernel, per operand layout
template <bool A_KMAJ, bool B_KMAJ>
inline int tc_launch_x3(const GemmTable& tab, const TcMaps& maps, const TcSegMaps& sm, const X3Sched& sched, int grid,
                        cudaStream_t stream, const char* label) {
  constexpr int slot = (A_KMAJ ? 0 : 1) + (B_KMAJ ? 0 : 2);
  {
    std::lock_guard<std::mutex> lock(device_mu());
    DeviceInfo* d = device_info();
    if (!d) return fail(TA3N_ERR_CUDA, "cudaGetDevice failed");
    if (!d->x3_configured[slot]) {
      TA3N_CUDA(cudaFuncSetAttribute(seg_gemm_tc_x3_kernel<A_KMAJ, B_KMAJ>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     x3_smem_bytes()));
      d->x3_configured[slot] = true;
    }
  }
  pre_launch(label, stream);
  launch_kernel(seg_gemm_tc_x3_kernel<A_KMAJ, B_KMAJ>, grid, TC_THREADS, x3_smem_bytes(), stream, tab, maps, sm, sched);
  return after_launch();
}

// Copy the groups `idx` of `plan` (with their segments) into a new plan.
inline GemmPlan sub_plan(const GemmPlan& plan, const std::vector<int>& idx) {
  GemmPlan out;
  out.a_kmaj = plan.a_kmaj;
  out.b_kmaj = plan.b_kmaj;
  out.load_flags = plan.load_flags;
  out.label = plan.label;
  for (int i : idx) {
    Group g = plan.groups[i];
    const int b = g.seg_begin;
    g.seg_begin = (int)out.segs.size();
    for (int k = 0; k < g.seg_count; ++k) out.segs.push_back(plan.segs[b + k]);
    out.groups.push_back(g);
  }
  return out;
}

// rank-3 maps for MN-major operands whose MN extent is a multiple of 32 in every group of the plan
inline void tc_rank3_flags(const GemmPlan& plan, bool* a3d, bool* b3d) {
  *a3d = !plan.a_kmaj;
  *b3d = !plan.b_kmaj;
  for (const Group& g : plan.groups) {
    if (g.M % 32 != 0) *a3d = false;
    if (g.N % 32 != 0) *b3d = false;
  }
}

inline double x3_makespan(const GemmPlan& plan, const std::vector<int>& ks, int sms,
                          std::vector<std::vector<std::pair<int, int>>>* assign = nullptr);

// The precise kernel's schedule for the groups [g_first, g_first + tab.n_groups) of `plan` staged in `tab`: the LPT
// lists of x3_makespan, one CTA per non-empty list.  Returns the grid size.
inline int x3_schedule(const GemmPlan& plan, size_t g_first, const GemmTable& tab, X3Sched* sched) {
  const int ctas = std::min(device_sm_count(), kX3MaxCtas);
  if (tab.total_tiles > kX3MaxTasks) {
    sched->listed = 0;
    return std::min(tab.total_tiles, ctas);
  }
  std::vector<int> idx, ks;
  for (int i = 0; i < tab.n_groups; ++i) {
    idx.push_back((int)g_first + i);
    ks.push_back(tab.g[i].ksplit);
  }
  std::vector<std::vector<std::pair<int, int>>> lists;
  x3_makespan(sub_plan(plan, idx), ks, ctas, &lists);
  sched->listed = 1;
  int grid = 0, n = 0;
  for (const auto& l : lists) {
    if (l.empty()) continue;
    sched->off[grid++] = (unsigned short)n;
    for (const auto& gt : l) sched->task[n++] = (unsigned short)(tab.g[gt.first].tile_begin + gt.second);
  }
  sched->off[grid] = (unsigned short)n;
  return grid;
}

// Launch `plan` (all groups eligible) on the tensor-core engine.
inline int launch_tc(const GemmPlan& plan_in, cudaStream_t stream, bool precise = false) {
  // longest-K groups first (see the tile remap in the kernel): LPT-style balance of the tensor pipe
  std::vector<int> order(plan_in.groups.size());
  for (size_t i = 0; i < order.size(); ++i) order[i] = (int)i;
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) {
    return plan_in.k_total(plan_in.groups[a]) / plan_in.groups[a].ksplit >
           plan_in.k_total(plan_in.groups[b]) / plan_in.groups[b].ksplit;
  });
  const GemmPlan plan = sub_plan(plan_in, order);
  bool a3d, b3d;
  tc_rank3_flags(plan, &a3d, &b3d);
  size_t gi = 0;
  while (gi < plan.groups.size()) {
    const size_t g_first = gi;
    GemmTable tab;
    TcMaps maps;
    TcSegMaps sm;
    memset(&tab, 0, sizeof(int) * 4);
    memset(&sm, 0, sizeof(sm));
    std::map<MapKey, int> local;
    int ng = 0, ns = 0, tiles = 0, nmaps = 0;
    bool any_split = false;
    while (gi < plan.groups.size() && ng < kMaxGroups) {
      const Group& src = plan.groups[gi];
      if (ns + src.seg_count > kMaxSegs) break;
      // tensor maps of this group's segments (deduplicated within the launch)
      std::vector<std::pair<MapKey, MapKey>> keys;
      int fresh = 0;
      std::map<MapKey, int> trial = local;
      for (int i = 0; i < src.seg_count; ++i) {
        MapKey ka, kb;
        tc_seg_keys(plan.segs[src.seg_begin + i], src, plan.a_kmaj, plan.b_kmaj, a3d, b3d, &ka, &kb, precise);
        for (const MapKey& k : {ka, kb})
          if (!trial.count(k)) trial[k] = nmaps + fresh++;
        keys.push_back({ka, kb});
      }
      if (nmaps + fresh > kMaxMaps) {
        if (ng == 0) return fail(TA3N_ERR_UNSUPPORTED, "tensor-core GEMM: one group needs %d tensor maps", fresh);
        break;
      }
      for (auto& kv : trial)
        if (!local.count(kv.first)) {
          TA3N_TRY(encode_map(kv.first, &maps.m[kv.second]));
          local[kv.first] = kv.second;
        }
      nmaps += fresh;
      Group g = src;
      for (int i = 0; i < src.seg_count; ++i) {
        tab.s[ns + i] = plan.segs[src.seg_begin + i];
        sm.a[ns + i] = (unsigned char)local[keys[i].first];
        sm.b[ns + i] = (unsigned char)local[keys[i].second];
      }
      g.seg_begin = ns;
      ns += src.seg_count;
      g.tiles_m = (g.M + TC_BM - 1) / TC_BM;
      g.tiles_n = (g.N + TC_BN - 1) / TC_BN;
      g.tile_begin = tiles;
      tiles += g.tiles_m * g.tiles_n * g.ksplit;
      g.fix_slot = -1;
      any_split |= g.ksplit > 1;
      tab.g[ng++] = g;
      ++gi;
    }
    tab.n_groups = ng;
    tab.total_tiles = tiles;
    tab.pad_ = (a3d ? 1 : 0) | (b3d ? 2 : 0);
    if (tiles > 0) {
      X3Sched sched;
      const int grid = precise ? x3_schedule(plan, g_first, tab, &sched) : 0;
      if (precise && plan.a_kmaj && plan.b_kmaj)
        TA3N_TRY((tc_launch_x3<true, true>(tab, maps, sm, sched, grid, stream, plan.label)));
      else if (precise && plan.a_kmaj && !plan.b_kmaj)
        TA3N_TRY((tc_launch_x3<true, false>(tab, maps, sm, sched, grid, stream, plan.label)));
      else if (precise && !plan.a_kmaj && !plan.b_kmaj)
        TA3N_TRY((tc_launch_x3<false, false>(tab, maps, sm, sched, grid, stream, plan.label)));
      else if (precise)
        TA3N_TRY((tc_launch_x3<false, true>(tab, maps, sm, sched, grid, stream, plan.label)));
      else if (plan.a_kmaj && plan.b_kmaj)
        TA3N_TRY((tc_launch_one<true, true>(tab, maps, sm, stream, plan.label)));
      else if (plan.a_kmaj && !plan.b_kmaj)
        TA3N_TRY((tc_launch_one<true, false>(tab, maps, sm, stream, plan.label)));
      else if (!plan.a_kmaj && !plan.b_kmaj)
        TA3N_TRY((tc_launch_one<false, false>(tab, maps, sm, stream, plan.label)));
      else
        TA3N_TRY((tc_launch_one<false, true>(tab, maps, sm, stream, plan.label)));
      if (any_split) {
        // vectorised reduce when every split group allows it (the forward layers), blocks for split groups only
        SplitGroups sgs;
        sgs.n = 0;
        bool vec = true;
        size_t mx4 = 0;
        for (int i = 0; i < ng; ++i) {
          const Group& g = tab.g[i];
          if (g.ksplit <= 1) continue;
          sgs.idx[sgs.n++] = (unsigned char)i;
          const bool ok = g.N % 4 == 0 && g.ldc % 4 == 0 && (reinterpret_cast<uintptr_t>(g.C) & 15u) == 0 &&
                          (reinterpret_cast<uintptr_t>(g.partial) & 15u) == 0 &&
                          (g.flags & ~(EPI_BIAS | EPI_RELU | EPI_DROP_RNG)) == 0 && g.ksplit <= 8;
          vec = vec && ok;
          mx4 = std::max(mx4, (size_t)g.M * g.N / 4);
        }
        if (vec && sgs.n > 0) {
          dim3 grid((unsigned)std::min<size_t>((mx4 + 255) / 256, 1024), sgs.n);
          pre_launch("splitk_reduce", stream);
          launch_kernel(splitk_reduce_v4_kernel, grid, 256, 0, stream, tab, sgs);
        } else {
          dim3 grid(splitk_reduce_blocks(tab), ng);
          pre_launch("splitk_reduce", stream);
          launch_kernel(splitk_reduce_kernel, grid, 256, 0, stream, tab);
        }
        TA3N_TRY(after_launch());
      }
    }
  }
  return TA3N_OK;
}

// ---- balanced split-K for the precise forward launches ------------------------------------------------------
// The precise kernel holds one CTA per SM and is bound by shared-memory bandwidth, so a launch costs what its
// longest CTA queue costs: the shared layer has 80 tiles of 64 slabs for 132 SMs, the forward batch 80
// tiles of 16 slabs next to tiles of up to 80.  Split factors per group are chosen by simulating the greedy (LPT)
// assignment of the resulting tasks to the SMs for a few target task lengths; partials go to the caller's scratch
// (ta3n_set_forward_scratch) and a fixed-order reduce pass applies the epilogue.  Deterministic.
struct ForwardScratch {
  void* ptr = nullptr;
  size_t bytes = 0;
};
inline ForwardScratch& forward_scratch() {
  static thread_local ForwardScratch s;
  return s;
}
inline int x3_plan_slabs(const GemmPlan& plan, const Group& g) {
  int n = 0;
  for (int k = 0; k < g.seg_count; ++k) n += (plan.segs[g.seg_begin + k].len + TC_BK - 1) / TC_BK;
  return n;
}
// Greedy (LPT) assignment of the tasks of `plan` (group gi split ks[gi] ways: tiles * ks[gi] tasks, numbered within the
// group) to `sms` SMs; returns the makespan.  `assign`, when given, receives the task list of each SM as (group, task)
// pairs, longest first: the precise kernel runs exactly this schedule.
inline double x3_makespan(const GemmPlan& plan, const std::vector<int>& ks, int sms,
                          std::vector<std::vector<std::pair<int, int>>>* assign) {
  struct Task {
    double len;
    int g, t;
  };
  std::vector<Task> tasks;
  for (size_t gi = 0; gi < plan.groups.size(); ++gi) {
    const Group& g = plan.groups[gi];
    const int tiles = ((g.M + TC_BM - 1) / TC_BM) * ((g.N + TC_BN - 1) / TC_BN);
    const double len = (double)x3_plan_slabs(plan, g) / ks[gi] + 4.0;      // + prologue / epilogue, in slab units
    for (int t = 0; t < tiles * ks[gi]; ++t) tasks.push_back({len, (int)gi, t});
  }
  std::sort(tasks.begin(), tasks.end(), [](const Task& a, const Task& b) {
    return a.len != b.len ? a.len > b.len : std::tie(a.g, a.t) < std::tie(b.g, b.t);
  });
  std::vector<double> load(sms, 0.0);
  if (assign) assign->assign(sms, {});
  for (const Task& t : tasks) {
    const auto it = std::min_element(load.begin(), load.end());
    *it += t.len;
    if (assign) (*assign)[it - load.begin()].push_back({t.g, t.t});
  }
  return *std::max_element(load.begin(), load.end());
}
inline void plan_splitk_balanced(GemmPlan& plan, Arena* arena, int sms) {
  if (!arena) return;
  double total = 0;
  for (const Group& g : plan.groups)
    total += (double)x3_plan_slabs(plan, g) * ((g.M + TC_BM - 1) / TC_BM) * ((g.N + TC_BN - 1) / TC_BN);
  std::vector<int> best(plan.groups.size(), 1);
  double best_cost = x3_makespan(plan, best, sms);
  for (double c : {1.1, 1.25, 1.5, 2.0, -2.0, -3.0, -4.0}) {      // negative: the same factor for every group
    const double target = std::max(8.0, total / sms * c);
    std::vector<int> ks(plan.groups.size(), 1);
    for (size_t gi = 0; gi < plan.groups.size(); ++gi) {
      const int slabs = x3_plan_slabs(plan, plan.groups[gi]);
      int k = c > 0 ? (int)std::ceil(slabs / target) : (int)(-c);
      k = std::max(1, std::min(k, 8));
      while (k > 1 && slabs / k < 8) --k;
      ks[gi] = k;
    }
    bool any = false;
    for (int k : ks) any |= k > 1;
    const double cost = x3_makespan(plan, ks, sms) + (any ? 8.0 : 0.0);      // the reduce pass
    if (cost < best_cost * 0.92) {
      best_cost = cost;
      best = ks;
    }
  }
  for (size_t gi = 0; gi < plan.groups.size(); ++gi) {
    Group& g = plan.groups[gi];
    if (best[gi] < 2) continue;
    float* p = arena->floats((size_t)best[gi] * g.M * g.N);
    if (!p) continue;                      // scratch too small: stay unsplit (still correct)
    g.ksplit = best[gi];
    g.partial = p;
  }
}

// TA3N_X3_DGRAD=1: the data-gradient GEMMs of the x3 engine at fp32 grade as well: TRN bias gradients at ~2e-6 instead
// of ~2.4e-4, at the cost of three products per K step on every data-gradient GEMM; the worst tensors (shared-layer
// gradients, set by ReLU-pattern differences and by the tf32 weight-gradient GEMM itself) do not improve -> off by
// default.
inline bool x3_dgrad_enabled() {
  static const bool on = []() {
    const char* e = getenv("TA3N_X3_DGRAD");
    return e && e[0] == '1';
  }();
  return on;
}

// Run a plan.  With the tf32 engine selected, every group the tensor-core kernel can take runs
// there; the rest (tiny heads, unaligned operands, ReLU-on-load) runs on the fp32 SIMT engine --
// still CUDA, never the CPU.
inline int run_gemm(GemmPlan& plan, cudaStream_t stream, Arena* splitk_arena = nullptr) {
  if (plan.groups.empty()) return TA3N_OK;
  for (auto& g : plan.groups)
    if (g.M <= 0 || g.N <= 0 || g.seg_count <= 0)
      return fail(TA3N_ERR_INVALID, "seg_gemm: empty group M=%d N=%d segs=%d", g.M, g.N, g.seg_count);
  const int engine = gemm_engine().load();
  if (engine == TA3N_GEMM_TF32_TCGEN05 || engine == TA3N_GEMM_TF32X3_TCGEN05) {
    // the precise kernel for the forward layers of the x3 engine (K-major operands); everything else plain tf32
    const bool precise = engine == TA3N_GEMM_TF32X3_TCGEN05 && (plan.precise || (plan.precise_dgrad && x3_dgrad_enabled()));
    std::vector<int> tc_idx, simt_idx;
    // x3 engine: the small weight-gradient GEMMs (the 256 x 256 layers of the video / relation discriminators,
    // <= 0.3 GFLOP each) run on the precise kernel.  Near the adversarial equilibrium their source and target
    // halves cancel, which amplifies the 3e-4 of a tf32 product to 4e-3 of the net gradient (cfg3).
    // (One 20-tile launch of the x3 kernel instead of the exact SIMT engine, which is several times slower here.)
    const bool small_exact = engine == TA3N_GEMM_TF32X3_TCGEN05 && !plan.a_kmaj && !plan.b_kmaj && !precise;
    std::vector<int> fine_idx;
    for (int i = 0; i < (int)plan.groups.size(); ++i) {
      const Group& g = plan.groups[i];
      const bool tiny = small_exact && (long)g.M * g.N <= 256L * 256L && 2.0 * g.M * g.N * (double)plan.k_total(g) <= 3e8;
      if (!tc_group_ok(plan, g))
        simt_idx.push_back(i);
      else
        (tiny ? fine_idx : tc_idx).push_back(i);
    }
    if (!fine_idx.empty()) {
      GemmPlan fine = sub_plan(plan, fine_idx);
      fine.label = "wgrad_small_x3";
      TA3N_TRY(launch_tc(fine, stream, true));
    }
    if (!tc_idx.empty()) {
      GemmPlan tc = sub_plan(plan, tc_idx);
      // only the forward plans: they run on ONE stream, in order, so they can share the scratch; precise data-gradient
      // plans (TA3N_X3_DGRAD=1) may run on forked streams (parallel_branches) and stay unsplit
      if (precise && plan.precise && splitk_arena == nullptr && forward_scratch().ptr != nullptr) {
        Arena scratch(forward_scratch().ptr, forward_scratch().bytes);
        plan_splitk_balanced(tc, &scratch, device_sm_count());
      } else {
        plan_splitk(tc, splitk_arena, TC_BM, TC_BN, TC_BK, 4);
      }
      TA3N_TRY(launch_tc(tc, stream, precise));
    }
    if (!simt_idx.empty()) {
      GemmPlan rest = sub_plan(plan, simt_idx);
      plan_splitk(rest, splitk_arena, SG_BM, SG_BN, SG_BK, 8);
      TA3N_TRY(launch_simt(rest, stream));
    }
    return TA3N_OK;
  }
  plan_splitk(plan, splitk_arena, SG_BM, SG_BN, SG_BK, 8);
  return launch_simt(plan, stream);
}

}  // namespace ta3n
