// step_kernel.cuh -- the fused training step of the path as ONE persistent kernel.
//
// main.py:418-576 for the shipped configuration (forward of VideoModel.forward models.py:545-722, the composed loss,
// backward to every parameter gradient) is a static graph of ~900 small tasks: 128x128 wgmma GEMM tiles
// (gemm_wgmma.cuh), per-video row tasks and column-sum tasks (step_rows.cuh).  Run as separate launches
// (25 kernels, every one sub-wave) the step is the SUM of per-launch critical paths plus a drain and a
// pipeline fill at every kernel boundary.  Here one CTA per SM pulls tasks from
// priority queues; a task becomes eligible when the arrival counters of the tasks that produce its inputs have reached
// their targets (release / acquire through global memory), so
//   * dependent stages overlap at 128-row granularity instead of at kernel boundaries,
//   * the frame branch, the weight-gradient tiles and the column sums (half of the work, needed by nobody on the
//     video-level chain) fill the SMs the latency-bound chain leaves idle,
//   * split-K tiles are folded by an "owner" tile that depends on its partial tiles -- deterministic, no reduce pass.
// Scheduling: the tasks live in kStepQueues queues (0 = the forward / data-gradient spine, 1..6 = the per-row-block
// chains between the TRN forward and the TRN data gradient, 7 = fillers: frame branch, weight gradients, column sums),
// each with a ticket cursor.  A CTA's scheduler warp looks at the head of every queue at once, and draws a ticket
// from the first queue whose head task is READY (arrival counters reached).  A CTA never blocks on a task: a ticket
// drawn in a race for a task that is not ready yet is parked and polled, while the CTA keeps taking other work -- an
// SM that cannot advance the critical chain takes a filler instead of waiting.  Progress needs the queue orders to be
// consistent with the dependencies (a head-only scheduler must be able to finish: checked by ta3n_step_describe and
// tests/test_step_plan.py); a bounded spin turns a violation into a trap instead of a hang.
// Results do not depend on which CTA runs a task: every output element is produced by exactly one task with a fixed
// summation order -> bit-identical reruns.
#pragma once

#include "gemm_wgmma.cuh"
#include "step_rows.cuh"

namespace ta3n {

// warps 0..7: the two wgmma consumer warpgroups of the GEMM tiles, the epilogue and the row tasks; 8 TMA producer;
// 9 scheduler
constexpr int kStepThreads = 320;
constexpr int kStepProducerWarp = 8, kStepSchedulerWarp = 9;
constexpr int kStepStages = 3;        // operand ring: 3 x 32 KB
constexpr int kStepSlots = 3;         // tasks a CTA holds at once (scheduled ahead of the one being finished)
constexpr int kStepScratchBytes = 40 * 1024;      // shared memory of the row tasks (outside the operand ring)
static_assert(8 * TC_EPI_STAGE_FLOATS * 4 <= kStepScratchBytes, "epilogue staging tiles live in the scratch area");
// ring + row-task scratch + accumulator tile
constexpr int kStepSmemBytes = kStepStages * TC_STAGE_BYTES + kStepScratchBytes + TC_ACC_BYTES + 1024;

constexpr int kStepQueues = 8;

enum : int { TASK_GEMM = 0, TASK_ROW = 1, TASK_COLSUM_PART = 2, TASK_COLSUM_REDUCE = 3, TASK_FINISH = 4, TASK_STOP = 5,
             TASK_FRAME = 6 };

struct StepTask {
  int type;
  int group;              // GEMM: group index; COLSUM_*: job index
  int m0, n0;             // GEMM: tile origin; ROW / FRAME: first video / frame row, count; COLSUM_PART: column block, row split
  int split, mode;        // GEMM: split index, TILE_* mode; ROW: ROW_* kind
  int wait_begin[2], wait_end[2], wait_val[2];     // wait until counters[i] >= val for i in [begin, end)
  int signal;             // counter bumped on completion (-1: none)
  int signal2;            // second counter (the stage total; -1: none)
  int split_counter;      // GEMM, TILE_SPLIT: arrival counter of the output tile (the last split to arrive reduces)
  int urgent;             // on the latency-critical chain: only an otherwise idle CTA may take it (no queueing behind
                          // tiles the CTA has already committed to)
};
static_assert(sizeof(StepTask) % 4 == 0 && sizeof(StepTask) / 4 <= 32, "staged by one warp");

struct StepGroup {
  Group g;
  int a_kmaj, b_kmaj, pad_flags, seg_begin;
};

struct StepHeader {
  int n_tasks, n_counters, n_groups, n_jobs;
  const StepTask* tasks;
  const StepGroup* groups;
  const SegLite* segs;
  const CUtensorMap* maps;
  const WColsumJob* jobs;
  const TailArgs* tail;
  int* counters;                 // [n_counters] arrival counters, then [kStepQueues] ticket cursors of the queues
  int queue_begin[kStepQueues + 1];   // tasks of queue q are [queue_begin[q], queue_begin[q + 1])
  unsigned long long* step_counter;   // dropout step counter, advanced by the FINISH task (may be null)
  unsigned long long* trace;     // optional [n_tasks][8]: {sm id | tag, started, accumulator ready, done, body done,
                                 // CTA synced, -, -} (globaltimer ns), followed by [M / 8][8] phase marks of the row tasks
};

struct StepSlot {                // one scheduled task: descriptor + (GEMM) the group and its segments
  StepTask task;
  int index;                     // position in the queue (trace)
  int flags;                     // a_kmaj | b_kmaj << 1 | pad_flags << 2
  int c_begin, n_iter;
  TileCtx ctx;
};

// NOTE: polls use ld.relaxed, never ld.acquire: ptxas implements a gpu-scope acquire as load + CCTL.IVALL, i.e. every
// poll invalidated the SM's whole L1, once per poll.
// The acquire is one fence after the poll has succeeded.
__device__ __forceinline__ void red_release(int* p, int v) {
  asm volatile("red.release.gpu.global.add.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void fence_proxy_async_all() { asm volatile("fence.proxy.async;" ::: "memory"); }
__device__ __forceinline__ unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ unsigned sm_id() {
  unsigned v;
  asm volatile("mov.u32 %0, %smid;" : "=r"(v));
  return v;
}

// Task slots in file-scope shared memory, so that the out-of-line epilogue below reads its group with LDS
__shared__ StepSlot g_slots[kStepSlots];

// The tile epilogue of slot s, one out-of-line copy per class (own register allocation, see step_rows.cuh)
template <int CLS>
__device__ __noinline__ void step_epilogue_cls(const int s, const float* acc, const int ew, const uint32_t stage) {
  const StepSlot& sl = g_slots[s];
  tc_epilogue_cls<8, CLS>(sl.ctx, sl.task.m0, sl.task.n0, sl.task.split, sl.n_iter, sl.task.mode, acc, ew, stage);
}
// TILE_REDUCE pass of slot s: the split-K partials of the tile, summed in split order, through the fused epilogue
template <int CLS>
__device__ __noinline__ void step_reduce_cls(const int s, const int ew, const uint32_t stage) {
  const StepSlot& sl = g_slots[s];
  tc_epilogue_cls<8, CLS>(sl.ctx, sl.task.m0, sl.task.n0, 0, 0, TILE_REDUCE, nullptr, ew, stage);
}
__device__ __forceinline__ void step_reduce(const int s, const int ew, const uint32_t stage) {
  if (epi_class(TILE_REDUCE, g_slots[s].ctx.g.flags) == EPI_CLS_PLAIN)
    step_reduce_cls<EPI_CLS_PLAIN>(s, ew, stage);
  else
    step_reduce_cls<EPI_CLS_FORWARD>(s, ew, stage);      // split groups never carry auxiliary operands
}
__device__ __forceinline__ void step_epilogue(const int s, const float* acc, const int ew, const uint32_t stage) {
  const int cls = epi_class(g_slots[s].task.mode, g_slots[s].ctx.g.flags);
  if (cls == EPI_CLS_PLAIN)
    step_epilogue_cls<EPI_CLS_PLAIN>(s, acc, ew, stage);
  else if (cls == EPI_CLS_FORWARD)
    step_epilogue_cls<EPI_CLS_FORWARD>(s, acc, ew, stage);
  else
    step_epilogue_cls<EPI_CLS_ALL>(s, acc, ew, stage);
}

__device__ __forceinline__ int ld_relaxed(const int* p) {
  int v;
  asm volatile("ld.relaxed.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// Is task `idx` runnable by this CTA now?  (arrival counters reached; row-type and urgent tasks only when the CTA is
// idle: they must not queue behind tiles it has already committed to)
__device__ __forceinline__ bool step_task_ready(const StepHeader& hd, const int idx, const bool idle) {
  const StepTask* t = hd.tasks + idx;
  if (!idle && (__ldg(&t->type) != TASK_GEMM || __ldg(&t->urgent) != 0)) return false;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int cb = __ldg(&t->wait_begin[r]), ce = __ldg(&t->wait_end[r]), val = __ldg(&t->wait_val[r]);
    for (int c = cb; c < ce; ++c)
      if (ld_relaxed(hd.counters + c) < val) return false;      // relaxed: the caller fences ONCE after the claim
  }
  return true;
}

constexpr int kStepDeferred = 8;      // tickets a CTA may hold for tasks that were not ready when it drew them

// Scheduler warp: the next task for this CTA.  Every queue has a ticket cursor; a CTA draws a ticket (atomicAdd: no two
// CTAs ever contend for the same task) only after seeing that the task at the cursor is READY.  When several CTAs draw
// at once the later tickets belong to tasks nobody has checked: such a task, if not ready, is parked in the CTA's
// deferred list and polled with the queue heads -- the CTA never blocks on it and keeps taking other work.
// Row / column-sum tasks and the GEMM tiles of the latency-critical chains (`urgent`) are taken only by a CTA with
// nothing else in flight: queued behind tiles a CTA has committed to they would wait while other SMs idle.  One CTA
// in four is RESERVED for the spine and the chains: it ignores the filler queue until every other queue is drained,
// so that a chain task that becomes ready finds an idle SM instead of waiting for a filler tile to finish.
// Returns the task index, or -1 when every queue is drained.
__device__ __forceinline__ int step_next_task(const StepHeader& hd, int* const cursors, const int lane,
                                              const volatile int* done_count, const uint32_t issued, int* deferred,
                                              int& n_def) {
  unsigned spins = 0;
  for (;;) {
    const bool allow_rows = (uint32_t)(*done_count) == issued;
    const bool reserved = (blockIdx.x & 3u) == 0u;
    int cand = -1;
    bool ready = false;
    if (lane < kStepQueues) {
      const int c = ld_relaxed(cursors + lane);
      if (c < hd.queue_begin[lane + 1] - hd.queue_begin[lane]) cand = hd.queue_begin[lane] + c;
    } else if (lane < kStepQueues + kStepDeferred) {
      if (lane - kStepQueues < n_def) cand = deferred[lane - kStepQueues];
    }
    const unsigned open = __ballot_sync(0xffffffffu, cand >= 0);
    if (reserved && lane == kStepQueues - 1 && (open & ((1u << (kStepQueues - 1)) - 1u)) != 0u) cand = -1;
    if (cand >= 0) ready = step_task_ready(hd, cand, allow_rows);
    const unsigned rm = __ballot_sync(0xffffffffu, ready);
    const unsigned rdef = rm >> kStepQueues;
    if (rdef != 0u) {                                       // a parked task has become ready: oldest commitment first
      const int k = __ffs(rdef) - 1;
      const int t = deferred[k];
      __syncwarp();
      if (lane == 0) deferred[k] = deferred[n_def - 1];
      --n_def;
      __syncwarp();
      return t;
    }
    const unsigned rq = rm & ((1u << kStepQueues) - 1u);
    if (rq != 0u && n_def < kStepDeferred) {
      const int q = __ffs(rq) - 1;
      const int seen = __shfl_sync(0xffffffffu, cand, q);
      int t = 0;
      if (lane == 0) t = hd.queue_begin[q] + atomicAdd(cursors + q, 1);
      t = __shfl_sync(0xffffffffu, t, 0);
      if (t >= hd.queue_begin[q + 1]) continue;             // the queue ran out between the look and the draw
      if (t == seen) return t;
      bool ok = false;
      if (lane == 0) ok = step_task_ready(hd, t, allow_rows);
      ok = __shfl_sync(0xffffffffu, ok ? 1 : 0, 0) != 0;
      if (ok) return t;
      if (lane == 0) deferred[n_def] = t;
      ++n_def;
      __syncwarp();
      continue;
    }
    if (open == 0u) return -1;                              // every queue drained, nothing parked
    __nanosleep(32);
    if (++spins > (1u << 24)) __trap();                     // ~ seconds: a task graph that cannot complete
  }
}

__global__ void __launch_bounds__(kStepThreads, 1) ta3n_step_kernel(const __grid_constant__ StepHeader hd) {
  extern __shared__ uint8_t step_smem_raw[];
  __shared__ __align__(8) TcShared sh;
  __shared__ __align__(8) uint64_t slot_full[kStepSlots];
  __shared__ __align__(8) uint64_t slot_empty[kStepSlots];
  StepSlot* const slots = g_slots;
  __shared__ int done_count;            // tasks this CTA has completed (scheduler: is anything still in flight?)
  __shared__ int split_rank;            // TILE_SPLIT: how many splits of the tile had arrived before this one
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(step_smem_raw) + 1023) & ~uintptr_t(1023));
  float* scratch = reinterpret_cast<float*>(smem + kStepStages * TC_STAGE_BYTES);
  float* acc_tile = reinterpret_cast<float*>(smem + kStepStages * TC_STAGE_BYTES + kStepScratchBytes);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tid = threadIdx.x;
  int* const cursors = hd.counters + hd.n_counters;
  __shared__ int deferred[kStepDeferred];

  // ---- one-time setup ----
  if (warp == kStepProducerWarp && lane == 0) {
    tc_pipe_init<kStepStages>(&sh);
    for (int s = 0; s < kStepSlots; ++s) {
      mbar_init(&slot_full[s], 1);
      mbar_init(&slot_empty[s], 1 + TC_CONSUMER_WARPS);       // producer + 8 consumer warps
    }
    done_count = 0;
    fence_barrier_init();
  }
  for (int i = tid; i < (int)(sizeof(TailArgs) / sizeof(int)); i += kStepThreads)
    reinterpret_cast<int*>(&g_tail)[i] = reinterpret_cast<const int*>(hd.tail)[i];
  __syncthreads();
  if (tid == 0) g_tail.dbg = hd.trace ? hd.trace + (size_t)hd.n_tasks * 8 : nullptr;      // row-task phase marks
  __syncthreads();
  // (no griddepcontrol here: the kernel is launched with plain stream ordering behind the memset of its counters,
  //  and must not release its dependents before it has finished)

  if (warp == kStepSchedulerWarp) {
    // =========================== scheduler: claim ready tasks, stage them ===========================
    int n_def = 0;
    for (uint32_t k = 0;; ++k) {
      const int s = (int)(k % kStepSlots);
      mbar_wait(&slot_empty[s], ((k / kStepSlots) & 1u) ^ 1u);
      StepSlot& sl = slots[s];
      const int t = step_next_task(hd, cursors, lane, &done_count, k, deferred, n_def);
      __threadfence();                     // acquire side of the arrival counters (relaxed polls above), once per task
      if (t < 0) {
        if (lane == 0) {
          sl.task.type = TASK_STOP;
          mbar_arrive(&slot_full[s]);
        }
        break;
      }
      if (lane < (int)(sizeof(StepTask) / sizeof(int)))
        reinterpret_cast<int*>(&sl.task)[lane] = __ldg(reinterpret_cast<const int*>(hd.tasks + t) + lane);
      __syncwarp();
      const int type = sl.task.type;
      if (type == TASK_GEMM) {
        const StepGroup* sg = hd.groups + sl.task.group;
        for (int i = lane; i < (int)(sizeof(Group) / sizeof(int)); i += 32)
          reinterpret_cast<int*>(&sl.ctx.g)[i] = __ldg(reinterpret_cast<const int*>(&sg->g) + i);
        const int sb = __ldg(&sg->seg_begin), sc = __ldg(&sg->g.seg_count);
        for (int i = lane; i < sc; i += 32) sl.ctx.seg[i] = hd.segs[sb + i];
        __syncwarp();
        if (lane == 0) {
          sl.flags = (__ldg(&sg->a_kmaj) ? 1 : 0) | (__ldg(&sg->b_kmaj) ? 2 : 0) | (__ldg(&sg->pad_flags) << 2);
          int c_begin, n_iter;
          tc_chunk_range(sl.ctx, sl.task.split, &c_begin, &n_iter);
          sl.c_begin = c_begin;
          sl.n_iter = n_iter;
        }
      }
      if (lane == 0) sl.index = t;
      __syncwarp();
      if (lane == 0) mbar_arrive(&slot_full[s]);
    }
  } else if (warp == kStepProducerWarp) {
    // =========================== TMA producer ===========================
    if (lane == 0) {
      uint32_t slabs = 0;
      for (uint32_t k = 0;; ++k) {
        const int s = (int)(k % kStepSlots);
        mbar_wait(&slot_full[s], (k / kStepSlots) & 1u);
        const StepSlot& sl = slots[s];
        const int type = sl.task.type;
        if (type == TASK_STOP) break;
        if (type == TASK_GEMM && sl.n_iter > 0) {
          fence_proxy_async_all();                       // operands written by other SMs' generic stores -> TMA reads
          tc_produce<kStepStages>(sl.ctx, hd.maps, (sl.flags & 1) != 0, (sl.flags & 2) != 0, sl.flags >> 2, sl.task.m0,
                                  sl.task.n0, sl.c_begin, sl.n_iter, smem, &sh, slabs);
          slabs += (uint32_t)sl.n_iter;
        }
        mbar_arrive(&slot_empty[s]);
      }
    }
  } else {
    // =========================== consumer / epilogue / row warps (0..7) ===========================
    const int ew = warp;
    const int rt = tid;
    uint32_t slabs = 0;
    for (uint32_t k = 0;; ++k) {
      const int s = (int)(k % kStepSlots);
      mbar_wait(&slot_full[s], (k / kStepSlots) & 1u);
      const StepSlot& sl = slots[s];
      const int type = sl.task.type;
      if (type == TASK_STOP) break;
      unsigned long long t_sched = 0, t_acc = 0, t_body = 0, t_sync = 0;
      bool publish = true;                 // a split-K tile that was not the last to arrive has nothing to announce
      if (hd.trace && rt == 0) t_sched = global_ns();
      if (type == TASK_GEMM) {
        if (sl.n_iter > 0) {            // (the previous task's readers of acc_tile are past the completion barrier)
          float d[64];
          tc_consume<kStepStages>((sl.flags & 1) != 0, (sl.flags & 2) != 0, sl.n_iter, smem, &sh, slabs, d);
          slabs += (uint32_t)sl.n_iter;
          tc_store_acc(acc_tile, d, tid);
          row_sync();
        }
        if (hd.trace && rt == 0) t_acc = global_ns();
        step_epilogue(s, acc_tile, ew, smem_u32(scratch + ew * TC_EPI_STAGE_FLOATS));
        if (sl.task.mode == TILE_SPLIT) {      // raw partial written: am I the last split of this tile?
          row_sync();
          if (rt == 0) {
            __threadfence();                   // release my partial (cumulative over the CTA: bar above) ...
            const int before = atomicAdd(hd.counters + sl.task.split_counter, 1);
            __threadfence();                   // ... acquire the others'
            split_rank = before;
          }
          row_sync();
          if (split_rank == sl.ctx.g.ksplit - 1) {
            step_reduce(s, ew, smem_u32(scratch + ew * TC_EPI_STAGE_FLOATS));
            publish = true;
          } else {
            publish = false;
          }
        }
      } else if (type == TASK_FRAME) {
        frame_task(sl.task.m0, sl.task.n0, rt);
      } else if (type == TASK_ROW) {
        video_row_task(sl.task.mode, sl.task.m0, sl.task.n0, rt);
      } else if (type == TASK_COLSUM_PART || type == TASK_COLSUM_REDUCE) {
        for (int i = rt; i < (int)(sizeof(WColsumJob) / sizeof(int)); i += kRowThreads)
          reinterpret_cast<int*>(&g_job)[i] = __ldg(reinterpret_cast<const int*>(hd.jobs + sl.task.group) + i);
        row_sync();
        if (type == TASK_COLSUM_PART)
          colsum_part_task(scratch, sl.task.m0, sl.task.n0, rt);
        else
          colsum_reduce_task(rt);
      } else if (type == TASK_FINISH) {
        if (rt == 0 && hd.step_counter) hd.step_counter[0] += 1ull;
      }
      if (hd.trace && rt == 0) t_body = global_ns();
      // ---- completion: every store of the task issued -> release its arrival counters ----
      const int sig = sl.task.signal, sig2 = sl.task.signal2, index = sl.index;
      const unsigned long long tag = ((unsigned long long)type << 16) | ((unsigned long long)(unsigned)sl.task.group << 24) |
                                     ((unsigned long long)sl.task.mode << 48) | ((unsigned long long)(unsigned)sl.n_iter << 52);
      row_sync();                        // every warp's stores are issued (CTA-scope order) ...
      if (hd.trace && rt == 0) t_sync = global_ns();
      if (rt == 0) {
        if (publish && (sig >= 0 || sig2 >= 0)) {
          __threadfence();               // ... one cumulative gpu-scope fence publishes them with the release below
          fence_proxy_async_all();
          if (sig >= 0) red_release(hd.counters + sig, 1);
          if (sig2 >= 0) red_release(hd.counters + sig2, 1);
        }
        *reinterpret_cast<volatile int*>(&done_count) = (int)(k + 1);
        if (hd.trace) {
          unsigned long long* tr = hd.trace + (size_t)index * 8;
          tr[0] = (unsigned long long)sm_id() | tag;
          tr[1] = t_sched;
          tr[2] = t_acc;
          tr[3] = global_ns();
          tr[4] = t_body;
          tr[5] = t_sync;
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&slot_empty[s]);
    }
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
