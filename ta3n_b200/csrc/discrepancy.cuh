// discrepancy.cuh -- discrepancy-based alignment, dis_DA 'DAN' / 'JAN' (main.py:455-505; loss.py:46-120).
//
// Per level (DAN) or for the joint pair of layers (JAN), over the 2s rows cat(source[:s], target[:s]) of a chunk:
//   L2_ij = sum_d (x_id - x_jd)^2                      direct differences, so the diagonal is exactly 0
//   bw    = sum L2 / ((2s)^2 - 2s) / mul^(num/2)        (detached: no gradient through it)
//   K_ij  = sum_{k<num} exp(-L2_ij / (bw mul^k))        JAN: K = K_0 (.) K_1, each layer with its own bw
//   loss  = mean over the s x s blocks of XX + YY - XY - YX = 1/s^2 sum_ij sgn_i sgn_j K_ij
// and the gradient of alpha * (level mean over chunks), through G_ij = d(alpha loss)/dL2_ij (symmetric):
//   dx_i = 4 sum_j G_ij (x_i - x_j)
// Three launches, sized for the buffers' row capacity; every block reads the real-row pair from the device and
// exits when its tile lies outside this batch's chunks, so the sequence is graph-capturable and needs no host sync.
// Both passes over a feature / row dimension stage 64-wide slices through shared memory and load the next slice into
// registers while the current one is consumed, so that the global-load latency overlaps the arithmetic.
//   dis_dist_kernel   L2 tiles (32 x 32, shared-memory staged) on and above the diagonal, each also stored
//                     transposed, + each tile's fp64 sum (twice that for a tile off the diagonal)
//   dis_coef_kernel   bandwidth (fixed-order fp64 sum of the tile sums), K, the loss tile sums (fp64), G over L2
//   dis_grad_kernel   dx rows (32 rows x 32 features per block), and block (0,0,0) folds the loss sums
// No float atomics: every sum has a fixed order, so replays are bit-identical.
#pragma once

#include "common.cuh"

namespace ta3n {

constexpr int kDisTile = 32;
constexpr int kDisThreads = 256;
constexpr int kDisChunk = 256;      // main.py:487: DAN cuts the rows into chunks of at most 256 per domain
constexpr int kDisK = 64;           // features (distance pass) / rows j (gradient pass) per shared-memory stage
constexpr int kDisLoads = kDisTile * kDisK / kDisThreads;     // values each thread stages per operand and stage

struct DisLayer {
  const float* xs;      // [>= s rows, d] source rows (nullptr: layer off)
  const float* xt;      // [>= s rows, d] target rows
  float* gs;            // gradient rows of xs / xt (same layout)
  float* gt;
  int d, num;
  float mul;
  int store;            // 1: the gradient is written, rows outside the chunks zeroed; 0: added
};

struct DisArgs {
  DisLayer layer[2];
  int joint;            // one chunk, K = the product of the layers' kernels (JAN; one layer: mmd_rbf unchunked)
  int Bs, Bt;           // row capacity of the source / target buffers
  int cap;              // rows per domain of one chunk at most
  int max_chunks;
  int ntile;            // tiles per side of a chunk matrix: ceil(2 cap / 32)
  const int* valid;     // {real source rows, real target rows} or nullptr (all rows real)
  const float* alpha;   // weight of the term in *loss (device) or nullptr (1)
  float* loss;          // += alpha * loss_d
  float* loss_d;        // = loss_d
  double* meter;        // optional {sum of loss_d * real source rows, last loss_d, sum of real source rows}
  float* mats;          // [2][max_chunks][2 cap][2 cap]: L2, overwritten by G
  double* l2_part;      // [2][max_chunks][ntile^2]
  double* loss_part;    // [2][max_chunks][ntile^2]
};

struct DisLive {
  int vs, s, nch;       // real source rows; rows per domain of a chunk; chunks (0: the term is 0 this batch)
};

__device__ __forceinline__ DisLive dis_live(const DisArgs& a) {
  const int vs = a.valid ? max(0, min(a.valid[0], a.Bs)) : a.Bs;
  const int vt = a.valid ? max(0, min(a.valid[1], a.Bt)) : a.Bt;
  const int n = min(vs, vt);
  DisLive v{vs, n, n > 0 ? 1 : 0};
  if (!a.joint && n > kDisChunk) {
    // a size above 256 that 256 does not divide has no chunking in the reference (its view() fails): contributes 0
    v.s = kDisChunk;
    v.nch = n % kDisChunk ? 0 : n / kDisChunk;
  }
  return v;
}

// row i of chunk c's matrix: source row c s + i for i < s, else target row c s + i - s
template <typename T>
__device__ __forceinline__ T* dis_row(T* xs, T* xt, int d, int c, int s, int i) {
  return i < s ? xs + (size_t)(c * s + i) * d : xt + (size_t)(c * s + i - s) * d;
}

// layer l by value, selected without indexing the parameter array dynamically (that copies it to local memory)
__device__ __forceinline__ DisLayer dis_layer(const DisArgs& a, int l) { return l ? a.layer[1] : a.layer[0]; }

__device__ __forceinline__ size_t dis_mat_stride(const DisArgs& a) { return (size_t)(2 * a.cap) * (2 * a.cap); }

// fixed-order block sum (kDisThreads threads); every thread gets the total
__device__ __forceinline__ double dis_block_sum(double v, double* red) {
  red[threadIdx.x] = v;
  __syncthreads();
#pragma unroll
  for (int o = kDisThreads / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  const double t = red[0];
  __syncthreads();
  return t;
}

// grid (ntile, ntile, 2 max_chunks): tile (y, x) of layer z / max_chunks, chunk z % max_chunks; blocks with y > x only
// take their share of the zeroing
__global__ void __launch_bounds__(kDisThreads) dis_dist_kernel(DisArgs a) {
  pdl_wait();
  __shared__ float A[kDisTile][kDisK + 1], B[kDisTile][kDisK + 1];
  __shared__ double red[kDisThreads];
  const DisLive v = dis_live(a);
  const int l = blockIdx.z / a.max_chunks, c = blockIdx.z % a.max_chunks;
  const DisLayer L = dis_layer(a, l);
  if (!L.xs) return;
  if (L.store) {
    // rows past the chunks carry no gradient this batch: zero them, spread over this layer's blocks
    const size_t nu = (size_t)v.nch * v.s;
    const size_t ns = ((size_t)a.Bs - nu) * L.d, nt = ((size_t)a.Bt - nu) * L.d;
    const size_t nb = (size_t)gridDim.x * gridDim.y * a.max_chunks;
    const size_t b = ((size_t)c * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
    for (size_t e = b * kDisThreads + threadIdx.x; e < ns + nt; e += nb * kDisThreads) {
      if (e < ns) L.gs[nu * L.d + e] = 0.f;
      else L.gt[nu * L.d + (e - ns)] = 0.f;
    }
  }
  const int m = 2 * v.s;
  const int i0 = blockIdx.y * kDisTile, j0 = blockIdx.x * kDisTile;
  if (c >= v.nch || i0 >= m || j0 >= m || i0 > j0) return;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  float acc[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
  float ra[kDisLoads], rb[kDisLoads];
  auto load = [&](int k0) {
#pragma unroll
    for (int u = 0; u < kDisLoads; ++u) {
      const int e = threadIdx.x + u * kDisThreads, r = e / kDisK, k = e % kDisK;
      const bool kin = k0 + k < L.d;
      ra[u] = (kin && i0 + r < m) ? dis_row(L.xs, L.xt, L.d, c, v.s, i0 + r)[k0 + k] : 0.f;
      rb[u] = (kin && j0 + r < m) ? dis_row(L.xs, L.xt, L.d, c, v.s, j0 + r)[k0 + k] : 0.f;
    }
  };
  load(0);
  for (int k0 = 0; k0 < L.d; k0 += kDisK) {
#pragma unroll
    for (int u = 0; u < kDisLoads; ++u) {
      const int e = threadIdx.x + u * kDisThreads;
      A[e / kDisK][e % kDisK] = ra[u];
      B[e / kDisK][e % kDisK] = rb[u];
    }
    __syncthreads();
    if (k0 + kDisK < L.d) load(k0 + kDisK);
    const int kn = min(kDisK, L.d - k0);
    for (int k = 0; k < kn; ++k) {
      const float a0 = A[ty][k], a1 = A[ty + 16][k], b0 = B[tx][k], b1 = B[tx + 16][k];
      float t;
      // (x_i - x_j)^2 == (x_j - x_i)^2 in the same k order: L2 is bitwise symmetric
      t = a0 - b0; acc[0][0] = fmaf(t, t, acc[0][0]);
      t = a0 - b1; acc[0][1] = fmaf(t, t, acc[0][1]);
      t = a1 - b0; acc[1][0] = fmaf(t, t, acc[1][0]);
      t = a1 - b1; acc[1][1] = fmaf(t, t, acc[1][1]);
    }
    __syncthreads();
  }
  float* mat = a.mats + (size_t)blockIdx.z * dis_mat_stride(a);
  const int ld = 2 * a.cap;
  double part = 0.0;
#pragma unroll
  for (int p = 0; p < 2; ++p)
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int i = i0 + ty + 16 * p, j = j0 + tx + 16 * q;
      A[ty + 16 * p][tx + 16 * q] = acc[p][q];
      if (i < m && j < m) {
        mat[(size_t)i * ld + j] = acc[p][q];
        part += (double)acc[p][q];
      }
    }
  if (i0 != j0) {
    // the mirror tile L2_ji = L2_ij (the same bits), written row by row from shared memory
    __syncthreads();
    for (int e = threadIdx.x; e < kDisTile * kDisTile; e += kDisThreads) {
      const int r = e / kDisTile, q = e % kDisTile;
      if (j0 + r < m && i0 + q < m) mat[(size_t)(j0 + r) * ld + i0 + q] = A[q][r];
    }
    part *= 2.0;
  }
  part = dis_block_sum(part, red);
  if (threadIdx.x == 0) a.l2_part[(size_t)blockIdx.z * a.ntile * a.ntile + blockIdx.y * a.ntile + blockIdx.x] = part;
}

// bandwidths of the reference's guassian_kernel (fp32 after the sum, as torch computes them): bw_k = bw mul^k
__device__ __forceinline__ float dis_bandwidth(const DisArgs& a, int z, int m, double* red) {
  const int ntl = (m + kDisTile - 1) / kDisTile;
  const double* part = a.l2_part + (size_t)z * a.ntile * a.ntile;
  double t = 0.0;
  for (int e = threadIdx.x; e < ntl * ntl; e += kDisThreads)
    if (e / ntl <= e % ntl) t += part[(e / ntl) * a.ntile + e % ntl];      // tiles on and above the diagonal
  t = dis_block_sum(t, red);
  return (float)(t / ((double)m * m - m));
}

struct DisKernelSum {
  float k, dk;          // sum_k exp(-L2 / bw_k) and its derivative in L2
};

__device__ __forceinline__ DisKernelSum dis_kernel_sum(float l2, float bw, int num, float mul) {
  DisKernelSum r{0.f, 0.f};
  float bk = bw;
  for (int k = 0; k < num; ++k) {
    const float e = expf(-l2 / bk);
    r.k += e;
    r.dk -= e / bk;
    bk *= mul;
  }
  return r;
}

// grid (ntile, ntile, joint ? 1 : 2 max_chunks).  DAN: one layer per block; joint: the product over the layers that
// are on (one layer alone is plain mmd_rbf without chunks); an absent layer's factor is exactly 1.
__global__ void __launch_bounds__(kDisThreads) dis_coef_kernel(DisArgs a) {
  pdl_wait();
  __shared__ double red[kDisThreads];
  const DisLive v = dis_live(a);
  const int l = a.joint ? 0 : blockIdx.z / a.max_chunks, c = a.joint ? 0 : blockIdx.z % a.max_chunks;
  const bool on[2] = {a.layer[0].xs && (a.joint || l == 0), a.layer[1].xs && (a.joint || l == 1)};
  if (!on[0] && !on[1]) return;
  const int m = 2 * v.s;
  const int i0 = blockIdx.y * kDisTile, j0 = blockIdx.x * kDisTile;
  if (c >= v.nch || i0 >= m || j0 >= m) return;
  float bw[2] = {0.f, 0.f};
  float* mat[2];
#pragma unroll
  for (int q = 0; q < 2; ++q) {
    mat[q] = a.mats + (size_t)(q * a.max_chunks + c) * dis_mat_stride(a);
    if (!on[q]) continue;
    // bw /= mul^(num // 2) (loss.py:57); mul^k by repeated products, as Python's float power of a small integer
    const float b = dis_bandwidth(a, q * a.max_chunks + c, m, red);
    float p = 1.f;
    for (int k = 0; k < a.layer[q].num / 2; ++k) p *= a.layer[q].mul;
    bw[q] = b / p;
  }
  const float al = a.alpha ? *a.alpha : 1.f;
  const float coef = (float)((double)al / ((double)v.nch * v.s * v.s));
  const int ld = 2 * a.cap;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  double part = 0.0;
#pragma unroll
  for (int p = 0; p < 2; ++p)
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int i = i0 + ty + 16 * p, j = j0 + tx + 16 * q;
      if (i >= m || j >= m) continue;
      const size_t o = (size_t)i * ld + j;
      const float sg = ((i < v.s) == (j < v.s)) ? 1.f : -1.f;
      DisKernelSum k0{1.f, 0.f}, k1{1.f, 0.f};
      if (on[0]) k0 = dis_kernel_sum(mat[0][o], bw[0], a.layer[0].num, a.layer[0].mul);
      if (on[1]) k1 = dis_kernel_sum(mat[1][o], bw[1], a.layer[1].num, a.layer[1].mul);
      part += (double)(sg * (k0.k * k1.k));
      if (on[0]) mat[0][o] = coef * sg * (k0.dk * k1.k);
      if (on[1]) mat[1][o] = coef * sg * (k0.k * k1.dk);
    }
  part = dis_block_sum(part, red);
  if (threadIdx.x == 0)
    a.loss_part[(size_t)blockIdx.z * a.ntile * a.ntile + blockIdx.y * a.ntile + blockIdx.x] = part;
}

// loss_d = sum over levels of (mean over chunks of 1/s^2 sum of the tile sums); one block, fixed order
__device__ void dis_finish(const DisArgs& a, const DisLive& v, double* red) {
  double tot = 0.0;
  const int m = 2 * v.s, ntl = (m + kDisTile - 1) / kDisTile;
  for (int l = 0; l < (a.joint ? 1 : 2); ++l) {
    if (!a.joint && !a.layer[l].xs) continue;
    double lv = 0.0;
    for (int c = 0; c < v.nch; ++c) {
      const double* part = a.loss_part + (size_t)(l * a.max_chunks + c) * a.ntile * a.ntile;
      double t = 0.0;
      for (int e = threadIdx.x; e < ntl * ntl; e += kDisThreads) t += part[(e / ntl) * a.ntile + e % ntl];
      lv += dis_block_sum(t, red) / ((double)v.s * v.s);
    }
    if (v.nch > 0) tot += lv / v.nch;
  }
  if (threadIdx.x == 0) {
    const float ld = (float)tot;
    if (v.nch > 0) a.loss[0] += (a.alpha ? *a.alpha : 1.f) * ld;
    a.loss_d[0] = ld;
    if (a.meter) {
      a.meter[0] += (double)ld * v.vs;
      a.meter[1] = (double)ld;
      a.meter[2] += (double)v.vs;
    }
  }
}

// grid (ceil(max d / 32), ntile, 2 max_chunks): rows [32 y, +32) of chunk z % max_chunks of layer z / max_chunks,
// features [32 x, +32)
__global__ void __launch_bounds__(kDisThreads) dis_grad_kernel(DisArgs a) {
  pdl_wait();
  __shared__ float Gs[kDisTile][kDisK + 1], Xj[kDisK][kDisTile + 1];
  __shared__ double red[kDisThreads];
  const DisLive v = dis_live(a);
  if (blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0) dis_finish(a, v, red);
  const int l = blockIdx.z / a.max_chunks, c = blockIdx.z % a.max_chunks;
  const DisLayer L = dis_layer(a, l);
  const int m = 2 * v.s;
  const int i0 = blockIdx.y * kDisTile, e0 = blockIdx.x * kDisTile;
  if (!L.xs || c >= v.nch || i0 >= m || e0 >= L.d) return;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const float* G = a.mats + (size_t)blockIdx.z * dis_mat_stride(a);
  const int ld = 2 * a.cap;
  float xi[2][2], acc[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
#pragma unroll
  for (int p = 0; p < 2; ++p)
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int i = i0 + ty + 16 * p, e = e0 + tx + 16 * q;
      xi[p][q] = (i < m && e < L.d) ? dis_row(L.xs, L.xt, L.d, c, v.s, i)[e] : 0.f;
    }
  float rg[kDisLoads], rx[kDisLoads];
  auto load = [&](int j0) {
#pragma unroll
    for (int u = 0; u < kDisLoads; ++u) {
      const int t = threadIdx.x + u * kDisThreads;
      const int r = t / kDisK, q = t % kDisK;                   // G rows i0 + r, columns j0 + q
      rg[u] = (i0 + r < m && j0 + q < m) ? G[(size_t)(i0 + r) * ld + j0 + q] : 0.f;
      const int rj = t / kDisTile, f = t % kDisTile;            // x rows j0 + rj, features e0 + f
      rx[u] = (j0 + rj < m && e0 + f < L.d) ? dis_row(L.xs, L.xt, L.d, c, v.s, j0 + rj)[e0 + f] : 0.f;
    }
  };
  load(0);
  for (int j0 = 0; j0 < m; j0 += kDisK) {
#pragma unroll
    for (int u = 0; u < kDisLoads; ++u) {
      const int t = threadIdx.x + u * kDisThreads;
      Gs[t / kDisK][t % kDisK] = rg[u];
      Xj[t / kDisTile][t % kDisTile] = rx[u];
    }
    __syncthreads();
    if (j0 + kDisK < m) load(j0 + kDisK);
    const int jn = min(kDisK, m - j0);
    for (int j = 0; j < jn; ++j) {
      const float g0 = Gs[ty][j], g1 = Gs[ty + 16][j], x0 = Xj[j][tx], x1 = Xj[j][tx + 16];
      acc[0][0] = fmaf(g0, xi[0][0] - x0, acc[0][0]);
      acc[0][1] = fmaf(g0, xi[0][1] - x1, acc[0][1]);
      acc[1][0] = fmaf(g1, xi[1][0] - x0, acc[1][0]);
      acc[1][1] = fmaf(g1, xi[1][1] - x1, acc[1][1]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int p = 0; p < 2; ++p)
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int i = i0 + ty + 16 * p, e = e0 + tx + 16 * q;
      if (i >= m || e >= L.d) continue;
      float* g = dis_row(L.gs, L.gt, L.d, c, v.s, i) + e;
      *g = L.store ? 4.f * acc[p][q] : *g + 4.f * acc[p][q];
    }
}

// host: buffer geometry for the row capacity (Bs, Bt); the workspace is the matrices then the two partial arrays
struct DisGeom {
  int cap, max_chunks, ntile;
  size_t mats, parts;     // floats of the matrices, doubles of one partial array
};

inline DisGeom dis_geom(int Bs, int Bt, int joint) {
  DisGeom g;
  const int nmin = std::min(Bs, Bt);
  g.cap = joint ? nmin : std::min(nmin, kDisChunk);
  g.max_chunks = (!joint && nmin > kDisChunk) ? nmin / kDisChunk : 1;
  g.ntile = (2 * g.cap + kDisTile - 1) / kDisTile;
  g.mats = (size_t)2 * g.max_chunks * (size_t)(2 * g.cap) * (2 * g.cap);
  g.parts = (size_t)2 * g.max_chunks * g.ntile * g.ntile;
  return g;
}

inline size_t dis_bytes(const DisGeom& g) {
  return ((g.mats * sizeof(float) + 255) / 256) * 256 + 2 * ((g.parts * sizeof(double) + 255) / 256) * 256;
}

}  // namespace ta3n
