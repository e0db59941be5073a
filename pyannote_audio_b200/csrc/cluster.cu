// Clustering on the device, fp64 like the reference (numpy/scipy promote to double):
//   * centroid-linkage agglomerative clustering  = scipy.cluster.hierarchy.linkage(X, "centroid", "euclidean")
//       call sites /root/reference/src/pyannote/audio/pipelines/clustering.py:597-603 (VBx) and :371-385 (AHC)
//   * fcluster(Z, t, criterion="distance")        (host, tree walk)      clustering.py:604, 385
//   * cdist(., ., "cosine")                       clustering.py:645-655
//   * VBx variational iterations                  utils/vbx.py:98-136 (called from clustering.py:608-616)
//   * constrained_argmax (3 x K assignment)       clustering.py:127-140
// Arithmetic that decides merges uses explicit round-to-nearest mul/add (no FMA contraction) in the same operation
// order as scipy's C code so that dendrogram heights agree to the last bit on ordinary inputs.
#include "../../include/b200diar.h"
#include "common.cuh"
#include "cluster.cuh"
#include <cfloat>
#include <algorithm>
#include <cmath>
#include <cooperative_groups.h>

namespace cg = cooperative_groups;

namespace b200 {

// ------------------------------------------------------------------------------------------------------
// pairwise Euclidean distances (full symmetric matrix with unused diagonal, or scipy's condensed triangle)
// ------------------------------------------------------------------------------------------------------
__global__ void normalize_rows_kernel(const double* __restrict__ x, double* __restrict__ y, int n, int dim) {
  const int i = blockIdx.x;
  __shared__ double red[32];
  double s = 0.0;
  for (int d = threadIdx.x; d < dim; d += blockDim.x) s += x[(size_t)i * dim + d] * x[(size_t)i * dim + d];
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < (blockDim.x + 31) / 32; ++w) t += red[w];
    red[0] = sqrt(t);
  }
  __syncthreads();
  const double nrm = red[0];
  for (int d = threadIdx.x; d < dim; d += blockDim.x) y[(size_t)i * dim + d] = x[(size_t)i * dim + d] / nrm;
}

// numpy's float32 `add.reduce` along a contiguous axis (pairwise summation, numpy/_core/src/umath/loops_utils.h.src):
// blocks of <= 128 elements are summed with 8 interleaved accumulators combined as ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)),
// longer runs are split in halves (rounded down to a multiple of 8) recursively.  Elements here are float(x[i])^2.
__device__ float np_pairwise_sumsq_f32(const double* __restrict__ x, int n) {
  if (n < 8) {
    float res = 0.f;
    for (int i = 0; i < n; ++i) { const float v = (float)x[i]; res = __fadd_rn(res, __fmul_rn(v, v)); }
    return res;
  }
  if (n <= 128) {
    float r[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { const float v = (float)x[j]; r[j] = __fmul_rn(v, v); }
    int i = 8;
    for (; i < n - (n % 8); i += 8) {
#pragma unroll
      for (int j = 0; j < 8; ++j) { const float v = (float)x[i + j]; r[j] = __fadd_rn(r[j], __fmul_rn(v, v)); }
    }
    float res = __fadd_rn(__fadd_rn(__fadd_rn(r[0], r[1]), __fadd_rn(r[2], r[3])),
                          __fadd_rn(__fadd_rn(r[4], r[5]), __fadd_rn(r[6], r[7])));
    for (; i < n; ++i) { const float v = (float)x[i]; res = __fadd_rn(res, __fmul_rn(v, v)); }
    return res;
  }
  int n2 = n / 2;
  n2 -= n2 % 8;
  return __fadd_rn(np_pairwise_sumsq_f32(x, n2), np_pairwise_sumsq_f32(x + n2, n - n2));
}

// rows holding float32 values (embeddings come out of the network as float32): exactly
//   x / np.linalg.norm(x, axis=1, keepdims=True)   in float32, as the reference computes it (pipelines/clustering.py:
// 597-599, 371-373 on float32 embeddings), then widened to the fp64 the linkage works in
__global__ void normalize_rows_np_f32_kernel(const double* __restrict__ x, double* __restrict__ y, int n, int dim) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double* r = x + (size_t)i * dim;
  const float nrm = __fsqrt_rn(np_pairwise_sumsq_f32(r, dim));
  for (int d = 0; d < dim; ++d) y[(size_t)i * dim + d] = (double)__fdiv_rn((float)r[d], nrm);
}

// packed row k of scipy's condensed distance vector (upper triangle, row-major): element j > k is row[j], with
// 64-bit offsets (the condensed index passes 2^31 at n ~ 65k)
__host__ __device__ __forceinline__ long long packed_row(int k, int n) {
  return (long long)k * n - (long long)k * (k + 1) / 2 - k - 1;
}

// kPacked = false: full symmetric n x n matrix, diagonal DBL_MAX; true: condensed upper triangle (scipy's pdist
// layout, n (n - 1) / 2 values).  The per-pair arithmetic is the same code for both layouts.
template <bool kPacked>
__global__ void pdist_kernel(const double* __restrict__ x, double* __restrict__ D, int n, int dim) {
  if (kPacked && blockIdx.x < blockIdx.y) return;          // tile entirely below the diagonal
  // 16x16 tile of pairs per block, operands staged through shared memory in chunks of 32 dims
  __shared__ double xi[16][33], xj[16][33];
  const int i = blockIdx.y * 16 + threadIdx.y, j = blockIdx.x * 16 + threadIdx.x;
  double s = 0.0;
  for (int d0 = 0; d0 < dim; d0 += 32) {
    const int tid = threadIdx.y * 16 + threadIdx.x;
    for (int e = tid; e < 16 * 32; e += 256) {
      const int r = e >> 5, c = e & 31;
      const int gi = blockIdx.y * 16 + r, gj = blockIdx.x * 16 + r;
      xi[r][c] = (gi < n && d0 + c < dim) ? x[(size_t)gi * dim + d0 + c] : 0.0;
      xj[r][c] = (gj < n && d0 + c < dim) ? x[(size_t)gj * dim + d0 + c] : 0.0;
    }
    __syncthreads();
#pragma unroll
    for (int c = 0; c < 32; ++c) {
      const double df = __dsub_rn(xi[threadIdx.y][c], xj[threadIdx.x][c]);
      s = __dadd_rn(s, __dmul_rn(df, df));
    }
    __syncthreads();
  }
  if (kPacked) {
    if (i < j && j < n) D[packed_row(i, n) + j] = sqrt(s);
  } else {
    if (i < n && j < n) D[(size_t)i * n + j] = (i == j) ? DBL_MAX : sqrt(s);
  }
}

// ------------------------------------------------------------------------------------------------------
// centroid linkage: single persistent CTA, nearest-neighbour candidates per row (upper triangle)
// ------------------------------------------------------------------------------------------------------
__device__ __forceinline__ double lw_centroid(double dxi, double dyi, double dxy, double nx, double ny) {
  // scipy/_hierarchy_distance_update.pxi::_centroid
  //   sqrt((((nx*dxi*dxi) + (ny*dyi*dyi)) - (nx*ny*dxy*dxy)/(nx+ny)) / (nx+ny))
  const double a = __dmul_rn(__dmul_rn(nx, dxi), dxi);
  const double b = __dmul_rn(__dmul_rn(ny, dyi), dyi);
  const double c = __ddiv_rn(__dmul_rn(__dmul_rn(__dmul_rn(nx, ny), dxy), dxy), __dadd_rn(nx, ny));
  return sqrt(__ddiv_rn(__dsub_rn(__dadd_rn(a, b), c), __dadd_rn(nx, ny)));
}

struct MinPair {
  double v;
  int i;
};
__device__ __forceinline__ MinPair min_pair(MinPair a, MinPair b) {
  if (b.v < a.v || (b.v == a.v && b.i < a.i)) return b;
  return a;
}
__device__ __forceinline__ MinPair warp_min(MinPair m) {
  for (int o = 16; o > 0; o >>= 1) {
    MinPair t;
    t.v = __shfl_xor_sync(0xffffffffu, m.v, o);
    t.i = __shfl_xor_sync(0xffffffffu, m.i, o);
    m = min_pair(m, t);
  }
  return m;
}

// nearest alive j > k of row k among the columns j = k + 1 + first, + stride, ...  (four independent loads in flight
// per thread); min_pair is an order-independent (value, index) minimum, so any split of a row gives the same answer.
// row[j] is d(k, j).  kL2: load through L2 only (the grid-wide kernel reads values other CTAs have just written).
template <bool kL2 = false>
__device__ __forceinline__ MinPair row_nn_part(const double* __restrict__ row, const unsigned char* alive, int n, int k,
                                               int first, int stride) {
  auto ld = [&](int j) { return kL2 ? __ldcg(row + j) : row[j]; };
  MinPair m{DBL_MAX, n};
  int j = k + 1 + first;
  for (; j + 3 * stride < n; j += 4 * stride) {
    const double v0 = ld(j), v1 = ld(j + stride), v2 = ld(j + 2 * stride), v3 = ld(j + 3 * stride);
    if (alive[j]) m = min_pair(m, MinPair{v0, j});
    if (alive[j + stride]) m = min_pair(m, MinPair{v1, j + stride});
    if (alive[j + 2 * stride]) m = min_pair(m, MinPair{v2, j + 2 * stride});
    if (alive[j + 3 * stride]) m = min_pair(m, MinPair{v3, j + 3 * stride});
  }
  for (; j < n; j += stride)
    if (alive[j]) m = min_pair(m, MinPair{ld(j), j});
  return m;
}

// nearest alive j > k of row k, computed by one warp
__device__ __forceinline__ void row_nn(const double* __restrict__ D, const unsigned char* alive, int n, int k, int lane,
                                       double* nn_d, int* nn_i) {
  const MinPair m = warp_min(row_nn_part(D + (size_t)k * n, alive, n, k, lane, 32));
  if (lane == 0) { nn_d[k] = m.v; nn_i[k] = m.i; }
}

struct LinkJob {
  int n;
  int row_off;        // offset of this problem in the per-row arrays
  int z_off;          // row offset into Z
  int pad;
  long long d_off;    // element offset of this problem's n x n distance matrix
};

constexpr int kLinkSmemRows = 4096;   // per-row state lives in shared memory up to this many rows

// one CTA per clustering problem (file): problems are independent, so a batch of files fills the machine.
// Per merge: (A) block-wide argmin over the nearest-neighbour candidates, (B) one fused pass that applies the
// Lance-Williams update to row/column y, maintains the candidates of the rows k < y and collects the new nearest
// neighbour of y from the values it has just computed (no re-scan of row y), (C) re-scan of the few rows whose
// candidate was x or y.  Arithmetic and tie rules are unchanged, so dendrograms still match scipy bit for bit.
__global__ void __launch_bounds__(1024) linkage_centroid_kernel(const LinkJob* __restrict__ jobs,
                                                                double* __restrict__ Dall, double* __restrict__ Zall,
                                                                double* __restrict__ nn_d_all,
                                                                int* __restrict__ nn_i_all, int* __restrict__ size_all,
                                                                int* __restrict__ id_all,
                                                                unsigned char* __restrict__ alive_all,
                                                                int* __restrict__ todo_all) {
  extern __shared__ unsigned char link_smem[];
  const LinkJob job = jobs[blockIdx.x];
  const int n = job.n;
  if (n < 2) return;
  double* __restrict__ D = Dall + job.d_off;
  double* __restrict__ Z = Zall + (size_t)job.z_off * 4;
  int* __restrict__ id = id_all + job.row_off;
  int* __restrict__ todo = todo_all + job.row_off + blockIdx.x;     // n + 1 entries per problem
  double* nn_d;
  int* nn_i;
  int* size;
  unsigned char* alive;
  if (n <= kLinkSmemRows) {            // generic pointers: shared or global
    nn_d = reinterpret_cast<double*>(link_smem);
    nn_i = reinterpret_cast<int*>(link_smem + (size_t)kLinkSmemRows * 8);
    size = reinterpret_cast<int*>(link_smem + (size_t)kLinkSmemRows * 12);
    alive = link_smem + (size_t)kLinkSmemRows * 16;
  } else {
    nn_d = nn_d_all + job.row_off;
    nn_i = nn_i_all + job.row_off;
    size = size_all + job.row_off;
    alive = alive_all + job.row_off;
  }
  __shared__ MinPair s_red[32];
  __shared__ int s_x, s_y, s_ntodo;
  __shared__ double s_dxy;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = tid; i < n; i += 1024) { size[i] = 1; id[i] = i; alive[i] = 1; }
  __syncthreads();
  for (int k = warp; k < n; k += 32) row_nn(D, alive, n, k, lane, nn_d, nn_i);
  __syncthreads();

  for (int m = 0; m < n - 1; ++m) {
    // A. global closest pair
    MinPair best{DBL_MAX, n};
    for (int i = tid; i < n; i += 1024)
      if (alive[i] && nn_i[i] < n) best = min_pair(best, MinPair{nn_d[i], i});
    best = warp_min(best);
    if (lane == 0) s_red[warp] = best;
    __syncthreads();
    if (warp == 0) {
      MinPair b = s_red[lane];
      b = warp_min(b);
      if (lane == 0) {
        s_x = b.i;
        s_y = nn_i[b.i];
        s_dxy = b.v;
        s_ntodo = 0;
      }
    }
    __syncthreads();
    const int x = s_x, y = s_y;                            // x < y: candidates only look right
    const double dxy = s_dxy;
    const double nx = size[x], ny = size[y];
    if (tid == 0) {
      const int ia = id[x], ib = id[y];
      Z[m * 4 + 0] = ia < ib ? ia : ib;
      Z[m * 4 + 1] = ia < ib ? ib : ia;
      Z[m * 4 + 2] = dxy;
      Z[m * 4 + 3] = nx + ny;
    }
    // B. Lance-Williams update (merged cluster lives in slot y, slot x dies) + candidate maintenance
    const double* rx = D + (size_t)x * n;
    double* ry = D + (size_t)y * n;
    MinPair ybest{DBL_MAX, n};
    for (int k = tid; k < n; k += 1024) {
      if (!alive[k] || k == x || k == y) continue;
      const double dn = lw_centroid(rx[k], ry[k], dxy, nx, ny);
      ry[k] = dn;
      D[(size_t)k * n + y] = dn;
      if (k > y) {
        ybest = min_pair(ybest, MinPair{dn, k});           // new nearest neighbour of y among j > y
      } else {
        const int cur = nn_i[k];
        if (cur == x || cur == y) {
          todo[atomicAdd(&s_ntodo, 1)] = k;                // its candidate vanished or changed: re-scan
        } else if (dn < nn_d[k] || (dn == nn_d[k] && y < cur)) {
          nn_d[k] = dn;
          nn_i[k] = y;
        }
      }
    }
    ybest = warp_min(ybest);
    __syncthreads();                                       // s_red free again, all reads of size/id done
    if (lane == 0) s_red[warp] = ybest;
    __syncthreads();
    if (warp == 0) {
      MinPair b = warp_min(s_red[lane]);
      if (lane == 0) {
        nn_d[y] = b.v;
        nn_i[y] = b.i;
        alive[x] = 0;
        size[y] = (int)(nx + ny);
        id[y] = n + m;
      }
    }
    __syncthreads();
    // C. rows whose candidate was x or y are re-scanned.  Usually a handful: R rows at a time share the block's 32
    // warps (W = 32 / R warps per row, every load of a row in flight at once) instead of one warp walking a whole
    // row through ~n / 128 dependent round trips to L2, which was most of a merge's latency
    const int nt = s_ntodo;
    if (nt > 0) {
      int R = 1;
      while (R < nt && R < 32) R <<= 1;                    // rows per pass, a power of two <= 32
      const int W = 32 / R, g = warp / W, wl = warp % W;
      for (int t0 = 0; t0 < nt; t0 += R) {
        const int t = t0 + g;
        const int k = t < nt ? todo[t] : -1;
        MinPair part{DBL_MAX, n};
        if (k >= 0) part = warp_min(row_nn_part(D + (size_t)k * n, alive, n, k, wl * 32 + lane, W * 32));
        if (W == 1) {
          if (k >= 0 && lane == 0) { nn_d[k] = part.v; nn_i[k] = part.i; }
        } else {
          if (lane == 0) s_red[warp] = part;
          __syncthreads();
          if (wl == 0 && k >= 0) {
            MinPair b = lane < W ? s_red[g * W + lane] : MinPair{DBL_MAX, n};
            b = warp_min(b);
            if (lane == 0) { nn_d[k] = b.v; nn_i[k] = b.i; }
          }
          __syncthreads();                                 // s_red is reused by the next pass / phase A
        }
      }
      __syncthreads();
    }
  }
}

// ------------------------------------------------------------------------------------------------------
// centroid linkage of one large problem on the whole GPU: a cooperative grid over the packed distances
// ------------------------------------------------------------------------------------------------------
constexpr int kLinkGridThreads = 512;        // one CTA per SM; 128 registers a thread keep the merge loop unspilled
constexpr int kLinkGridMaxCtas = 1024;
// scratch after the job table: per-CTA partial minima of phases A and B (2 x kLinkGridMaxCtas) and the re-scan count
constexpr size_t kLinkGridScratch = 2 * kLinkGridMaxCtas * sizeof(MinPair) + 256;

// (value, index) minimum over the CTA, returned to every thread (every warp reduces the warp minima itself)
__device__ __forceinline__ MinPair block_min(MinPair m, MinPair* s_red, int n) {
  constexpr int kWarps = kLinkGridThreads / 32;
  m = warp_min(m);
  __syncthreads();                                         // s_red free again
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = m;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  return warp_min(lane < kWarps ? s_red[lane] : MinPair{DBL_MAX, n});
}

// The merges of linkage_centroid_kernel, each split over every CTA with three grid-wide barriers:
//   (A) per-CTA minima of the nearest-neighbour candidates; after the barrier every CTA reduces the partials to the
//       same closest pair (x, y);
//   (B) the Lance-Williams update of every alive k and the maintenance of the candidates of rows k < y, spread over
//       the grid; per-CTA minima of y's new neighbour among k > y; rows whose candidate was x or y are queued;
//   (C) each queued row is re-scanned by one CTA; CTA 0 installs y's candidate, size and id.
// Every reduction is the order-independent min_pair over the same values, and the arithmetic is lw_centroid, so Z is
// bit-identical to the one-CTA kernel's.  Per-row state lives in global memory; P is the condensed upper triangle.
__global__ void __launch_bounds__(kLinkGridThreads, 1)
linkage_centroid_grid_kernel(double* P, int n, double* Z, double* nn_d, int* nn_i, int* size, int* id,
                             unsigned char* alive, int* todo, int* ntodo, MinPair* part) {
  cg::grid_group grid = cg::this_grid();
  __shared__ MinPair s_red[kLinkGridThreads / 32];
  const int tid = threadIdx.x, lane = tid & 31, nb = gridDim.x;
  const int gtid = blockIdx.x * kLinkGridThreads + tid, gthreads = nb * kLinkGridThreads;
  const int gwarp = gtid >> 5, gwarps = gthreads >> 5;
  for (int i = gtid; i < n; i += gthreads) { size[i] = 1; id[i] = i; alive[i] = 1; }
  grid.sync();
  for (int k = gwarp; k < n; k += gwarps) {
    const MinPair m = warp_min(row_nn_part<true>(P + packed_row(k, n), alive, n, k, lane, 32));
    if (lane == 0) { nn_d[k] = m.v; nn_i[k] = m.i; }
  }
  grid.sync();

  for (int m = 0; m < n - 1; ++m) {
    // A. global closest pair
    MinPair best{DBL_MAX, n};
    for (int i = gtid; i < n; i += gthreads)
      if (alive[i] && nn_i[i] < n) best = min_pair(best, MinPair{nn_d[i], i});
    best = block_min(best, s_red, n);
    if (tid == 0) part[blockIdx.x] = best;
    if (gtid == 0) *ntodo = 0;                             // every read of the previous merge's count is done
    grid.sync();
    MinPair b{DBL_MAX, n};
    for (int c = lane; c < nb; c += 32) b = min_pair(b, part[c]);
    b = warp_min(b);
    const int x = b.i, y = nn_i[x];                        // x < y: candidates only look right
    const double dxy = b.v;
    const double nx = size[x], ny = size[y];
    if (gtid == 0) {
      const int ia = id[x], ib = id[y];
      Z[(size_t)m * 4 + 0] = ia < ib ? ia : ib;
      Z[(size_t)m * 4 + 1] = ia < ib ? ib : ia;
      Z[(size_t)m * 4 + 2] = dxy;
      Z[(size_t)m * 4 + 3] = nx + ny;
      alive[x] = 0;                                        // row x is skipped below by its own thread either way
    }
    // B. Lance-Williams update (merged cluster lives in slot y, slot x dies) + candidate maintenance
    MinPair ybest{DBL_MAX, n};
    for (int k = gtid; k < n; k += gthreads) {
      if (!alive[k] || k == x || k == y) continue;
      const double dxk = P[k < x ? packed_row(k, n) + x : packed_row(x, n) + k];
      double* pyk = P + (k < y ? packed_row(k, n) + y : packed_row(y, n) + k);
      const double dn = lw_centroid(dxk, *pyk, dxy, nx, ny);
      *pyk = dn;
      if (k > y) {
        ybest = min_pair(ybest, MinPair{dn, k});           // new nearest neighbour of y among j > y
      } else {
        const int cur = nn_i[k];
        if (cur == x || cur == y) {
          todo[atomicAdd(ntodo, 1)] = k;                   // its candidate vanished or changed: re-scan
        } else if (dn < nn_d[k] || (dn == nn_d[k] && y < cur)) {
          nn_d[k] = dn;
          nn_i[k] = y;
        }
      }
    }
    ybest = block_min(ybest, s_red, n);
    if (tid == 0) part[nb + blockIdx.x] = ybest;
    grid.sync();
    // C. y's candidate from the partials of B; queued rows re-scanned, one CTA per row
    if (blockIdx.x == 0 && tid < 32) {
      MinPair yb{DBL_MAX, n};
      for (int c = lane; c < nb; c += 32) yb = min_pair(yb, part[nb + c]);
      yb = warp_min(yb);
      if (lane == 0) {
        nn_d[y] = yb.v;
        nn_i[y] = yb.i;
        size[y] = (int)(nx + ny);
        id[y] = n + m;
      }
    }
    const int nt = *ntodo;
    for (int t = blockIdx.x; t < nt; t += nb) {            // uniform over the CTA
      const int k = todo[t];
      const MinPair r = block_min(row_nn_part<true>(P + packed_row(k, n), alive, n, k, tid, kLinkGridThreads), s_red, n);
      if (tid == 0) { nn_d[k] = r.v; nn_i[k] = r.i; }
    }
    grid.sync();
  }
}

// ------------------------------------------------------------------------------------------------------
// cosine cdist
// ------------------------------------------------------------------------------------------------------
__global__ void cdist_cosine_kernel(const double* __restrict__ a, int m, const double* __restrict__ b, int k, int dim,
                                    double* __restrict__ d) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= m * k) return;
  const int i = idx / k, j = idx % k;
  const double *u = a + (size_t)i * dim, *v = b + (size_t)j * dim;
  double uv = 0, uu = 0, vv = 0;
  for (int t = 0; t < dim; ++t) {
    uv += u[t] * v[t];
    uu += u[t] * u[t];
    vv += v[t] * v[t];
  }
  double c = uv / (sqrt(uu) * sqrt(vv));
  if (fabs(c) > 1.0) c = copysign(1.0, c);
  d[idx] = 1.0 - c;
}

// ------------------------------------------------------------------------------------------------------
// VBx: one persistent CTA per clustering problem runs all iterations (utils/vbx.py:98-136)
// ------------------------------------------------------------------------------------------------------
struct VbxJob {
  int n, S;
  int fea_off;        // row offset into fea / rho / G / lpx
  int pad;
  long long gam_off;  // element offset into gamma
  int pi_off;         // element offset into pi / Ng / cst
  int mod_off;        // row offset (in units of D) into alpha / invL  (= pi_off)
};

__device__ __forceinline__ double block_sum_1024(double v, double* red) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double t = 0.0;
  if (threadIdx.x < 32) {
    t = red[threadIdx.x];
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if (threadIdx.x == 0) red[32] = t;
  }
  __syncthreads();
  return red[32];
}

constexpr int kVbxCtas = 8;        // thread-block cluster per problem; phases separated by cluster barriers
constexpr int kVbxTileD = 128;     // PLDA dimension the shared-memory speaker-model phase is written for
constexpr int kVbxTileRows = 32;   // frames staged per tile

__device__ __forceinline__ void vbx_cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

__global__ void __cluster_dims__(kVbxCtas, 1, 1) __launch_bounds__(1024)
vbx_kernel(const VbxJob* __restrict__ jobs, const double* __restrict__ fea_all, const double* __restrict__ phi, int D,
           double Fa, double Fb, int max_iters, double epsilon, double* __restrict__ gamma_all,
           double* __restrict__ pi_all, double* __restrict__ rho_all, double* __restrict__ G_all,
           double* __restrict__ lpx_all, double* __restrict__ alpha_all, double* __restrict__ invL_all,
           double* __restrict__ cst_all, double* __restrict__ praw_all, double* __restrict__ part_all,
           int* __restrict__ iters_all) {
  const int prob = blockIdx.x / kVbxCtas;
  uint32_t rank;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(rank));
  const VbxJob job = jobs[prob];
  const int n = job.n, S = job.S;
  if (n <= 0 || S <= 0) return;                            // uniform over the cluster
  const double* X = fea_all + (size_t)job.fea_off * D;
  double* rho = rho_all + (size_t)job.fea_off * D;
  double* G = G_all + job.fea_off;
  double* lpx = lpx_all + job.fea_off;
  double* gamma = gamma_all + job.gam_off;
  double* pi = pi_all + job.pi_off;
  double* cst = cst_all + job.pi_off;
  double* praw = praw_all + job.pi_off;
  double* part = part_all + (size_t)prob * 2 * kVbxCtas;
  double* alpha = alpha_all + (size_t)job.mod_off * D;
  double* invL = invL_all + (size_t)job.mod_off * D;
  __shared__ double red[33];
  __shared__ double s_rho[kVbxTileRows][kVbxTileD];        // 32 KB: rho rows of the speaker-model phase
  __shared__ double s_gam[kVbxTileRows][8];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int gtid = (int)rank * 1024 + tid, gthreads = kVbxCtas * 1024;
  const int gwarp = (int)rank * 32 + warp, gwarps = kVbxCtas * 32;
  const double FaFb = Fa / Fb;

  // rho = X * sqrt(phi);  G = -0.5 * (|x|^2 + D log(2 pi))    (one warp per frame)
  for (int i = gwarp; i < n; i += gwarps) {
    double s = 0.0;
    for (int d = lane; d < D; d += 32) {
      const double x = X[(size_t)i * D + d];
      s += x * x;
      rho[(size_t)i * D + d] = x * sqrt(phi[d]);
    }
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) G[i] = -0.5 * (s + D * log(2.0 * M_PI));
  }
  for (int s = gtid; s < S; s += gthreads) pi[s] = 1.0 / S;
  vbx_cluster_sync();

  double prev = 0.0;
  int it = 0;
  for (; it < max_iters; ++it) {
    // speaker models: one (s, d) pair per thread, frames summed in order
    if (D == kVbxTileD) {
      // a CTA's 1024 threads are 8 speakers x 128 dimensions, and every speaker needs the same rho rows: the rows (and
      // the 8 gamma columns) are staged once per CTA in shared memory, 32 frames at a time, instead of each warp
      // streaming its own copy from L2 (8 x the bytes into the SM, which bounded this phase).  Per thread the frames
      // are still summed in ascending order with the same operations: bit-identical to the loop below.
      for (int ebase = (int)rank * 1024; ebase < S * D; ebase += gthreads) {        // uniform over the CTA
        const int e = ebase + tid, s0 = ebase / kVbxTileD;
        const int ns = S - s0 < 8 ? S - s0 : 8;
        const bool ok = e < S * D;
        const int sl = tid / kVbxTileD, d = tid % kVbxTileD;
        double ng = 0.0, acc = 0.0;
        for (int i0 = 0; i0 < n; i0 += kVbxTileRows) {
          const int cnt = n - i0 < kVbxTileRows ? n - i0 : kVbxTileRows;
          __syncthreads();                                 // the previous tile has been consumed
          for (int q = tid; q < cnt * kVbxTileD; q += 1024)
            s_rho[q / kVbxTileD][q % kVbxTileD] = rho[(size_t)(i0 + q / kVbxTileD) * D + q % kVbxTileD];
          for (int q = tid; q < cnt * 8; q += 1024)
            s_gam[q >> 3][q & 7] = (q & 7) < ns ? gamma[(size_t)(i0 + (q >> 3)) * S + s0 + (q & 7)] : 0.0;
          __syncthreads();
          if (ok) {
#pragma unroll 8
            for (int ii = 0; ii < cnt; ++ii) {
              const double g = s_gam[ii][sl];
              ng += g;
              acc += g * s_rho[ii][d];
            }
          }
        }
        if (ok) {
          const double il = 1.0 / (1.0 + FaFb * ng * phi[d]);
          invL[e] = il;
          alpha[e] = FaFb * il * acc;
        }
      }
    } else {
      for (int e = gtid; e < S * D; e += gthreads) {
        const int s = e / D, d = e - s * D;
        double ng = 0.0, acc = 0.0;
#pragma unroll 4
        for (int i = 0; i < n; ++i) {
          const double g = gamma[(size_t)i * S + s];
          ng += g;
          acc += g * rho[(size_t)i * D + d];
        }
        const double il = 1.0 / (1.0 + FaFb * ng * phi[d]);
        invL[e] = il;
        alpha[e] = FaFb * il * acc;
      }
    }
    vbx_cluster_sync();
    for (int s = gwarp; s < S; s += gwarps) {
      double c = 0.0;
      for (int d = lane; d < D; d += 32) {
        const double al = alpha[s * D + d];
        c += (invL[s * D + d] + al * al) * phi[d];
      }
      for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
      if (lane == 0) cst[s] = -0.5 * c;
    }
    vbx_cluster_sync();
    // responsibilities: one warp per frame
    for (int i = gwarp; i < n; i += gwarps) {
      double mx = -DBL_MAX;
      for (int s = 0; s < S; ++s) {
        double dot = 0.0;
        for (int d = lane; d < D; d += 32) dot += rho[(size_t)i * D + d] * alpha[s * D + d];
        for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
        const double v = Fa * (dot + cst[s] + G[i]) + log(pi[s] + 1e-8);
        if (lane == 0) gamma[(size_t)i * S + s] = v;
        mx = fmax(mx, v);
      }
      __syncwarp();
      double se = 0.0;
      for (int s = lane; s < S; s += 32) se += exp(gamma[(size_t)i * S + s] - mx);
      for (int o = 16; o > 0; o >>= 1) se += __shfl_xor_sync(0xffffffffu, se, o);
      const double lse = log(se) + mx;
      for (int s = lane; s < S; s += 32) gamma[(size_t)i * S + s] = exp(gamma[(size_t)i * S + s] - lse);
      if (lane == 0) lpx[i] = lse;
    }
    vbx_cluster_sync();
    // priors (one warp per speaker) and the two ELBO sums (per-CTA partials, combined in rank order)
    for (int s = gwarp; s < S; s += gwarps) {
      double c = 0.0;
      for (int i = lane; i < n; i += 32) c += gamma[(size_t)i * S + s];
      for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
      if (lane == 0) praw[s] = c;
    }
    double l = 0.0;
    for (int i = gtid; i < n; i += gthreads) l += lpx[i];
    l = block_sum_1024(l, red);
    double r = 0.0;
    for (int e = gtid; e < S * D; e += gthreads) r += log(invL[e]) - invL[e] - alpha[e] * alpha[e] + 1.0;
    r = block_sum_1024(r, red);
    if (tid == 0) { part[2 * rank] = l; part[2 * rank + 1] = r; }
    vbx_cluster_sync();
    double tot = 0.0;
    for (int s = 0; s < S; ++s) tot += praw[s];
    for (int s = gtid; s < S; s += gthreads) pi[s] = praw[s] / tot;
    l = 0.0; r = 0.0;
    for (int k = 0; k < kVbxCtas; ++k) { l += part[2 * k]; r += part[2 * k + 1]; }
    const double E = l + Fb * 0.5 * r;                     // ELBO (vbx.py:130); identical in every thread
    vbx_cluster_sync();                                    // pi visible, part/praw reusable
    if (it > 0 && E - prev < epsilon) { ++it; break; }
    prev = E;
  }
  if (tid == 0 && rank == 0) iters_all[prob] = it;
}

// ------------------------------------------------------------------------------------------------------
// constrained assignment: maximise sum of soft[c][s][k] over injective maps of (up to 3) speakers to clusters
// ------------------------------------------------------------------------------------------------------
// The reference solves it with scipy.optimize.linear_sum_assignment(maximize=True) (clustering.py:127-140).  Chunks
// with inactive speakers have rows that are all one constant, so optima are tied exactly and the answer is whichever
// optimum the solver reaches.  The kernel therefore runs the same solver: the shortest augmenting path method of
// Crouse (2016) on the negated costs, transposed when there are fewer clusters than speakers, columns scanned from the
// last to the first, and ties of the path minimum resolved towards a free column.  It also makes the same choice on
// near-ties, because it does the same additions and subtractions in the same order.
constexpr int kAssignMaxK = 127;     // cluster ids are int8

__device__ void assign_lsap(const double* __restrict__ p, int K, signed char* __restrict__ h) {
  const bool tr = K < 3;             // tall 3 x K cost matrix: solve its transpose (clusters pick speakers)
  const int nr = tr ? K : 3, nc = tr ? 3 : K;
  double u[3], v[kAssignMaxK], spc[kAssignMaxK];
  int col4row[3], row4col[kAssignMaxK], path[kAssignMaxK], rem[kAssignMaxK];
  bool SR[3], SC[kAssignMaxK];
  for (int i = 0; i < nr; ++i) { u[i] = 0.0; col4row[i] = -1; }
  for (int j = 0; j < nc; ++j) { v[j] = 0.0; row4col[j] = -1; path[j] = -1; }
  for (int cur = 0; cur < nr; ++cur) {
    for (int i = 0; i < nr; ++i) SR[i] = false;
    for (int j = 0; j < nc; ++j) { SC[j] = false; spc[j] = INFINITY; rem[j] = nc - j - 1; }
    int nrem = nc, i = cur, sink = -1;
    double minv = 0.0;
    while (sink == -1) {
      int index = -1;
      double lowest = INFINITY;
      SR[i] = true;
      for (int it = 0; it < nrem; ++it) {
        const int j = rem[it];
        const double cost = -(tr ? p[j * K + i] : p[i * K + j]);
        const double r = __dsub_rn(__dsub_rn(__dadd_rn(minv, cost), u[i]), v[j]);
        if (r < spc[j]) { path[j] = i; spc[j] = r; }
        if (spc[j] < lowest || (spc[j] == lowest && row4col[j] == -1)) { lowest = spc[j]; index = it; }
      }
      minv = lowest;
      const int j = rem[index];
      if (row4col[j] == -1) sink = j;
      else i = row4col[j];
      SC[j] = true;
      rem[index] = rem[--nrem];
    }
    u[cur] = __dadd_rn(u[cur], minv);
    for (int a = 0; a < nr; ++a)
      if (SR[a] && a != cur) u[a] = __dadd_rn(u[a], __dsub_rn(minv, spc[col4row[a]]));
    for (int b = 0; b < nc; ++b)
      if (SC[b]) v[b] = __dsub_rn(v[b], __dsub_rn(minv, spc[b]));
    for (int j = sink;;) {           // augment along the path back to the current row
      const int a = path[j];
      row4col[j] = a;
      const int t = col4row[a];
      col4row[a] = j;
      j = t;
      if (a == cur) break;
    }
  }
  h[0] = h[1] = h[2] = -2;
  if (tr) {
    for (int k = 0; k < K; ++k) h[col4row[k]] = (signed char)k;
  } else {
    for (int s = 0; s < 3; ++s) h[s] = (signed char)col4row[s];
  }
}

__global__ void assign_kernel(const double* __restrict__ soft, int C, int K, int constrained,
                              signed char* __restrict__ hard) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const double* p = soft + (size_t)c * 3 * K;
  signed char* h = hard + c * 3;
  if (!constrained) {
    // np.argmax: the first maximum, and a NaN counts as the maximum (the first NaN wins)
    for (int s = 0; s < 3; ++s) {
      int best = 0;
      for (int k = 1; k < K && !isnan(p[s * K + best]); ++k)
        if (isnan(p[s * K + k]) || p[s * K + k] > p[s * K + best]) best = k;
      h[s] = (signed char)best;
    }
    return;
  }
  assign_lsap(p, K, h);
}

// ------------------------------------------------------------------------------------------------------
// host wrappers
// ------------------------------------------------------------------------------------------------------
size_t linkage_workspace_bytes_batched(const int* row_offsets, int nfiles, int dim, int grid_min) {
  size_t d = 0;
  bool grid = false;
  const int ntot = row_offsets[nfiles];
  for (int f = 0; f < nfiles; ++f) {
    const size_t n = row_offsets[f + 1] - row_offsets[f];
    if ((long long)n >= grid_min) grid = true;
    else d += n * n;
  }
  return align_up(d * 8, 256) + align_up((size_t)ntot * dim * 8, 256) + (size_t)(ntot + nfiles + 64) * 40 +
         (size_t)nfiles * sizeof(LinkJob) + 8192 + (grid ? kLinkGridScratch : 0);
}

// the packed distances of the largest whole-GPU problem: allocated for the call, shared by its large problems
size_t linkage_grid_bytes(const int* row_offsets, int nfiles, int grid_min) {
  size_t big = 0;
  for (int f = 0; f < nfiles; ++f) {
    const size_t n = row_offsets[f + 1] - row_offsets[f];
    if ((long long)n >= grid_min && 4 * n * (n - 1) > big) big = 4 * n * (n - 1);
  }
  return big;
}

// a stream-ordered device allocation freed when the scope ends (after the work queued on `st` before the free)
struct StreamFree {
  void* p;
  cudaStream_t st;
  ~StreamFree() {
    if (p) cudaFreeAsync(p, st);
  }
};

int linkage_centroid_batched(const double* x, const int* row_offsets, int nfiles, int dim, int normalize, double* Z,
                             void* ws, cudaStream_t st, int grid_min) {
  const int ntot = row_offsets[nfiles];
  std::vector<LinkJob> jobs(nfiles);
  std::vector<int> big;                  // problems for the whole-GPU path: no CTA of the batched kernel (n = 0)
  size_t d = 0;
  int z = 0;
  for (int f = 0; f < nfiles; ++f) {
    const int n = row_offsets[f + 1] - row_offsets[f];
    const bool grid = n >= grid_min;
    if (grid) big.push_back(f);
    jobs[f].n = grid ? 0 : n;
    jobs[f].row_off = row_offsets[f];
    jobs[f].z_off = z;
    jobs[f].pad = 0;
    jobs[f].d_off = (long long)d;
    if (!grid) d += (size_t)n * n;
    z += n > 1 ? n - 1 : 0;
  }
  double* P = nullptr;
  const size_t p_bytes = linkage_grid_bytes(row_offsets, nfiles, grid_min);
  if (p_bytes) {
    const cudaError_t e = cudaMallocAsync((void**)&P, p_bytes, st);
    if (e != cudaSuccess) {
      cudaGetLastError();
      int nmax = 0;
      for (int f : big) nmax = std::max(nmax, row_offsets[f + 1] - row_offsets[f]);
      set_error("linkage: %d observations need %llu bytes of device memory for their packed distances "
                "(4 n (n - 1)): %s", nmax, (unsigned long long)p_bytes, cudaGetErrorString(e));
      return e == cudaErrorMemoryAllocation ? B200_ERR_OOM : B200_ERR_CUDA;
    }
  }
  StreamFree free_p{P, st};              // every return below releases the packed distances
  char* p = (char*)ws;
  double* D = (double*)p; p += align_up(d * 8, 256);
  double* xn = (double*)p; p += align_up((size_t)ntot * dim * 8, 256);
  double* nn_d = (double*)p; p += align_up((size_t)ntot * 8, 256);
  int* nn_i = (int*)p; p += align_up((size_t)ntot * 4, 256);
  int* size = (int*)p; p += align_up((size_t)ntot * 4, 256);
  int* id = (int*)p; p += align_up((size_t)ntot * 4, 256);
  int* todo = (int*)p; p += align_up((size_t)(ntot + nfiles + 1) * 4, 256);
  unsigned char* alive = (unsigned char*)p; p += align_up((size_t)ntot, 256);
  LinkJob* djobs = (LinkJob*)p;
  B200_CUDA_OK(cudaMemcpyAsync(djobs, jobs.data(), sizeof(LinkJob) * nfiles, cudaMemcpyHostToDevice, st));
  const double* src = x;
  int rc;
  if (normalize && ntot > 0) {
    if ((rc = normalize == 2 ? launch(normalize_rows_np_f32_kernel, ceil_div(ntot, 64), 64, 0, st, x, xn, ntot, dim)
                             : launch(normalize_rows_kernel, ntot, 128, 0, st, x, xn, ntot, dim)))
      return rc;
    src = xn;
  }
  for (int f = 0; f < nfiles; ++f) {
    const int n = jobs[f].n;
    if (n < 2) continue;
    dim3 grid(ceil_div(n, 16), ceil_div(n, 16));
    if ((rc = launch(pdist_kernel<false>, grid, dim3(16, 16), 0, st, src + (size_t)jobs[f].row_off * dim,
                     D + jobs[f].d_off, n, dim)))
      return rc;
  }
  const size_t link_smem_bytes = (size_t)kLinkSmemRows * 17;
  if ((rc = launch(linkage_centroid_kernel, nfiles, 1024, link_smem_bytes, st, djobs, D, Z, nn_d, nn_i, size, id, alive,
                   todo)))
    return rc;
  if (big.empty()) return B200_OK;

  // large problems, one after another: packed distances, then a cooperative grid of one CTA per SM
  MinPair* part = (MinPair*)(p + align_up((size_t)nfiles * sizeof(LinkJob), 256));
  int* ntodo = (int*)(part + 2 * kLinkGridMaxCtas);
  int dev = 0, sms = 0, per_sm = 0;
  B200_CUDA_OK(cudaGetDevice(&dev));
  B200_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  B200_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, linkage_centroid_grid_kernel, kLinkGridThreads, 0));
  B200_CHECK(per_sm >= 1, B200_ERR_CUDA, "linkage: the whole-GPU kernel does not fit on an SM");
  const int nb = std::min(sms, kLinkGridMaxCtas);
  for (int f : big) {
    const int n = row_offsets[f + 1] - row_offsets[f], ro = row_offsets[f];
    dim3 grid(ceil_div(n, 16), ceil_div(n, 16));
    if ((rc = launch(pdist_kernel<true>, grid, dim3(16, 16), 0, st, src + (size_t)ro * dim, P, n, dim))) return rc;
    if ((rc = launch<true>(linkage_centroid_grid_kernel, nb, kLinkGridThreads, 0, st, P, n,
                           Z + (size_t)jobs[f].z_off * 4, nn_d + ro, nn_i + ro, size + ro, id + ro, alive + ro,
                           todo + ro + f, ntodo, part)))
      return rc;
  }
  free_p.p = nullptr;
  B200_CUDA_OK(cudaFreeAsync(P, st));
  return B200_OK;
}

// ------------------------------------------------------------------------------------------------------
// PLDA transform (core/plda.py:50-63 over utils/vbx.py:211-217): one CTA per embedding
//   y  = sqrt(Din)  * l2(x - mean1);   z = sqrt(Dout) * l2(lda^T y - mean2);   fea = (z - mu) . plda_tr^T [:, :L]
// lda is [Din][Dout] row-major, trT is [Dout][L] row-major (= plda_tr.T[:, :L]); everything fp64 like numpy.
// ------------------------------------------------------------------------------------------------------
__device__ __forceinline__ double block_sum_256(double v, double* red) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double t = 0.0;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += red[w];
  return t;
}

__global__ void __launch_bounds__(256) plda_transform_kernel(const double* __restrict__ x, int Din, int Dout, int L,
                                                              const double* __restrict__ mean1,
                                                              const double* __restrict__ mean2,
                                                              const double* __restrict__ lda,
                                                              const double* __restrict__ mu,
                                                              const double* __restrict__ trT,
                                                              double* __restrict__ fea) {
  extern __shared__ double plda_sm[];
  double* y = plda_sm;            // [Din]
  double* z = plda_sm + Din;      // [Dout]
  __shared__ double red[8];
  const int i = blockIdx.x, tid = threadIdx.x;
  double s = 0.0;
  for (int d = tid; d < Din; d += blockDim.x) {
    const double v = x[(size_t)i * Din + d] - mean1[d];
    y[d] = v;
    s += v * v;
  }
  const double n1 = sqrt(block_sum_256(s, red));
  const double sc1 = sqrt((double)Din);
  for (int d = tid; d < Din; d += blockDim.x) y[d] = sc1 * (y[d] / n1);
  __syncthreads();
  s = 0.0;
  for (int j = tid; j < Dout; j += blockDim.x) {
    double a = 0.0;
    for (int d = 0; d < Din; ++d) a += lda[(size_t)d * Dout + j] * y[d];
    a -= mean2[j];
    z[j] = a;
    s += a * a;
  }
  const double n2 = sqrt(block_sum_256(s, red));
  const double sc2 = sqrt((double)Dout);
  for (int j = tid; j < Dout; j += blockDim.x) z[j] = sc2 * (z[j] / n2) - mu[j];
  __syncthreads();
  for (int k = tid; k < L; k += blockDim.x) {
    double a = 0.0;
    for (int j = 0; j < Dout; ++j) a += z[j] * trT[(size_t)j * L + k];
    fea[(size_t)i * L + k] = a;
  }
}

int plda_transform(const double* x, int n, int Din, int Dout, int L, const double* mean1, const double* mean2,
                   const double* lda, const double* mu, const double* trT, double* fea, cudaStream_t st) {
  return launch(plda_transform_kernel, n, 256, (size_t)(Din + Dout) * sizeof(double), st, x, Din, Dout, L, mean1, mean2,
                lda, mu, trT, fea);
}

// ------------------------------------------------------------------------------------------------------
// VBx centroids (pipelines/clustering.py:620-621):  W = q[:, kept];  centroids = W^T train / sum_i W
// one CTA per kept speaker, threads over the embedding dimension (coalesced rows of `train`)
// ------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) weighted_centroids_kernel(const double* __restrict__ q, int n, int S,
                                                                  const int* __restrict__ kept,
                                                                  const double* __restrict__ train, int dim,
                                                                  double* __restrict__ centroids) {
  const int k = blockIdx.x, col = kept[k];
  __shared__ double red[8];
  double wsum = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) wsum += q[(size_t)i * S + col];
  wsum = block_sum_256(wsum, red);
  for (int d = threadIdx.x; d < dim; d += blockDim.x) {
    double a = 0.0;
    for (int i = 0; i < n; ++i) a += q[(size_t)i * S + col] * train[(size_t)i * dim + d];
    centroids[(size_t)k * dim + d] = a / wsum;
  }
}

int weighted_centroids(const double* q, int n, int S, const int* kept, int K, const double* train, int dim,
                       double* centroids, cudaStream_t st) {
  return launch(weighted_centroids_kernel, K, 256, 0, st, q, n, S, kept, train, dim, centroids);
}

int cdist_cosine(const double* a, int m, const double* b, int k, int dim, double* d, cudaStream_t st) {
  return launch(cdist_cosine_kernel, ceil_div(m * k, 128), 128, 0, st, a, m, b, k, dim, d);
}

size_t vbx_workspace_bytes_batched(const int* n, const int* S, int nfiles, int D) {
  size_t ntot = 0, stot = 0;
  for (int f = 0; f < nfiles; ++f) { ntot += n[f]; stot += S[f]; }
  return (ntot * D + 2 * ntot + 2 * stot * D + 2 * stot + 64 + (size_t)nfiles * 2 * kVbxCtas) * 8 +
         (size_t)nfiles * (sizeof(VbxJob) + 4) + 8192;
}

// fea [sum n][D], gamma concatenated per problem ([n_f][S_f] row-major), pi concatenated ([S_f])
int vbx_run_batched(const double* fea, const double* phi, const int* n, const int* S, int nfiles, int D, double Fa,
                    double Fb, int max_iters, double epsilon, double* gamma, double* pi, int* iters_host, void* ws,
                    cudaStream_t st) {
  std::vector<VbxJob> jobs(nfiles);
  size_t ntot = 0, stot = 0, gtot = 0;
  for (int f = 0; f < nfiles; ++f) {
    jobs[f].n = n[f]; jobs[f].S = S[f]; jobs[f].fea_off = (int)ntot; jobs[f].pad = 0;
    jobs[f].gam_off = (long long)gtot; jobs[f].pi_off = (int)stot; jobs[f].mod_off = (int)stot;
    ntot += n[f]; stot += S[f]; gtot += (size_t)n[f] * S[f];
  }
  double* p = (double*)ws;
  double* rho = p; p += ntot * D;
  double* G = p; p += ntot;
  double* lpx = p; p += ntot;
  double* alpha = p; p += stot * D;
  double* invL = p; p += stot * D;
  double* cst = p; p += stot + 8;
  double* praw = p; p += stot + 8;
  double* part = p; p += (size_t)nfiles * 2 * kVbxCtas;
  VbxJob* djobs = (VbxJob*)p;
  int* iters = (int*)(djobs + nfiles);
  B200_CUDA_OK(cudaMemcpyAsync(djobs, jobs.data(), sizeof(VbxJob) * nfiles, cudaMemcpyHostToDevice, st));
  const int rc = launch(vbx_kernel, nfiles * kVbxCtas, 1024, 0, st, djobs, fea, phi, D, Fa, Fb, max_iters, epsilon,
                        gamma, pi, rho, G, lpx, alpha, invL, cst, praw, part, iters);
  if (rc) return rc;
  if (iters_host) {
    B200_CUDA_OK(cudaMemcpyAsync(iters_host, iters, sizeof(int) * nfiles, cudaMemcpyDeviceToHost, st));
    B200_CUDA_OK(cudaStreamSynchronize(st));
  }
  return B200_OK;
}

int assign_clusters(const double* soft, int C, int K, int constrained, signed char* hard, cudaStream_t st) {
  return launch(assign_kernel, ceil_div(C, 128), 128, 0, st, soft, C, K, constrained, hard);
}

// fcluster(Z, t, criterion="distance") -- scipy/_hierarchy.pyx cluster_dist -> cluster_monocrit
int fcluster_distance(const double* Z, int n, double t, int* T) {
  if (n == 1) { T[0] = 1; return B200_OK; }
  std::vector<double> MD(n - 1);
  for (int i = 0; i < n - 1; ++i) {
    double m = Z[i * 4 + 2];
    const int l = (int)Z[i * 4 + 0], r = (int)Z[i * 4 + 1];
    if (l >= n) m = std::fmax(m, MD[l - n]);
    if (r >= n) m = std::fmax(m, MD[r - n]);
    MD[i] = m;
  }
  std::vector<int> curr(n);
  std::vector<unsigned char> visited(2 * n, 0);
  int k = 0, n_cluster = 0, leader = -1;
  curr[0] = 2 * n - 2;
  while (k >= 0) {
    const int root = curr[k] - n;
    const int lc = (int)Z[root * 4 + 0], rc = (int)Z[root * 4 + 1];
    if (leader == -1 && MD[root] <= t) { leader = root; ++n_cluster; }
    if (lc >= n && !visited[lc]) { visited[lc] = 1; curr[++k] = lc; continue; }
    if (rc >= n && !visited[rc]) { visited[rc] = 1; curr[++k] = rc; continue; }
    if (lc < n) { if (leader == -1) ++n_cluster; T[lc] = n_cluster; }
    if (rc < n) { if (leader == -1) ++n_cluster; T[rc] = n_cluster; }
    if (leader == root) leader = -1;
    --k;
  }
  return B200_OK;
}

}  // namespace b200
