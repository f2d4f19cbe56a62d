// Device-side ordering of the observations for the bundle adjustment kernels.
//
// The reference keeps observations in per-shot maps and lets Ceres' Program order the residual
// blocks (bundle_adjuster.cc:866-915).  Here the raw observation list (any order) is turned, on the
// device, into the layout the kernels want:
//   * observations sorted by (point, shot)                      -> CSR by point (pt_start)
//   * this rank's points (p % world == rank), ordered so that points seen by exactly the same
//     shots are adjacent                                         -> segments of ba_schur_seg
//   * free-point offsets, local point coordinates, the map back to the caller's indices.
// One radix sort of 64-bit keys over the observations, one over the points, three scans; the host
// only reads back a few counts (OrderCounts).
#pragma once
#include <thrust/iterator/counting_iterator.h>

#include <cub/cub.cuh>

#include "common.cuh"

namespace osfm {

struct OrderCounts {
  int err;      // bit 0: observation names a shot that doesn't exist, bit 1: a point that doesn't exist
  int npf;      // free local points
  int nseg;     // segments of the fast Schur path
  int p_fast;   // local points on the fast path (they come first)
  long long n_local;  // observations of this rank's points
  long long n_fast;   // observations of the fast-path points
  unsigned long long pair_bound;  // sum over ALL points of k (k + 1) / 2
};

constexpr unsigned long long ORD_SLOW = 1ULL << 63;
constexpr int ORD_SEG_MAX_POINTS = 64;

struct OrdMax {
  __host__ __device__ int operator()(int a, int b) const { return a > b ? a : b; }
};

// key = (point << 32) | shot, value = position in the caller's list
__global__ void ord_make_keys(long long n, const int* __restrict__ shot, const int* __restrict__ point, int S,
                              int Pfull, unsigned long long* __restrict__ keys, int* __restrict__ vals,
                              OrderCounts* oc) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int s = shot[i], p = point[i];
  int e = 0;
  if (s < 0 || s >= S) e |= 1;
  if (p < 0 || p >= Pfull) e |= 2;
  if (e) atomicOr(&oc->err, e);
  keys[i] = e ? ~0ULL : (((unsigned long long)(unsigned)p << 32) | (unsigned)s);
  vals[i] = (int)i;
}

// g_start[p] = first sorted position of point p (p = 0..Pfull); optional split of the keys
__global__ void ord_point_starts(const unsigned long long* __restrict__ keys, long long n, int Pfull,
                                 long long* __restrict__ g_start) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p > Pfull) return;
  const unsigned long long want = (unsigned long long)(unsigned)p << 32;
  long long lo = 0, hi = n;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (keys[mid] < want) lo = mid + 1; else hi = mid;
  }
  g_start[p] = lo;
}
__global__ void ord_split_keys(const unsigned long long* __restrict__ keys, long long n, int* __restrict__ g_shot,
                               int* __restrict__ g_point) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  g_shot[i] = (int)(unsigned)(keys[i] & 0xffffffffULL);
  g_point[i] = (int)(unsigned)(keys[i] >> 32);
}
__global__ void ord_pair_bound(const long long* __restrict__ g_start, int Pfull, OrderCounts* oc) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  unsigned long long v = 0;
  if (p < Pfull) {
    const unsigned long long k = (unsigned long long)(g_start[p + 1] - g_start[p]);
    v = k * (k + 1) / 2;
  }
  for (int o = 16; o; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0 && v) atomicAdd(&oc->pair_bound, v);
}

// per local point: signature of its shot list and whether the fast Schur path takes it
__global__ void ord_signatures(const unsigned long long* __restrict__ keys, const long long* __restrict__ g_start,
                               const int* __restrict__ pt_const, int P, int world, int rank, int wc, int use_seg,
                               int kmax, int na, int wcmax, unsigned long long* __restrict__ key2,
                               int* __restrict__ val2) {
  const int lp = blockIdx.x * blockDim.x + threadIdx.x;
  if (lp >= P) return;
  const int p = lp * world + rank;
  const long long b = g_start[p], e = g_start[p + 1];
  // pt_const: bit 0 = constant point, bit 1 = the point has a prior (kept off the segment path: only the
  // per-point kernel ba_schur adds prior rows to V_p / g_p)
  unsigned long long h = 1469598103934665603ULL;
  for (long long j = b; j < e; ++j) {
    h ^= (keys[j] & 0xffffffffULL) + 0x9e3779b97f4a7c15ULL;
    h *= 1099511628211ULL;
  }
  // the constant flag hashes as one more element of the list, 2^32, which no shot index takes.  (Folded into the
  // initial value instead, it cancelled against the first shot: a constant point seen by shots (1, ...) hashed like
  // a free point seen by (2, ...), and the two groups split each other's runs into more segments.)
  if (pt_const[p] & 1) {
    h ^= (1ULL << 32) + 0x9e3779b97f4a7c15ULL;
    h *= 1099511628211ULL;
  }
  const long long k = e - b;
  const bool eligible = use_seg && k >= 1 && k <= kmax && k * wc <= na && wc <= wcmax && !(pt_const[p] & 2);
  key2[lp] = (eligible ? 0ULL : ORD_SLOW) | (h >> 1);
  val2[lp] = lp;
}

// np = new local index: observation count, free flag, inverse map, caller's index
__global__ void ord_counts(const int* __restrict__ order, const long long* __restrict__ g_start,
                           const int* __restrict__ pt_const, int P, int world, int rank, long long* __restrict__ kk,
                           int* __restrict__ free_flag, int* __restrict__ inv_order, int* __restrict__ global_of) {
  const int np = blockIdx.x * blockDim.x + threadIdx.x;
  if (np > P) return;
  if (np == P) { kk[np] = 0; free_flag[np] = 0; return; }
  const int op = order[np];
  const int p = op * world + rank;
  kk[np] = g_start[p + 1] - g_start[p];
  free_flag[np] = (pt_const[p] & 1) ? 0 : 1;
  inv_order[op] = np;
  global_of[np] = p;
}
__global__ void ord_finish_points(int P, const int* __restrict__ free_flag, const int* __restrict__ free_scan,
                                  const long long* __restrict__ pt_start, const int* __restrict__ global_of,
                                  const double* __restrict__ pts_full, int* __restrict__ pt_poff,
                                  double* __restrict__ pts0, double* __restrict__ pts1, OrderCounts* oc) {
  const int np = blockIdx.x * blockDim.x + threadIdx.x;
  if (np > P) return;
  if (np == P) { oc->npf = free_scan[P]; oc->n_local = pt_start[P]; return; }
  pt_poff[np] = free_flag[np] ? free_scan[np] : -1;
  const int g = global_of[np];
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const double x = pts_full[3 * (size_t)g + j];
    pts0[3 * (size_t)np + j] = x;
    pts1[3 * (size_t)np + j] = x;
  }
}

// sorted position j -> slot in the new point order
__global__ void ord_gather_obs(const unsigned long long* __restrict__ keys, const int* __restrict__ vals,
                               long long n_valid, const long long* __restrict__ g_start,
                               const int* __restrict__ inv_order, const long long* __restrict__ pt_start, int world,
                               int rank, const double* __restrict__ raw_xy, const double* __restrict__ raw_sigma,
                               long long* __restrict__ obs_orig, int* __restrict__ obs_shot,
                               int* __restrict__ obs_point, double* __restrict__ obs_x, double* __restrict__ obs_y,
                               double* __restrict__ obs_isig) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n_valid) return;
  const unsigned long long key = keys[j];
  const int p = (int)(unsigned)(key >> 32);
  if (p % world != rank) return;
  const int np = inv_order[p / world];
  const long long d = pt_start[np] + (j - g_start[p]);
  const int i = vals[j];
  obs_orig[d] = i;
  obs_shot[d] = (int)(unsigned)(key & 0xffffffffULL);
  obs_point[d] = np;
  const double2 xy = reinterpret_cast<const double2*>(raw_xy)[i];
  obs_x[d] = xy.x;
  obs_y[d] = xy.y;
  obs_isig[d] = 1.0 / raw_sigma[i];  // projection_errors.h:21
}

// head[np] = np when point np cannot share a segment with np - 1 (or is off the fast path), else -1
__global__ void ord_seg_heads(int P, const unsigned long long* __restrict__ key2s, const int* __restrict__ order,
                              const long long* __restrict__ g_start, const unsigned long long* __restrict__ keys,
                              const int* __restrict__ pt_const, int world, int rank, int* __restrict__ head) {
  const int np = blockIdx.x * blockDim.x + threadIdx.x;
  if (np >= P) return;
  bool same = np > 0 && !(key2s[np] & ORD_SLOW) && key2s[np] == key2s[np - 1];
  if (same) {
    const int pa = order[np - 1] * world + rank, pb = order[np] * world + rank;
    const long long a0 = g_start[pa], b0 = g_start[pb];
    const long long k = g_start[pb + 1] - b0;
    same = (g_start[pa + 1] - a0) == k && (pt_const[pa] & 1) == (pt_const[pb] & 1);
    for (long long t = 0; t < k && same; ++t) same = (keys[a0 + t] & 0xffffffffULL) == (keys[b0 + t] & 0xffffffffULL);
  }
  head[np] = same ? -1 : np;
}
// a segment starts at the head of a run and every ORD_SEG_MAX_POINTS points after it
__global__ void ord_seg_flags(int P, const unsigned long long* __restrict__ key2s, const int* __restrict__ run_head,
                              char* __restrict__ flags) {
  const int np = blockIdx.x * blockDim.x + threadIdx.x;
  if (np >= P) return;
  flags[np] = (!(key2s[np] & ORD_SLOW) && ((np - run_head[np]) % ORD_SEG_MAX_POINTS) == 0) ? 1 : 0;
}
__global__ void ord_seg_finish(int P, const unsigned long long* __restrict__ key2s,
                               const long long* __restrict__ pt_start, int* __restrict__ seg_start,
                               const int* __restrict__ num_selected, OrderCounts* oc) {
  if (blockIdx.x || threadIdx.x) return;
  int lo = 0, hi = P;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (key2s[mid] < ORD_SLOW) lo = mid + 1; else hi = mid;
  }
  const int nsel = P > 0 ? *num_selected : 0;
  seg_start[nsel] = lo;
  oc->nseg = nsel;
  oc->p_fast = lo;
  oc->n_fast = pt_start[lo];
}

// results: local points back to the caller's indices
__global__ void ord_scatter_points(int P, const double* __restrict__ pts_local, const int* __restrict__ global_of,
                                   double* __restrict__ pts_full) {
  const int np = blockIdx.x * blockDim.x + threadIdx.x;
  if (np >= P) return;
  const int g = global_of[np];
#pragma unroll
  for (int j = 0; j < 3; ++j) pts_full[3 * (size_t)g + j] = pts_local[3 * (size_t)np + j];
}

}  // namespace osfm
