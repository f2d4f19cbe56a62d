// Reduced camera system of bundle adjustment, block-sparse and resident in L2.
//
// S = (U + D_c) - sum_p W_p (V_p + D_p)^-1 W_p^T is stored as variable-size dense blocks, one per
// pair of *parameter blocks* (camera intrinsics C, rig instance 6, rig camera 6) that share at
// least one point.  The structure depends only on the observation graph, so it is built once
// per run() on the device:
//   1. every point inserts the block pairs of its observations into a hash set (atomicCAS),
//   2. the unique keys are sorted (cub radix sort) -> deterministic layout on every rank,
//   3. value offsets are assigned: upper blocks (bi <= bj) first — the part that is accumulated
//      with atomics and all-reduced — then the mirrored lower blocks,
//   4. block-row lists (CSR over blocks, both triangles) are emitted for the PCG mat-vec.
// For the 500-camera / 2M-observation scene this is ~16 MB instead of a 162 MB dense matrix, i.e.
// the Schur atomics and every PCG mat-vec hit the 50 MB L2 of an H100 instead of HBM.
//
// Included by ba.cu only (shares BAView / Scalars / block_reduce_sum).
#pragma once
#include <cub/cub.cuh>

#include "ba_pcg_plan.h"

namespace osfm {

constexpr unsigned long long BSR_EMPTY = ~0ull;

struct BsrView {
  const unsigned long long* tkeys;  // hash table: key = bi * nblk + bj
  const int* tvals;                 // value offset of the block
  unsigned tmask;
  int nblk;
  const int* blk_off;               // reduced-vector offset of each parameter block
  const int* blk_sz;
};

__device__ __forceinline__ unsigned bsr_hash(unsigned long long k) {
  k ^= k >> 33; k *= 0xff51afd7ed558ccdULL; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ULL; k ^= k >> 33;
  return (unsigned)k;
}
__device__ __forceinline__ int bsr_lookup(const BsrView& h, int bi, int bj) {
  const unsigned long long key = (unsigned long long)bi * (unsigned)h.nblk + (unsigned)bj;
  unsigned slot = bsr_hash(key) & h.tmask;
  for (;;) {
    const unsigned long long k = h.tkeys[slot];
    if (k == key) return h.tvals[slot];
    if (k == BSR_EMPTY) return -1;
    slot = (slot + 1) & h.tmask;
  }
}
__device__ __forceinline__ void bsr_insert(unsigned long long* tkeys, unsigned tmask, unsigned long long key) {
  unsigned slot = bsr_hash(key) & tmask;
  for (;;) {
    const unsigned long long k = tkeys[slot];
    if (k == key) return;
    if (k == BSR_EMPTY) {
      const unsigned long long old = atomicCAS(&tkeys[slot], BSR_EMPTY, key);
      if (old == BSR_EMPTY || old == key) return;
    }
    slot = (slot + 1) & tmask;
  }
}

// Parameter blocks of one observation: [camera | rig instance | rig camera], -1 = constant / absent.
struct ObsBlk {
  int blk[3];
  int C;
  __device__ __forceinline__ int slot_of(int c) const { return c < C ? 0 : (c < C + 6 ? 1 : 2); }
  __device__ __forceinline__ int lstart(int s) const { return s == 0 ? 0 : (s == 1 ? C : C + 6); }
  __device__ __forceinline__ int size(int s) const { return s == 0 ? C : 6; }
};
struct BlkMaps {
  const int *cam_blk, *inst_blk, *rc_blk;
};
__device__ __forceinline__ ObsBlk obs_blocks(const BAView& v, const BlkMaps& bm, int shot) {
  ObsBlk ob;
  const int cam = v.shot_cam[shot];
  ob.C = v.cam_np[cam];
  ob.blk[0] = bm.cam_blk[cam];
  ob.blk[1] = bm.inst_blk[v.shot_inst[shot]];
  ob.blk[2] = v.shot_use_rc[shot] ? bm.rc_blk[v.shot_rc[shot]] : -1;
  return ob;
}

// ---- structure discovery ----------------------------------------------------------------
// One thread per observation a (global CSR by point): pairs (a, b >= a) of the same point.
__global__ void bsr_enum_pairs(BAView v, BlkMaps bm, const int* __restrict__ g_obs_shot,
                               const long long* __restrict__ g_pt_start, const int* __restrict__ g_obs_point,
                               long long n_obs, unsigned long long* tkeys, unsigned tmask, int nblk) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_obs) return;
  const int p = g_obs_point[i];
  const ObsBlk oa = obs_blocks(v, bm, g_obs_shot[i]);
  const long long e = g_pt_start[p + 1];
  for (long long j = i; j < e; ++j) {
    const ObsBlk ob = obs_blocks(v, bm, g_obs_shot[j]);
#pragma unroll
    for (int s1 = 0; s1 < 3; ++s1) {
      if (oa.blk[s1] < 0) continue;
#pragma unroll
      for (int s2 = 0; s2 < 3; ++s2) {
        if (ob.blk[s2] < 0) continue;
        const int lo = min(oa.blk[s1], ob.blk[s2]), hi = max(oa.blk[s1], ob.blk[s2]);
        bsr_insert(tkeys, tmask, (unsigned long long)lo * (unsigned)nblk + (unsigned)hi);
      }
    }
  }
}
// every parameter block owns its diagonal block (priors / damping live there)
__global__ void bsr_insert_diagonal(unsigned long long* tkeys, unsigned tmask, int nblk) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < nblk) bsr_insert(tkeys, tmask, (unsigned long long)b * (unsigned)nblk + (unsigned)b);
}
// compact the table into a list of upper keys; off-diagonal ones also emit their mirror (bit 63 set
// so that one sort puts all upper blocks before all lower blocks)
__global__ void bsr_compact(const unsigned long long* tkeys, unsigned tsize, int nblk, unsigned long long* out,
                            unsigned* count) {
  const unsigned s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= tsize) return;
  const unsigned long long k = tkeys[s];
  if (k == BSR_EMPTY) return;
  const unsigned bi = (unsigned)(k / (unsigned)nblk), bj = (unsigned)(k % (unsigned)nblk);
  if (bi == bj) {
    out[atomicAdd(count, 1u)] = k;
  } else {
    const unsigned o = atomicAdd(count, 2u);
    out[o] = k;
    out[o + 1] = (1ull << 63) | ((unsigned long long)bj * (unsigned)nblk + bi);
  }
}
__global__ void bsr_block_areas(const unsigned long long* keys, int n, int nblk, const int* blk_sz, int* area) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long k = keys[i] & ~(1ull << 63);
  area[i] = blk_sz[k / (unsigned)nblk] * blk_sz[k % (unsigned)nblk];
}
// table values for every stored block (lower keys are inserted here), plus the plain (bi,bj) key list
__global__ void bsr_fill_table(const unsigned long long* skeys, const int* offs, int n, unsigned long long* tkeys,
                               int* tvals, unsigned tmask, unsigned long long* plain) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long key = skeys[i] & ~(1ull << 63);
  plain[i] = key;
  unsigned slot = bsr_hash(key) & tmask;
  for (;;) {
    const unsigned long long k = tkeys[slot];
    if (k == key) break;
    if (k == BSR_EMPTY) {
      const unsigned long long old = atomicCAS(&tkeys[slot], BSR_EMPTY, key);
      if (old == BSR_EMPTY || old == key) break;
    }
    slot = (slot + 1) & tmask;
  }
  tvals[slot] = offs[i];
}
// block-row lists from the keys sorted by (bi, bj): columns, offsets, row pointers
__global__ void bsr_rows(const unsigned long long* rkeys, int n, BsrView h, int* row_ptr, int* row_col, int* row_off) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n) return;
  const int nblk = h.nblk;
  const int bi = i < n ? (int)(rkeys[i] / (unsigned)nblk) : nblk;
  const int prev = i > 0 ? (int)(rkeys[i - 1] / (unsigned)nblk) : -1;
  for (int b = prev + 1; b <= bi; ++b) row_ptr[b] = i;  // also fills empty rows and row_ptr[nblk]
  if (i < n) {
    const int bj = (int)(rkeys[i] % (unsigned)nblk);
    row_col[i] = bj;
    row_off[i] = bsr_lookup(h, bi, bj);
  }
}
// upper-block list for the finish kernel: (bi, bj, offset, mirror offset or -1)
__global__ void bsr_upper_list(const unsigned long long* skeys, const int* offs, int n_upper, BsrView h, int4* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_upper) return;
  const int bi = (int)(skeys[i] / (unsigned)h.nblk), bj = (int)(skeys[i] % (unsigned)h.nblk);
  out[i] = make_int4(bi, bj, offs[i], bi == bj ? -1 : bsr_lookup(h, bj, bi));
}
__global__ void bsr_diag_offsets(BsrView h, int* diag_off) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < h.nblk) diag_off[b] = bsr_lookup(h, b, b);
}

__global__ void bsr_prior_offsets(const int* pr_blk, const int* pr_local, int n, const int* diag_off, const int* blk_sz,
                                  int* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = diag_off[pr_blk[i]] + pr_local[i] * blk_sz[pr_blk[i]] + pr_local[i];
}

// ---------------------------------------------------------------------------
// Schur complement.  One CTA per point (observations of a point are contiguous).
//   U   += Jc_s^T Jc_s,  g_c += Jc_s^T r              (every observation)
//   V    = sum Jp_s^T Jp_s + D_p ; g_p = sum Jp_s^T r   (free points)
//   S   -= W_a V^-1 W_b^T,  rhs -= W_a V^-1 g_p         (all pairs a <= b)
// Only upper blocks (bi <= bj; upper triangle inside diagonal blocks) are written, with fp64
// atomics that resolve in L2; ba_finish_system mirrors them after the optional all-reduce.
// Js = J diag(scale); diag = LM diagonal before division by the radius.
// ---------------------------------------------------------------------------
constexpr int SCHUR_THREADS = 128;
constexpr int SCHUR_KC = 16;  // observations staged per chunk

// Rank rule of the covariance pass (ba_cov.cuh): J is rank deficient when a Cholesky pivot is <= COV_TAU times
// the original diagonal entry.  Point side: the pivots of the scaled, undamped [[a b c] [b d e] [c e f]] = V
// (the negated tests also catch NaN).  Raises flag COV_F_POINT_RANK of the pass.
constexpr double COV_TAU = 1e-10;
constexpr int COV_F_POINT_RANK = 0;
__device__ __forceinline__ bool point_rank_deficient(double a, double b, double c, double d, double e, double f) {
  if (!(a > COV_TAU * a)) return true;
  const double p1 = d - b * b / a;
  if (!(p1 > COV_TAU * d)) return true;
  const double q = e - b * c / a;
  const double p2 = f - c * c / a - q * q / p1;
  return !(p2 > COV_TAU * f);
}

// rank_flag != null (covariance pass, inv_radius = 0): the pivot test above on every free point's V
__global__ void __launch_bounds__(SCHUR_THREADS)
    ba_schur(BAView v, BlkMaps bm, BsrView h, const double* __restrict__ scale, const double* __restrict__ diag,
             double inv_radius, double* __restrict__ Sval, double* __restrict__ rhs, double* __restrict__ Vinv,
             double* __restrict__ gpo, int p_off, PointPriorView pp, const double* __restrict__ pts,
             int* __restrict__ rank_flag) {
  extern __shared__ double sm[];
  const int wc = v.wc, nres = v.nres, nc = v.nc;
  double* Ya = sm;                                   // [KC][wc][3]
  double* Wb = Ya + SCHUR_KC * wc * 3;               // [KC][wc][3]
  int* ga_col = reinterpret_cast<int*>(Wb + SCHUR_KC * wc * 3);  // [KC][wc] packed (blk, slot, size, row) or -1
  int* gb_col = ga_col + SCHUR_KC * wc;
  int* oba = gb_col + SCHUR_KC * wc;                 // [KC][4]: blk0, blk1, blk2, C
  int* obb = oba + SCHUR_KC * 4;
  int* offt = obb + SCHUR_KC * 4;                    // [KC][KC][9] value offsets of (min blk, max blk)
  __shared__ double sVi[9], sg[3], sVig[3];

  const int p = p_off + blockIdx.x;
  const long long b0 = v.pt_start[p], e0 = v.pt_start[p + 1];
  const int k = (int)(e0 - b0);
  const int pf = v.pt_poff[p];
  if (k == 0 && pf < 0) return;   // a free point without observations still needs V^-1 = (D_p + prior)^-1
  const size_t N = (size_t)v.N;
  const int tid = threadIdx.x;

  // ---- U and g_c: thread per (observation, local column c1) ----
  for (int idx = tid; idx < k * wc; idx += SCHUR_THREADS) {
    const int a = idx / wc, c1 = idx % wc;
    const long long i = b0 + a;
    const ObsBlk ob = obs_blocks(v, bm, v.obs_shot[i]);
    if (c1 >= ob.C + 12) continue;
    const int s1 = ob.slot_of(c1);
    const int B1 = ob.blk[s1];
    if (B1 < 0) continue;
    const int r1 = c1 - ob.lstart(s1);
    const int g1 = h.blk_off[B1] + r1;
    const double sc1 = scale[g1];
    double j1[3], rr[3];
    for (int q = 0; q < nres; ++q) {
      j1[q] = v.Jc[((size_t)q * wc + c1) * N + i] * sc1;
      rr[q] = v.r[q * N + i];
    }
    double g = 0.0;
    for (int q = 0; q < nres; ++q) g += j1[q] * rr[q];
    atomicAdd(&rhs[g1], g);
#pragma unroll
    for (int s2 = 0; s2 < 3; ++s2) {
      const int B2 = ob.blk[s2];
      if (B2 < B1) continue;  // B2 < 0, or the mirrored entry is produced by the other thread
      const int off = bsr_lookup(h, B1, B2);
      const int sz2 = ob.size(s2), l2 = ob.lstart(s2);
      const int g2base = h.blk_off[B2];
      for (int r2 = (B1 == B2 ? r1 : 0); r2 < sz2; ++r2) {
        const double sc2 = scale[g2base + r2];
        double val = 0.0;
        for (int q = 0; q < nres; ++q) val += j1[q] * v.Jc[((size_t)q * wc + l2 + r2) * N + i] * sc2;
        atomicAdd(&Sval[off + r1 * sz2 + r2], val);
      }
    }
  }
  if (pf < 0) return;

  // ---- V, g_p: warp 0 (a point has few observations), shuffle reduction ----
  const double sp0 = scale[nc + 3 * pf], sp1 = scale[nc + 3 * pf + 1], sp2 = scale[nc + 3 * pf + 2];
  if (tid < 32) {
    double acc[9];
#pragma unroll
    for (int j = 0; j < 9; ++j) acc[j] = 0.0;
    for (int a = tid; a < k; a += 32) {
      const long long i = b0 + a;
      for (int q = 0; q < nres; ++q) {
        const double x = v.Jp[((size_t)q * 3 + 0) * N + i] * sp0;
        const double y = v.Jp[((size_t)q * 3 + 1) * N + i] * sp1;
        const double z = v.Jp[((size_t)q * 3 + 2) * N + i] * sp2;
        const double rq = v.r[q * N + i];
        acc[0] += x * x; acc[1] += x * y; acc[2] += x * z; acc[3] += y * y; acc[4] += y * z; acc[5] += z * z;
        acc[6] += x * rq; acc[7] += y * rq; acc[8] += z * rq;
      }
    }
#pragma unroll
    for (int j = 0; j < 9; ++j) {
#pragma unroll
      for (int o = 16; o; o >>= 1) acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], o);
    }
    if (tid == 0) {
      if (pp.d) {  // point prior rows (diagonal): V_jj += (d_j s_j)^2, g_j += d_j s_j r_j
        const size_t g = (size_t)pp.global_of[p];
        const double sps[3] = {sp0, sp1, sp2};
        const int vi[3] = {0, 3, 5};
#pragma unroll
        for (int j = 0; j < 3; ++j) {
          const double dj = pp.d[3 * g + j] * sps[j];
          if (dj == 0.0) continue;
          acc[vi[j]] += dj * dj;
          acc[6 + j] += dj * pp.d[3 * g + j] * (pts[3 * (size_t)p + j] - pp.x0[3 * g + j]);
        }
      }
      const double a = acc[0] + diag[nc + 3 * pf] * inv_radius, b = acc[1], c = acc[2];
      const double d = acc[3] + diag[nc + 3 * pf + 1] * inv_radius, e = acc[4];
      const double f = acc[5] + diag[nc + 3 * pf + 2] * inv_radius;
      if (rank_flag && point_rank_deficient(a, b, c, d, e, f)) *rank_flag = 1;
      const double A = d * f - e * e, B = c * e - b * f, Cc = b * e - c * d;
      const double id = 1.0 / (a * A + b * B + c * Cc);
      sVi[0] = A * id; sVi[1] = B * id; sVi[2] = Cc * id;
      sVi[3] = B * id; sVi[4] = (a * f - c * c) * id; sVi[5] = (b * c - a * e) * id;
      sVi[6] = Cc * id; sVi[7] = sVi[5]; sVi[8] = (a * d - b * b) * id;
      sg[0] = acc[6]; sg[1] = acc[7]; sg[2] = acc[8];
      for (int j = 0; j < 3; ++j) sVig[j] = sVi[j * 3] * sg[0] + sVi[j * 3 + 1] * sg[1] + sVi[j * 3 + 2] * sg[2];
      const size_t NP = (size_t)v.npf;
      Vinv[0 * NP + pf] = sVi[0]; Vinv[1 * NP + pf] = sVi[1]; Vinv[2 * NP + pf] = sVi[2];
      Vinv[3 * NP + pf] = sVi[4]; Vinv[4 * NP + pf] = sVi[5]; Vinv[5 * NP + pf] = sVi[8];
      gpo[0 * NP + pf] = sg[0]; gpo[1 * NP + pf] = sg[1]; gpo[2 * NP + pf] = sg[2];
    }
  }
  __syncthreads();

  // ---- pairs, tiled KC x KC over (a-chunk <= b-chunk) ----
  for (int a0 = 0; a0 < k; a0 += SCHUR_KC) {
    const int na = min(SCHUR_KC, k - a0);
    __syncthreads();
    for (int idx = tid; idx < na * wc; idx += SCHUR_THREADS) {
      const int a = idx / wc, c1 = idx % wc;
      const long long i = b0 + a0 + a;
      const ObsBlk ob = obs_blocks(v, bm, v.obs_shot[i]);
      if (c1 == 0) { oba[a * 4] = ob.blk[0]; oba[a * 4 + 1] = ob.blk[1]; oba[a * 4 + 2] = ob.blk[2]; oba[a * 4 + 3] = ob.C; }
      int g1 = -1, m1 = -1;
      if (c1 < ob.C + 12) {
        const int s1 = ob.slot_of(c1);
        if (ob.blk[s1] >= 0) {
          const int r1 = c1 - ob.lstart(s1);
          g1 = h.blk_off[ob.blk[s1]] + r1;
          m1 = (ob.blk[s1] << 12) | (s1 << 10) | (ob.size(s1) << 5) | r1;
        }
      }
      ga_col[a * wc + c1] = m1;
      double w0 = 0.0, w1 = 0.0, w2 = 0.0;
      if (g1 >= 0) {
        const double s1 = scale[g1];
        for (int q = 0; q < nres; ++q) {
          const double jc = v.Jc[((size_t)q * wc + c1) * N + i] * s1;
          w0 += jc * v.Jp[((size_t)q * 3 + 0) * N + i] * sp0;
          w1 += jc * v.Jp[((size_t)q * 3 + 1) * N + i] * sp1;
          w2 += jc * v.Jp[((size_t)q * 3 + 2) * N + i] * sp2;
        }
        atomicAdd(&rhs[g1], -(w0 * sVig[0] + w1 * sVig[1] + w2 * sVig[2]));
      }
      double* y = Ya + (a * wc + c1) * 3;
      y[0] = w0 * sVi[0] + w1 * sVi[3] + w2 * sVi[6];
      y[1] = w0 * sVi[1] + w1 * sVi[4] + w2 * sVi[7];
      y[2] = w0 * sVi[2] + w1 * sVi[5] + w2 * sVi[8];
    }
    for (int bb0 = a0; bb0 < k; bb0 += SCHUR_KC) {
      const int nb = min(SCHUR_KC, k - bb0);
      __syncthreads();
      for (int idx = tid; idx < nb * wc; idx += SCHUR_THREADS) {
        const int b = idx / wc, c2 = idx % wc;
        const long long i = b0 + bb0 + b;
        const ObsBlk ob = obs_blocks(v, bm, v.obs_shot[i]);
        if (c2 == 0) { obb[b * 4] = ob.blk[0]; obb[b * 4 + 1] = ob.blk[1]; obb[b * 4 + 2] = ob.blk[2]; obb[b * 4 + 3] = ob.C; }
        int g2 = -1, m2 = -1;
        if (c2 < ob.C + 12) {
          const int s2 = ob.slot_of(c2);
          if (ob.blk[s2] >= 0) {
            const int r2 = c2 - ob.lstart(s2);
            g2 = h.blk_off[ob.blk[s2]] + r2;
            m2 = (ob.blk[s2] << 12) | (s2 << 10) | (ob.size(s2) << 5) | r2;
          }
        }
        gb_col[b * wc + c2] = m2;
        double w0 = 0.0, w1 = 0.0, w2 = 0.0;
        if (g2 >= 0) {
          const double s2 = scale[g2];
          for (int q = 0; q < nres; ++q) {
            const double jc = v.Jc[((size_t)q * wc + c2) * N + i] * s2;
            w0 += jc * v.Jp[((size_t)q * 3 + 0) * N + i] * sp0;
            w1 += jc * v.Jp[((size_t)q * 3 + 1) * N + i] * sp1;
            w2 += jc * v.Jp[((size_t)q * 3 + 2) * N + i] * sp2;
          }
        }
        double* w = Wb + (b * wc + c2) * 3;
        w[0] = w0; w[1] = w1; w[2] = w2;
      }
      __syncthreads();
      // value offsets of the (min block, max block) of every (a, slot) x (b, slot) combination
      for (int idx = tid; idx < na * nb * 9; idx += SCHUR_THREADS) {
        const int ab = idx / 9, ss = idx % 9;
        const int a = ab / nb, b = ab % nb;
        const int B1 = oba[a * 4 + ss / 3], B2 = obb[b * 4 + ss % 3];
        offt[(a * SCHUR_KC + b) * 9 + ss] = (B1 < 0 || B2 < 0) ? -1 : bsr_lookup(h, min(B1, B2), max(B1, B2));
      }
      __syncthreads();
      // thread <-> one (b, c2) column of the staged b-chunk (its W row lives in registers); it walks
      // all (a <= b, c1): Y_a[c1] is a warp-uniform shared-memory broadcast and consecutive threads
      // hit consecutive addresses of S (coalesced L2 atomics).
      for (int item = tid; item < nb * wc; item += SCHUR_THREADS) {
        const int m2 = gb_col[item];
        if (m2 < 0) continue;
        const int b = item / wc;
        const int B2 = m2 >> 12, s2 = (m2 >> 10) & 3, sz2 = (m2 >> 5) & 31, r2 = m2 & 31;
        const double w0 = Wb[item * 3], w1 = Wb[item * 3 + 1], w2 = Wb[item * 3 + 2];
        const int gb = bb0 + b;
        for (int a = 0; a < na; ++a) {
          const int ga = a0 + a;
          if (ga > gb) break;
          const int* offrow = offt + (a * SCHUR_KC + b) * 9 + s2;
          const int* ma = ga_col + a * wc;
          const double* ya = Ya + a * wc * 3;
          for (int c1 = 0; c1 < wc; ++c1) {
            const int m1 = ma[c1];
            if (m1 < 0) continue;
            const int B1 = m1 >> 12, s1 = (m1 >> 10) & 3, sz1 = (m1 >> 5) & 31, r1 = m1 & 31;
            double val = ya[c1 * 3] * w0 + ya[c1 * 3 + 1] * w1 + ya[c1 * 3 + 2] * w2;
            int pos;
            if (B1 < B2) {
              pos = r1 * sz2 + r2;
            } else if (B1 > B2) {
              if (ga == gb) continue;  // same observation: produced by the mirrored (c2, c1) visit
              pos = r2 * sz1 + r1;
            } else {
              if (ga == gb) {
                if (r2 < r1) continue;
                pos = r1 * sz1 + r2;
              } else {
                if (r1 == r2) val *= 2.0;  // (a,b) and (b,a) land on the same diagonal entry
                pos = min(r1, r2) * sz1 + max(r1, r2);
              }
            }
            atomicAdd(&Sval[offrow[s1 * 3] + pos], -val);
          }
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------
// Segmented Schur complement (fast path), three kernels.
//
// Points are ordered on the host so that points observed by exactly the same shots are contiguous
// ("segment").  Every point of a segment scatters into the same entries of S, so the segment's update
//   S_seg += sum_p ( U_p - Y_p W_p^T ),   Y_p, W_p: (k*wc) x 3
// is a small dense product that can be accumulated in registers and flushed with one L2 atomic per
// entry per *segment* instead of per point (9.5x fewer on the 500-camera scene).
//   A0  ba_point_blocks : one thread per point        -> V^-1, g_p, V^-1 g_p
//   A1  ba_obs_rows     : one thread per (obs, column) -> scaled Jacobian row, W row, Y = W V^-1 row
//                         (coalesced plane reads, massively parallel), g_c / rhs atomics
//   B   ba_schur_seg    : one CTA per segment: streams the contiguous rows of its points into shared
//                         memory, accumulates in registers, flushes
// Splitting the irregular gathers (A) from the dense accumulation (B) is what makes B short: earlier
// single-kernel versions were latency-bound at 2 CTAs/SM.
// Eligible: k <= 16, k * wc <= SEG_NA, wc <= 16; everything else goes through ba_schur.
// ---------------------------------------------------------------------------
constexpr int SEG_NA = 96;                 // max camera-side columns of a segment (k * wc)
constexpr int SEG_SPLIT = 4;                // row quarters per column
constexpr int SEG_THREADS = SEG_SPLIT * SEG_NA;
constexpr int SEG_KMAX = 16;
constexpr int SEG_WCMAX = 16;
constexpr int SEG_PCHUNK = 8;              // points staged per chunk

// A0: V^-1, g_p, V^-1 g_p of the points [0, p_count); rank_flag as in ba_schur.
// One thread per point, but the plane values are not read by it: a thread's observations are contiguous, so a
// warp's loads would be 80 bytes apart (one 32-byte sector per lane and load, 8x the bytes the kernel needs).  The
// CTA's points own one contiguous observation range; it is staged through shared memory in tiles of PB_TILE
// observations with coalesced loads, and every thread sums its own observations out of the tile in the same order.
constexpr int PB_THREADS = 128;
constexpr int PB_TILE = 256;
// Damps the scaled V (upper triangle xx xy xz yy yz zz) and g_p (V[6..8]) of free point pf, tests its rank, stores
// V^-1, g_p and V^-1 g_p.
__device__ __forceinline__ void point_block_finish(const BAView& v, int pf, const double (&V)[9], const double* __restrict__ diag,
                                                   double inv_radius, double* __restrict__ Vinv, double* __restrict__ gpo,
                                                   double* __restrict__ Vig, int* __restrict__ rank_flag) {
  const int nc = v.nc;
  const double a = V[0] + diag[nc + 3 * pf] * inv_radius, b = V[1], c = V[2];
  const double d = V[3] + diag[nc + 3 * pf + 1] * inv_radius, e = V[4];
  const double f = V[5] + diag[nc + 3 * pf + 2] * inv_radius;
  if (rank_flag && point_rank_deficient(a, b, c, d, e, f)) *rank_flag = 1;
  const double A = d * f - e * e, B = c * e - b * f, Cc = b * e - c * d;
  const double id = 1.0 / (a * A + b * B + c * Cc);
  const double i00 = A * id, i01 = B * id, i02 = Cc * id, i11 = (a * f - c * c) * id, i12 = (b * c - a * e) * id,
               i22 = (a * d - b * b) * id;
  const size_t NP = (size_t)v.npf;
  Vinv[0 * NP + pf] = i00; Vinv[1 * NP + pf] = i01; Vinv[2 * NP + pf] = i02;
  Vinv[3 * NP + pf] = i11; Vinv[4 * NP + pf] = i12; Vinv[5 * NP + pf] = i22;
  gpo[0 * NP + pf] = V[6]; gpo[1 * NP + pf] = V[7]; gpo[2 * NP + pf] = V[8];
  Vig[0 * NP + pf] = i00 * V[6] + i01 * V[7] + i02 * V[8];
  Vig[1 * NP + pf] = i01 * V[6] + i11 * V[7] + i12 * V[8];
  Vig[2 * NP + pf] = i02 * V[6] + i12 * V[7] + i22 * V[8];
}
__global__ void __launch_bounds__(PB_THREADS)
    ba_point_blocks(BAView v, int p_count, const double* __restrict__ scale, const double* __restrict__ diag,
                    double inv_radius, double* __restrict__ Vinv, double* __restrict__ gpo, double* __restrict__ Vig,
                    int* __restrict__ rank_flag) {
  __shared__ double tile[12][PB_TILE];   // r (nres) + Jp (3 nres) rows, nres <= 3
  const int p0 = blockIdx.x * PB_THREADS;
  const int p = p0 + threadIdx.x;
  const int p_end = min(p0 + PB_THREADS, p_count);
  const int pf = p < p_count ? v.pt_poff[p] : -1;
  const size_t N = (size_t)v.N;
  const int nc = v.nc, nres = v.nres, nrows = 4 * nres;
  double sp0 = 0.0, sp1 = 0.0, sp2 = 0.0;
  long long my_lo = 0, my_hi = 0;
  if (pf >= 0) {
    sp0 = scale[nc + 3 * pf]; sp1 = scale[nc + 3 * pf + 1]; sp2 = scale[nc + 3 * pf + 2];
    my_lo = v.pt_start[p]; my_hi = v.pt_start[p + 1];
  }
  double V[9];
#pragma unroll
  for (int j = 0; j < 9; ++j) V[j] = 0.0;
  const long long o_lo = v.pt_start[p0], o_hi = v.pt_start[p_end];
  for (long long t0 = o_lo; t0 < o_hi; t0 += PB_TILE) {
    const int len = (int)min((long long)PB_TILE, o_hi - t0);
    __syncthreads();   // the previous tile is consumed
    for (int idx = threadIdx.x; idx < nrows * PB_TILE; idx += PB_THREADS) {
      const int row = idx / PB_TILE, el = idx - row * PB_TILE;
      if (el < len) tile[row][el] = row < nres ? v.r[(size_t)row * N + t0 + el] : v.Jp[(size_t)(row - nres) * N + t0 + el];
    }
    __syncthreads();
    const long long i0 = max(my_lo, t0), i1 = min(my_hi, t0 + len);
    for (long long i = i0; i < i1; ++i) {
      const int el = (int)(i - t0);
      for (int q = 0; q < nres; ++q) {
        const double x = tile[nres + q * 3 + 0][el] * sp0;
        const double y = tile[nres + q * 3 + 1][el] * sp1;
        const double z = tile[nres + q * 3 + 2][el] * sp2;
        const double rq = tile[q][el];
        V[0] += x * x; V[1] += x * y; V[2] += x * z; V[3] += y * y; V[4] += y * z; V[5] += z * z;
        V[6] += x * rq; V[7] += y * rq; V[8] += z * rq;
      }
    }
  }
  if (pf < 0) return;
  point_block_finish(v, pf, V, diag, inv_radius, Vinv, gpo, Vig, rank_flag);
}

// A1: rows of every (observation i < n_obs, local column c2) in plane layout rows[(c2*3 + j) * n_obs + i]
// (coalesced for this kernel, 640-byte runs for a segment in kernel B): rowsJ scaled Jacobian,
// rowsW = Js^T Jp, rowsY = W V^-1; rhs += Js^T r - W V^-1 g_p.  Thread index: i fastest.
__global__ void __launch_bounds__(256)
    ba_obs_rows(BAView v, BlkMaps bm, BsrView h, long long n_obs, const double* __restrict__ scale,
                const double* __restrict__ Vinv, const double* __restrict__ Vig, double* __restrict__ rowsJ,
                double* __restrict__ rowsW, double* __restrict__ rowsY, double* __restrict__ rhs) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int wc = v.wc;
  if (idx >= n_obs * wc) return;
  const int c2 = (int)(idx / n_obs);
  const long long i = idx - (long long)c2 * n_obs;
  const size_t N = (size_t)v.N;
  const ObsBlk ob = obs_blocks(v, bm, v.obs_shot[i]);
  int g = -1;
  if (c2 < ob.C + 12) {
    const int s2 = ob.slot_of(c2);
    if (ob.blk[s2] >= 0) g = h.blk_off[ob.blk[s2]] + c2 - ob.lstart(s2);
  }
  double js[3] = {0.0, 0.0, 0.0}, w[3] = {0.0, 0.0, 0.0}, y[3] = {0.0, 0.0, 0.0};
  if (g >= 0) {
    const double sc = scale[g];
    const int pf = v.pt_poff[v.obs_point[i]];
    double gr = 0.0;
    double sp0 = 0.0, sp1 = 0.0, sp2 = 0.0;
    if (pf >= 0) { sp0 = scale[v.nc + 3 * pf]; sp1 = scale[v.nc + 3 * pf + 1]; sp2 = scale[v.nc + 3 * pf + 2]; }
    for (int q = 0; q < v.nres; ++q) {
      const double jc = v.Jc[((size_t)q * wc + c2) * N + i] * sc;
      js[q] = jc;
      gr += jc * v.r[q * N + i];
      if (pf >= 0) {
        w[0] += jc * v.Jp[((size_t)q * 3 + 0) * N + i] * sp0;
        w[1] += jc * v.Jp[((size_t)q * 3 + 1) * N + i] * sp1;
        w[2] += jc * v.Jp[((size_t)q * 3 + 2) * N + i] * sp2;
      }
    }
    if (pf >= 0) {
      const size_t NP = (size_t)v.npf;
      const double i00 = Vinv[0 * NP + pf], i01 = Vinv[1 * NP + pf], i02 = Vinv[2 * NP + pf];
      const double i11 = Vinv[3 * NP + pf], i12 = Vinv[4 * NP + pf], i22 = Vinv[5 * NP + pf];
      y[0] = w[0] * i00 + w[1] * i01 + w[2] * i02;
      y[1] = w[0] * i01 + w[1] * i11 + w[2] * i12;
      y[2] = w[0] * i02 + w[1] * i12 + w[2] * i22;
      gr -= w[0] * Vig[0 * NP + pf] + w[1] * Vig[1 * NP + pf] + w[2] * Vig[2 * NP + pf];
    }
    atomicAdd(&rhs[g], gr);
  }
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const size_t o = ((size_t)c2 * 3 + j) * (size_t)n_obs + (size_t)i;
    rowsJ[o] = js[j]; rowsW[o] = w[j]; rowsY[o] = y[j];
  }
}

struct SegSmem {
  double Ys[SEG_PCHUNK][SEG_NA][3];
  double Ws[SEG_PCHUNK][SEG_NA][3];
  double Js[SEG_PCHUNK][SEG_NA][3];
  int meta[SEG_NA];
  int gcol[SEG_NA];
  int oblk[SEG_KMAX][4];
  int offt[SEG_KMAX * SEG_KMAX * 9];
};
// the chunk buffers are dead when the accumulators are flushed: a (SEG_NA/2) x SEG_NA tile aliases them
static_assert(sizeof(double) * (SEG_NA / 2) * SEG_NA <= sizeof(double) * 3 * SEG_PCHUNK * SEG_NA * 3, "tile must fit");

// B: one CTA per segment.  WC = compile-time camera-side width (0 = runtime, up to SEG_WCMAX).
template <int WC>
__global__ void __launch_bounds__(SEG_THREADS, 2)
    ba_schur_seg(BAView v, BlkMaps bm, BsrView h, const int* __restrict__ seg_start, long long n_obs,
                 const double* __restrict__ rowsJ, const double* __restrict__ rowsW,
                 const double* __restrict__ rowsY, double* __restrict__ Sval) {
  extern __shared__ __align__(16) unsigned char seg_raw[];
  SegSmem& sm = *reinterpret_cast<SegSmem*>(seg_raw);
  double* tile = reinterpret_cast<double*>(seg_raw);  // [SEG_NA][SEG_NA], valid after the last chunk

  const int wc = WC ? WC : v.wc;
  const int p_begin = seg_start[blockIdx.x], p_end = seg_start[blockIdx.x + 1];
  const long long o0 = v.pt_start[p_begin];
  const int k = (int)(v.pt_start[p_begin + 1] - o0);
  const int ncols = k * wc;
  const int tid = threadIdx.x;
  const int split = tid / SEG_NA;          // which quarter of the rows
  const int item = tid - split * SEG_NA;   // my column (b, c2)
  const int half = split;                  // (split 0 also owns the structure setup and U)
  const bool active = item < ncols;
  const int b = active ? item / wc : 0;
  const bool pfree = v.pt_poff[p_begin] >= 0;   // same for the whole segment (part of the signature)

  // ---- structure of the segment (from its first point) ----
  if (half == 0 && active) {
    const int c2 = item - b * wc;
    const ObsBlk ob = obs_blocks(v, bm, v.obs_shot[o0 + b]);
    if (c2 == 0) { sm.oblk[b][0] = ob.blk[0]; sm.oblk[b][1] = ob.blk[1]; sm.oblk[b][2] = ob.blk[2]; sm.oblk[b][3] = ob.C; }
    int g = -1, m = -1;
    if (c2 < ob.C + 12) {
      const int s2 = ob.slot_of(c2);
      if (ob.blk[s2] >= 0) {
        const int r2 = c2 - ob.lstart(s2);
        g = h.blk_off[ob.blk[s2]] + r2;
        m = (ob.blk[s2] << 12) | (s2 << 10) | (ob.size(s2) << 5) | r2;
      }
    }
    sm.gcol[item] = g;
    sm.meta[item] = m;
  }
  __syncthreads();
  for (int idx = tid; idx < k * k * 9; idx += SEG_THREADS) {
    const int ab = idx / 9, ss = idx - ab * 9;
    const int a = ab / k, bb = ab - a * k;
    const int B1 = sm.oblk[a][ss / 3], B2 = sm.oblk[bb][ss % 3];
    sm.offt[(a * SEG_KMAX + bb) * 9 + ss] = (B1 < 0 || B2 < 0) ? -1 : bsr_lookup(h, min(B1, B2), max(B1, B2));
  }

  constexpr int ROWS = SEG_NA / SEG_SPLIT;
  constexpr int PASS_ROWS = SEG_NA / 2;
  constexpr int WCU = WC ? WC : SEG_WCMAX;
  double acc[ROWS];
#pragma unroll
  for (int e = 0; e < ROWS; ++e) acc[e] = 0.0;
  double uacc[WCU];
#pragma unroll
  for (int e = 0; e < WCU; ++e) uacc[e] = 0.0;
  const int row0 = split * ROWS;

  for (int pc0 = p_begin; pc0 < p_end; pc0 += SEG_PCHUNK) {
    const int np = min(SEG_PCHUNK, p_end - pc0);
    __syncthreads();  // previous chunk fully consumed
    // rows of the chunk: for every plane (c2, j) a run of np*k consecutive observations
    {
      const long long ibase = v.pt_start[pc0];
      const int run = np * k;
      for (int t = tid; t < wc * 3 * run; t += SEG_THREADS) {
        const int plane = t / run, off = t - plane * run;   // off = lp * k + b
        const int c2 = plane / 3, j = plane - c2 * 3;
        const int lp = off / k, bb = off - lp * k;
        const size_t src = (size_t)plane * (size_t)n_obs + (size_t)(ibase + off);
        sm.Js[lp][bb * wc + c2][j] = rowsJ[src];
        if (pfree) {
          sm.Ws[lp][bb * wc + c2][j] = rowsW[src];
          sm.Ys[lp][bb * wc + c2][j] = rowsY[src];
        }
      }
    }
    __syncthreads();
    if (pfree && active) {
      for (int lp = 0; lp < np; ++lp) {
        const double w0 = sm.Ws[lp][item][0], w1 = sm.Ws[lp][item][1], w2 = sm.Ws[lp][item][2];
#pragma unroll
        for (int e = 0; e < ROWS; ++e)
          acc[e] -= sm.Ys[lp][row0 + e][0] * w0 + sm.Ys[lp][row0 + e][1] * w1 + sm.Ys[lp][row0 + e][2] * w2;
      }
    }
    // U_b = Js_b^T Js_b: column (b, c2) against the wc rows of the same observation
    if (half == 0 && active) {
      for (int lp = 0; lp < np; ++lp) {
        const double j0 = sm.Js[lp][item][0], j1 = sm.Js[lp][item][1], j2 = sm.Js[lp][item][2];
#pragma unroll
        for (int c1 = 0; c1 < WCU; ++c1) {
          if (c1 < wc) {
            const double* jr = sm.Js[lp][b * wc + c1];
            uacc[c1] += jr[0] * j0 + jr[1] * j1 + jr[2] * j2;
          }
        }
      }
    }
  }

  // ---- accumulators -> shared tile [row - h*ROWS][column], one row-half at a time; U is added on the
  //      same-observation rows; then a rolled flush loop (small code) issues the atomics ----
  for (int hpass = 0; hpass < 2; ++hpass) {
    __syncthreads();  // chunk buffers / previous pass no longer needed: the tile aliases them
    if (active && row0 / PASS_ROWS == hpass) {
#pragma unroll
      for (int e = 0; e < ROWS; ++e) tile[(row0 - hpass * PASS_ROWS + e) * SEG_NA + item] = pfree ? acc[e] : 0.0;
    }
    __syncthreads();
    if (half == 0 && active) {
#pragma unroll
      for (int c1 = 0; c1 < WCU; ++c1) {
        const int row = b * wc + c1;
        if (c1 < wc && row >= hpass * PASS_ROWS && row < (hpass + 1) * PASS_ROWS)
          tile[(row - hpass * PASS_ROWS) * SEG_NA + item] += uacc[c1];
      }
    }
    __syncthreads();
    const int rbeg = hpass * PASS_ROWS, rend = min(ncols, (hpass + 1) * PASS_ROWS);
    for (int t = tid; t < (rend - rbeg) * ncols; t += SEG_THREADS) {
      const int lr = t / ncols, col = t - lr * ncols;
      const int row = rbeg + lr;
      const int m1 = sm.meta[row], m2 = sm.meta[col];
      if (m1 < 0 || m2 < 0) continue;
      const int a = row / wc, bb = col / wc;
      if (a > bb) continue;
      const int B1 = m1 >> 12, s1 = (m1 >> 10) & 3, sz1 = (m1 >> 5) & 31, r1 = m1 & 31;
      const int B2 = m2 >> 12, s2 = (m2 >> 10) & 3, sz2 = (m2 >> 5) & 31, r2 = m2 & 31;
      double val = tile[lr * SEG_NA + col];
      int pos;
      if (B1 < B2) {
        pos = r1 * sz2 + r2;
      } else if (B1 > B2) {
        if (a == bb) continue;
        pos = r2 * sz1 + r1;
      } else {
        if (a == bb) {
          if (r2 < r1) continue;
          pos = r1 * sz1 + r2;
        } else {
          if (r1 == r2) val *= 2.0;
          pos = min(r1, r2) * sz1 + max(r1, r2);
        }
      }
      atomicAdd(&Sval[sm.offt[(a * SEG_KMAX + bb) * 9 + s1 * 3 + s2] + pos], val);
    }
  }
}

// ---------------------------------------------------------------------------
// Segment Schur complement on the fp64 tensor cores, fused with the row construction.
// One CTA per segment.  Per chunk of SM_PCH points the CTA builds, straight from the residual /
// Jacobian planes, the operands   Yt[k][col] = -(W V^-1)(col, k),  Wt[k][col] = W(col, k),
// Jt[k][col] = Js(col, k)   (k = 3 * point-in-chunk + component, col = shot-in-segment * wc + local
// column) in shared memory, then accumulates the UPPER tiles of
//     S_seg = sum_p ( U_p - Y_p W_p^T )            (symmetric: Y W^T = W V^-1 W^T)
// with mma.m8n8k4.f64: C(ti,tj) += Yt^T(ti) Wt(tj), plus Jt^T Jt masked to the same shot for the
// tiles that touch a diagonal block (U).  The accumulators are flushed once per segment, from the
// fragments, with fp64 atomics that resolve in L2; g_c - W V^-1 g_p goes to the right-hand side once
// per segment column.  Leading dimension SM_LD = 4 (mod 16) makes the fragment loads conflict-free.
// Replaces ba_obs_rows + ba_schur_seg (no materialised rows: the planes are read once).
// ---------------------------------------------------------------------------
constexpr int SM_PCH = 8;
constexpr int SM_KC = 3 * SM_PCH;
constexpr int SM_LD = 100;
constexpr int SM_THREADS = 384;
constexpr int SM_NT = SEG_NA / 8;                    // 12 tiles per side
constexpr int SM_NEAR = (2 * SM_NT - 1 + SM_THREADS / 32 - 1) / (SM_THREADS / 32);                       // 2 near-diagonal tiles per warp
constexpr int SM_SLOTS = SM_NEAR + ((SM_NT - 1) * (SM_NT - 2) / 2 + SM_THREADS / 32 - 1) / (SM_THREADS / 32);  // + 5 far tiles
struct SegMmaSmem {
  double Yt[SM_KC][SM_LD];
  double Wt[SM_KC][SM_LD];
  double Jt[SM_KC][SM_LD];
  double G[SM_PCH][SEG_NA];   // per (point of the chunk, column): its share of the reduced right-hand side
  double obsd[SM_PCH * SEG_KMAX][12];  // per observation of the chunk: r[3], (Jp * point scale)[3][3]
  double ptd[SM_PCH][9];               // per point of the chunk: V^-1 (6), V^-1 g_p (3)
  double scol[SEG_NA];                 // Jacobi scale of every column
  unsigned char lp_of[SM_PCH * SEG_KMAX], bb_of[SM_PCH * SEG_KMAX];  // observation-in-chunk -> (point, shot)
  int meta[SEG_NA];
  int gcol[SEG_NA];
  int oblk[SEG_KMAX][4];
  int offt[SEG_KMAX * SEG_KMAX * 9];
};

// Per-segment tables (constant over the LM iterations of a run, built once by ba_seg_tables before the first
// linearisation; scol by ba_seg_scales once the Jacobi scale is known, or by ba_seg_tables when it is given one):
//   [ gcol (ncols) | meta (ncols) | offt (k (k + 1) / 2 shot pairs a <= b, 9 slot pairs each) ] ints, then
//   scol (ncols doubles, 8-byte aligned).  tab_off[s] = offset of segment s in ints.
__host__ __device__ inline int seg_pair_index(int a, int b, int k) { return a * k - a * (a - 1) / 2 + (b - a); }
__host__ __device__ inline long long seg_table_ints(int k, int wc) {
  const int ncols = k * wc;
  long long n = 2LL * ncols + 9LL * (k * (k + 1) / 2);
  n += n & 1;              // doubles start on an 8-byte boundary
  return n + 2LL * ncols;  // scol
}
// tab_off[s] for every segment (then an exclusive scan on the host side via cub)
__global__ void ba_seg_table_sizes(BAView v, const int* __restrict__ seg_start, int nseg, long long* __restrict__ sizes) {
  const int sidx = blockIdx.x * blockDim.x + threadIdx.x;
  if (sidx > nseg) return;
  if (sidx == nseg) { sizes[sidx] = 0; return; }
  const int p0 = seg_start[sidx];
  const int k = (int)(v.pt_start[p0 + 1] - v.pt_start[p0]);
  sizes[sidx] = seg_table_ints(k, v.wc);
}
__global__ void __launch_bounds__(128)
    ba_seg_tables(BAView v, BlkMaps bm, BsrView h, const int* __restrict__ seg_start, const double* __restrict__ scale,
                  const long long* __restrict__ tab_off, int* __restrict__ tab) {
  __shared__ int oblk[SEG_KMAX][4];
  const int wc = v.wc;
  const int p0 = seg_start[blockIdx.x];
  const long long o0 = v.pt_start[p0];
  const int k = (int)(v.pt_start[p0 + 1] - o0);
  const int ncols = k * wc;
  int* T = tab + tab_off[blockIdx.x];
  int* gcol = T;
  int* meta = T + ncols;
  int* offt = T + 2 * ncols;
  long long nints = 2LL * ncols + 9LL * (k * (k + 1) / 2);
  nints += nints & 1;
  double* scol = reinterpret_cast<double*>(T + nints);
  for (int t = threadIdx.x; t < ncols; t += blockDim.x) {
    const int b = t / wc, c2 = t - b * wc;
    const ObsBlk ob = obs_blocks(v, bm, v.obs_shot[o0 + b]);
    if (c2 == 0) { oblk[b][0] = ob.blk[0]; oblk[b][1] = ob.blk[1]; oblk[b][2] = ob.blk[2]; oblk[b][3] = ob.C; }
    int g = -1, m = -1;
    if (c2 < ob.C + 12) {
      const int s2 = ob.slot_of(c2);
      if (ob.blk[s2] >= 0) {
        const int r2 = c2 - ob.lstart(s2);
        g = h.blk_off[ob.blk[s2]] + r2;
        m = (ob.blk[s2] << 12) | (s2 << 10) | (ob.size(s2) << 5) | r2;
      }
    }
    gcol[t] = g;
    meta[t] = m;
    if (scale) scol[t] = g >= 0 ? scale[g] : 0.0;
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < k * k * 9; idx += blockDim.x) {
    const int ab = idx / 9, ss = idx - ab * 9;
    const int a = ab / k, bb = ab - a * k;
    if (a > bb) continue;
    const int B1 = oblk[a][ss / 3], B2 = oblk[bb][ss % 3];
    offt[seg_pair_index(a, bb, k) * 9 + ss] = (B1 < 0 || B2 < 0) ? -1 : bsr_lookup(h, min(B1, B2), max(B1, B2));
  }
}

// The Jacobi scale of every segment column (scol of the tables above), from gcol: once the scale is known, and again
// when it changes (the covariance pass).  One CTA per segment.
__global__ void __launch_bounds__(128)
    ba_seg_scales(BAView v, const int* __restrict__ seg_start, const double* __restrict__ scale,
                  const long long* __restrict__ tab_off, int* __restrict__ tab) {
  const int p0 = seg_start[blockIdx.x];
  const int k = (int)(v.pt_start[p0 + 1] - v.pt_start[p0]);
  const int ncols = k * v.wc;
  const int* gcol = tab + tab_off[blockIdx.x];
  long long nints = 2LL * ncols + 9LL * (k * (k + 1) / 2);
  nints += nints & 1;
  double* scol = reinterpret_cast<double*>(tab + tab_off[blockIdx.x] + nints);
  for (int t = threadIdx.x; t < ncols; t += blockDim.x) scol[t] = gcol[t] >= 0 ? scale[gcol[t]] : 0.0;
}

__device__ __forceinline__ void dmma884(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
               : "+d"(c0), "+d"(c1)
               : "d"(a), "d"(b));
}

template <int WC>
__global__ void __launch_bounds__(SM_THREADS, 2)
    ba_schur_mma(BAView v, const int* __restrict__ seg_start, const long long* __restrict__ tab_off,
                 const int* __restrict__ tab, const double* __restrict__ scale, const double* __restrict__ Vinv, const double* __restrict__ Vig, double* __restrict__ Sval,
                 double* __restrict__ rhs, unsigned long long* prof) {
  extern __shared__ __align__(16) unsigned char seg_raw[];
  SegMmaSmem& sm = *reinterpret_cast<SegMmaSmem*>(seg_raw);
  // prof != null (OSFM_BA_TRACE): thread 0 adds its clocks per phase: structure, block offsets, loads, rows, mma, flush
  long long tk = prof ? clock64() : 0;
  auto mark = [&](int slot) {
    if (prof && threadIdx.x == 0) {
      const long long now = clock64();
      atomicAdd(&prof[slot], (unsigned long long)(now - tk));
      tk = now;
    }
  };
  const int wc = WC ? WC : v.wc;
  const int p_begin = seg_start[blockIdx.x], p_end = seg_start[blockIdx.x + 1];
  const long long o0 = v.pt_start[p_begin];
  const int k = (int)(v.pt_start[p_begin + 1] - o0);
  const int ncols = k * wc;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bool pfree = v.pt_poff[p_begin] >= 0;   // same for the whole segment (part of the signature)
  const size_t N = (size_t)v.N;
  const int nres = v.nres;

  // ---- tables of the segment (ba_seg_tables) -> shared memory; zero the operand buffers once ----
  {
    const int* T = tab + tab_off[blockIdx.x];
    const int npair9 = 9 * (k * (k + 1) / 2);
    for (int t = tid; t < 2 * ncols + npair9; t += SM_THREADS) {
      const int val = T[t];
      if (t < ncols) sm.gcol[t] = val;
      else if (t < 2 * ncols) sm.meta[t - ncols] = val;
      else sm.offt[t - 2 * ncols] = val;
    }
    long long nints = 2LL * ncols + npair9;
    nints += nints & 1;
    const double* scol = reinterpret_cast<const double*>(T + nints);
    if (tid < SEG_NA) {
      sm.scol[tid] = tid < ncols ? scol[tid] : 0.0;
      if (tid >= ncols) { sm.gcol[tid] = -1; sm.meta[tid] = -1; }
    }
  }
  if (tid < SM_PCH * SEG_KMAX) {
    const int lp = tid / k;
    sm.lp_of[tid] = (unsigned char)lp;
    sm.bb_of[tid] = (unsigned char)(tid - lp * k);
  }
  // every (row < 3 np, column < ncols) entry of the operand buffers is rewritten by each chunk; only the padding
  // columns [ncols, SM_LD) the 8-wide tiles can touch have to read as zero (zeroing all 57 KB cost 5k clocks per
  // segment)
  {
    const int padc = SM_LD - ncols;
    for (int t = tid; t < 3 * SM_KC * padc; t += SM_THREADS) {
      const int arr = t / (SM_KC * padc), rem = t - arr * (SM_KC * padc);
      const int kk = rem / padc, cc = ncols + rem - kk * padc;
      (arr == 0 ? sm.Yt : arr == 1 ? sm.Wt : sm.Jt)[kk][cc] = 0.0;
    }
  }
  mark(0);

  // ---- my tiles of the upper triangle of nt x nt 8x8 tiles.  Slots 0..SM_NEAR-1 take the tiles that can
  //      touch a diagonal (same-shot) block, (t, t) and (t, t + 1): they also accumulate Jt^T Jt in d[];
  //      the other slots take the tiles with tj >= ti + 2 (Y W^T only). ----
  const int nt = (ncols + 7) >> 3;
  const int n_near = 2 * nt - 1, n_far = (nt - 1) * (nt - 2) / 2;
  int tile_ij[SM_SLOTS];   // ti | tj << 8, or -1
  double c[SM_SLOTS][2], d[SM_NEAR][2];
#pragma unroll
  for (int sidx = 0; sidx < SM_SLOTS; ++sidx) {
    c[sidx][0] = 0.0; c[sidx][1] = 0.0;
    int ti = -1, tj = -1;
    if (sidx < SM_NEAR) {
      d[sidx][0] = 0.0; d[sidx][1] = 0.0;
      const int t = warp + sidx * (SM_THREADS / 32);
      if (t < nt) { ti = t; tj = t; }
      else if (t < n_near) { ti = t - nt; tj = ti + 1; }
    } else {
      int t = warp + (sidx - SM_NEAR) * (SM_THREADS / 32);
      if (t < n_far) {
        ti = 0;
        while (t >= nt - 2 - ti) { t -= nt - 2 - ti; ++ti; }
        tj = ti + 2 + t;
      }
    }
    tile_ij[sidx] = ti < 0 ? -1 : (ti | (tj << 8));
  }
  const int fr = lane >> 2, fk = lane & 3;   // fragment row / k of this lane
  double racc = 0.0;                         // reduced right-hand side of column tid (tid < ncols)

  for (int pc0 = p_begin; pc0 < p_end; pc0 += SM_PCH) {
    const int np = min(SM_PCH, p_end - pc0);
    const long long ibase = v.pt_start[pc0];
    const int run = np * k;
    __syncthreads();  // previous chunk fully consumed (and the structure tables are complete)
    mark(pc0 == p_begin ? 1 : 4);
    if (np < SM_PCH) {  // short last chunk: the k rows beyond it must read as zero
      const int kz0 = 3 * np, kz1 = (3 * np + 3) & ~3;
      for (int t = tid; t < (kz1 - kz0) * SM_LD; t += SM_THREADS) {
        const int kk = kz0 + t / SM_LD, cc = t % SM_LD;
        sm.Yt[kk][cc] = 0.0; sm.Wt[kk][cc] = 0.0; sm.Jt[kk][cc] = 0.0;
      }
    }
    // items (c2 = item >> 7, observation = item & 127): coalesced plane reads of the camera-side Jacobian, issued
    // first so that their latency overlaps the per-observation / per-point loads below
    constexpr int ITEMS = ((WC ? WC : SEG_WCMAX) * 128 + SM_THREADS - 1) / SM_THREADS;
    double jall[ITEMS][3];
#pragma unroll
    for (int it = 0; it < ITEMS; ++it) {
      const int t = tid + it * SM_THREADS;
      const int c2 = t >> 7, off = t & 127;
#pragma unroll
      for (int q = 0; q < 3; ++q)
        jall[it][q] = (c2 < wc && off < run && q < nres) ? v.Jc[((size_t)q * wc + c2) * N + (size_t)(ibase + off)] : 0.0;
    }
    // per-observation / per-point data of the chunk, loaded once (not once per camera-side column)
    if (tid < run) {
      const size_t i = (size_t)(ibase + tid);
      const int pf = v.pt_poff[pc0 + sm.lp_of[tid]];
      double sp[3] = {0.0, 0.0, 0.0};
      if (pfree) { sp[0] = scale[v.nc + 3 * pf]; sp[1] = scale[v.nc + 3 * pf + 1]; sp[2] = scale[v.nc + 3 * pf + 2]; }
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        const bool on = q < nres;
        sm.obsd[tid][q] = on ? v.r[q * N + i] : 0.0;
#pragma unroll
        for (int j = 0; j < 3; ++j) sm.obsd[tid][3 + 3 * q + j] = (on && pfree) ? v.Jp[((size_t)q * 3 + j) * N + i] * sp[j] : 0.0;
      }
    } else if (tid >= SM_THREADS - SM_PCH && pfree) {
      const int lp = tid - (SM_THREADS - SM_PCH);
      if (lp < np) {
        const int pf = v.pt_poff[pc0 + lp];
        const size_t NP = (size_t)v.npf;
#pragma unroll
        for (int e = 0; e < 6; ++e) sm.ptd[lp][e] = Vinv[e * NP + pf];
#pragma unroll
        for (int e = 0; e < 3; ++e) sm.ptd[lp][6 + e] = Vig[e * NP + pf];
      }
    }
    __syncthreads();
    mark(2);
#pragma unroll
    for (int it = 0; it < ITEMS; ++it) {
      const int t = tid + it * SM_THREADS;
      const int c2 = t >> 7, off = t & 127;
      if (c2 >= wc || off >= run) continue;
      const int lp = sm.lp_of[off], bb = sm.bb_of[off];
      const int col = bb * wc + c2;
      const double sc = sm.scol[col];
      const double* od = sm.obsd[off];
      double js[3], w[3] = {0.0, 0.0, 0.0}, y[3] = {0.0, 0.0, 0.0}, gr = 0.0;
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        js[q] = jall[it][q] * sc;
        gr += js[q] * od[q];
#pragma unroll
        for (int j = 0; j < 3; ++j) w[j] += js[q] * od[3 + 3 * q + j];
      }
      if (pfree) {
        const double* pd = sm.ptd[lp];
        y[0] = w[0] * pd[0] + w[1] * pd[1] + w[2] * pd[2];
        y[1] = w[0] * pd[1] + w[1] * pd[3] + w[2] * pd[4];
        y[2] = w[0] * pd[2] + w[1] * pd[4] + w[2] * pd[5];
        gr -= w[0] * pd[6] + w[1] * pd[7] + w[2] * pd[8];
      }
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        sm.Jt[3 * lp + j][col] = js[j];
        sm.Wt[3 * lp + j][col] = w[j];
        sm.Yt[3 * lp + j][col] = -y[j];
      }
      sm.G[lp][col] = gr;
    }
    __syncthreads();
    mark(3);
    if (tid < ncols)
      for (int lp = 0; lp < np; ++lp) racc += sm.G[lp][tid];
    const int ksteps = (3 * np + 3) >> 2;
#pragma unroll
    for (int sidx = 0; sidx < SM_SLOTS; ++sidx) {
      if (tile_ij[sidx] < 0) continue;
      // A-fragment row / B-fragment column of this lane, at k = fk
      const int arow = fk * SM_LD + 8 * (tile_ij[sidx] & 255) + fr, bcol = fk * SM_LD + 8 * (tile_ij[sidx] >> 8) + fr;
      if (pfree) {
        const double* yk = &sm.Yt[0][0] + arow;
        const double* wk = &sm.Wt[0][0] + bcol;
#pragma unroll 2
        for (int ks = 0; ks < ksteps; ++ks) dmma884(c[sidx][0], c[sidx][1], yk[ks * 4 * SM_LD], wk[ks * 4 * SM_LD]);
      }
      if (sidx < SM_NEAR) {   // Js^T Js; the flush keeps it only where row and column belong to the same shot
        const double* ja = &sm.Jt[0][0] + arow;
        const double* jb = &sm.Jt[0][0] + bcol;
#pragma unroll 2
        for (int ks = 0; ks < ksteps; ++ks) dmma884(d[sidx][0], d[sidx][1], ja[ks * 4 * SM_LD], jb[ks * 4 * SM_LD]);
      }
    }
  }

  // ---- flush: right-hand side once per column, the tiles straight from the fragments ----
  mark(4);
  if (tid < ncols && sm.gcol[tid] >= 0) atomicAdd(&rhs[sm.gcol[tid]], racc);
#pragma unroll
  for (int sidx = 0; sidx < SM_SLOTS; ++sidx) {
    if (tile_ij[sidx] < 0) continue;
    const int ti = tile_ij[sidx] & 255, tj = tile_ij[sidx] >> 8;
    const int row = 8 * ti + fr;
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int col = 8 * tj + 2 * fk + e;
      if (row >= ncols || col >= ncols) continue;
      const int m1 = sm.meta[row], m2 = sm.meta[col];
      if (m1 < 0 || m2 < 0) continue;
      const int a = row / wc, bb = col / wc;
      if (a > bb) continue;
      const int B1 = m1 >> 12, s1 = (m1 >> 10) & 3, sz1 = (m1 >> 5) & 31, r1 = m1 & 31;
      const int B2 = m2 >> 12, s2 = (m2 >> 10) & 3, sz2 = (m2 >> 5) & 31, r2 = m2 & 31;
      double val = c[sidx][e];
      if (sidx < SM_NEAR && a == bb) val += d[sidx < SM_NEAR ? sidx : 0][e];
      int pos;
      if (B1 < B2) {
        pos = r1 * sz2 + r2;
      } else if (B1 > B2) {
        if (a == bb) continue;
        pos = r2 * sz1 + r1;
      } else {
        if (a == bb) {
          if (r2 < r1) continue;
          pos = r1 * sz1 + r2;
        } else {
          if (r1 == r2) val *= 2.0;
          pos = min(r1, r2) * sz1 + max(r1, r2);
        }
      }
      atomicAdd(&Sval[sm.offt[seg_pair_index(a, bb, k) * 9 + s1 * 3 + s2] + pos], val);
    }
  }
  mark(5);
}

// Priors (after the all-reduce): diagonal entries of the diagonal blocks.
__global__ void ba_prior_system(PriorView pv, Params p, const double* scale, const int* __restrict__ prior_diag_off,
                                double* Sval, double* rhs) {
  const int row = blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= pv.n_cam_rows + pv.n_pos_rows) return;
  double r, d;
  int col;
  prior_row(pv, p, row, &r, &col, &d);
  const double ds = d * scale[col];
  atomicAdd(&Sval[prior_diag_off[row]], ds * ds);
  atomicAdd(&rhs[col], ds * r);
}

// One warp per upper block: LM damping on the diagonal, mirror inside diagonal blocks, transposed
// copy of off-diagonal blocks into their lower slots.
__global__ void __launch_bounds__(256)
    ba_finish_system(const int4* __restrict__ upper, int n_upper, BsrView h, double* Sval,
                     const double* __restrict__ diag, double inv_radius) {
  const int w = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (w >= n_upper) return;
  const int4 u = upper[w];
  const int szi = h.blk_sz[u.x], szj = h.blk_sz[u.y];
  if (u.x == u.y) {
    const int g0 = h.blk_off[u.x];
    for (int e = lane; e < szi * szi; e += 32) {
      const int r = e / szi, c = e % szi;
      if (r == c) Sval[u.z + e] += diag[g0 + r] * inv_radius;
      else if (c < r) Sval[u.z + e] = Sval[u.z + c * szi + r];
    }
  } else {
    for (int e = lane; e < szi * szj; e += 32) {
      const int r = e / szj, c = e % szj;
      Sval[u.w + c * szi + r] = Sval[u.z + e];
    }
  }
}

// ---------------------------------------------------------------------------
// PCG on S y = rhs.  Block-Jacobi preconditioner over *groups* of parameter blocks (a camera and the
// rig instance that is its only user form one group: intrinsics and pose of a shot are strongly
// coupled), one persistent kernel over all SMs, two grid barriers per iteration.
//
// Mat-vec layout ("block-row ELL", rebuilt from the block values every LM iteration by
// pcg_convert): for block row b with n scalar rows and M = sum of its blocks' column counts,
// Spcg[rowbase[b] + r*M + q] is entry (r, q) and colidx[cbase[b] + q] its global column, so a warp
// streams one scalar row with fully coalesced loads.
// ---------------------------------------------------------------------------
constexpr int MAXB = 16;

struct PcgLayout {
  const int* row_of;     // [nc] block row of every scalar row
  const int* row_M;      // [nblk]
  const long long* rowbase;  // [nblk] offset into Spcg
  const int* cbase;      // [nblk] offset into colidx
  const int* colidx;
  int ngroups;
  const int* grp_b1;     // [ngroups] first block of the group
  const int* grp_b2;     // [ngroups] second block or -1
};

// M of every block row and the in-row column offset of every stored block
__global__ void pcg_row_sizes(const int* __restrict__ row_ptr, const int* __restrict__ row_col, BsrView h, int* row_M,
                              int* qoff, int* blk_row) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= h.nblk) return;
  int acc = 0;
  for (int e = row_ptr[b]; e < row_ptr[b + 1]; ++e) {
    qoff[e] = acc;
    blk_row[e] = b;
    acc += h.blk_sz[row_col[e]];
  }
  row_M[b] = acc;
}
__global__ void pcg_fill_colidx(const int* __restrict__ row_col, const int* __restrict__ qoff,
                                const int* __restrict__ blk_row, int n_all, BsrView h, const int* __restrict__ cbase,
                                int* colidx, int* row_of) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_all) return;
  const int b = blk_row[e], cb = row_col[e];
  const int m = h.blk_sz[cb], co = h.blk_off[cb];
  for (int j = 0; j < m; ++j) colidx[cbase[b] + qoff[e] + j] = co + j;
  if (cb == b) {
    const int n = h.blk_sz[b], o = h.blk_off[b];
    for (int r = 0; r < n; ++r) row_of[o + r] = b;
  }
}
// one warp per stored block: scatter its values into the block-row ELL layout
__global__ void __launch_bounds__(256)
    pcg_convert(const double* __restrict__ Sval, const int* __restrict__ row_col, const int* __restrict__ row_off,
                const int* __restrict__ qoff, const int* __restrict__ blk_row, int n_all, BsrView h,
                const int* __restrict__ row_M, const long long* __restrict__ rowbase, double* __restrict__ Spcg) {
  const int e = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (e >= n_all) return;
  const int b = blk_row[e];
  const int n = h.blk_sz[b], m = h.blk_sz[row_col[e]], M = row_M[b];
  const double* src = Sval + row_off[e];
  double* dst = Spcg + rowbase[b] + qoff[e];
  for (int t = lane; t < n * m; t += 32) {
    const int r = t / m, j = t - r * m;
    dst[(size_t)r * M + j] = src[t];
  }
}

// Cholesky-inverts the diagonal matrix of every preconditioner group into Minv[g][MAXB*MAXB].  One warp per group,
// the factor in shared memory: lane 0 takes the pivot of column j, lanes j + 1 .. n - 1 its rows below, then lane c
// solves for column c of the inverse (every value is computed by one lane in the order of the serial algorithm).
constexpr int PFG_WARPS = 4;
__global__ void __launch_bounds__(32 * PFG_WARPS)
    pcg_factor_groups(const double* __restrict__ Sval, BsrView h, const int* __restrict__ diag_off,
                      const int* __restrict__ grp_b1, const int* __restrict__ grp_b2, int ngroups,
                      double* __restrict__ Minv) {
  __shared__ double Ls[PFG_WARPS][MAXB * MAXB];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = blockIdx.x * PFG_WARPS + w;
  if (g >= ngroups) return;   // warp-uniform
  double* L = Ls[w];
  const int b1 = grp_b1[g], b2 = grp_b2[g];
  const int n1 = h.blk_sz[b1], n2 = b2 >= 0 ? h.blk_sz[b2] : 0;
  const int n = n1 + n2;
  const double* D1 = Sval + diag_off[b1];
  for (int t = lane; t < n1 * n1; t += 32) {
    const int i = t / n1, j = t - i * n1;
    if (j <= i) L[i * MAXB + j] = D1[t];
  }
  if (b2 >= 0) {
    const double* D2 = Sval + diag_off[b2];
    for (int t = lane; t < n2 * n2; t += 32) {
      const int i = t / n2, j = t - i * n2;
      if (j <= i) L[(n1 + i) * MAXB + n1 + j] = D2[t];
    }
    const int o12 = bsr_lookup(h, min(b1, b2), max(b1, b2));
    for (int t = lane; t < n2 * n1; t += 32) {
      const int i = t / n1, j = t - i * n1;
      // lower-left part = block (b2 rows, b1 cols); the stored upper block is (min, max)
      double v = 0.0;
      if (o12 >= 0) v = b1 < b2 ? Sval[o12 + j * n2 + i] : Sval[o12 + i * n1 + j];
      L[(n1 + i) * MAXB + j] = v;
    }
  }
  __syncwarp();
  for (int j = 0; j < n; ++j) {
    if (lane == 0) {
      double d = L[j * MAXB + j];
      for (int k = 0; k < j; ++k) d -= L[j * MAXB + k] * L[j * MAXB + k];
      L[j * MAXB + j] = sqrt(fmax(d, 1e-300));
    }
    __syncwarp();
    const int i = j + 1 + lane;
    if (i < n) {
      double s = L[i * MAXB + j];
      for (int k = 0; k < j; ++k) s -= L[i * MAXB + k] * L[j * MAXB + k];
      L[i * MAXB + j] = s / L[j * MAXB + j];
    }
    __syncwarp();
  }
  if (lane >= n) return;
  const int c = lane;
  double* out = Minv + (size_t)g * MAXB * MAXB;
  double y[MAXB];
  for (int i = 0; i < n; ++i) {
    double s = (i == c) ? 1.0 : 0.0;
    for (int k = 0; k < i; ++k) s -= L[i * MAXB + k] * y[k];
    y[i] = s / L[i * MAXB + i];
  }
  for (int i = n - 1; i >= 0; --i) {
    double s = y[i];
    for (int k = i + 1; k < n; ++k) s -= L[k * MAXB + i] * y[k];
    y[i] = s / L[i * MAXB + i];
  }
  for (int i = 0; i < n; ++i) out[i * MAXB + c] = y[i];
}

constexpr int PCG_MAX_CTAS = 256;
constexpr int PCG_FLAG_STRIDE = 32;
struct PcgState {
  // header: what the host reads back after a solve
  int iterations;
  int converged;
  double rr_final;                     // |r|^2 at exit (NaN -> the step is rejected)
  int deflated;                        // pcg_pipelined: 1 = solved with gauge deflation (0 when W^T S W was singular)
  long long prof[8];                  // CTA 0 / thread 0 clock64 totals per phase (OSFM_BA_TRACE)
  // per-CTA partial sums of the reduction riding on the barrier (double-buffered by generation parity; read and
  // written as 16-byte vectors, hence the alignment)
  alignas(16) double slot[2][PCG_MAX_CTAS][4];
  // wide payload of the deflated solver: 3 dot products + PCG_ND projections (double-buffered by generation parity)
  double slotx[2][PCG_MAX_CTAS][12];
  // the in-loop dot products of pcg_pipelined as flagged words (pcg_post_wide / pcg_collect_wide, pcg_post3 /
  // pcg_collect3): PCG_NW doubles per CTA, two words each, by value so that one warp reads a value of 32 CTAs in four
  // lines; double-buffered by exchange parity
  alignas(16) unsigned long long slotf[2][PCG_NW][PCG_MAX_CTAS][2];
  // their totals (pcg_collect_wide), one 128-byte line each: every CTA reads all of them
  alignas(128) unsigned long long totf[2][PCG_NW][16];
  // per-CTA arrival generation, one 128-byte line each (packed flags contend for one line on
  // every arrival; one line per CTA does not)
  unsigned flags[PCG_MAX_CTAS * PCG_FLAG_STRIDE];
};
constexpr size_t PCG_STATE_HEADER = offsetof(PcgState, slot);

// Where the resident variant keeps things in shared memory (byte offsets; host-computed, uniform).
struct PcgResident {
  const int* row_lo;   // [grid + 1] scalar-row range of every CTA (balanced by stored entries)
  int off_S, off_cols, off_rows;  // p at 0
  int max_rows;
};

__device__ __forceinline__ double ldcg_d(const double* p) { return __ldcg(p); }

// Grid barrier + all-reduce of NV = 2 or 3 doubles for a fully resident grid (grid <= #SMs, 1 CTA / SM).
// Every CTA publishes its partial sums in its own slot (double-buffered by generation parity) and
// release-stores its flag; every CTA then polls all flags (thread t polls CTA t) and sums the slots
// in a fixed order, so all CTAs get bit-identical totals and the result does not depend on timing.
// NV = 2 ignores c and leaves C unwritten: classic PCG reduces two sums, and carrying a third costs it registers.
template <int NV>
__device__ __forceinline__ void grid_reduce(PcgState* st, unsigned nblocks, unsigned& gen, double a, double b, double c,
                                            double& A, double& B, double& C, double (*red)[3]) {
  static_assert(NV == 2 || NV == 3, "two or three sums");
  ++gen;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
    if (NV == 3) c += __shfl_xor_sync(0xffffffffu, c, o);
  }
  if (lane == 0) { red[warp][0] = a; red[warp][1] = b; if (NV == 3) red[warp][2] = c; }
  __syncthreads();  // also: every global write of this CTA happens-before thread 0's release below
  if (threadIdx.x == 0) {
    double sa = 0.0, sb = 0.0, sc = 0.0;
    for (int w = 0; w < nwarps; ++w) { sa += red[w][0]; sb += red[w][1]; if (NV == 3) sc += red[w][2]; }
    double* sl = st->slot[gen & 1][blockIdx.x];
    __stcg(reinterpret_cast<double2*>(sl), make_double2(sa, sb));
    if (NV == 3) __stcg(sl + 2, sc);
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(&st->flags[blockIdx.x * PCG_FLAG_STRIDE]), "r"(gen) : "memory");
  }
  double va = 0.0, vb = 0.0, vc = 0.0;
  if (threadIdx.x < nblocks) {
    const long long t0 = clock64();
    unsigned cur;
    do {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(cur) : "l"(&st->flags[threadIdx.x * PCG_FLAG_STRIDE]) : "memory");
      if (clock64() - t0 > 8000000000LL) __trap();  // a protocol bug must not hang the GPU
    } while ((int)(cur - gen) < 0);  // monotonic: a fast CTA may already have published generation gen + 1
    const double* sl = st->slot[gen & 1][threadIdx.x];
    const double2 ab = __ldcg(reinterpret_cast<const double2*>(sl));
    va = ab.x; vb = ab.y;
    if (NV == 3) vc = __ldcg(sl + 2);
  }
  __syncthreads();  // red[] is free again; the acquires above order every thread's later loads
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    va += __shfl_xor_sync(0xffffffffu, va, o);
    vb += __shfl_xor_sync(0xffffffffu, vb, o);
    if (NV == 3) vc += __shfl_xor_sync(0xffffffffu, vc, o);
  }
  if (lane == 0) { red[warp][0] = va; red[warp][1] = vb; if (NV == 3) red[warp][2] = vc; }
  __syncthreads();
  double sa = 0.0, sb = 0.0, sc = 0.0;
  const int wmax = (int)((nblocks + 31) >> 5);
  for (int w = 0; w < wmax; ++w) { sa += red[w][0]; sb += red[w][1]; if (NV == 3) sc += red[w][2]; }
  A = sa; B = sb;
  if (NV == 3) C = sc;
  __syncthreads();
}

// z_G = Minv_G r_G for one group (one warp); returns this lane's contributions to r.z and r.r
__device__ __forceinline__ void pcg_apply_group(const BsrView& h, const PcgLayout& L, const double* Minv, int g, int lane,
                                                double rn, double* z, double* a_rz, double* a_rr, int n, int o_lane) {
  const double* M = Minv + (size_t)g * MAXB * MAXB;
  double s = 0.0;
  for (int j = 0; j < n; ++j) {
    const double rj = __shfl_sync(0xffffffffu, rn, j);
    if (lane < n) s += M[lane * MAXB + j] * rj;
  }
  if (lane < n) {
    z[o_lane] = s;
    *a_rz += s * rn;
    *a_rr += rn * rn;
  }
}

// RES = true: the CTA's slice of S (contiguous scalar rows, balanced by entries), its column indices
// (uint16) and the search direction p live in shared memory for the whole solve; an iteration then
// moves only the vectors through L2 (2 * nc doubles per CTA).  RES = false streams S from L2 / HBM.
template <bool RES>
__global__ void __launch_bounds__(PCG_THREADS, 1)
    pcg_persistent(const double* __restrict__ Spcg, PcgLayout L, BsrView h, const double* __restrict__ Minv,
                   const double* __restrict__ rhs, double* x, double* r, double* z, double* p0, double* p1, double* Ap,
                   PcgState* st, int nc, int max_iter, double tol2_rel, PcgResident R) {
  extern __shared__ __align__(16) unsigned char pcg_smem[];
  __shared__ double red[PCG_THREADS / 32][3];
  const int warps_per_cta = blockDim.x >> 5;
  const int warp = threadIdx.x >> 5;
  const int gw = blockIdx.x * warps_per_cta + warp;
  const int nw = gridDim.x * warps_per_cta;
  const int lane = threadIdx.x & 31;
  double* pbuf[2] = {p0, p1};
  unsigned bar_gen = 0;

  double* p_s = reinterpret_cast<double*>(pcg_smem);
  double* S_s = reinterpret_cast<double*>(pcg_smem + R.off_S);
  unsigned short* cols_s = reinterpret_cast<unsigned short*>(pcg_smem + R.off_cols);
  int* row_soff = reinterpret_cast<int*>(pcg_smem + R.off_rows);
  int* row_coff = row_soff + R.max_rows;
  int* row_len = row_coff + R.max_rows;
  int lo = 0, hi = 0;
  if (RES) {
    lo = R.row_lo[blockIdx.x];
    hi = R.row_lo[blockIdx.x + 1];
    if (hi > lo) {
      const int b_lo = L.row_of[lo], b_hi = L.row_of[hi - 1];
      const long long s_base = L.rowbase[b_lo] + (long long)(lo - h.blk_off[b_lo]) * L.row_M[b_lo];
      const long long s_end = L.rowbase[b_hi] + (long long)(hi - h.blk_off[b_hi]) * L.row_M[b_hi];
      const int c_base = L.cbase[b_lo], c_end = L.cbase[b_hi] + L.row_M[b_hi];
      for (int t = threadIdx.x; t < (int)(s_end - s_base); t += blockDim.x) S_s[t] = __ldcs(Spcg + s_base + t);
      for (int t = threadIdx.x; t < c_end - c_base; t += blockDim.x) cols_s[t] = (unsigned short)L.colidx[c_base + t];
      for (int t = threadIdx.x; t < hi - lo; t += blockDim.x) {
        const int i = lo + t, b = L.row_of[i], M = L.row_M[b];
        row_soff[t] = (int)(L.rowbase[b] + (long long)(i - h.blk_off[b]) * M - s_base);
        row_coff[t] = L.cbase[b] - c_base;
        row_len[t] = M;
      }
    }
  }

  // ---- init: x = 0, r = rhs, z = M^-1 r, p_old = 0, rz, bb ----
  double rz_cur, bb;
  {
    double a_rz = 0.0, a_rr = 0.0;
    for (int g = gw; g < L.ngroups; g += nw) {
      const int b1 = L.grp_b1[g], b2 = L.grp_b2[g];
      const int n1 = h.blk_sz[b1], n2 = b2 >= 0 ? h.blk_sz[b2] : 0, n = n1 + n2;
      const int o = lane < n1 ? h.blk_off[b1] + lane : (lane < n ? h.blk_off[b2] + lane - n1 : 0);
      double rn = 0.0;
      if (lane < n) {
        rn = rhs[o];
        x[o] = 0.0;
        r[o] = rn;
      }
      pcg_apply_group(h, L, Minv, g, lane, rn, z, &a_rz, &a_rr, n, o);
      if (lane < n) p0[o] = 0.0;
    }
    double unused;
    grid_reduce<2>(st, gridDim.x, bar_gen, a_rz, a_rr, 0.0, rz_cur, bb, unused, red);
  }
  const double tol2 = tol2_rel * bb;
  double rr = bb;
  int it = 0;
  if (bb > 0.0) {
    double beta = 0.0;  // p_1 = z_0
    for (; it < max_iter; ++it) {
      const int cur = it & 1, nxt = cur ^ 1;
      const double* pold = pbuf[cur];
      double* pnew = pbuf[nxt];
      // ---- phase A: p = z + beta p_old (on the fly), Ap = S p, pAp ----
      double a_pAp = 0.0;
      const long long tk0 = clock64();
      long long tk1 = tk0;
      if (RES) {
        for (int c = threadIdx.x; c < nc; c += blockDim.x) p_s[c] = ldcg_d(&z[c]) + beta * ldcg_d(&pold[c]);
        __syncthreads();
        tk1 = clock64();
        for (int t = warp; t < hi - lo; t += warps_per_cta) {
          const double* vals = S_s + row_soff[t];
          const unsigned short* cols = cols_s + row_coff[t];
          const int M = row_len[t];
          double s0 = 0.0, s1 = 0.0;
          int q = lane;
          for (; q + 32 < M; q += 64) {
            s0 += vals[q] * p_s[cols[q]];
            s1 += vals[q + 32] * p_s[cols[q + 32]];
          }
          if (q < M) s0 += vals[q] * p_s[cols[q]];
          double s = s0 + s1;
#pragma unroll
          for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
          if (lane == 0) {
            const int i = lo + t;
            const double pi = p_s[i];
            pnew[i] = pi;
            Ap[i] = s;
            a_pAp += s * pi;
          }
        }
      } else {
        for (int i = gw; i < nc; i += nw) {
          const int b = L.row_of[i];
          const int rr_ = i - h.blk_off[b];
          const int M = L.row_M[b];
          const double* vals = Spcg + L.rowbase[b] + (size_t)rr_ * M;
          const int* cols = L.colidx + L.cbase[b];
          double s = 0.0;
          for (int q = lane; q < M; q += 32) {
            const int c = cols[q];
            s += vals[q] * (ldcg_d(&z[c]) + beta * ldcg_d(&pold[c]));
          }
#pragma unroll
          for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
          if (lane == 0) {
            const double pi = ldcg_d(&z[i]) + beta * ldcg_d(&pold[i]);
            pnew[i] = pi;
            Ap[i] = s;
            a_pAp += s * pi;
          }
        }
      }
      double pAp, unused;
      const long long tk2 = clock64();
      grid_reduce<2>(st, gridDim.x, bar_gen, a_pAp, 0.0, 0.0, pAp, unused, unused, red);
      const long long tk3 = clock64();
      // ---- phase B: x += alpha p ; r -= alpha Ap ; z = M^-1 r ; rz_new, rr ----
      const double alpha = rz_cur / pAp;
      double a_rz = 0.0, a_rr = 0.0;
      for (int g = gw; g < L.ngroups; g += nw) {
        const int b1 = L.grp_b1[g], b2 = L.grp_b2[g];
        const int n1 = h.blk_sz[b1], n2 = b2 >= 0 ? h.blk_sz[b2] : 0, n = n1 + n2;
        const int o = lane < n1 ? h.blk_off[b1] + lane : (lane < n ? h.blk_off[b2] + lane - n1 : 0);
        double rn = 0.0;
        if (lane < n) {
          x[o] += alpha * ldcg_d(&pnew[o]);
          rn = r[o] - alpha * ldcg_d(&Ap[o]);
          r[o] = rn;
        }
        pcg_apply_group(h, L, Minv, g, lane, rn, z, &a_rz, &a_rr, n, o);
      }
      double rz_new;
      const long long tk4 = clock64();
      grid_reduce<2>(st, gridDim.x, bar_gen, a_rz, a_rr, 0.0, rz_new, rr, unused, red);
      if (blockIdx.x == 0 && threadIdx.x == 0) {
        const long long tk5 = clock64();
        st->prof[0] += tk1 - tk0; st->prof[1] += tk2 - tk1; st->prof[2] += tk3 - tk2; st->prof[3] += tk4 - tk3;
        st->prof[4] += tk5 - tk4;
      }
      if (!(rr == rr) || rr <= tol2) { ++it; break; }  // NaN (step will be rejected) or converged
      beta = rz_new / rz_cur;
      rz_cur = rz_new;
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) { st->iterations = it; st->rr_final = rr; st->converged = (rr <= tol2) ? 1 : 0; }
}


// ---------------------------------------------------------------------------
// Pipelined PCG (Ghysels & Vanroose 2014, preconditioned pipelined CG): the global reduction of an
// iteration's dot products runs during its mat-vec, which does not need them.  There is no grid barrier
// in the loop: the dot products and m travel as flagged words (flag_put / flag_wait_all), a CTA starts its
// mat-vec as soon as the entries of m its columns need have arrived and collects the totals after it.
// Every CTA owns whole
// preconditioner groups: their rows of S, the groups' inverse blocks and all eight recurrence
// vectors of those rows stay in shared memory / registers for the whole solve; the only vector that
// moves through L2 is m = M^-1 w (nc flagged pairs, double-buffered by iteration parity): a
// CTA gathers, per column list of its block rows, the entries of m those columns need into a packed copy
// (mp), so the rows then stream S and mp from shared memory without bank conflicts.  The two block rows
// of a group usually store the same block columns (a camera and the rig instance of its only shot); they
// then share one column list and one packed copy.
// The recurrences drift from the true residual earlier than classic CG; the kernel reports
// converged = 0 on stagnation / breakdown and the host re-solves with pcg_persistent.
// ---------------------------------------------------------------------------
struct PcgPipe {   // the layout of plan_pcg_pipelined (ba_pcg_plan.h)
  const int* grp_lo;  // [grid + 1] group range of every CTA
  const char* grp_shared;  // [ngroups] 1 = the two block rows of the group have one column list
  int off_S, off_Minv, off_vec, off_cols, off_rows;  // byte offsets into dynamic shared memory; mp at 0
  int off_defl;       // [2][PCG_ND][max_rows] doubles: own rows of W and of S W
  const double* Wdef; // [PCG_ND][nc] deflation vectors (scaled variables), or null: plain PCG
  int max_cols;
  int max_rows, max_groups;
};

// Deflation vectors of the reduced system: the similarity gauge of the rig instances at the current poses.
// Instance block = [r (camera -> world angle-axis) | t (camera origin)], x_cam = R(-r) (X - t).  Under the world map
// X -> s Q X + T:  t -> s Q t + T,  R(r) -> Q R(r), i.e. to first order
//   translation e_a:  dt = e_a;   rotation w = e_a:  dr = J_l(r)^-1 e_a, dt = e_a x t;   scale:  dt = t,
// in the Jacobi-scaled variables (x = scale * x_scaled).  Intrinsics, rig cameras and ext blocks do not move.
// When nothing fixes the gauge these seven directions carry the smallest eigenvalues of the reduced system
// (only the LM damping acts on them); with priors / fixed shots they are ordinary vectors and deflating them is harmless.
__global__ void pcg_gauge_vectors(int NI, const int* __restrict__ inst_poff, const double* __restrict__ inst,
                                  const double* __restrict__ scale, int nc, double* __restrict__ W) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= NI) return;
  const int c0 = inst_poff[i];
  if (c0 < 0) return;
  const double r[3] = {inst[6 * (size_t)i], inst[6 * (size_t)i + 1], inst[6 * (size_t)i + 2]};
  const double t[3] = {inst[6 * (size_t)i + 3], inst[6 * (size_t)i + 4], inst[6 * (size_t)i + 5]};
  // J_l^-1 = I - K / 2 + g K^2,  K = [r]x,  g = 1 / th^2 - (1 + cos th) / (2 th sin th)
  const double th2 = r[0] * r[0] + r[1] * r[1] + r[2] * r[2];
  double g = 1.0 / 12.0;
  if (th2 > 1e-8) {
    const double th = sqrt(th2);
    g = 1.0 / th2 - (1.0 + cos(th)) / (2.0 * th * sin(th));
  }
  const double K[9] = {0.0, -r[2], r[1], r[2], 0.0, -r[0], -r[1], r[0], 0.0};
  double J[9];
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < 3; ++b) {
      double k2 = 0.0;
      for (int c = 0; c < 3; ++c) k2 += K[a * 3 + c] * K[c * 3 + b];
      J[a * 3 + b] = (a == b ? 1.0 : 0.0) - 0.5 * K[a * 3 + b] + g * k2;
    }
  double inv_s[6];
  for (int j = 0; j < 6; ++j) inv_s[j] = 1.0 / scale[c0 + j];
  for (int a = 0; a < 3; ++a) {
    W[(size_t)a * nc + c0 + 3 + a] = inv_s[3 + a];                                   // translation
    for (int b = 0; b < 3; ++b) W[(size_t)(3 + a) * nc + c0 + b] = J[b * 3 + a] * inv_s[b];   // rotation: dr
    // e_a x t
    const int a1 = (a + 1) % 3, a2 = (a + 2) % 3;
    W[(size_t)(3 + a) * nc + c0 + 3 + a1] = -t[a2] * inv_s[3 + a1];
    W[(size_t)(3 + a) * nc + c0 + 3 + a2] = t[a1] * inv_s[3 + a2];
    W[(size_t)6 * nc + c0 + 3 + a] = t[a] * inv_s[3 + a];                            // scale
  }
}

// warp i sums value i over the CTAs' rows of gather: lane l takes CTAs l, l + 32, ... in order, then a fixed tree
__device__ __forceinline__ void wide_column_sums(unsigned nblocks, double* vals /* [PCG_NW] */, const double* gather) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (warp < PCG_NW) {
    double sa = 0.0;
    for (unsigned c = lane; c < nblocks; c += 32) sa += gather[c * PCG_NW + warp];
#pragma unroll
    for (int o = 16; o; o >>= 1) sa += __shfl_xor_sync(0xffffffffu, sa, o);
    if (lane == 0) vals[warp] = sa;
  }
  __syncthreads();
}

// The grid_reduce barrier with PCG_NW doubles per CTA.  Built for latency, the only thing that matters here, and around one
// measurement: arguments and results must not live in local memory -- every poll of the barrier invalidates L1
// (ld.acquire -> CCTL.IVALL), so a stack array written before the call and read inside it is an L2 round trip (the
// version with in[] / out[] arrays spent 2.9k + 2.5k clocks per call on that).  Protocol: the owners of the CTA's rows
// (threads < nactive) have written their PCG_NW contributions to inrow[thread][.] in shared memory; warp i sums
// column i and publishes it in the CTA's slot; thread 0 releases the flag; thread t < nblocks acquires CTA t's flag,
// loads its slot with independent 16-byte loads and drops it into gather[t][.]; warp i sums column i over the CTAs
// in a fixed order (bit-identical totals in every CTA) into vals[i], which the caller reads.  Not inlined: the kernel
// calls it from six places and the loop body has to stay resident in the instruction cache.  The loop of pcg_pipelined
// exchanges its dot products through flagged words instead (pcg_post_wide / pcg_collect_wide below); this barrier
// serves the once-per-solve exchanges, where the plain stores it orders are what the caller reads next.
__device__ __noinline__ void grid_reduce_wide(PcgState* st, unsigned nblocks, unsigned* gen_io, double* vals /* [PCG_NW] */,
                                              double* gather /* [nblocks][PCG_NW] */, const double* inrow /* [nactive][PCG_NW] */,
                                              int nactive) {
  const unsigned gen = ++(*gen_io);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();   // inrow is complete
  if (warp < PCG_NW) {
    double sa = 0.0;
    for (int r = lane; r < nactive; r += 32) sa += inrow[r * PCG_NW + warp];
#pragma unroll
    for (int o = 16; o; o >>= 1) sa += __shfl_xor_sync(0xffffffffu, sa, o);
    if (lane == 0) __stcg(&st->slotx[gen & 1][blockIdx.x][warp], sa);
  }
  __syncthreads();  // the slot (and every other global write of this CTA) happens-before thread 0's release
  if (threadIdx.x == 0)
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(&st->flags[blockIdx.x * PCG_FLAG_STRIDE]), "r"(gen) : "memory");
  if (threadIdx.x < nblocks) {
    const long long t0 = clock64();
    unsigned cur;
    do {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(cur) : "l"(&st->flags[threadIdx.x * PCG_FLAG_STRIDE]) : "memory");
      if (clock64() - t0 > 8000000000LL) __trap();
    } while ((int)(cur - gen) < 0);
    const double2* sl = reinterpret_cast<const double2*>(st->slotx[gen & 1][threadIdx.x]);
    double2 v[PCG_NW / 2];
#pragma unroll
    for (int i = 0; i < PCG_NW / 2; ++i) v[i] = __ldcg(sl + i);
    double2* dst = reinterpret_cast<double2*>(gather + threadIdx.x * PCG_NW);
#pragma unroll
    for (int i = 0; i < PCG_NW / 2; ++i) dst[i] = v[i];
  }
  __syncthreads();
  wide_column_sums(nblocks, vals, gather);
}
static_assert(PCG_THREADS / 32 >= PCG_NW, "a warp per value of the wide barrier");

// Flagged words (the LL protocol of NCCL): a double travels as two 8-byte words {low 32 bits | gen << 32} and
// {high 32 bits | gen << 32}.  Each word is single-copy atomic, so a reader that sees gen in both words has the value
// that was stored with it -- no fence before the store, no acquire on the load, and a relaxed load polls without
// invalidating L1 (ld.acquire does, CCTL.IVALL).  The pair is stored as one v2 store, but nothing relies on 16-byte
// atomicity (the PTX memory model does not promise it): the words are checked one by one.  A reader must never find
// the generation it waits for in a word before that word is meant for it: the callers zero the buffers before a solve
// and count gen up from 1 within it.
__device__ __forceinline__ void flag_put(unsigned long long* p, double v, unsigned gen) {
  const unsigned long long b = (unsigned long long)__double_as_longlong(v), g = (unsigned long long)gen << 32;
  asm volatile("st.relaxed.gpu.global.v2.b64 [%0], {%1, %2};" ::"l"(p), "l"((b & 0xffffffffull) | g), "l"((b >> 32) | g)
               : "memory");
}
__device__ __forceinline__ ulonglong2 flag_ld(const unsigned long long* p) {
  ulonglong2 w;
  asm volatile("ld.relaxed.gpu.global.v2.b64 {%0, %1}, [%2];" : "=l"(w.x), "=l"(w.y) : "l"(p));
  return w;
}
__device__ __forceinline__ bool flag_ok(ulonglong2 w, unsigned gen) {
  return (unsigned)(w.x >> 32) == gen && (unsigned)(w.y >> 32) == gen;
}
__device__ __forceinline__ double flag_val(ulonglong2 w) {
  return __longlong_as_double((long long)((w.x & 0xffffffffull) | (w.y << 32)));
}
// Waits until the N loaded pairs w[i] (of addr(i)) all carry gen.  The late ones are re-loaded together, so a wait costs
// one round trip per poll however many of them were late -- one by one, every stale pair behind the first late one
// would cost another.  grid_reduce's clock budget.  A pair the caller has no address for is set to carry gen.
template <int N, class Addr>
__device__ __forceinline__ void flag_wait_all(ulonglong2 (&w)[N], Addr addr, unsigned gen) {
  bool ok = true;
#pragma unroll
  for (int i = 0; i < N; ++i) ok = ok && flag_ok(w[i], gen);
  if (ok) return;
  const long long t0 = clock64();
  do {
#pragma unroll
    for (int i = 0; i < N; ++i)
      if (!flag_ok(w[i], gen)) w[i] = flag_ld(addr(i));
    if (clock64() - t0 > 8000000000LL) __trap();  // a protocol bug must not hang the GPU
    ok = true;
#pragma unroll
    for (int i = 0; i < N; ++i) ok = ok && flag_ok(w[i], gen);
  } while (!ok);
}

// The two halves of the wide barrier for the loop of pcg_pipelined, with its PCG_NW doubles per CTA in flagged words
// (st->slotf[gen & 1]).  pcg_post_wide: warp i sums column i of inrow (same order as grid_reduce_wide) and stores it;
// no fence, no flag, no wait.  pcg_collect_wide, called later: value i is summed over the CTAs by ONE warp of the grid
// (warp i / nblocks of CTA i % nblocks), in grid_reduce_wide's order -- lane l takes CTAs l, l + 32, ... in order, then
// a fixed tree -- and published as a flagged total, which every CTA then reads: bit-identical totals everywhere, but
// every CTA reads PCG_NW totals instead of every slot of the grid (132 x 132 x 160 bytes per iteration on C4, read
// from the same few hundred lines at once, which made the collection cost more than the barrier it replaced).
// Reuse: a slot (and a total) of gen + 2 is written only after its writer has read the totals of gen + 1; they exist
// only once every CTA has posted gen + 1, which each does after it has read the totals of gen, and those were
// published after every slot of gen had been read.  No reader of gen can see it overwritten.
__device__ __noinline__ void pcg_post_wide(PcgState* st, unsigned gen, const double* inrow /* [nactive][PCG_NW] */,
                                           int nactive) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();   // inrow is complete
  if (warp < PCG_NW) {
    double sa = 0.0;
    for (int r = lane; r < nactive; r += 32) sa += inrow[r * PCG_NW + warp];
#pragma unroll
    for (int o = 16; o; o >>= 1) sa += __shfl_xor_sync(0xffffffffu, sa, o);
    if (lane == 0) flag_put(st->slotf[gen & 1][warp][blockIdx.x], sa, gen);
  }
}
__device__ __noinline__ void pcg_collect_wide(PcgState* st, unsigned nblocks, unsigned gen, double* vals /* [PCG_NW] */) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned i = warp * nblocks + blockIdx.x;   // the value this warp sums, if any
  if (i < PCG_NW) {
    const unsigned long long(*sl)[2] = st->slotf[gen & 1][i];
    const unsigned long long none = (unsigned long long)gen << 32;   // past the last CTA: nothing to wait for
    constexpr int K = PCG_MAX_CTAS / 32;
    ulonglong2 v[K];
#pragma unroll
    for (int k = 0; k < K; ++k) v[k] = lane + 32 * k < (int)nblocks ? flag_ld(sl[lane + 32 * k]) : make_ulonglong2(none, none);
    flag_wait_all(v, [&](int k) { return sl[lane + 32 * k]; }, gen);
    double sa = 0.0;
#pragma unroll
    for (int k = 0; k < K; ++k)
      if (lane + 32 * k < (int)nblocks) sa += flag_val(v[k]);
#pragma unroll
    for (int o = 16; o; o >>= 1) sa += __shfl_xor_sync(0xffffffffu, sa, o);
    if (lane == 0) flag_put(st->totf[gen & 1][i], sa, gen);
  }
  if (threadIdx.x < PCG_NW) {
    ulonglong2 t[1] = {flag_ld(st->totf[gen & 1][threadIdx.x])};
    flag_wait_all(t, [&](int) { return st->totf[gen & 1][threadIdx.x]; }, gen);
    vals[threadIdx.x] = flag_val(t[0]);
  }
  __syncthreads();
}
static_assert(PCG_MAX_CTAS % 32 == 0 && PCG_NW <= PCG_THREADS / 32, "pcg_collect_wide: whole warps of slots, a warp per value");

// grid_reduce<3> split the same way, for the loop of pcg_pipelined without deflation: the same sums in the same order
// (bit-identical totals), the CTA's three values in flagged words of st->slotf[gen & 1] instead of a released slot.
__device__ __forceinline__ void pcg_post3(PcgState* st, unsigned gen, double a, double b, double c, double (*red)[3]) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
    c += __shfl_xor_sync(0xffffffffu, c, o);
  }
  if (lane == 0) { red[warp][0] = a; red[warp][1] = b; red[warp][2] = c; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double sa = 0.0, sb = 0.0, sc = 0.0;
    for (int w = 0; w < nwarps; ++w) { sa += red[w][0]; sb += red[w][1]; sc += red[w][2]; }
    flag_put(st->slotf[gen & 1][0][blockIdx.x], sa, gen);
    flag_put(st->slotf[gen & 1][1][blockIdx.x], sb, gen);
    flag_put(st->slotf[gen & 1][2][blockIdx.x], sc, gen);
  }
  __syncthreads();   // red[] is read by thread 0 above and rewritten by pcg_collect3
}
__device__ __forceinline__ void pcg_collect3(PcgState* st, unsigned nblocks, unsigned gen, double& A, double& B, double& C,
                                             double (*red)[3]) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double va = 0.0, vb = 0.0, vc = 0.0;
  if (threadIdx.x < nblocks) {
    const auto sl = st->slotf[gen & 1];
    ulonglong2 v[3] = {flag_ld(sl[0][threadIdx.x]), flag_ld(sl[1][threadIdx.x]), flag_ld(sl[2][threadIdx.x])};
    flag_wait_all(v, [&](int i) { return sl[i][threadIdx.x]; }, gen);
    va = flag_val(v[0]); vb = flag_val(v[1]); vc = flag_val(v[2]);
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    va += __shfl_xor_sync(0xffffffffu, va, o);
    vb += __shfl_xor_sync(0xffffffffu, vb, o);
    vc += __shfl_xor_sync(0xffffffffu, vc, o);
  }
  if (lane == 0) { red[warp][0] = va; red[warp][1] = vb; red[warp][2] = vc; }
  __syncthreads();
  double sa = 0.0, sb = 0.0, sc = 0.0;
  const int wmax = (int)((nblocks + 31) >> 5);
  for (int w = 0; w < wmax; ++w) { sa += red[w][0]; sb += red[w][1]; sc += red[w][2]; }
  A = sa; B = sb; C = sc;
  __syncthreads();
}

__global__ void __launch_bounds__(PCG_THREADS, 1)
    pcg_pipelined(const double* __restrict__ Spcg, PcgLayout L, BsrView h, const double* __restrict__ Minv,
                  const double* __restrict__ rhs, double* x_out, unsigned long long* mflag, PcgState* st,
                  int nc, int max_iter, double tol2_rel, PcgPipe R) {
  extern __shared__ __align__(16) unsigned char pcg_smem[];
  __shared__ double red[PCG_THREADS / 32][3];
  __shared__ int s_nrows, s_ncols;
  const int nwarps = blockDim.x >> 5, warp = threadIdx.x >> 5, lane = threadIdx.x & 31, tid = threadIdx.x;
  double* mp_s = reinterpret_cast<double*>(pcg_smem);  // packed m per owned block row: mp_s[coff + q] = m[cols[q]]
  double* S_s = reinterpret_cast<double*>(pcg_smem + R.off_S);
  double* Minv_s = reinterpret_cast<double*>(pcg_smem + R.off_Minv);
  double* w_s = reinterpret_cast<double*>(pcg_smem + R.off_vec);  // input of the group solves
  double* n_s = w_s + R.max_rows;                                  // mat-vec output
  double* g_s = n_s + R.max_rows;                                  // group-solve output (u, then m of the own rows)
  unsigned short* cols_s = reinterpret_cast<unsigned short*>(pcg_smem + R.off_cols);
  int* row_soff = reinterpret_cast<int*>(pcg_smem + R.off_rows);
  int* row_coff = row_soff + R.max_rows;
  int* row_len = row_coff + R.max_rows;
  int* row_gidx = row_len + R.max_rows;
  int* grp_row0 = row_gidx + R.max_rows;  // [max_groups + 1]
  int* grp_moff = grp_row0 + R.max_groups + 1;  // [max_groups + 1] offset of the group's n x n inverse in Minv_s
  // mat-vec units: up to three consecutive rows with one column list (they share its packed m)
  int* unit_soff = grp_moff + R.max_groups + 1;  // [max_rows] each
  int* unit_coff = unit_soff + R.max_rows;
  int* unit_len = unit_coff + R.max_rows;
  int* unit_lr0 = unit_len + R.max_rows;
  int* unit_nr = unit_lr0 + R.max_rows;
  __shared__ double part_s[PCG_THREADS / 8][3];   // per 8-lane group: partial sums of its unit's rows
  __shared__ int s_nunits;
  // deflation (R.Wdef != null): own rows of W and A W, (W^T A W)^-1, W^T b projected through it
  __shared__ double redw[PCG_THREADS / 32][PCG_NW];
  __shared__ double Einv_s[PCG_ND * PCG_ND], c0_s[PCG_ND], tc_s[PCG_ND];
  __shared__ int s_defl;
  double* Wd_s = reinterpret_cast<double*>(pcg_smem + R.off_defl);
  double* AW_s = Wd_s + PCG_ND * R.max_rows;
  double* gather_s = AW_s + PCG_ND * R.max_rows;   // [gridDim.x][PCG_NW]: the slots of all CTAs on the wide barrier
  double* inrow_s = gather_s + PCG_NW * gridDim.x; // [max_rows][PCG_NW]: what the owners of the rows put on it
  double* wide_s = &redw[0][0];                    // [PCG_NW]: its totals
  const int MR = R.max_rows;
  unsigned bar_gen = 0;

  const int g_lo = R.grp_lo[blockIdx.x], g_hi = R.grp_lo[blockIdx.x + 1], ng = g_hi - g_lo;
  if (tid == 0) {
    int lr = 0, s_off = 0, c_off = 0, m_off = 0;
    for (int g = g_lo; g < g_hi; ++g) {
      grp_row0[g - g_lo] = lr;
      grp_moff[g - g_lo] = m_off;
      const int lr0 = lr;
      for (int k = 0; k < 2; ++k) {
        const int b = k ? L.grp_b2[g] : L.grp_b1[g];
        if (b < 0) continue;
        const int n = h.blk_sz[b], M = L.row_M[b];
        if (k && R.grp_shared[g]) c_off -= M;   // the second block row reads the first one's column list
        for (int r = 0; r < n; ++r, ++lr) {
          row_soff[lr] = s_off + r * M;
          row_coff[lr] = c_off;
          row_len[lr] = M;
          row_gidx[lr] = h.blk_off[b] + r;
        }
        s_off += n * M;
        c_off += M;
      }
      m_off += (lr - lr0) * (lr - lr0);
    }
    grp_row0[ng] = lr;
    grp_moff[ng] = m_off;
    s_nrows = lr;
    s_ncols = c_off;
    int nu = 0;
    for (int r0 = 0; r0 < lr;) {
      int nr = 1;  // rows r0 .. r0 + nr - 1 with one column list, consecutive in S_s (across the block rows of a group)
      while (nr < 3 && r0 + nr < lr && row_coff[r0 + nr] == row_coff[r0] && row_soff[r0 + nr] == row_soff[r0] + nr * row_len[r0]) ++nr;
      unit_soff[nu] = row_soff[r0]; unit_coff[nu] = row_coff[r0]; unit_len[nu] = row_len[r0]; unit_lr0[nu] = r0; unit_nr[nu] = nr;
      ++nu;
      r0 += nr;
    }
    s_nunits = nu;
  }
  __syncthreads();
  const int nrows = s_nrows, ncols = s_ncols;
  for (int lr = warp; lr < nrows; lr += nwarps) {
    const int i = row_gidx[lr], b = L.row_of[i], M = row_len[lr];
    const double* src = Spcg + L.rowbase[b] + (long long)(i - h.blk_off[b]) * M;
    for (int q = lane; q < M; q += 32) S_s[row_soff[lr] + q] = __ldcs(src + q);
    // the first row of a block row that owns its column list (not the second block row of a shared group)
    if (i == h.blk_off[b] && (lr == 0 || row_coff[lr] != row_coff[lr - 1])) {
      const int* csrc = L.colidx + L.cbase[b];
      for (int q = lane; q < M; q += 32) cols_s[row_coff[lr] + q] = (unsigned short)csrc[q];
    }
  }
  for (int gl = warp; gl < ng; gl += nwarps) {   // the group inverses, packed at n x n
    const int n = grp_row0[gl + 1] - grp_row0[gl];
    const double* src = Minv + (size_t)(g_lo + gl) * MAXB * MAXB;
    for (int t = lane; t < n * n; t += 32) Minv_s[grp_moff[gl] + t] = src[(t / n) * MAXB + t % n];
  }

  // group solve: g_s[rows of g] = Minv_g * w_s[rows of g], published as flagged words of generation gen in the m buffer
  // of its parity (mflag[gen & 1][column][2], zeroed before the solve)
  auto group_solve = [&](unsigned gen) {
    unsigned long long* publish = mflag + (size_t)(gen & 1) * 2 * nc;
    for (int gl = warp; gl < ng; gl += nwarps) {
      const int r0 = grp_row0[gl], n = grp_row0[gl + 1] - r0;
      const double* M = Minv_s + grp_moff[gl];
      double sv = 0.0;
      if (lane < n)
        for (int j = 0; j < n; ++j) sv += M[lane * n + j] * w_s[r0 + j];
      if (lane < n) {
        g_s[r0 + lane] = sv;
        flag_put(publish + 2 * row_gidx[r0 + lane], sv, gen);
      }
    }
  };
  // n_s[lr] = (S m)[row lr], m packed per block row in mp_s.  The mat-vec is bound by shared-memory
  // bandwidth, so a lane multiplies one loaded m entry into up to three rows (a unit) and the 64
  // eight-lane groups of the CTA split the units' columns among them; partial sums meet in part_s.
  auto matvec = [&]() {
    const int nunits = s_nunits;
    const int gidx = tid >> 3, l = tid & 7, ngroups8 = blockDim.x >> 3;
    const int gpu = max(1, ngroups8 / nunits);   // groups per unit
    for (int ub = 0; ub < nunits; ub += ngroups8) {   // one pass unless a CTA has more than 64 units
      const int upass = min(nunits - ub, ngroups8 / gpu);   // units handled in this pass
      const int ul = gidx / gpu, sub = gidx - ul * gpu;
      const int u = ub + ul;
      double a0 = 0.0, a1 = 0.0, a2 = 0.0;
      const bool on = ul < upass;
      if (on) {
        const int M = unit_len[u], nr = unit_nr[u];
        const double* v0 = S_s + unit_soff[u];
        const double* v1 = v0 + (nr > 1 ? M : 0);
        const double* v2 = v0 + (nr > 2 ? 2 * M : 0);
        const double* mp = mp_s + unit_coff[u];
        const int step = gpu * 8;
        int q = sub * 8 + l;
        for (; q + step < M; q += 2 * step) {
          const double m0 = mp[q], m1 = mp[q + step];
          a0 += v0[q] * m0; a1 += v1[q] * m0; a2 += v2[q] * m0;
          a0 += v0[q + step] * m1; a1 += v1[q + step] * m1; a2 += v2[q + step] * m1;
        }
        if (q < M) { const double m0 = mp[q]; a0 += v0[q] * m0; a1 += v1[q] * m0; a2 += v2[q] * m0; }
      }
#pragma unroll
      for (int o = 4; o; o >>= 1) {
        a0 += __shfl_xor_sync(0xffffffffu, a0, o);
        a1 += __shfl_xor_sync(0xffffffffu, a1, o);
        a2 += __shfl_xor_sync(0xffffffffu, a2, o);
      }
      if (l == 0) { part_s[gidx][0] = a0; part_s[gidx][1] = a1; part_s[gidx][2] = a2; }
      __syncthreads();
      if (tid < upass * 3) {
        const int uu = tid / 3, r = tid - uu * 3;
        const int u2 = ub + uu;
        if (r < unit_nr[u2]) {
          double sv = 0.0;
          for (int g2 = 0; g2 < gpu; ++g2) sv += part_s[uu * gpu + g2][r];
          n_s[unit_lr0[u2] + r] = sv;
        }
      }
      __syncthreads();
    }
  };
  // mp_s[e] = src[cols_s[e]] for every column entry of the owned block rows (gathers from L2, 8 in flight)
  auto stage = [&](const double* src) {
    const int bd = blockDim.x;
    for (int e = tid; e < ncols; e += 8 * bd) {
      double a[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) a[k] = (e + k * bd < ncols) ? ldcg_d(src + cols_s[e + k * bd]) : 0.0;
#pragma unroll
      for (int k = 0; k < 8; ++k)
        if (e + k * bd < ncols) mp_s[e + k * bd] = a[k];
    }
  };
  // the same for the m that group_solve(gen) published: each entry is waited for on its own, so the gathers of a CTA
  // need only the CTAs that own its columns to have published, not the whole grid
  auto stage_m = [&](unsigned gen) {
    const unsigned long long* src = mflag + (size_t)(gen & 1) * 2 * nc;
    const int bd = blockDim.x;
    for (int e = tid; e < ncols; e += 8 * bd) {
      const unsigned long long none = (unsigned long long)gen << 32;   // past the end: nothing to wait for
      ulonglong2 a[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) a[k] = e + k * bd < ncols ? flag_ld(src + 2 * cols_s[e + k * bd]) : make_ulonglong2(none, none);
      flag_wait_all(a, [&](int k) { return src + 2 * cols_s[e + k * bd]; }, gen);
#pragma unroll
      for (int k = 0; k < 8; ++k)
        if (e + k * bd < ncols) mp_s[e + k * bd] = flag_val(a[k]);
    }
  };

  // ---- deflation set-up: A W (PCG_ND mat-vecs, no barrier: W is known everywhere), E = W^T A W, W^T b ----
  // Deflated CG (Saad, Yeung, Erhel, Guyomarc'h 2000) in its projected form: with Q = W E^-1 W^T and P = I - A Q solve
  // P A y = P b by (pipelined) PCG, then x = Q b + (I - Q A) y.  P A is symmetric positive semi-definite and the true
  // residual b - A x equals the residual of the projected system, so the stopping rule is unchanged.  The projection
  // of a mat-vec, A m -> A m - A W E^-1 (A W)^T m, needs the PCG_ND numbers (A W)^T m of the vector m the barrier
  // exchanges anyway: they ride on that barrier, an iteration still costs one.
  const bool mine = tid < nrows;
  const int gi = mine ? row_gidx[tid] : 0;
  const double bi = mine ? rhs[gi] : 0.0;
  bool defl = R.Wdef != nullptr;
  double bb;
  if (defl) {
    __syncthreads();   // S_s / cols_s of my rows were loaded by other warps
#pragma unroll 1
    for (int j = 0; j < PCG_ND; ++j) {
      if (mine) Wd_s[j * MR + tid] = R.Wdef[(size_t)j * nc + gi];
      stage(R.Wdef + (size_t)j * nc);
      __syncthreads();
      matvec();
      __syncthreads();
      if (mine) AW_s[j * MR + tid] = n_s[tid];
      __syncthreads();
    }
    // 28 entries of the symmetric E, W^T b (7), b^T b: four wide reductions
    double E[PCG_ND * PCG_ND], wb[PCG_ND];
    // the 36 totals wait in Einv_s (49 doubles, written only once thread 0 has read them): an array of them in
    // registers, live across the grid_reduce_wide calls, does not fit the kernel's 128 registers
    double* collected = Einv_s;
    for (int pass = 0; pass < 4; ++pass) {
#pragma unroll
      for (int q = 0; q < PCG_NW; ++q) {
        const int idx = pass * PCG_NW + q;   // 0..27: E(a <= b) row-major upper; 28..34: W^T b; 35: b^T b
        double val = 0.0;
        if (mine) {
          if (idx < 28) {
            int a = 0, rem = idx;
            while (rem >= PCG_ND - a) { rem -= PCG_ND - a; ++a; }
            const int b2 = a + rem;
            val = Wd_s[a * MR + tid] * AW_s[b2 * MR + tid];
          } else if (idx < 35) {
            val = Wd_s[(idx - 28) * MR + tid] * bi;
          } else if (idx == 35) {
            val = bi * bi;
          }
        }
        if (mine) inrow_s[tid * PCG_NW + q] = val;
      }
      grid_reduce_wide(st, gridDim.x, &bar_gen, wide_s, gather_s, inrow_s, nrows);
      if (tid < PCG_NW && pass * PCG_NW + tid < 36) collected[pass * PCG_NW + tid] = wide_s[tid];
      __syncthreads();   // wide_s / inrow_s are rewritten by the next pass
    }
    bb = collected[35];
    __syncthreads();   // every thread has read bb before thread 0 rewrites Einv_s
    if (tid == 0) {
      // every CTA factorises the same 7 x 7 matrix: identical decisions everywhere
      int idx = 0;
      for (int a = 0; a < PCG_ND; ++a)
        for (int b2 = a; b2 < PCG_ND; ++b2) { E[a * PCG_ND + b2] = collected[idx]; E[b2 * PCG_ND + a] = collected[idx]; ++idx; }
      for (int a = 0; a < PCG_ND; ++a) wb[a] = collected[28 + a];
      double Lc[PCG_ND * PCG_ND];
      bool ok = true;
      double dmax = 0.0;
      for (int a = 0; a < PCG_ND; ++a) dmax = fmax(dmax, E[a * PCG_ND + a]);
      for (int j = 0; j < PCG_ND && ok; ++j) {
        double dd = E[j * PCG_ND + j];
        for (int k2 = 0; k2 < j; ++k2) dd -= Lc[j * PCG_ND + k2] * Lc[j * PCG_ND + k2];
        if (!(dd > 1e-12 * dmax) || !(dmax > 0.0)) { ok = false; break; }
        dd = sqrt(dd);
        Lc[j * PCG_ND + j] = dd;
        for (int i2 = j + 1; i2 < PCG_ND; ++i2) {
          double sv2 = E[i2 * PCG_ND + j];
          for (int k2 = 0; k2 < j; ++k2) sv2 -= Lc[i2 * PCG_ND + k2] * Lc[j * PCG_ND + k2];
          Lc[i2 * PCG_ND + j] = sv2 / dd;
        }
      }
      if (ok) {
        for (int cidx = 0; cidx < PCG_ND; ++cidx) {   // E^-1 column by column
          double y[PCG_ND];
          for (int i2 = 0; i2 < PCG_ND; ++i2) {
            double sv2 = (i2 == cidx) ? 1.0 : 0.0;
            for (int k2 = 0; k2 < i2; ++k2) sv2 -= Lc[i2 * PCG_ND + k2] * y[k2];
            y[i2] = sv2 / Lc[i2 * PCG_ND + i2];
          }
          for (int i2 = PCG_ND - 1; i2 >= 0; --i2) {
            double sv2 = y[i2];
            for (int k2 = i2 + 1; k2 < PCG_ND; ++k2) sv2 -= Lc[k2 * PCG_ND + i2] * y[k2];
            y[i2] = sv2 / Lc[i2 * PCG_ND + i2];
          }
          for (int i2 = 0; i2 < PCG_ND; ++i2) Einv_s[i2 * PCG_ND + cidx] = y[i2];
        }
        for (int a = 0; a < PCG_ND; ++a) {
          double sv2 = 0.0;
          for (int b2 = 0; b2 < PCG_ND; ++b2) sv2 += Einv_s[a * PCG_ND + b2] * wb[b2];
          c0_s[a] = sv2;
        }
      }
      s_defl = ok ? 1 : 0;
    }
    __syncthreads();
    defl = s_defl != 0;   // dependent / vanishing vectors (e.g. every rig instance fixed): plain PCG
  }
  // tc_s = E^-1 t for the PCG_ND projections the wide barrier left in wide_s[3..]: seven threads, not all 512 (49 DFMA
  // each) -- and no per-thread copy of the result in registers (the kernel sits at its 128-register limit)
  auto coarse = [&]() {
    if (tid < PCG_ND) {
      double sv2 = 0.0;
#pragma unroll
      for (int b2 = 0; b2 < PCG_ND; ++b2) sv2 += Einv_s[tid * PCG_ND + b2] * wide_s[3 + b2];
      tc_s[tid] = sv2;
    }
    __syncthreads();
  };
  // sum_j (A W)_j[row] c_j for the own row
  auto aw_dot = [&](const double* c) -> double {
    double sv2 = 0.0;
#pragma unroll
    for (int j = 0; j < PCG_ND; ++j) sv2 += AW_s[j * MR + tid] * c[j];
    return sv2;
  };

  // ---- init: y = 0, r = P b, u = M^-1 r, w = P A u, m = M^-1 w ----
  double xr = 0.0, rr_ = bi, u = 0.0, w = 0.0, z = 0.0, q = 0.0, sv_ = 0.0, p = 0.0;
  if (defl && mine) rr_ = bi - aw_dot(c0_s);
  if (mine) w_s[tid] = rr_;
  __syncthreads();
  // Generations of the flagged exchanges: u = M^-1 r is 1, the m of loop iteration it and the dot products posted in it
  // are it + 2.  Every flagged buffer (mflag, st->slotf, st->totf) is zeroed with the rest of PcgState before the solve, so no
  // word left by an earlier solve, run or handle can carry a generation this solve waits for.
  group_solve(1);
  if (defl) {
    __syncthreads();   // g_s of my row was written by the warp that solved its group
    if (mine) {
      double* ir = inrow_s + tid * PCG_NW;
      ir[0] = 0.0; ir[1] = 0.0; ir[2] = 0.0;
#pragma unroll
      for (int j = 0; j < PCG_ND; ++j) ir[3 + j] = AW_s[j * MR + tid] * g_s[tid];
    }
    grid_reduce_wide(st, gridDim.x, &bar_gen, wide_s, gather_s, inrow_s, nrows);
    coarse();
  } else {
    double d0, d1, d2;
    grid_reduce<3>(st, gridDim.x, bar_gen, 0.0, 0.0, mine ? rr_ * rr_ : 0.0, d0, d1, d2, red);
    bb = d2;
  }
  const double tol2 = tol2_rel * bb;
  double rr = bb;
  int it = 0, converged = 0;
  if (bb > 0.0) {
    if (mine) u = g_s[tid];
    stage_m(1);   // already visible: the barrier above ordered it
    __syncthreads();
    matvec();
    __syncthreads();
    if (mine) { w = n_s[tid] - (defl ? aw_dot(tc_s) : 0.0); w_s[tid] = w; }
    __syncthreads();
    group_solve(2);
    double gamma_prev = 1.0, alpha_prev = 1.0, best = bb;
    int since_best = 0;
    // Ghysels-Vanroose order: an iteration posts its dot products, then stages m and runs the mat-vec -- which do not
    // need them -- and only then collects the totals, which by then have mostly arrived.  The exit tests therefore run
    // after a mat-vec the exiting iteration does not use; every CTA takes them on bit-identical totals, so all leave
    // together and none waits for an m that is not coming.
    // Reuse of the two m buffers: m of generation gen + 2 overwrites gen.  Its writer has read the totals of gen + 1
    // first, which exist only once every CTA has posted gen + 1, and a CTA posts that only after it has staged gen, so
    // no CTA is still reading gen.
    for (;; ++it) {
      const unsigned gen = (unsigned)it + 2u;
      const long long tk0 = clock64();
      if (defl) {
        __syncthreads();   // g_s (m of my row) comes from another warp's group solve
        if (mine) {
          double* ir = inrow_s + tid * PCG_NW;
          ir[0] = rr_ * u; ir[1] = w * u; ir[2] = rr_ * rr_;
#pragma unroll
          for (int j = 0; j < PCG_ND; ++j) ir[3 + j] = AW_s[j * MR + tid] * g_s[tid];   // (A W)^T m of the m being exchanged
        }
        pcg_post_wide(st, gen, inrow_s, nrows);
      } else
        pcg_post3(st, gen, mine ? rr_ * u : 0.0, mine ? w * u : 0.0, mine ? rr_ * rr_ : 0.0, red);
      const long long tk1 = clock64();
      stage_m(gen);
      __syncthreads();
      const long long tk2 = clock64();
      matvec();
      __syncthreads();
      const long long tk3 = clock64();
      double gamma, delta;
      if (defl) {
        pcg_collect_wide(st, gridDim.x, gen, wide_s);
        gamma = wide_s[0]; delta = wide_s[1]; rr = wide_s[2];
        coarse();
      } else
        pcg_collect3(st, gridDim.x, gen, gamma, delta, rr, red);
      const long long tk4 = clock64();
      if (!(rr == rr)) break;
      if (rr <= tol2) { converged = 1; break; }
      if (rr < best) { best = rr; since_best = 0; } else if (++since_best > 150) break;  // stagnation
      if (it >= max_iter) break;
      const double beta = it > 0 ? gamma / gamma_prev : 0.0;
      const double alpha = it > 0 ? gamma / (delta - beta * gamma / alpha_prev) : gamma / delta;
      if (mine) {
        const double mo = g_s[tid], nn = n_s[tid] - (defl ? aw_dot(tc_s) : 0.0);   // P A m
        z = nn + beta * z;
        q = mo + beta * q;
        sv_ = w + beta * sv_;
        p = u + beta * p;
        xr += alpha * p;
        rr_ -= alpha * sv_;
        u -= alpha * q;
        w -= alpha * z;
        w_s[tid] = w;
      }
      __syncthreads();
      group_solve(gen + 1);
      gamma_prev = gamma;
      alpha_prev = alpha;
      if (blockIdx.x == 0 && tid == 0) {   // OSFM_BA_TRACE: post, stage (with the waits for m), mat-vec, collect, update
        const long long tk5 = clock64();
        st->prof[0] += tk1 - tk0; st->prof[1] += tk2 - tk1; st->prof[2] += tk3 - tk2; st->prof[3] += tk4 - tk3;
        st->prof[4] += tk5 - tk4;
      }
    }
  } else {
    converged = 1;
  }
  if (defl) {
    // x = Q b + y - Q A y = y + W (c0 - E^-1 (A W)^T y)
    if (mine) {
      double* ir = inrow_s + tid * PCG_NW;
      ir[0] = 0.0; ir[1] = 0.0; ir[2] = 0.0;
#pragma unroll
      for (int j = 0; j < PCG_ND; ++j) ir[3 + j] = AW_s[j * MR + tid] * xr;
    }
    grid_reduce_wide(st, gridDim.x, &bar_gen, wide_s, gather_s, inrow_s, nrows);
    coarse();
    if (mine) {
      double add = 0.0;
#pragma unroll
      for (int j = 0; j < PCG_ND; ++j) add += Wd_s[j * MR + tid] * (c0_s[j] - tc_s[j]);
      xr += add;
    }
  }
  if (mine) x_out[gi] = xr;
  // The residual above is the recurred one, which drifts from b - S x in pipelined CG: check the true residual of the
  // returned x with one more exchange and mat-vec, and hand the solve to the classic kernel if it is not what was claimed.
  if (converged && bb > 0.0) {
    double d0, d1, d2;
    grid_reduce<3>(st, gridDim.x, bar_gen, 0.0, 0.0, 0.0, d0, d1, d2, red);   // x of every CTA is visible
    stage(x_out);
    __syncthreads();
    matvec();
    __syncthreads();
    const double tr = mine ? bi - n_s[tid] : 0.0;
    grid_reduce<3>(st, gridDim.x, bar_gen, 0.0, 0.0, tr * tr, d0, d1, d2, red);
    rr = d2;
    if (!(rr <= 4.0 * tol2)) converged = 0;
  }
  if (blockIdx.x == 0 && tid == 0) {
    st->iterations = it; st->rr_final = rr; st->converged = converged; st->deflated = defl ? 1 : 0;
  }
}

}  // namespace osfm
