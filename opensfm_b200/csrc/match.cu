// Brute-force descriptor matching on H100 (sm_90a).
//
// Replaces the OpenCV call under opensfm/matching.py:723-777
// (`cv2.DescriptorMatcher.knnMatch(k=2)` + Lowe ratio test) for float32 L2
// ("BruteForce") and uint8 Hamming ("BruteForce-Hamming") descriptors.
//
// Semantics reproduced from cv2 (SURVEY.md §8c, pinned by tests against live cv2):
//  * L2 candidates are ranked by sqrt(float32 sum of squared differences);
//    Hamming by the integer bit count;
//  * ties -> lowest train index (cv2 inserts with a strict `<`);
//  * masked-out trains are skipped; a query with < 2 candidates has no match
//    (matching.py:752);
//  * ratio test `m.distance < ratio * n.distance` in double on the float32
//    distances (matching.py:754).
//
// Kernels in this file:
//  bf_top2_simt        Hamming SIMT tile kernel (XOR + popcount)
//  bf_top2_f32_cv<MT>  float32 SIMT tile kernel in cv2's summation order
//  bf_top2_finalize    merge train chunks per query + ratio test
//  bf_symmetric        keep (i,j) iff j's match is i (matching.py:775-777)
// The wgmma tensor-core distance kernels live in match_tc.cu.
#include <algorithm>
#include <cmath>
#include <map>
#include <vector>

#include "common.cuh"
#include "match_common.cuh"

namespace osfm {

// ---------------------------------------------------------------------------
// Hamming SIMT tile kernel
// ---------------------------------------------------------------------------
constexpr int BM = 64;       // queries per CTA tile
constexpr int BN = 64;       // trains per inner tile
constexpr int DK = 16;       // u32 words per k-step
constexpr int LDS_STRIDE = 68;

__global__ void __launch_bounds__(256) bf_top2_simt(const MatchJob* __restrict__ jobs,
                                                    const int* __restrict__ tile_prefix, int njobs,
                                                    Top2* __restrict__ partial) {
  __shared__ __align__(16) uint32_t As[DK][LDS_STRIDE];
  __shared__ __align__(16) uint32_t Bs[DK][LDS_STRIDE];
  __shared__ Top2 cand[BM][16];

  const MatchTile tile = decode_tile<BM>(jobs, tile_prefix, njobs, blockIdx.x);
  const MatchJob& job = tile.job;
  const int q0 = tile.q0, t_begin = tile.t_begin, t_end = tile.t_end, chunk = tile.chunk;
  const int D = job.dim_padded;  // words per row (multiple of DK)
  const uint32_t* __restrict__ Q = static_cast<const uint32_t*>(job.q);
  const uint32_t* __restrict__ T = static_cast<const uint32_t*>(job.t);

  const int tid = threadIdx.x;
  const int ty = tid >> 4, tx = tid & 15;

  Top2 best[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) best[i] = top2_empty();

  for (int t0 = t_begin; t0 < t_end; t0 += BN) {
    int acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = 0;

    for (int k0 = 0; k0 < D; k0 += DK) {
      // 64 rows x 16 elems = 256 x 16-byte vectors per operand: one per thread
      {
        const int row = tid & 63, kq = tid >> 6;  // kq 0..3 -> elems kq*4..kq*4+3
        const int gq = q0 + row, gt = t0 + row;
        uint4 va = make_uint4(0, 0, 0, 0), vb = make_uint4(0, 0, 0, 0);
        if (gq < job.nq) va = *reinterpret_cast<const uint4*>(Q + (size_t)gq * D + k0 + kq * 4);
        if (gt < t_end) vb = *reinterpret_cast<const uint4*>(T + (size_t)gt * D + k0 + kq * 4);
        const uint32_t* ea = reinterpret_cast<const uint32_t*>(&va);
        const uint32_t* eb = reinterpret_cast<const uint32_t*>(&vb);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          As[kq * 4 + e][row] = ea[e];
          Bs[kq * 4 + e][row] = eb[e];
        }
      }
      __syncthreads();
#pragma unroll
      for (int k = 0; k < DK; ++k) {
        const uint4 a4 = *reinterpret_cast<const uint4*>(&As[k][ty * 4]);
        const uint4 b4 = *reinterpret_cast<const uint4*>(&Bs[k][tx * 4]);
        const uint32_t* a = reinterpret_cast<const uint32_t*>(&a4);
        const uint32_t* b = reinterpret_cast<const uint32_t*>(&b4);
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] += __popc(a[i] ^ b[j]);
      }
      __syncthreads();
    }
    // fold this tile's 4x4 results into the thread-local top-2 of each row
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int gq = q0 + ty * 4 + i;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int gt = t0 + tx * 4 + j;
        if (gq >= job.nq || gt >= t_end) continue;
        if (!job_allows(job, gq, gt)) continue;
        top2_insert(best[i], (float)acc[i][j], gt);
      }
    }
  }
  // merge the 16 threads that share a query row
#pragma unroll
  for (int i = 0; i < 4; ++i) cand[ty * 4 + i][tx] = best[i];
  __syncthreads();
  if (tid < BM) {
    const int gq = q0 + tid;
    if (gq < job.nq) {
      Top2 m = top2_empty();
      for (int x = 0; x < 16; ++x) top2_merge(m, cand[tid][x]);
      partial[job.partial_off + (size_t)chunk * job.nq + gq] = m;
    }
  }
}

// ---------------------------------------------------------------------------
// General float32 descriptors, bit-exact with cv2's summation order (cv_tile_d2, match_common.cuh).
// MT = micro-tile edge per thread (4 -> 64x64 CTA tile, 2 -> 32x32 for long descriptors).
// ---------------------------------------------------------------------------
template <int MT>
__global__ void __launch_bounds__(256) bf_top2_f32_cv(const MatchJob* __restrict__ jobs,
                                                      const int* __restrict__ tile_prefix, int njobs,
                                                      Top2* __restrict__ partial) {
  constexpr int TS = 16 * MT;      // rows per tile side
  constexpr int LD = TS + 4;       // floats per element row (keeps 16-byte alignment, staggers banks)
  extern __shared__ __align__(16) float fx_smem[];
  __shared__ Top2 cand[TS][16];

  const MatchTile tile = decode_tile<TS>(jobs, tile_prefix, njobs, blockIdx.x);
  const MatchJob& job = tile.job;
  const int q0 = tile.q0, t_begin = tile.t_begin, t_end = tile.t_end, chunk = tile.chunk;
  const int D = job.dim_padded;
  const int nblk = job.dim / 16;   // full 16-element blocks of the TRUE dimension; the rest is cv2's scalar tail
  const float* __restrict__ Q = static_cast<const float*>(job.q);
  const float* __restrict__ T = static_cast<const float*>(job.t);
  float* As = fx_smem;
  float* Bs = fx_smem + (size_t)D * LD;

  const int tid = threadIdx.x;
  const int ty = tid >> 4, tx = tid & 15;
  cv_load_tile<TS, LD>(As, Q, q0, job.nq, D);

  Top2 best[MT];
#pragma unroll
  for (int i = 0; i < MT; ++i) best[i] = top2_empty();

  for (int t0 = t_begin; t0 < t_end; t0 += TS) {
    __syncthreads();  // previous tile's readers are done (and As is complete on the first pass)
    cv_load_tile<TS, LD>(Bs, T, t0, t_end, D);
    __syncthreads();
    float d2[MT][MT];
    cv_tile_d2<MT, LD>(As, Bs, D, nblk, ty, tx, d2);
#pragma unroll
    for (int i = 0; i < MT; ++i) {
      const int gq = q0 + ty * MT + i;
#pragma unroll
      for (int j = 0; j < MT; ++j) {
        const int gt = t0 + tx * MT + j;
        if (gq >= job.nq || gt >= t_end) continue;
        if (!job_allows(job, gq, gt)) continue;
        top2_insert(best[i], __fsqrt_rn(d2[i][j]), gt);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < MT; ++i) cand[ty * MT + i][tx] = best[i];
  __syncthreads();
  if (tid < TS) {
    const int gq = q0 + tid;
    if (gq < job.nq) {
      Top2 m = top2_empty();
      for (int x = 0; x < 16; ++x) top2_merge(m, cand[tid][x]);
      partial[job.partial_off + (size_t)chunk * job.nq + gq] = m;
    }
  }
}
constexpr int FX_MAX_DIM_T64 = 320;   // padded elements: 2 * 320 * 68 * 4 B = 174 KB of shared memory
constexpr int FX_MAX_DIM_T32 = 704;   // 2 * 704 * 36 * 4 B = 203 KB

static void launch_simt(Matcher& m, int njobs, int ntiles, int) {
  bf_top2_simt<<<(unsigned)ntiles, 256, 0, m.stream>>>(m.d_jobs.p, m.d_prefix.p, njobs, m.d_partial.p);
  OSFM_LAUNCH_CHECK();
}
template <int MT>
static void launch_f32_cv(Matcher& m, int njobs, int ntiles, int smem) {
  constexpr int max_dim = MT == 4 ? FX_MAX_DIM_T64 : FX_MAX_DIM_T32;
  m.opt_in_smem(bf_top2_f32_cv<MT>, 2 * max_dim * (16 * MT + 4) * (int)sizeof(float));
  bf_top2_f32_cv<MT><<<(unsigned)ntiles, 256, smem, m.stream>>>(m.d_jobs.p, m.d_prefix.p, njobs, m.d_partial.p);
  OSFM_LAUNCH_CHECK();
}

// The SIMT kernels split the trains until there are four tiles per SM.  The float32 kernel keeps whole rows in
// shared memory, so its tile edge follows the longest padded row of the submission.
static KernelPlan simt_plan(bool u8, int max_dim_padded) {
  if (u8) return {BM, BM, 4, false, 0, launch_simt};
  if (max_dim_padded > FX_MAX_DIM_T32)
    throw ArgError("float32 descriptors longer than 704 elements are not supported by the exact matcher");
  const int tile = max_dim_padded > FX_MAX_DIM_T64 ? 32 : 64;
  const int smem = 2 * max_dim_padded * (tile + 4) * (int)sizeof(float);
  return {tile, tile, 4, false, smem, tile == 64 ? launch_f32_cv<4> : launch_f32_cv<2>};
}

// ---------------------------------------------------------------------------
// Merge chunks + ratio test.  grid = (ceil(max_nq/256), njobs)
// ---------------------------------------------------------------------------
// squared != 0: the partials hold squared distances (tensor-core L2 kernel; only used when float32 sqrt is
// injective on them, so merging in d^2 is merging in cv2's ranking) and are sqrt'd here.
__global__ void bf_top2_finalize(const MatchJob* __restrict__ jobs, const Top2* __restrict__ partial,
                                 int32_t* __restrict__ match_buf, double ratio, int squared) {
  const MatchJob job = jobs[blockIdx.y];
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= job.nq) return;
  Top2 m = top2_empty();
  for (int c = 0; c < job.nchunks; ++c) top2_merge(m, partial[job.partial_off + (size_t)c * job.nq + q]);
  if (squared) {
    m.s1 = __fsqrt_rn(m.s1);
    m.s2 = __fsqrt_rn(m.s2);
  }
  int out = -1;
  // matching.py:752-755: two candidates and m.distance < ratio * n.distance (double)
  if (m.i1 >= 0 && m.i2 >= 0 && (double)m.s1 < ratio * (double)m.s2) out = m.i1;
  match_buf[job.match_off + q] = out;
}

// matching.py:775-777: intersect matches_ij with the transposed matches_ji.
// grid = (ceil(max_na/256), npairs); job 2p is a->b, job 2p+1 is b->a.
__global__ void bf_symmetric(const MatchJob* __restrict__ jobs, const int32_t* __restrict__ match_buf,
                             int32_t* __restrict__ out, const long long* __restrict__ out_off) {
  const MatchJob fwd = jobs[2 * blockIdx.y];
  const MatchJob bwd = jobs[2 * blockIdx.y + 1];
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= fwd.nq) return;
  const int j = match_buf[fwd.match_off + q];
  int res = -1;
  if (j >= 0 && match_buf[bwd.match_off + j] == q) res = j;
  out[out_off[blockIdx.y] + q] = res;
}

// ---------------------------------------------------------------------------
// Compact result lists.  The per-query results (train index or -1) of every pair become the (query, train) rows the
// reference returns (matching.py:749-756), packed pair after pair in query order, on the device: the host reads
// back only the matches (about a sixth of the queries) and never touches the per-query arrays -- building the
// same lists with numpy cost 100 ms for 2389 pairs, four times the matching itself.
//   bf_pair_counts   one CTA per pair: number of matches
//   bf_pair_scan     exclusive scan of the counts (one CTA; <= 30000 pairs)
//   bf_pair_compact  one CTA per pair: ordered compaction with block scans
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256) bf_pair_counts(const int32_t* __restrict__ res, const long long* __restrict__ out_off,
                                                      int* __restrict__ counts) {
  __shared__ int wsum[8];
  const long long b = out_off[blockIdx.x], e = out_off[blockIdx.x + 1];
  int c = 0;
  for (long long i = b + threadIdx.x; i < e; i += 256) c += res[i] >= 0;
  for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int w = 0; w < 8; ++w) t += wsum[w];
    counts[blockIdx.x] = t;
  }
}
__global__ void __launch_bounds__(1024) bf_pair_scan(const int* __restrict__ counts, int npairs, long long* __restrict__ coff) {
  __shared__ long long wtot[32];
  __shared__ long long carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int base = 0; base < npairs; base += 1024) {
    const int i = base + threadIdx.x;
    long long v = i < npairs ? counts[i] : 0, incl = v;
    for (int o = 1; o < 32; o <<= 1) {
      const long long up = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += up;
    }
    if (lane == 31) wtot[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      long long w = wtot[lane], wi = w;
      for (int o = 1; o < 32; o <<= 1) {
        const long long up = __shfl_up_sync(0xffffffffu, wi, o);
        if (lane >= o) wi += up;
      }
      wtot[lane] = wi - w;   // exclusive warp offsets
    }
    __syncthreads();
    const long long excl = carry + wtot[warp] + incl - v;
    if (i < npairs) coff[i] = excl;
    __syncthreads();
    if (threadIdx.x == 1023) carry = excl + v;
    __syncthreads();
  }
  if (threadIdx.x == 0) coff[npairs] = carry;
}
__global__ void __launch_bounds__(256) bf_pair_compact(const int32_t* __restrict__ res, const long long* __restrict__ out_off,
                                                       const long long* __restrict__ coff, int32_t* __restrict__ pairs) {
  __shared__ int wsum[8];
  __shared__ int base_s;
  const long long b = out_off[blockIdx.x], e = out_off[blockIdx.x + 1];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) base_s = 0;
  __syncthreads();
  for (long long t0 = b; t0 < e; t0 += 256) {
    const long long i = t0 + threadIdx.x;
    const int j = i < e ? res[i] : -1;
    const unsigned m = __ballot_sync(0xffffffffu, j >= 0);
    if (lane == 0) wsum[warp] = __popc(m);
    __syncthreads();
    int off = base_s;
    for (int w = 0; w < warp; ++w) off += wsum[w];
    if (j >= 0) {
      const long long o = coff[blockIdx.x] + off + __popc(m & ((1u << lane) - 1u));
      pairs[2 * o] = (int32_t)(i - b);
      pairs[2 * o + 1] = j;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      int t = 0;
      for (int w = 0; w < 8; ++w) t += wsum[w];
      base_s += t;
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------
// Descriptor upload helpers
// ---------------------------------------------------------------------------
// Pads rows to dim_padded with zeros (distance-neutral).  One thread per padded element.
template <class T>
__global__ void pad_rows_kernel(const T* __restrict__ src, int n, int dim, T* __restrict__ dst, int dim_padded) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (size_t)n * dim_padded) return;
  const int r = idx / dim_padded, c = idx % dim_padded;
  dst[idx] = c < dim ? src[(size_t)r * dim + c] : T(0);
}

// ---------------------------------------------------------------------------
// Guided matching: epipolar mask of a pair as a bitmask, built on the device.
//
// matching.compute_inliers_bearing_epipolar (opensfm/matching.py:847-868) ->
// geometry::EpipolarAngleTwoBearingsMany (opensfm/src/geometry/src/triangulation.cc:195-219), fp64 on float32
// bearings:  t^ = t / |t|,  b2w_j = R b2_j,  e1_i = (t^ x b1_i)^,  e2_j = (t^ x b2w_j)^,
//            sym_ij = (|e1_i . b2w_j| + |b1_i . e2_j|) / 2,   mask_ij = (pi/2 - acos(sym_ij)) < threshold.
// epi_vectors: the per-feature vectors in fp64 (and their float32 roundings).
// epi_mask_bits: one warp per 32 x 32 block; the test runs in float32 against sin(threshold) with a guard band
// (|error| of the float32 evaluation < 1e-6), and only elements inside the band evaluate the reference's fp64
// expression with acos -- so the decision is the reference's for every element, at float32 cost.
// Both layouts are written from one evaluation: F[i][j / 32] (queries of image 1) and T[j][i / 32] (the
// transposed mask the symmetric pass needs, matching.py:774).
// ---------------------------------------------------------------------------
struct EpiPair {
  const float *b1, *b2;     // bearings n x 3
  double* v1;               // [n1][6] : b1, e1     (fp64)
  double* v2;               // [n2][6] : b2w, e2
  uint32_t *F, *T;
  int n1, n2, w1, w2;       // w2 = words per row of F (over n2), w1 = words per row of T (over n1)
  double pose[12];
};
__global__ void epi_vectors(const EpiPair* __restrict__ pairs) {
  const EpiPair& p = pairs[blockIdx.y];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  // Eigen's normalized() (Dot.h): a vector whose squared norm is 0 comes back unchanged.  So t = 0 gives zero
  // epipolar vectors (symmetric_epi = 0: every element passes a positive threshold) and a bearing parallel to t
  // a zero e, never a division by zero.
  auto normalize = [](double v[3]) {
    const double z = v[0] * v[0] + v[1] * v[1] + v[2] * v[2];
    if (z > 0.0) {
      const double n = sqrt(z);
      v[0] /= n; v[1] /= n; v[2] /= n;
    }
  };
  double t[3] = {p.pose[9], p.pose[10], p.pose[11]};
  normalize(t);
  auto emit = [&](double* out, const double b[3]) {
    double e[3] = {t[1] * b[2] - t[2] * b[1], t[2] * b[0] - t[0] * b[2], t[0] * b[1] - t[1] * b[0]};
    normalize(e);
    out[0] = b[0]; out[1] = b[1]; out[2] = b[2];
    out[3] = e[0]; out[4] = e[1]; out[5] = e[2];
  };
  if (i < p.n1) {
    const double b[3] = {(double)p.b1[3 * i], (double)p.b1[3 * i + 1], (double)p.b1[3 * i + 2]};
    emit(p.v1 + 6 * (size_t)i, b);
  }
  if (i < p.n2) {
    const double a[3] = {(double)p.b2[3 * i], (double)p.b2[3 * i + 1], (double)p.b2[3 * i + 2]};
    const double* R = p.pose;
    const double b[3] = {R[0] * a[0] + R[1] * a[1] + R[2] * a[2], R[3] * a[0] + R[4] * a[1] + R[5] * a[2],
                         R[6] * a[0] + R[7] * a[1] + R[8] * a[2]};
    emit(p.v2 + 6 * (size_t)i, b);
  }
}
__global__ void __launch_bounds__(256) epi_mask_bits(const EpiPair* __restrict__ pairs, double threshold) {
  // One CTA = 256 x 256 elements = 8 x 8 blocks of 32 x 32; warp w owns column block w and walks the 8 row blocks.
  // The 32 rows of a block ([b1 | e1] as float32) sit in shared memory and are read by every lane (broadcast);
  // the row words (F) and column words (T) of the whole CTA tile are staged in shared memory and written as full
  // 32-byte runs -- one word per (row, block) scattered straight to HBM made the kernel store-bound at 7e11
  // elements/s.
  __shared__ __align__(16) float rows[32][8];
  __shared__ uint32_t sF[256][8], sT[256][8];
  const EpiPair& p = pairs[blockIdx.z];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int jb0 = blockIdx.x * 8, ib0 = blockIdx.y * 8;
  if (jb0 >= p.w2 || ib0 >= p.w1) return;   // CTA-uniform (pairs of different sizes share the grid)
  const int jb = jb0 + wib;
  const int j = jb * 32 + lane;
  const float NaNf = __int_as_float(0x7fc00000);
  float cj[6] = {NaNf, NaNf, NaNf, NaNf, NaNf, NaNf};
  if (j < p.n2) for (int e = 0; e < 6; ++e) cj[e] = (float)p.v2[6 * (size_t)j + e];
  // The reference tests asin(sym) = pi/2 - acos(sym) < threshold; asin lies in [-pi/2, pi/2], where sin is
  // increasing, so the clamped threshold decides the same.  Past pi/2 the test is sym < 1: the band around 1 goes
  // to fp64, where sym > 1 gives acos = NaN and fails, as in the reference.
  const float s_thr = (float)sin(fmin(fmax(threshold, -M_PI / 2.0), M_PI / 2.0));
  const float lo = s_thr - 2e-6f, hi = s_thr + 2e-6f;
  for (int ibl = 0; ibl < 8; ++ibl) {
    const int ib = ib0 + ibl;
    __syncthreads();   // previous row block consumed
    if (threadIdx.x < 192) {
      const int r = threadIdx.x / 6, e = threadIdx.x - r * 6;
      const int gi = ib * 32 + r;
      rows[r][e] = gi < p.n1 ? (float)p.v1[6 * (size_t)gi + e] : NaNf;
    }
    __syncthreads();
    uint32_t colbits = 0;
#pragma unroll 4
    for (int r = 0; r < 32; ++r) {
      const float4 ra = *reinterpret_cast<const float4*>(&rows[r][0]);   // b1.x, b1.y, b1.z, e1.x
      const float2 rb = *reinterpret_cast<const float2*>(&rows[r][4]);   // e1.y, e1.z
      const float sym = 0.5f * (fabsf(ra.w * cj[0] + rb.x * cj[1] + rb.y * cj[2]) + fabsf(ra.x * cj[3] + ra.y * cj[4] + ra.z * cj[5]));
      bool in = sym < lo;               // NaN (missing row / column, degenerate epipolar plane) compares false
      if (!(sym < lo) && sym < hi) {    // inside the guard band: the reference's own fp64 expression
        const double* a = p.v1 + 6 * (size_t)(ib * 32 + r);
        const double* c = p.v2 + 6 * (size_t)j;
        const double sd = (fabs(a[3] * c[0] + a[4] * c[1] + a[5] * c[2]) + fabs(a[0] * c[3] + a[1] * c[4] + a[2] * c[5])) / 2.0;
        in = (M_PI / 2.0 - acos(sd)) < threshold;
      }
      const uint32_t rowbits = __ballot_sync(0xffffffffu, in);
      if (lane == 0) sF[ibl * 32 + r][wib] = rowbits;
      if (in) colbits |= 1u << r;
    }
    sT[wib * 32 + lane][ibl] = colbits;
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < 256 * 8; idx += 256) {
    const int r = idx >> 3, w = idx & 7;
    const int gi = ib0 * 32 + r, gj = jb0 * 32 + r;
    if (gi < p.n1 && jb0 + w < p.w2) p.F[(size_t)gi * p.w2 + jb0 + w] = sF[r][w];
    if (gj < p.n2 && ib0 + w < p.w1) p.T[(size_t)gj * p.w1 + ib0 + w] = sT[r][w];
  }
}

// ---------------------------------------------------------------------------
// Matcher object (its methods run under the C ABI's with_handle, which makes the device current)
// ---------------------------------------------------------------------------
Matcher::Matcher(int dev) : DeviceStream(dev) {
  cudaDeviceProp prop;
  OSFM_CUDA(cudaGetDeviceProperties(&prop, device));
  num_sms = prop.multiProcessorCount;
}

Matcher::~Matcher() {
  cudaStreamSynchronize(stream);
  for (auto& sl : slabs) cudaFree(sl.base);
}

void* Matcher::slab_alloc(size_t bytes, int* slab_idx) {
  bytes = align256(bytes);
  // first fit in the released ranges, then the bump pointers, then a new slab
  for (size_t i = 0; i < slabs.size(); ++i) {
    Slab& sl = slabs[i];
    for (size_t r = 0; r < sl.free_ranges.size(); ++r) {
      if (sl.free_ranges[r].second < bytes) continue;
      void* p = sl.base + sl.free_ranges[r].first;
      if (sl.free_ranges[r].second == bytes) sl.free_ranges.erase(sl.free_ranges.begin() + r);
      else { sl.free_ranges[r].first += bytes; sl.free_ranges[r].second -= bytes; }
      ++sl.live;
      *slab_idx = (int)i;
      return p;
    }
  }
  for (size_t i = 0; i < slabs.size(); ++i) {
    Slab& sl = slabs[i];
    if (sl.cap - sl.used >= bytes) {
      void* p = sl.base + sl.used;
      sl.used += bytes;
      ++sl.live;
      *slab_idx = (int)i;
      return p;
    }
  }
  // 16 MB first, doubling up to 512 MB: one-shot matchers stay small, resident image sets need few cudaMallocs
  size_t cap = (size_t)16 << 20;
  for (size_t i = 0; i < slabs.size() && cap < ((size_t)512 << 20); ++i) cap *= 2;
  cap = std::max(cap, bytes);
  Slab sl;
  OSFM_CUDA(cudaMalloc(&sl.base, cap));
  sl.cap = cap;
  sl.used = bytes;
  sl.live = 1;
  slabs.push_back(sl);
  *slab_idx = (int)slabs.size() - 1;
  return sl.base;
}

void Matcher::slab_release(int idx, void* ptr, size_t bytes) {   // callers synchronise the stream before releasing
  if (idx < 0) return;
  Slab& sl = slabs[idx];
  if (--sl.live == 0) { sl.used = 0; sl.free_ranges.clear(); return; }
  bytes = align256(bytes);
  if (!ptr || bytes == 0) return;
  size_t off = (size_t)(static_cast<char*>(ptr) - sl.base);
  auto& fr = sl.free_ranges;
  auto it = std::lower_bound(fr.begin(), fr.end(), std::make_pair(off, (size_t)0));
  it = fr.insert(it, std::make_pair(off, bytes));
  if (it + 1 != fr.end() && it->first + it->second == (it + 1)->first) { it->second += (it + 1)->second; fr.erase(it + 1); }
  if (it != fr.begin() && (it - 1)->first + (it - 1)->second == it->first) { (it - 1)->second += it->second; it = fr.erase(it) - 1; }
  if (it->first + it->second == sl.used) { sl.used = it->first; fr.erase(it); }   // the tail goes back to the bump pointer
}

// exactness flags / max norms of the sets added since the last call (one D2H copy for all of them)
void Matcher::refresh_info() {
  if (pending.empty()) return;
  h_info.resize(2 * (size_t)next_slot);
  OSFM_CUDA(cudaMemcpyAsync(h_info.data(), d_info.p, sizeof(int) * 2 * (size_t)next_slot, cudaMemcpyDeviceToHost, stream));
  OSFM_CUDA(cudaStreamSynchronize(stream));
  for (int id : pending) {
    auto it = sets.find(id);
    if (it == sets.end() || !it->second.info_pending) continue;
    DescSet& s = it->second;
    s.tc_ok = h_info[2 * s.slot] == 0;
    std::memcpy(&s.tc_max_norm, &h_info[2 * s.slot + 1], sizeof(float));
    s.info_pending = false;
  }
  pending.clear();
}

void Matcher::free_set(DescSet& s) {
  release(s.rows);
  release(s.bearings);
  release(s.vlad);
  release(s.bow_words);
  release(s.bow_hist);
  if (s.slot >= 0) {
    cudaMemsetAsync(d_info.p + 2 * s.slot, 0, 2 * sizeof(int), stream);
    free_slots.push_back(s.slot);
  }
  s.tc_ok = false;
  s.slot = -1;
}

// widen uint8 rows to zero-padded float32 rows (uint8-stored L2 descriptors that do not take the tensor-core path)
__global__ void widen_rows_kernel(const uint8_t* __restrict__ src, int n, int dim, float* __restrict__ dst, int dim_padded) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (size_t)n * dim_padded) return;
  const int r = idx / dim_padded, c = idx % dim_padded;
  dst[idx] = c < dim ? (float)src[(size_t)r * dim + c] : 0.0f;
}

int Matcher::add_async(const void* host, int n, int dim, bool u8, bool u8_as_l2) {
  if (n < 0 || dim <= 0) throw ArgError("descriptor matrix must be n x dim with dim > 0");
  if (!host && n > 0) throw ArgError("null descriptor pointer");
  DescSet s;
  s.n = n;
  s.dim = dim;
  s.u8 = u8;
  if (u8 && u8_as_l2) throw ArgError("a descriptor set is either Hamming or uint8-stored L2");
  const size_t esz = u8 ? 1 : 4;          // element size of the resident rows
  const size_t hsz = (u8 || u8_as_l2) ? 1 : 4;  // element size of the host rows
  // padded row length in bytes: multiple of DK elements (64 B for both types)
  const int row_bytes = (int)(((size_t)dim * esz + 63) / 64 * 64);
  s.dim_padded = row_bytes / 4;  // in 4-byte elements
  s.row_bytes = row_bytes;
  const bool tc = tc_capable(dim, u8);
  const bool h8 = u8 && h8_capable(dim);     // Hamming on the tensor cores: +-1 fp8 operands
  const size_t data_bytes = align256((size_t)std::max(n, 1) * row_bytes);
  s.rows_padded = (tc || h8) ? tc_rows_padded(n) : 0;
  const size_t tc_bytes = tc ? tc_operand_bytes(s.rows_padded) : h8 ? h8_operand_bytes(s.rows_padded) : 0;
  slab_new(s.rows, data_bytes + tc_bytes, n);
  if (tc) {
    if (d_info.p == nullptr) {
      d_info.reserve(2 * (size_t)MAX_SLOTS);
      OSFM_CUDA(cudaMemsetAsync(d_info.p, 0, sizeof(int) * 2 * (size_t)MAX_SLOTS, stream));
    }
    if (!free_slots.empty()) { s.slot = free_slots.back(); free_slots.pop_back(); }
    else if (next_slot < MAX_SLOTS) s.slot = next_slot++;
    else { release(s.rows); throw std::runtime_error("too many resident descriptor sets"); }
  }
  if (n > 0) {
    const bool dense = !u8_as_l2 && (size_t)dim * esz == (size_t)row_bytes;  // the upload already is the padded copy
    const void* src = s.rows.p;
    if (dense) {
      OSFM_CUDA(cudaMemcpyAsync(s.rows.p, host, (size_t)n * row_bytes, cudaMemcpyHostToDevice, stream));
    } else {
      staging.reserve(std::max<size_t>((size_t)n * dim * hsz, (size_t)4 << 20));
      OSFM_CUDA(cudaMemcpyAsync(staging.p, host, (size_t)n * dim * hsz, cudaMemcpyHostToDevice, stream));
      src = staging.p;
    }
    if (tc) {
      // one fused pass: padded copy (if needed) + exactness + norms + bf16 operands (match_tc.cu)
      prepare_tc(s, src, u8_as_l2, dense ? nullptr : reinterpret_cast<float*>(s.rows.p));
    } else if (u8_as_l2) {
      const size_t total = (size_t)n * s.dim_padded;
      widen_rows_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(staging.p, n, dim, (float*)s.rows.p, s.dim_padded);
      OSFM_LAUNCH_CHECK();
    } else if (!dense) {
      const size_t total = (size_t)n * row_bytes / esz;
      const int threads = 256;
      const unsigned blocks = (unsigned)((total + threads - 1) / threads);
      if (u8)
        pad_rows_kernel<uint8_t><<<blocks, threads, 0, stream>>>(staging.p, n, dim, (uint8_t*)s.rows.p, row_bytes);
      else
        pad_rows_kernel<float><<<blocks, threads, 0, stream>>>((const float*)staging.p, n, dim, (float*)s.rows.p, row_bytes / 4);
      OSFM_LAUNCH_CHECK();
    }
    if (h8) prepare_h8(s, reinterpret_cast<const uint8_t*>(s.rows.p), row_bytes);
  } else {
    // a set without rows is trivially exact: its jobs have no query tiles or no train tiles, so it must not move
    // the rest of a submission off the tensor cores
    s.tc_ok = tc || h8;
  }
  const int id = next_id++;
  sets[id] = s;
  if (s.info_pending) pending.push_back(id);
  return id;
}

void Matcher::set_bearings(int id, const float* host_n_by_3) {
  auto it = sets.find(id);
  if (it == sets.end()) throw ArgError("unknown descriptor set id");
  if (!host_n_by_3) throw ArgError("null bearings");
  DescSet& s = it->second;
  if (!s.bearings.p) slab_new(s.bearings, sizeof(float) * 3 * (size_t)std::max(s.n, 1), s.n);
  if (s.n > 0) {
    OSFM_CUDA(cudaMemcpyAsync(s.bearings.p, host_n_by_3, sizeof(float) * 3 * (size_t)s.n, cudaMemcpyHostToDevice, stream));
    OSFM_CUDA(cudaStreamSynchronize(stream));
  }
}

int Matcher::add(const void* host, int n, int dim, bool u8, bool u8_as_l2) {
  const int id = add_async(host, n, dim, u8, u8_as_l2);
  OSFM_CUDA(cudaStreamSynchronize(stream));  // the caller may reuse its buffer
  return id;
}

void Matcher::remove(int id) {
  auto it = sets.find(id);
  if (it == sets.end()) throw ArgError("unknown descriptor set id");
  OSFM_CUDA(cudaStreamSynchronize(stream));
  free_set(it->second);
  sets.erase(it);
}

void Matcher::clear() {
  OSFM_CUDA(cudaStreamSynchronize(stream));
  for (auto& kv : sets) free_set(kv.second);
  sets.clear();
}

// ---------------------------------------------------------------------------
// A submission, step by step: build_jobs, plan_guided_masks, choose_kernel, cut_chunks, then upload and launch
// (Matcher::match_pairs_async).
// ---------------------------------------------------------------------------
// What the jobs of a submission have in common.
struct JobSummary {
  bool any_u8 = false, any_f32 = false;
  bool all_tc = true;   // every pair bf16-exact and norm-bounded: the tensor-core L2 kernel ranks as cv2 does
  bool all_h8 = true;   // every set has the fp8 operands of the tensor-core Hamming kernel
  int max_nq = 0, max_dim_padded = 0;
};

// m.h_jobs: one job per pair and direction (job 2p is a->b, 2p+1 is b->a when symmetric); m.h_out_off: the first
// result of every pair.
static JobSummary build_jobs(Matcher& m, int npairs, const int* ids_a, const int* ids_b, bool symmetric,
                             const uint8_t* dmask) {
  const int ndir = symmetric ? 2 : 1;
  m.h_jobs.assign(npairs * ndir, MatchJob());
  m.h_out_off.assign(npairs + 1, 0);
  JobSummary js;
  for (int p = 0; p < npairs; ++p) {
    auto ia = m.sets.find(ids_a[p]), ib = m.sets.find(ids_b[p]);
    if (ia == m.sets.end() || ib == m.sets.end()) throw ArgError("unknown descriptor set id in pair list");
    const DescSet& A = ia->second;
    const DescSet& B = ib->second;
    // matching.py:737: assert f1.dtype.type == f2.dtype.type
    if (A.u8 != B.u8 || A.dim != B.dim) throw ArgError("descriptor sets of a pair differ in dtype or dimension");
    js.any_u8 |= A.u8;
    js.any_f32 |= !A.u8;
    js.max_dim_padded = std::max(js.max_dim_padded, A.dim_padded);
    // d^2 <= (|a| + |b|)^2 <= 2 (|a|^2 + |b|^2) must stay below 2^22 for the d^2-space ranking of the
    // tensor-core kernel to equal cv2's sqrt-space ranking (float32 sqrt injective on integers < 2^22)
    js.all_tc &= (!A.u8 && A.tc_ok && B.tc_ok && 2.0f * (A.tc_max_norm + B.tc_max_norm) < 4194304.0f);
    js.all_h8 &= (A.u8 && A.tc_ok && B.tc_ok);
    m.h_out_off[p + 1] = m.h_out_off[p] + A.n;
    for (int d = 0; d < ndir; ++d) {
      MatchJob& j = m.h_jobs[p * ndir + d];
      const DescSet& Qs = d == 0 ? A : B;
      const DescSet& Ts = d == 0 ? B : A;
      j.q = Qs.rows.p; j.t = Ts.rows.p;
      j.q_tc = Qs.tc_q; j.t_tc = Ts.tc_t;
      j.q_norm = Qs.tc_norm; j.t_norm = Ts.tc_norm;
      j.nq = Qs.n; j.nt = Ts.n;
      j.dim = A.dim;
      j.dim_padded = A.dim_padded;
      j.mask = dmask;
      if (dmask) {
        // forward: mask[q*n2 + t]; backward reads the transpose (matching.py:774)
        j.mask_sq = d == 0 ? B.n : 1;
        j.mask_st = d == 0 ? 1 : B.n;
      }
      js.max_nq = std::max(js.max_nq, j.nq);
    }
  }
  if (js.any_u8 && js.any_f32) throw ArgError("mixed float32 / uint8 pairs in one submission");
  return js;
}

// Guided matching: places both layouts of every pair's bitmask in m.d_mask_bits and its epipolar vectors in
// m.d_epi_vec, and points the jobs at their masks.  Returns the records epi_vectors / epi_mask_bits fill them from.
static std::vector<EpiPair> plan_guided_masks(Matcher& m, int npairs, const int* ids_a, const int* ids_b,
                                              bool symmetric, const double* pose12) {
  const int ndir = symmetric ? 2 : 1;
  size_t words = 0, vecs = 0;
  std::vector<EpiPair> epi(npairs);
  for (int p = 0; p < npairs; ++p) {   // offsets first: the buffers are sized by the whole submission
    const DescSet& A = m.sets.find(ids_a[p])->second;
    const DescSet& B = m.sets.find(ids_b[p])->second;
    if (!A.bearings.p || !B.bearings.p) throw ArgError("guided matching needs bearings for both images (osfm_matcher_set_bearings)");
    EpiPair& e = epi[p];
    e.b1 = A.bearings.p; e.b2 = B.bearings.p; e.n1 = A.n; e.n2 = B.n;
    e.w1 = (A.n + 31) / 32; e.w2 = (B.n + 31) / 32;
    e.F = reinterpret_cast<uint32_t*>(words); words += (size_t)A.n * e.w2;
    e.T = reinterpret_cast<uint32_t*>(words); words += (size_t)B.n * e.w1;
    e.v1 = reinterpret_cast<double*>(vecs); vecs += 6 * (size_t)A.n;
    e.v2 = reinterpret_cast<double*>(vecs); vecs += 6 * (size_t)B.n;
    std::memcpy(e.pose, pose12 + 12 * (size_t)p, sizeof(double) * 12);
  }
  if (words > ((size_t)1 << 29)) throw ArgError("guided submission needs more than 2 GiB of mask bits: split the pair list");
  m.d_mask_bits.reserve(std::max<size_t>(words, 1));
  m.d_epi_vec.reserve(std::max<size_t>(vecs, 1));
  for (int p = 0; p < npairs; ++p) {   // offsets -> pointers
    EpiPair& e = epi[p];
    e.F = m.d_mask_bits.p + reinterpret_cast<size_t>(e.F);
    e.T = m.d_mask_bits.p + reinterpret_cast<size_t>(e.T);
    e.v1 = m.d_epi_vec.p + reinterpret_cast<size_t>(e.v1);
    e.v2 = m.d_epi_vec.p + reinterpret_cast<size_t>(e.v2);
    for (int d = 0; d < ndir; ++d) {
      MatchJob& j = m.h_jobs[p * ndir + d];
      j.mask_bits = d == 0 ? e.F : e.T;
      j.mask_words = d == 0 ? e.w2 : e.w1;
    }
    m.last_masks.push_back(EpiMasks{e.F, e.T, e.n1, e.n2, e.w1, e.w2});
  }
  return epi;
}

// choice (osfm_matcher_set_kernel): 0 takes the tensor cores wherever they rank as cv2 does, 1 the SIMT kernels,
// 2 the tensor-core L2 kernel or an error.
static DistKernel choose_kernel(int choice, const JobSummary& js, bool byte_mask, bool guided, int npairs) {
  if (choice == 2) {
    if (!js.all_tc || byte_mask)
      throw ArgError("tensor-core kernel forced but descriptors are not bf16-exact / norm-bounded, or a mask is set");
    return DistKernel::TC_L2;
  }
  if (choice == 0 && js.all_tc && !byte_mask && js.any_f32 && tc_available())
    return DistKernel::TC_L2;   // (guided pairs too: the tensor-core epilogue applies the bitmask)
  if (choice == 0 && js.all_h8 && js.any_u8 && !byte_mask && !guided && npairs > 0 && tc_available())
    return DistKernel::TC_HAMMING;   // Hamming as a +-1 fp8 contraction
  return DistKernel::SIMT;
}

struct TileCounts {
  long long tiles = 0, partials = 0, matches = 0;
};
// Query tiles of the kernel's height; when they are too few to fill the GPU, the trains of every job are split into
// chunks (whole multiples of chunk_unit).  Lays out the partials and results of the jobs, and m.h_prefix: the first
// tile of every job, then the total.
static TileCounts cut_chunks(Matcher& m, const KernelPlan& k) {
  const int njobs = (int)m.h_jobs.size();
  long long total_qtiles = 0;
  for (auto& j : m.h_jobs) { j.qtiles = (j.nq + k.tile_m - 1) / k.tile_m; total_qtiles += j.qtiles; }
  const long long target = (long long)m.num_sms * k.ctas_per_sm;
  m.h_prefix.assign(njobs + 1, 0);
  TileCounts c;
  for (int i = 0; i < njobs; ++i) {
    MatchJob& j = m.h_jobs[i];
    int nchunks = 1;
    if (total_qtiles < target && total_qtiles > 0) {
      const int want = (int)((target + total_qtiles - 1) / total_qtiles);
      const int maxc = std::max(1, (j.nt + k.chunk_unit - 1) / k.chunk_unit);
      nchunks = std::min(want, maxc);
    }
    int chunk_len = (j.nt + nchunks - 1) / nchunks;
    chunk_len = std::max(k.chunk_unit, (chunk_len + k.chunk_unit - 1) / k.chunk_unit * k.chunk_unit);
    nchunks = std::max(1, (j.nt + chunk_len - 1) / chunk_len);
    j.nchunks = nchunks;
    j.chunk_len = chunk_len;
    j.partial_off = c.partials;
    c.partials += (long long)nchunks * j.nq;
    j.match_off = c.matches;
    c.matches += j.nq;
    m.h_prefix[i] = (int)c.tiles;
    c.tiles += (long long)j.qtiles * nchunks;
    if (c.tiles > 0x7fffffffLL) throw ArgError("too many tiles in one submission");
  }
  m.h_prefix[njobs] = (int)c.tiles;
  return c;
}

void Matcher::match_pairs_async(int npairs, const int* ids_a, const int* ids_b, double ratio, bool symmetric,
                                const uint8_t* dmask, const double* pose12, double epi_threshold) {
  refresh_info();
  if (npairs < 0) throw ArgError("npairs < 0");
  if (npairs > 30000) throw ArgError("at most 30000 pairs per submission");
  last_masks.clear();
  const JobSummary js = build_jobs(*this, npairs, ids_a, ids_b, symmetric, dmask);
  const int njobs = (int)h_jobs.size();
  const bool guided = pose12 != nullptr;
  std::vector<EpiPair> epi;
  if (guided) {
    if (dmask) throw ArgError("guided matching builds its own mask");
    epi = plan_guided_masks(*this, npairs, ids_a, ids_b, symmetric, pose12);
  }
  const DistKernel kernel = choose_kernel(kernel_choice, js, dmask != nullptr, guided, npairs);
  last_kernel = (int)kernel;
  last_total_results = h_out_off[npairs];
  last_npairs = npairs;
  const KernelPlan plan = kernel == DistKernel::SIMT ? simt_plan(js.any_u8, js.max_dim_padded) : tc_plan(kernel, guided);
  const TileCounts counts = cut_chunks(*this, plan);

  // ---- upload and launch ----
  d_jobs.reserve(njobs + 1);
  d_prefix.reserve(njobs + 1);
  d_out_off.reserve(npairs + 1);
  d_partial.reserve(std::max<long long>(counts.partials, 1));
  d_match.reserve(std::max<long long>(counts.matches, 1));
  d_out.reserve(std::max<long long>(last_total_results, 1));
  p_jobs.reserve(njobs + 1);
  p_prefix.reserve(njobs + 1);
  p_out_off.reserve(npairs + 1);
  // previous batch may still be reading the pinned staging buffers
  OSFM_CUDA(cudaStreamSynchronize(stream));
  std::copy(h_jobs.begin(), h_jobs.end(), p_jobs.p);
  std::copy(h_prefix.begin(), h_prefix.end(), p_prefix.p);
  std::copy(h_out_off.begin(), h_out_off.end(), p_out_off.p);

  OSFM_CUDA(cudaEventRecord(ev[0], stream));
  if (njobs > 0) {
    OSFM_CUDA(cudaMemcpyAsync(d_jobs.p, p_jobs.p, sizeof(MatchJob) * njobs, cudaMemcpyHostToDevice, stream));
    OSFM_CUDA(cudaMemcpyAsync(d_prefix.p, p_prefix.p, sizeof(int) * (njobs + 1), cudaMemcpyHostToDevice, stream));
    OSFM_CUDA(cudaMemcpyAsync(d_out_off.p, p_out_off.p, sizeof(long long) * (npairs + 1), cudaMemcpyHostToDevice,
                              stream));
  }
  if (guided && npairs > 0) {
    // EpiPair records travel through the (otherwise idle) epi pose buffers: sizeof(EpiPair) is a multiple of 8
    static_assert(sizeof(EpiPair) % sizeof(double) == 0, "EpiPair packs into doubles");
    const size_t nd = sizeof(EpiPair) / sizeof(double) * (size_t)npairs;
    d_epi_pose.reserve(nd); p_epi_pose.reserve(nd);
    std::memcpy(p_epi_pose.p, epi.data(), sizeof(EpiPair) * (size_t)npairs);
    OSFM_CUDA(cudaMemcpyAsync(d_epi_pose.p, p_epi_pose.p, sizeof(EpiPair) * (size_t)npairs, cudaMemcpyHostToDevice, stream));
    const EpiPair* dp = reinterpret_cast<const EpiPair*>(d_epi_pose.p);
    int max_n = 1, max_w1 = 1, max_w2 = 1;
    for (const EpiPair& e : epi) { max_n = std::max({max_n, e.n1, e.n2}); max_w1 = std::max(max_w1, e.w1); max_w2 = std::max(max_w2, e.w2); }
    epi_vectors<<<dim3((max_n + 127) / 128, npairs), 128, 0, stream>>>(dp);
    OSFM_LAUNCH_CHECK();
    epi_mask_bits<<<dim3((max_w2 + 7) / 8, (max_w1 + 7) / 8, npairs), 256, 0, stream>>>(dp, epi_threshold);
    OSFM_LAUNCH_CHECK();
  }
  OSFM_CUDA(cudaEventRecord(ev[1], stream));
  if (counts.tiles > 0) plan.launch(*this, njobs, (int)counts.tiles, plan.smem);
  OSFM_CUDA(cudaEventRecord(ev[2], stream));
  if (njobs > 0 && js.max_nq > 0) {
    dim3 grid((js.max_nq + 255) / 256, njobs);
    bf_top2_finalize<<<grid, 256, 0, stream>>>(d_jobs.p, d_partial.p, d_match.p, ratio, plan.squared ? 1 : 0);
    OSFM_LAUNCH_CHECK();
    if (symmetric) {
      dim3 g2((js.max_nq + 255) / 256, npairs);
      bf_symmetric<<<g2, 256, 0, stream>>>(d_jobs.p, d_match.p, d_out.p, d_out_off.p);
      OSFM_LAUNCH_CHECK();
    }
  }
  results_in_match_buf = !symmetric;
  OSFM_CUDA(cudaEventRecord(ev[3], stream));
}

void Matcher::get_epipolar_masks(int pair, uint32_t* F, uint32_t* T) {
  if (last_masks.empty()) throw ArgError("the last submission was not guided");
  if (pair < 0 || pair >= (int)last_masks.size()) throw ArgError("pair index out of range");
  if (!F || !T) throw ArgError("null output");
  const EpiMasks& e = last_masks[pair];
  const size_t fw = (size_t)e.n1 * e.w2, tw = (size_t)e.n2 * e.w1;
  if (fw) OSFM_CUDA(cudaMemcpyAsync(F, e.F, sizeof(uint32_t) * fw, cudaMemcpyDeviceToHost, stream));
  if (tw) OSFM_CUDA(cudaMemcpyAsync(T, e.T, sizeof(uint32_t) * tw, cudaMemcpyDeviceToHost, stream));
  OSFM_CUDA(cudaStreamSynchronize(stream));
}

void Matcher::fetch(int32_t* out, int64_t capacity) {
  if (capacity < last_total_results) throw ArgError("output buffer too small for the last batch");
  if (last_total_results > 0) {
    // one-way results are laid out per job == per pair in d_match (match_off == out_off)
    const int32_t* src = results_in_match_buf ? d_match.p : d_out.p;
    OSFM_CUDA(cudaMemcpyAsync(out, src, sizeof(int32_t) * last_total_results, cudaMemcpyDeviceToHost, stream));
  }
  OSFM_CUDA(cudaStreamSynchronize(stream));
}

// offsets_out[npairs + 1]: first row of every pair in the packed list; pairs_out: (query, train) int32 rows.
// Returns the number of rows; throws if capacity_rows is too small.
long long Matcher::fetch_pairs(long long* offsets_out, int32_t* pairs_out, long long capacity_rows) {
  const int npairs = last_npairs;
  if (npairs == 0) { if (offsets_out) offsets_out[0] = 0; return 0; }
  const int32_t* src = results_in_match_buf ? d_match.p : d_out.p;
  d_pair_counts.reserve(npairs + 1);
  d_pair_off.reserve(npairs + 2);
  d_pairs.reserve(2 * (size_t)std::max<long long>(last_total_results, 1));
  bf_pair_counts<<<npairs, 256, 0, stream>>>(src, d_out_off.p, d_pair_counts.p);
  OSFM_LAUNCH_CHECK();
  bf_pair_scan<<<1, 1024, 0, stream>>>(d_pair_counts.p, npairs, d_pair_off.p);
  OSFM_LAUNCH_CHECK();
  bf_pair_compact<<<npairs, 256, 0, stream>>>(src, d_out_off.p, d_pair_off.p, d_pairs.p);
  OSFM_LAUNCH_CHECK();
  OSFM_CUDA(cudaMemcpyAsync(offsets_out, d_pair_off.p, sizeof(long long) * (npairs + 1), cudaMemcpyDeviceToHost, stream));
  OSFM_CUDA(cudaStreamSynchronize(stream));
  const long long total = offsets_out[npairs];
  if (total > capacity_rows) throw ArgError("output buffer too small for the packed match lists");
  if (total > 0) {
    OSFM_CUDA(cudaMemcpyAsync(pairs_out, d_pairs.p, sizeof(int32_t) * 2 * (size_t)total, cudaMemcpyDeviceToHost, stream));
    OSFM_CUDA(cudaStreamSynchronize(stream));
  }
  return total;
}

void Matcher::last_ms(float* total, float* kernel) {
  OSFM_CUDA(cudaEventSynchronize(ev[3]));
  if (total) OSFM_CUDA(cudaEventElapsedTime(total, ev[0], ev[3]));
  if (kernel) OSFM_CUDA(cudaEventElapsedTime(kernel, ev[1], ev[2]));
}

void Matcher::one_shot(const void* f1, int n1, const void* f2, int n2, int dim, bool u8, double ratio,
                       const uint8_t* mask, bool symmetric, int32_t* out) {
  if (n1 < 0 || n2 < 0) throw ArgError("negative descriptor count");
  if (!out && n1 > 0) throw ArgError("null output");
  const int a = add(f1, n1, dim, u8);
  int b = -1;
  try {
    b = add(f2, n2, dim, u8);
    const uint8_t* dmask = nullptr;
    if (mask && n1 > 0 && n2 > 0) {
      mask_buf.reserve((size_t)n1 * n2);
      OSFM_CUDA(cudaMemcpyAsync(mask_buf.p, mask, (size_t)n1 * n2, cudaMemcpyHostToDevice, stream));
      dmask = mask_buf.p;
    }
    match_pairs_async(1, &a, &b, ratio, symmetric, dmask);
    fetch(out, n1);
  } catch (...) {
    if (b >= 0) remove(b);
    remove(a);
    throw;
  }
  remove(b);
  remove(a);
}

}  // namespace osfm

// ---------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------
using osfm::Matcher;

extern "C" {

int osfm_matcher_create(int device, osfm_matcher** out) { return osfm::create_handle(device, out); }
int osfm_matcher_destroy(osfm_matcher* m) { return osfm::destroy_handle(m); }

int osfm_bf_match_f32(osfm_matcher* m, const float* f1, int n1, const float* f2, int n2, int dim,
                      double lowes_ratio, const uint8_t* mask, int symmetric, int32_t* out_match) {
  return osfm::with_handle(
      m, [&](Matcher& M) { M.one_shot(f1, n1, f2, n2, dim, false, lowes_ratio, mask, symmetric != 0, out_match); });
}

int osfm_bf_match_u8(osfm_matcher* m, const uint8_t* f1, int n1, const uint8_t* f2, int n2, int nbytes,
                     double lowes_ratio, const uint8_t* mask, int symmetric, int32_t* out_match) {
  return osfm::with_handle(
      m, [&](Matcher& M) { M.one_shot(f1, n1, f2, n2, nbytes, true, lowes_ratio, mask, symmetric != 0, out_match); });
}

static int add_one(osfm_matcher* m, const void* desc, int n, int dim, bool u8, int* out_id, bool u8_as_l2 = false) {
  return osfm::with_handle(m, [&](Matcher& M) {
    if (!out_id) throw osfm::ArgError("null out_id");
    *out_id = M.add(desc, n, dim, u8, u8_as_l2);
  });
}
int osfm_matcher_add_f32(osfm_matcher* m, const float* desc, int n, int dim, int* out_id) {
  return add_one(m, desc, n, dim, false, out_id);
}
int osfm_matcher_add_u8(osfm_matcher* m, const uint8_t* desc, int n, int nbytes, int* out_id) {
  return add_one(m, desc, n, nbytes, true, out_id);
}

static int add_batch(osfm_matcher* m, int count, const void* const* desc, const int* n, int dim, bool u8, int* out_ids,
                     bool u8_as_l2 = false) {
  return osfm::with_handle(m, [&](Matcher& M) {
    if (count < 0 || (count > 0 && (!desc || !n || !out_ids))) throw osfm::ArgError("bad batch arguments");
    int done = 0;
    try {
      for (; done < count; ++done) out_ids[done] = M.add_async(desc[done], n[done], dim, u8, u8_as_l2);
      OSFM_CUDA(cudaStreamSynchronize(M.stream));
    } catch (...) {
      cudaStreamSynchronize(M.stream);
      for (int i = 0; i < done; ++i) M.remove(out_ids[i]);
      throw;
    }
  });
}
int osfm_matcher_add_batch_f32(osfm_matcher* m, int count, const float* const* desc, const int* n, int dim, int* out_ids) {
  return add_batch(m, count, reinterpret_cast<const void* const*>(desc), n, dim, false, out_ids);
}
int osfm_matcher_add_batch_u8(osfm_matcher* m, int count, const uint8_t* const* desc, const int* n, int nbytes,
                              int* out_ids) {
  return add_batch(m, count, reinterpret_cast<const void* const*>(desc), n, nbytes, true, out_ids);
}

int osfm_matcher_add_u8_l2(osfm_matcher* m, const uint8_t* desc, int n, int dim, int* out_id) {
  return add_one(m, desc, n, dim, false, out_id, true);
}
int osfm_matcher_add_batch_u8_l2(osfm_matcher* m, int count, const uint8_t* const* desc, const int* n, int dim,
                                 int* out_ids) {
  return add_batch(m, count, reinterpret_cast<const void* const*>(desc), n, dim, false, out_ids, true);
}

int osfm_matcher_remove(osfm_matcher* m, int id) {
  return osfm::with_handle(m, [&](Matcher& M) { M.remove(id); });
}

int osfm_matcher_clear(osfm_matcher* m) {
  return osfm::with_handle(m, [&](Matcher& M) { M.clear(); });
}

int osfm_matcher_match_pairs_async(osfm_matcher* m, int npairs, const int* ids_a, const int* ids_b,
                                   double lowes_ratio, int symmetric) {
  return osfm::with_handle(m, [&](Matcher& M) {
    if (npairs > 0 && (!ids_a || !ids_b)) throw osfm::ArgError("null pair list");
    M.match_pairs_async(npairs, ids_a, ids_b, lowes_ratio, symmetric != 0, nullptr);
  });
}

int osfm_matcher_set_bearings(osfm_matcher* m, int id, const float* bearings_n_by_3) {
  return osfm::with_handle(m, [&](Matcher& M) { M.set_bearings(id, bearings_n_by_3); });
}

int osfm_matcher_match_pairs_guided_async(osfm_matcher* m, int npairs, const int* ids_a, const int* ids_b,
                                          const double* pose12, double threshold, double lowes_ratio, int symmetric) {
  return osfm::with_handle(m, [&](Matcher& M) {
    if (npairs > 0 && (!ids_a || !ids_b || !pose12)) throw osfm::ArgError("null pair list / poses");
    // any threshold is the reference's comparison `angle < threshold`: at or below 0 nothing passes
    if (std::isnan(threshold)) throw osfm::ArgError("guided matching threshold is NaN");
    M.match_pairs_async(npairs, ids_a, ids_b, lowes_ratio, symmetric != 0, nullptr, pose12, threshold);
  });
}

int osfm_matcher_get_epipolar_masks(osfm_matcher* m, int pair, uint32_t* F, uint32_t* T) {
  return osfm::with_handle(m, [&](Matcher& M) { M.get_epipolar_masks(pair, F, T); });
}

int osfm_matcher_sync(osfm_matcher* m) {
  return osfm::with_handle(m, [&](Matcher& M) { OSFM_CUDA(cudaStreamSynchronize(M.stream)); });
}

int osfm_matcher_fetch(osfm_matcher* m, int32_t* out_match, int64_t capacity) {
  return osfm::with_handle(m, [&](Matcher& M) { M.fetch(out_match, capacity); });
}

int osfm_matcher_fetch_pairs(osfm_matcher* m, int64_t* offsets_out, int32_t* pairs_out, int64_t capacity_rows,
                             int64_t* total_rows) {
  return osfm::with_handle(m, [&](Matcher& M) {
    if (!offsets_out || !total_rows || (capacity_rows > 0 && !pairs_out)) throw osfm::ArgError("null output");
    static_assert(sizeof(long long) == sizeof(int64_t), "offsets are 64-bit");
    *total_rows = M.fetch_pairs(reinterpret_cast<long long*>(offsets_out), pairs_out, capacity_rows);
  });
}

int osfm_matcher_last_device_ms(osfm_matcher* m, float* ms_total, float* ms_distance_kernel) {
  return osfm::with_handle(m, [&](Matcher& M) { M.last_ms(ms_total, ms_distance_kernel); });
}

int osfm_matcher_set_kernel(osfm_matcher* m, int which) {
  return osfm::with_handle(m, [&](Matcher& M) {
    if (which < 0 || which > 2) throw osfm::ArgError("kernel must be 0, 1 or 2");
    M.kernel_choice = which;
  });
}

// returns the kernel, not an error code, and 0 when the call fails (a null matcher, for one)
int osfm_matcher_last_kernel(osfm_matcher* m) {
  int kernel = 0;
  osfm::with_handle(m, [&](Matcher& M) { kernel = M.last_kernel; });
  return kernel;
}

int osfm_matcher_device_bytes(osfm_matcher* m, int64_t* reserved, int64_t* in_use) {
  return osfm::with_handle(m, [&](Matcher& M) {
    if (!reserved || !in_use) throw osfm::ArgError("null argument");
    int64_t cap = 0, used = 0;
    for (const auto& sl : M.slabs) {
      cap += (int64_t)sl.cap;
      used += (int64_t)sl.used;
      for (const auto& fr : sl.free_ranges) used -= (int64_t)fr.second;
    }
    *reserved = cap;
    *in_use = used;
  });
}

}  // extern "C"
