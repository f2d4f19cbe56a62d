// RELPOSE: five-point relative-pose RANSAC of many image pairs at once, for the two-view bootstrap of the incremental
// reconstruction.
//
// Replaces, for every pair, pyrobust's ransac_relative_pose with RANSAC scoring (robust/robust_estimator.h,
// relative_pose_model.h) as multiview.relative_pose_ransac calls it.  The restatement the results are checked
// against, and the rules it follows, are in oracle/relative_pose_oracle.py; the solvers are relative_pose.cuh.
//
// One CTA per pair (rp_ransac), largest pairs first.  Thread 0 draws the 5-row sample from the shared mt19937(42)
// stream (ransac_stream.cuh), solves the five-point problem and decomposes each essential; the whole CTA then
// scores the up to 10 models of the sample in one pass over the rows, and the decisions the reference takes model by
// model (replace the best, local optimisation, stop) are replayed in model order from those counts.  A model's
// inlier rows are listed, in ascending order, only when it becomes the best one with at least 5 inliers: local
// optimisation samples from that list, thread 0 fits EssentialNPoints to the sample and the CTA counts its inliers.
// A pair of at most RANSAC_STAGE_ROWS rows is staged in shared memory (both bearings); a larger one is read through
// L2 via its row indices.  A last pass writes the inlier mask of the result.  The sample stream, the row passes, the
// launch plan and the argument checks are those of ransac_stream.cuh.
#include <math_constants.h>

#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <vector>

#include "common.cuh"
#include "ransac_stream.cuh"
#include "relative_pose.cuh"

namespace osfm {
namespace {

constexpr int RP_MIN_SAMPLE = 5;
constexpr int RP_MAX_SAMPLE = 12;          // local optimisation samples min(12, inliers / 2) rows (at least 5)
constexpr int RP_MAX_MODELS = relpose::MAX_MODELS;
constexpr int RP_LO_ITERATIONS = 10;

struct RpArgs {
  const double* bearings;        // 3 per entry, normalised
  const long long* pair_start;
  const long long* row_a;        // first image's bearing of row r
  const long long* row_b;        // second image's bearing of row r
  const int* order;              // pairs of this launch
  double threshold;              // 1 - cos(angle)
  int iterations;
  StreamSource src;
  int* best_rows;                // per row: the best model's inlier rows, ascending
  double* lo_model;              // 12 per pair
  int* ransac_inliers;
  unsigned char* mask;           // per row
};

struct RpShared {
  StreamState st;
  double x1[RP_MAX_SAMPLE * 3], x2[RP_MAX_SAMPLE * 3];
  double models[RP_MAX_MODELS][12];
  double cand[12];
  double best[12];
  int idx[RP_MAX_SAMPLE];
  int nm;
  int counts[RP_MAX_MODELS];
  int cand_count, best_count;
  int stop;
  int warp_n[RP_MAX_MODELS][RANSAC_WARPS];
};

__device__ __forceinline__ bool rp_inlier(const double* M, const double* x, const double* y, double t) {
  return fabs(relpose::evaluate(M, x, y)) < t;
}

// RelativePose::Evaluate's inlier test of RANSAC scoring: |1 - agreement| below t = 1 - cos(threshold)
struct RpErrorTest {
  double t;
  __device__ __forceinline__ bool operator()(const double* M, const double* x, const double* y) const {
    return rp_inlier(M, x, y, t);
  }
};

// inliers (by `test`) of the nm models at M (12 apart, in shared memory) into counts, in one pass over the rows;
// warp_n is RP_MAX_MODELS x RANSAC_WARPS ints of shared scratch
template <class Test>
__device__ void rp_count(int* warp_n, const RansacRows& rows, const double* M, int nm, Test test, int* counts) {
  int c[RP_MAX_MODELS];
#pragma unroll
  for (int j = 0; j < RP_MAX_MODELS; ++j) c[j] = 0;
  for (int i = threadIdx.x; i < rows.n; i += RANSAC_THREADS) {
    double x[3], y[3];
    rows.get(i, x, y);
#pragma unroll
    for (int j = 0; j < RP_MAX_MODELS; ++j)
      if (j < nm) c[j] += test(M + 12 * j, x, y) ? 1 : 0;
  }
  ransac_sums(c, nm, warp_n, counts);
}

// thread 0's solvers, out of line so that their registers and stack do not weigh on the CTA's passes over the rows
__device__ __noinline__ int rp_five_point(const double* x1, const double* x2, double* models) {
  double Es[9 * RP_MAX_MODELS], margin;
  const int ne = relpose::five_point(x1, x2, Es, &margin);
  for (int e = 0; e < ne; ++e) relpose::pose_from_essential(Es + 9 * e, RP_MIN_SAMPLE, x1, x2, models + 12 * e, &margin);
  return ne;
}

__device__ __noinline__ int rp_n_points(int k, const double* x1, const double* x2, double* out) {
  double E[9], margin;
  if (!relpose::n_points(k, x1, x2, E, &margin)) return 0;
  relpose::pose_from_essential(E, k, x1, x2, out, &margin);
  return 1;
}

__global__ void __launch_bounds__(RANSAC_THREADS) rp_ransac(RpArgs a, int staged) {
  __shared__ RpShared s;
  const int pair = a.order[blockIdx.x];
  const long long off = a.pair_start[pair];
  const RansacRows rows =
      ransac_rows(a.bearings, a.bearings, a.row_a + off, a.row_b + off, (int)(a.pair_start[pair + 1] - off), staged);
  const int n = rows.n;
  int* best_rows = a.best_rows + off;
  const double t = a.threshold;
  if (threadIdx.x == 0) {
    s.st.reset();
    s.best_count = 0;
    s.stop = 0;
    for (int k = 0; k < 12; ++k) s.best[k] = 0.0;
  }
  __syncthreads();

  for (int it = 0; it < a.iterations; ++it) {
    if (threadIdx.x == 0) {
      stream_sample(s.st, a.src, pair, RP_MIN_SAMPLE, n, s.idx);
      for (int k = 0; k < RP_MIN_SAMPLE; ++k) rows.get(s.idx[k], s.x1 + 3 * k, s.x2 + 3 * k);
      s.nm = rp_five_point(s.x1, s.x2, &s.models[0][0]);
    }
    __syncthreads();
    const int nm = s.nm;
    if (nm > 0) rp_count(&s.warp_n[0][0], rows, &s.models[0][0], nm, RpErrorTest{t}, s.counts);
    // the models in order: std::max(score, best) keeps the new one on ties, then LO, then ShouldStop
    for (int j = 0; j < nm; ++j) {
      const int c = s.counts[j];
      if (c >= s.best_count) {
        __syncthreads();
        if (threadIdx.x == 0) {
          for (int k = 0; k < 12; ++k) s.best[k] = s.models[j][k];
          s.best_count = c;
        }
        if (c >= RP_MIN_SAMPLE) {
          ransac_compact<12>(rows, s.models[j], RpErrorTest{t}, s.warp_n[0], best_rows);
          for (int lo = 0; lo < RP_LO_ITERATIONS; ++lo) {
            if (threadIdx.x == 0) {
              const int m = s.best_count;
              const int size = max(min(RP_MAX_SAMPLE, (int)(m * 0.5)), RP_MIN_SAMPLE);
              stream_sample(s.st, a.src, pair, size, m, s.idx);
              for (int k = 0; k < size; ++k) rows.get(best_rows[s.idx[k]], s.x1 + 3 * k, s.x2 + 3 * k);
              s.nm = rp_n_points(size, s.x1, s.x2, s.cand);
            }
            __syncthreads();
            if (s.nm > 0) {
              rp_count(&s.warp_n[0][0], rows, s.cand, 1, RpErrorTest{t}, &s.cand_count);
              if (s.cand_count >= s.best_count) {
                ransac_compact<12>(rows, s.cand, RpErrorTest{t}, s.warp_n[0], best_rows);
                if (threadIdx.x == 0) {
                  for (int k = 0; k < 12; ++k) s.best[k] = s.cand[k];
                  s.best_count = s.cand_count;
                }
              }
            }
            __syncthreads();
          }
        }
        __syncthreads();
      }
      if (threadIdx.x == 0) s.stop = ransac_should_stop(s.best_count, n, it, RP_MIN_SAMPLE);
      __syncthreads();
      const bool stop = s.stop;
      __syncthreads();
      if (stop) break;
    }
    const bool stop = s.stop;
    __syncthreads();
    if (stop) break;
  }

  // the inlier mask of the result (pyrobust's inliers_indices)
  double M[12];
  for (int k = 0; k < 12; ++k) M[k] = s.best[k];
  for (int i = threadIdx.x; i < n; i += RANSAC_THREADS) {
    double x[3], y[3];
    rows.get(i, x, y);
    a.mask[off + i] = rp_inlier(M, x, y, t) ? 1 : 0;
  }
  if (threadIdx.x == 0) {
    a.ransac_inliers[pair] = s.best_count;
    for (int k = 0; k < 12; ++k) a.lo_model[12LL * pair + k] = M[k];
    stream_record(s.st, a.src, pair);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// rp_two_view: the rest of two_view_reconstruction_general after RANSAC, per pair, from rp_ransac's lo_model
// ---------------------------------------------------------------------------------------------------------------
constexpr int TV_CONFIGS = 2;              // the pose, and its transpose when the Necker reversal is checked
constexpr int TV_MIN_REFINE = 6;           // refined when more than 5 rows are inliers; kept when more than 5 remain
constexpr double TV_GRADIENT_TOLERANCE = 1e-10;
constexpr double TV_PARAMETER_TOLERANCE = 1e-8;
constexpr double TV_COST_THRESHOLD = 2.220446049250313e-16;
constexpr double TV_INITIAL_TRUST_REGION = 1e4;
constexpr double TV_MIN_DIAGONAL = 1e-6, TV_MAX_DIAGONAL = 1e32;

// float(rand_k) / float(RAND_MAX) of the first 100 glibc rand() outputs after srand(42): RelativePoseCost's table
__constant__ float tv_pick_fraction[relpose::REFINE_PICKED];

struct TvArgs {
  const double* bearings;
  const long long* pair_start;
  const long long* row_a;
  const long long* row_b;
  const int* order;
  const double* lo_model;        // rp_ransac's, 12 per pair
  const double* plane_pose;      // 12 per pair: the plane motion [R_p | t_p], NaN when there is none
  double threshold;              // chord
  int refine_iterations;
  int configurations;            // 1, or 2 with the transposed pose
  double reversal_ratio;
  int* lists;                    // 2 per row: each configuration's first inlier rows, ascending
  double* pose;                  // 24 per pair: each configuration's final [R | t]
  int* counts;                   // 3 per pair: final inliers of each configuration, then of the plane motion
  int* chosen;                   // per pair: the 5-point configuration kept, -1 for none
  unsigned char* mask5;          // per row: the 5-point result's inliers
  unsigned char* maskp;          // per row: the plane result's inliers
};

struct TvBearingTest {
  double thr;
  __device__ __forceinline__ bool operator()(const double* M, const double* x, const double* y) const {
    return relpose::bearing_inlier(M, x, y, thr);
  }
};

__device__ __forceinline__ double tv_warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// RelativePoseCost at p over the warp, the picked rows across lanes: returns f . f; with JAC also the unscaled
// normal equations A = J^T J (upper triangle, row by row) and je = J^T (-f).  Every lane gets the sums.
template <bool JAC>
__device__ double tv_evaluate(const RansacRows& rows, const int* list, int count, const double* p, double* A,
                              double* je) {
  const int lane = threadIdx.x & 31;
  double ff = 0.0;
  if (JAC) {
    for (int k = 0; k < 21; ++k) A[k] = 0.0;
    for (int k = 0; k < 6; ++k) je[k] = 0.0;
  }
  for (int k = lane; k <= relpose::REFINE_PICKED; k += 32) {
    double x[3], y[3];
    if (k < relpose::REFINE_PICKED) {
      const int idx = (int)__fmul_rn(tv_pick_fraction[k], (float)count);
      rows.get(list[idx], x, y);
    }
    if (JAC) {
      relpose::Dual6 P[6];
      for (int i = 0; i < 6; ++i) {
        P[i] = relpose::Dual6(p[i]);
        P[i].d[i] = 1.0;
      }
      const relpose::Dual6 f =
          k < relpose::REFINE_PICKED ? relpose::refine_residual(P, x, y) : relpose::refine_norm_residual(P);
      ff += f.v * f.v;
      int e = 0;
      for (int i = 0; i < 6; ++i) {
        je[i] -= f.d[i] * f.v;
        for (int j = i; j < 6; ++j) A[e++] += f.d[i] * f.d[j];
      }
    } else {
      const double f = k < relpose::REFINE_PICKED ? relpose::refine_residual(p, x, y) : relpose::refine_norm_residual(p);
      ff += f * f;
    }
  }
  if (JAC) {
    for (int k = 0; k < 21; ++k) A[k] = tv_warp_sum(A[k]);
    for (int k = 0; k < 6; ++k) je[k] = tv_warp_sum(je[k]);
  }
  return tv_warp_sum(ff);
}

// TinySolver's scaled normal equations jtj = S A S (full), g = S je, from the packed A; returns max |g|
__device__ __forceinline__ double tv_scale(const double* A, const double* je, const double* s, double* jtj, double* g) {
  int e = 0;
  for (int i = 0; i < 6; ++i)
    for (int j = i; j < 6; ++j, ++e) jtj[i * 6 + j] = jtj[j * 6 + i] = s[i] * A[e] * s[j];
  double gmax = 0.0;
  for (int i = 0; i < 6; ++i) {
    g[i] = s[i] * je[i];
    gmax = fmax(gmax, fabs(g[i]));
  }
  return gmax;
}

// y = M^{-1} b for the symmetric positive definite 6 x 6 M (destroyed), by Cholesky
__device__ __forceinline__ void tv_cholesky_solve(double* M, const double* b, double* y) {
  for (int j = 0; j < 6; ++j) {
    double d = M[j * 6 + j];
    for (int k = 0; k < j; ++k) d -= M[j * 6 + k] * M[j * 6 + k];
    d = sqrt(d);
    M[j * 6 + j] = d;
    for (int i = j + 1; i < 6; ++i) {
      double v = M[i * 6 + j];
      for (int k = 0; k < j; ++k) v -= M[i * 6 + k] * M[j * 6 + k];
      M[i * 6 + j] = v / d;
    }
  }
  double z[6];
  for (int i = 0; i < 6; ++i) {
    double v = b[i];
    for (int k = 0; k < i; ++k) v -= M[i * 6 + k] * z[k];
    z[i] = v / M[i * 6 + i];
  }
  for (int i = 5; i >= 0; --i) {
    double v = z[i];
    for (int k = i + 1; k < 6; ++k) v -= M[k * 6 + i] * y[k];
    y[i] = v / M[i * 6 + i];
  }
}

// RelativePoseRefinement of the pose B (in shared memory) on the picked inlier rows, by one warp: TinySolver with
// max_num_iterations = iterations (rules in oracle/two_view_oracle.py); every lane runs the same control, lane 0
// writes the result.
__device__ __noinline__ void tv_refine(const RansacRows& rows, const int* list, int count, int iterations, double* B) {
  double x[6], A[21], je[6], s[6], jtj[36], g[6];
  relpose::refine_parameters(B, x);
  double cost = 0.5 * tv_evaluate<true>(rows, list, count, x, A, je);
  int e = 0;
  for (int i = 0; i < 6; ++i) {
    s[i] = 1.0 / (1.0 + sqrt(A[e]));
    e += 6 - i;
  }
  double gmax = tv_scale(A, je, s, jtj, g);
  if (!(gmax < TV_GRADIENT_TOLERANCE)) {
    double u = 1.0 / TV_INITIAL_TRUST_REGION, v = 2.0;
    for (int it = 1; it < iterations; ++it) {
      double reg[36], step[6], dx[6], xn[6];
      for (int k = 0; k < 36; ++k) reg[k] = jtj[k];
      for (int i = 0; i < 6; ++i) reg[i * 7] += u * fmin(fmax(jtj[i * 7], TV_MIN_DIAGONAL), TV_MAX_DIAGONAL);
      tv_cholesky_solve(reg, g, step);
      double dn = 0.0, xnorm = 0.0;
      for (int i = 0; i < 6; ++i) {
        dx[i] = s[i] * step[i];
        dn += dx[i] * dx[i];
        xnorm += x[i] * x[i];
      }
      if (sqrt(dn) < TV_PARAMETER_TOLERANCE * (sqrt(xnorm) + TV_PARAMETER_TOLERANCE)) break;
      for (int i = 0; i < 6; ++i) xn[i] = x[i] + dx[i];
      const double cost_change = 2.0 * cost - tv_evaluate<false>(rows, list, count, xn, nullptr, nullptr);
      double model_change = 0.0;
      for (int i = 0; i < 6; ++i) {
        double h = 0.0;
        for (int j = 0; j < 6; ++j) h += jtj[i * 6 + j] * step[j];
        model_change += step[i] * (2.0 * g[i] - h);
      }
      const double rho = cost_change / model_change;
      if (rho > 0.0) {
        for (int i = 0; i < 6; ++i) x[i] = xn[i];
        cost = 0.5 * tv_evaluate<true>(rows, list, count, x, A, je);
        gmax = tv_scale(A, je, s, jtj, g);
        if (gmax < TV_GRADIENT_TOLERANCE || cost < TV_COST_THRESHOLD) break;
        const double t = 2.0 * rho - 1.0;
        u *= fmax(1.0 / 3.0, 1.0 - t * t * t);
        v = 2.0;
      } else {
        u *= v;
        v *= 2.0;
      }
    }
  }
  __syncwarp();
  if ((threadIdx.x & 31) == 0) relpose::refine_pose(x, B);
  __syncwarp();
}

__global__ void __launch_bounds__(RANSAC_THREADS) rp_two_view(TvArgs a, int staged) {
  __shared__ int warp_n[TV_CONFIGS + 1][RANSAC_WARPS];
  __shared__ double B[TV_CONFIGS + 1][12];   // the configurations' poses, then the plane motion's
  __shared__ int counts[TV_CONFIGS + 1];
  __shared__ int first[TV_CONFIGS];
  __shared__ int chosen;
  const int pair = a.order[blockIdx.x];
  const long long off = a.pair_start[pair];
  const RansacRows rows =
      ransac_rows(a.bearings, a.bearings, a.row_a + off, a.row_b + off, (int)(a.pair_start[pair + 1] - off), staged);
  const int n = rows.n;
  if (threadIdx.x == 0) {
    // multiview.relative_pose_ransac's [R^T | -R^T t] of lo_model = [R | t], then its transpose (R^T, -R^T t)
    const double* L = a.lo_model + 12LL * pair;
    for (int i = 0; i < 3; ++i) {
      for (int j = 0; j < 3; ++j) B[0][i * 4 + j] = L[j * 4 + i];
      B[0][i * 4 + 3] = -(L[i] * L[3] + L[4 + i] * L[7] + L[8 + i] * L[11]);
    }
    for (int i = 0; i < 3; ++i) {
      for (int j = 0; j < 3; ++j) B[1][i * 4 + j] = a.configurations > 1 ? B[0][j * 4 + i] : CUDART_NAN;
      B[1][i * 4 + 3] = a.configurations > 1 ? -(B[0][i] * B[0][3] + B[0][4 + i] * B[0][7] + B[0][8 + i] * B[0][11])
                                             : CUDART_NAN;
    }
    // the plane motion's inliers are those of (R_p^T, -R_p^T t_p)
    const double* P = a.plane_pose + 12LL * pair;
    for (int i = 0; i < 3; ++i) {
      for (int j = 0; j < 3; ++j) B[2][i * 4 + j] = P[j * 4 + i];
      B[2][i * 4 + 3] = -(P[i] * P[3] + P[4 + i] * P[7] + P[8 + i] * P[11]);
    }
  }
  __syncthreads();
  const TvBearingTest test{a.threshold};
  int* lists = a.lists + 2 * off;
  for (int c = 0; c < a.configurations; ++c) {
    const int m = ransac_compact<12>(rows, B[c], test, warp_n[0], lists + (long long)c * n);
    if (threadIdx.x == 0) first[c] = m;
  }
  __syncthreads();
  // one warp per configuration: the two of a Necker check are refined at once
  const int warp = threadIdx.x >> 5;
  if (warp < a.configurations && first[warp] >= TV_MIN_REFINE)
    tv_refine(rows, lists + (long long)warp * n, first[warp], a.refine_iterations, B[warp]);
  __syncthreads();
  rp_count(&warp_n[0][0], rows, &B[0][0], TV_CONFIGS + 1, test, counts);
  if (threadIdx.x == 0) {
    // two_view_reconstruction_5pt: keep a configuration with more than 5 inliers; of two, none when
    // min / max > reversal_ratio, else the larger, the transposed one on a tie
    const bool k0 = counts[0] >= TV_MIN_REFINE, k1 = a.configurations > 1 && counts[1] >= TV_MIN_REFINE;
    int c = k0 ? 0 : (k1 ? 1 : -1);
    if (k0 && k1) {
      const double ratio = (double)min(counts[0], counts[1]) / (double)max(counts[0], counts[1]);
      c = ratio > a.reversal_ratio ? -1 : (counts[0] > counts[1] ? 0 : 1);
    }
    chosen = c;
  }
  __syncthreads();
  const int c = chosen;
  for (int i = threadIdx.x; i < n; i += RANSAC_THREADS) {
    double x[3], y[3];
    rows.get(i, x, y);
    a.mask5[off + i] = c >= 0 && test(B[c], x, y) ? 1 : 0;
    a.maskp[off + i] = test(B[2], x, y) ? 1 : 0;
  }
  if (threadIdx.x == 0) {
    for (int k = 0; k < 12 * TV_CONFIGS; ++k) a.pose[24LL * pair + k] = B[k / 12][k % 12];
    for (int k = 0; k <= TV_CONFIGS; ++k) a.counts[3LL * pair + k] = counts[k];
    a.chosen[pair] = c;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// rp_match_filter: robust_match_calibrated after its RANSAC, per pair, from rp_ransac's lo_model
// ---------------------------------------------------------------------------------------------------------------
constexpr int RM_ROUNDS = 3;               // the bearing inliers at 4, 2 and 1 times the threshold, each refined
constexpr int RM_MIN_INLIERS = 8;          // a round with fewer inliers empties the pair

struct RmArgs {
  const double* bearings;
  const long long* pair_start;
  const long long* row_a;
  const long long* row_b;
  const int* order;
  const double* lo_model;        // rp_ransac's, 12 per pair
  double threshold;              // chord
  int refine_iterations;
  int* lists;                    // per row: the current round's inlier rows, ascending
  double* pose;                  // 12 per pair: the refined [R | t], NaN when the pair ends empty
  int* counts;                   // 4 per pair: inliers of each round, then of the final pass; -1 for a pass not run
  unsigned char* mask;           // per row: the final inliers
};

__global__ void __launch_bounds__(RANSAC_THREADS) rp_match_filter(RmArgs a, int staged) {
  __shared__ int warp_n[RANSAC_WARPS];
  __shared__ double B[12];
  __shared__ int final_count;
  const int pair = a.order[blockIdx.x];
  const long long off = a.pair_start[pair];
  const RansacRows rows =
      ransac_rows(a.bearings, a.bearings, a.row_a + off, a.row_b + off, (int)(a.pair_start[pair + 1] - off), staged);
  const int n = rows.n;
  if (threadIdx.x == 0) {
    // multiview.relative_pose_ransac's [R^T | -R^T t] of lo_model = [R | t]
    const double* L = a.lo_model + 12LL * pair;
    for (int i = 0; i < 3; ++i) {
      for (int j = 0; j < 3; ++j) B[i * 4 + j] = L[j * 4 + i];
      B[i * 4 + 3] = -(L[i] * L[3] + L[4 + i] * L[7] + L[8 + i] * L[11]);
    }
  }
  __syncthreads();
  int* list = a.lists + off;
  int* counts = a.counts + 4LL * pair;
  // matching.py's relax loop; every thread gets the same count, so the CTA leaves the loop together
  bool empty = false;
  int round = 0;
  for (; round < RM_ROUNDS && !empty; ++round) {
    const int m = ransac_compact<12>(rows, B, TvBearingTest{(double)(4 >> round) * a.threshold}, warp_n, list);
    if (threadIdx.x == 0) counts[round] = m;
    empty = m < RM_MIN_INLIERS;
    if (!empty) {
      if (threadIdx.x < 32) tv_refine(rows, list, m, a.refine_iterations, B);
      __syncthreads();
    }
  }
  const TvBearingTest test{a.threshold};
  int c[1] = {0};
  for (int i = threadIdx.x; i < n; i += RANSAC_THREADS) {
    bool in = false;
    if (!empty) {
      double x[3], y[3];
      rows.get(i, x, y);
      in = test(B, x, y);
    }
    a.mask[off + i] = in ? 1 : 0;
    c[0] += in ? 1 : 0;
  }
  if (!empty) ransac_sums(c, 1, warp_n, &final_count);
  if (threadIdx.x == 0) {
    for (int k = 0; k < 12; ++k) a.pose[12LL * pair + k] = empty ? CUDART_NAN : B[k];
    for (int r = round; r < RM_ROUNDS; ++r) counts[r] = -1;
    counts[RM_ROUNDS] = empty ? -1 : final_count;
  }
}

// the first `count` outputs of glibc's rand() after srand(seed) (random_r's TYPE_3 additive generator)
void glibc_rand(unsigned seed, int count, std::vector<int>& out) {
  std::vector<int32_t> r(344 + (size_t)count);
  r[0] = (int32_t)seed;
  for (int i = 1; i < 31; ++i) {
    // 16807 * r[i - 1] % 2147483647 by Schrage's method, as srandom_r computes it
    const int32_t hi = r[i - 1] / 127773, lo = r[i - 1] % 127773;
    int32_t w = 16807 * lo - 2836 * hi;
    if (w < 0) w += 2147483647;
    r[i] = w;
  }
  for (int i = 31; i < 34; ++i) r[i] = r[i - 31];
  for (int i = 34; i < 344 + count; ++i) r[i] = (int32_t)((uint32_t)r[i - 31] + (uint32_t)r[i - 3]);
  out.resize((size_t)count);
  for (int k = 0; k < count; ++k) out[k] = (int)((uint32_t)r[344 + k] >> 1);
}

struct RelPose : DeviceStream<3> {
  RansacBatch batch;
  DevBuf<double> d_bearings, d_lo;
  DevBuf<int> d_ransac;
  DevBuf<unsigned char> d_mask;

  // the stage after RANSAC: two-view or match filter
  bool stage_timed = false;
  DevBuf<double> d_plane, d_tv_pose;
  DevBuf<int> d_tv_lists, d_tv_counts, d_tv_chosen;
  DevBuf<unsigned char> d_mask_plane;
  bool fractions_ready = false;

  explicit RelPose(int dev) : DeviceStream(dev) {}

  void run(int64_t num_bearings, const double* bearings, int64_t num_pairs, const int64_t* pair_start,
           const int64_t* row_a, const int64_t* row_b, double threshold, int iterations, double* lo_model,
           int32_t* ransac_inliers, uint8_t* inlier_mask);
  void two_view(int64_t num_bearings, const double* bearings, int64_t num_pairs, const int64_t* pair_start,
                const int64_t* row_a, const int64_t* row_b, double threshold, int ransac_iterations,
                int refine_iterations, int check_reversal, double reversal_ratio, const double* plane_pose,
                double* lo_model, int32_t* ransac_inliers, double* pose, int32_t* counts, int32_t* chosen,
                uint8_t* mask_5pt, uint8_t* mask_plane);
  void robust_match(int64_t num_bearings, const double* bearings, int64_t num_pairs, const int64_t* pair_start,
                    const int64_t* row_a, const int64_t* row_b, double threshold, int ransac_iterations,
                    int refine_iterations, double* lo_model, int32_t* ransac_inliers, double* pose, int32_t* counts,
                    uint8_t* mask);

 private:
  void check(int64_t num_bearings, const double* bearings, int64_t num_pairs, const int64_t* pair_start,
             const int64_t* row_a, const int64_t* row_b, double threshold, int iterations,
             int min_rows = RP_MIN_SAMPLE) {
    stage_timed = false;
    batch.check("relative pose", "pair", "rows", min_rows, num_pairs, pair_start, threshold, iterations,
                {{row_a, bearings, num_bearings, "bearing"}, {row_b, bearings, num_bearings, "bearing"}}, true);
  }
  // RelativePoseCost's row picks (tv_pick_fraction), uploaded once per handle before the first refinement
  void upload_pick_fractions() {
    if (fractions_ready) return;
    std::vector<int> r;
    glibc_rand(42, relpose::REFINE_PICKED, r);
    float frac[relpose::REFINE_PICKED];
    for (int k = 0; k < relpose::REFINE_PICKED; ++k) frac[k] = (float)r[k] / (float)RAND_MAX;
    OSFM_CUDA(cudaMemcpyToSymbolAsync(tv_pick_fraction, frac, sizeof(frac), 0, cudaMemcpyHostToDevice, stream));
    OSFM_CUDA(cudaStreamSynchronize(stream));
    fractions_ready = true;
  }
  // the launches of one RANSAC call (after the argument checks), up to ev[1]; the batch's plan serves the stage
  // after it
  void launch_ransac(int64_t num_bearings, const double* bearings, int64_t num_pairs, const int64_t* pair_start,
                     const int64_t* row_a, const int64_t* row_b, double threshold, int iterations);
};

void RelPose::launch_ransac(int64_t num_bearings, const double* bearings, int64_t num_pairs,
                            const int64_t* pair_start, const int64_t* row_a, const int64_t* row_b, double threshold,
                            int iterations) {
  batch.plan(stream, num_pairs, pair_start, {row_a, row_b});
  const int64_t R = pair_start[num_pairs];
  upload(d_bearings, bearings, (size_t)num_bearings * 3);
  d_mask.reserve((size_t)R);
  d_lo.reserve((size_t)num_pairs * 12);
  d_ransac.reserve((size_t)num_pairs);

  RpArgs a;
  a.bearings = d_bearings.p;
  a.pair_start = batch.d_start.p;
  a.row_a = batch.d_rows[0].p;
  a.row_b = batch.d_rows[1].p;
  a.threshold = 1.0 - std::cos(threshold);
  a.iterations = iterations;
  a.src = batch.source();
  a.best_rows = batch.d_best_rows.p;
  a.lo_model = d_lo.p;
  a.ransac_inliers = d_ransac.p;
  a.mask = d_mask.p;

  OSFM_CUDA(cudaEventRecord(ev[0], stream));
  if (num_bearings > 0) {
    ransac_normalize<<<(unsigned)((num_bearings + 255) / 256), 256, 0, stream>>>(d_bearings.p, num_bearings);
    OSFM_LAUNCH_CHECK();
  }
  batch.launch(rp_ransac, a, stream);
  OSFM_CUDA(cudaEventRecord(ev[1], stream));
}

void RelPose::run(int64_t num_bearings, const double* bearings, int64_t num_pairs, const int64_t* pair_start,
                  const int64_t* row_a, const int64_t* row_b, double threshold, int iterations, double* lo_model,
                  int32_t* ransac_inliers, uint8_t* inlier_mask) {
  check(num_bearings, bearings, num_pairs, pair_start, row_a, row_b, threshold, iterations);
  if (num_pairs > 0 && (!lo_model || !ransac_inliers || !inlier_mask)) throw ArgError("relative pose: null arrays");
  if (num_pairs == 0) return;
  launch_ransac(num_bearings, bearings, num_pairs, pair_start, row_a, row_b, threshold, iterations);
  const int64_t R = pair_start[num_pairs];
  download(lo_model, d_lo.p, (size_t)num_pairs * 12);
  download(ransac_inliers, d_ransac.p, (size_t)num_pairs);
  download(inlier_mask, d_mask.p, (size_t)R);
  OSFM_CUDA(cudaStreamSynchronize(stream));
  batch.done = num_pairs;
}

void RelPose::two_view(int64_t num_bearings, const double* bearings, int64_t num_pairs, const int64_t* pair_start,
                       const int64_t* row_a, const int64_t* row_b, double threshold, int ransac_iterations,
                       int refine_iterations, int check_reversal, double reversal_ratio, const double* plane_pose,
                       double* lo_model, int32_t* ransac_inliers, double* pose, int32_t* counts, int32_t* chosen,
                       uint8_t* mask_5pt, uint8_t* mask_plane) {
  check(num_bearings, bearings, num_pairs, pair_start, row_a, row_b, threshold, ransac_iterations);
  if (refine_iterations < 1) throw ArgError("two-view: refine_iterations must be at least 1");
  if (check_reversal != 0 && check_reversal != 1) throw ArgError("two-view: check_reversal must be 0 or 1");
  if (std::isnan(reversal_ratio)) throw ArgError("two-view: reversal_ratio is NaN");
  if (num_pairs > 0 && (!plane_pose || !lo_model || !ransac_inliers || !pose || !counts || !chosen || !mask_5pt ||
                        !mask_plane))
    throw ArgError("two-view: null arrays");
  if (num_pairs == 0) return;
  upload_pick_fractions();
  const int64_t R = pair_start[num_pairs];
  upload(d_plane, plane_pose, (size_t)num_pairs * 12);
  d_tv_lists.reserve((size_t)R * 2);
  d_tv_pose.reserve((size_t)num_pairs * 24);
  d_tv_counts.reserve((size_t)num_pairs * 3);
  d_tv_chosen.reserve((size_t)num_pairs);
  d_mask_plane.reserve((size_t)R);
  launch_ransac(num_bearings, bearings, num_pairs, pair_start, row_a, row_b, threshold, ransac_iterations);

  TvArgs a;
  a.bearings = d_bearings.p;
  a.pair_start = batch.d_start.p;
  a.row_a = batch.d_rows[0].p;
  a.row_b = batch.d_rows[1].p;
  a.lo_model = d_lo.p;
  a.plane_pose = d_plane.p;
  a.threshold = threshold;
  a.refine_iterations = refine_iterations;
  a.configurations = check_reversal ? 2 : 1;
  a.reversal_ratio = reversal_ratio;
  a.lists = d_tv_lists.p;
  a.pose = d_tv_pose.p;
  a.counts = d_tv_counts.p;
  a.chosen = d_tv_chosen.p;
  a.mask5 = d_mask.p;             // rp_ransac's mask is not returned by this call
  a.maskp = d_mask_plane.p;
  batch.launch(rp_two_view, a, stream);
  OSFM_CUDA(cudaEventRecord(ev[2], stream));
  download(lo_model, d_lo.p, (size_t)num_pairs * 12);
  download(ransac_inliers, d_ransac.p, (size_t)num_pairs);
  download(pose, d_tv_pose.p, (size_t)num_pairs * 24);
  download(counts, d_tv_counts.p, (size_t)num_pairs * 3);
  download(chosen, d_tv_chosen.p, (size_t)num_pairs);
  download(mask_5pt, d_mask.p, (size_t)R);
  download(mask_plane, d_mask_plane.p, (size_t)R);
  OSFM_CUDA(cudaStreamSynchronize(stream));
  batch.done = num_pairs;
  stage_timed = true;
}

void RelPose::robust_match(int64_t num_bearings, const double* bearings, int64_t num_pairs,
                           const int64_t* pair_start, const int64_t* row_a, const int64_t* row_b, double threshold,
                           int ransac_iterations, int refine_iterations, double* lo_model, int32_t* ransac_inliers,
                           double* pose, int32_t* counts, uint8_t* mask) {
  check(num_bearings, bearings, num_pairs, pair_start, row_a, row_b, threshold, ransac_iterations, RM_MIN_INLIERS);
  if (refine_iterations < 1) throw ArgError("robust match: refine_iterations must be at least 1");
  if (num_pairs > 0 && (!lo_model || !ransac_inliers || !pose || !counts || !mask))
    throw ArgError("robust match: null arrays");
  if (num_pairs == 0) return;
  upload_pick_fractions();
  const int64_t R = pair_start[num_pairs];
  d_tv_lists.reserve((size_t)R);
  d_tv_pose.reserve((size_t)num_pairs * 12);
  d_tv_counts.reserve((size_t)num_pairs * 4);
  launch_ransac(num_bearings, bearings, num_pairs, pair_start, row_a, row_b, threshold, ransac_iterations);

  RmArgs a;
  a.bearings = d_bearings.p;
  a.pair_start = batch.d_start.p;
  a.row_a = batch.d_rows[0].p;
  a.row_b = batch.d_rows[1].p;
  a.lo_model = d_lo.p;
  a.threshold = threshold;
  a.refine_iterations = refine_iterations;
  a.lists = d_tv_lists.p;
  a.pose = d_tv_pose.p;
  a.counts = d_tv_counts.p;
  a.mask = d_mask.p;              // rp_ransac's mask is not returned by this call
  batch.launch(rp_match_filter, a, stream);
  OSFM_CUDA(cudaEventRecord(ev[2], stream));
  download(lo_model, d_lo.p, (size_t)num_pairs * 12);
  download(ransac_inliers, d_ransac.p, (size_t)num_pairs);
  download(pose, d_tv_pose.p, (size_t)num_pairs * 12);
  download(counts, d_tv_counts.p, (size_t)num_pairs * 4);
  download(mask, d_mask.p, (size_t)R);
  OSFM_CUDA(cudaStreamSynchronize(stream));
  batch.done = num_pairs;
  stage_timed = true;
}

}  // namespace
}  // namespace osfm

struct osfm_relpose : osfm::Handle<osfm::RelPose> {
  using Handle::Handle;
  static constexpr const char* null_message = "null relative pose";
};

extern "C" {

int osfm_relpose_create(int device, osfm_relpose** out) { return osfm::create_handle(device, out); }
int osfm_relpose_destroy(osfm_relpose* h) { return osfm::destroy_handle(h); }

int osfm_relpose_run(osfm_relpose* h, int64_t num_bearings, const double* bearings, int64_t num_pairs,
                     const int64_t* pair_start, const int64_t* row_a, const int64_t* row_b, double threshold,
                     int iterations, double* lo_model, int32_t* ransac_inliers, uint8_t* inlier_mask) {
  return osfm::with_handle(h, [&](osfm::RelPose& K) {
    K.run(num_bearings, bearings, num_pairs, pair_start, row_a, row_b, threshold, iterations, lo_model,
          ransac_inliers, inlier_mask);
  });
}

int osfm_relpose_two_view(osfm_relpose* h, int64_t num_bearings, const double* bearings, int64_t num_pairs,
                          const int64_t* pair_start, const int64_t* row_a, const int64_t* row_b, double threshold,
                          int ransac_iterations, int refine_iterations, int check_reversal, double reversal_ratio,
                          const double* plane_pose, double* lo_model, int32_t* ransac_inliers, double* pose,
                          int32_t* counts, int32_t* chosen, uint8_t* mask_5pt, uint8_t* mask_plane) {
  return osfm::with_handle(h, [&](osfm::RelPose& K) {
    K.two_view(num_bearings, bearings, num_pairs, pair_start, row_a, row_b, threshold, ransac_iterations,
               refine_iterations, check_reversal, reversal_ratio, plane_pose, lo_model, ransac_inliers, pose, counts,
               chosen, mask_5pt, mask_plane);
  });
}

int osfm_relpose_robust_match(osfm_relpose* h, int64_t num_bearings, const double* bearings, int64_t num_pairs,
                              const int64_t* pair_start, const int64_t* row_a, const int64_t* row_b,
                              double threshold, int ransac_iterations, int refine_iterations, double* lo_model,
                              int32_t* ransac_inliers, double* pose, int32_t* counts, uint8_t* mask) {
  return osfm::with_handle(h, [&](osfm::RelPose& K) {
    K.robust_match(num_bearings, bearings, num_pairs, pair_start, row_a, row_b, threshold, ransac_iterations,
                   refine_iterations, lo_model, ransac_inliers, pose, counts, mask);
  });
}

int osfm_relpose_last_stage_ms(osfm_relpose* h, float* ransac_ms, float* stage_ms) {
  return osfm::with_handle(h, [&](osfm::RelPose& K) {
    if (!ransac_ms || !stage_ms) throw osfm::ArgError("null ms");
    *ransac_ms = *stage_ms = 0.f;
    if (K.batch.done) OSFM_CUDA(cudaEventElapsedTime(ransac_ms, K.ev[0], K.ev[1]));
    if (K.stage_timed) OSFM_CUDA(cudaEventElapsedTime(stage_ms, K.ev[1], K.ev[2]));
  });
}

int osfm_relpose_set_stream_prefix(osfm_relpose* h, int64_t length) {
  return osfm::with_handle(h, [&](osfm::RelPose& K) { K.batch.set_stream_prefix(length); });
}

int osfm_relpose_set_trace(osfm_relpose* h, int capacity) {
  return osfm::with_handle(h, [&](osfm::RelPose& K) { K.batch.set_trace(capacity); });
}

int osfm_relpose_get_trace(osfm_relpose* h, int32_t* count, int64_t* stream_used, int32_t* indices) {
  return osfm::with_handle(
      h, [&](osfm::RelPose& K) { K.batch.get_trace(K.stream, "relative pose", count, stream_used, indices); });
}

int osfm_relpose_last_device_ms(osfm_relpose* h, float* ms) {
  return osfm::with_handle(h, [&](osfm::RelPose& K) {
    if (!ms) throw osfm::ArgError("null ms");
    *ms = 0.f;
    if (K.batch.done) OSFM_CUDA(cudaEventElapsedTime(ms, K.ev[0], K.ev[K.stage_timed ? 2 : 1]));
  });
}

}  // extern "C"
