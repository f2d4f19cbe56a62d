// ROTRANSAC: rotation-only RANSAC of many image pairs at once, to rank them for the reconstruction bootstrap.
//
// Replaces, for every pair of compute_image_pairs (opensfm/reconstruction.py:208-244), pyrobust's
// ransac_relative_rotation with RANSAC scoring (opensfm/src/robust/robust_estimator.h, relative_rotation_model.h)
// followed by the chord-inlier count of _two_view_rotation_inliers (reconstruction.py:377-384).  The restatement the
// results are checked against, and the rules it follows, are in oracle/rotation_ransac_oracle.py.
//
// One CTA per pair (rr_ransac), largest pairs first.  Thread 0 draws the sample indices from the shared mt19937(42)
// stream and solves the 3x3 rotation; the whole CTA evaluates the model's errors, counts inliers and, when the
// model becomes the best one, writes its inlier rows in ascending order (the list local optimisation samples from).
// A pair of at most RANSAC_STAGE_ROWS rows is staged in shared memory; a larger one is read through L2 via its row
// indices.  A last pass writes the chord-inlier mask and counts.
//
// The sample stream, the row passes, the launch plan and the argument checks are those of ransac_stream.cuh.
#include <cmath>

#include "absolute_pose.cuh"
#include "common.cuh"
#include "ransac_stream.cuh"

namespace osfm {
namespace {

constexpr int RR_MIN_SAMPLE = 3;
constexpr int RR_MAX_SAMPLE = 12;          // local optimisation samples min(12, inliers / 2) rows (at least 3)
constexpr int RR_LO_ITERATIONS = 10;

struct RrArgs {
  const double* bearings;        // 3 per entry
  const long long* pair_start;
  const long long* row_a;        // bearing of row r in the first image
  const long long* row_b;        // ... and in the second
  const int* order;              // pairs of this launch
  double chord_threshold, ransac_threshold;
  int iterations;
  StreamSource src;
  int* best_rows;                // per row: the best model's inlier rows, ascending
  double* lo_model;              // 9 per pair
  int* ransac_inliers;
  int* chord_inliers;
  unsigned char* chord_mask;     // per row
};

struct RrShared {
  StreamState st;
  double sample[RR_MAX_SAMPLE][6];
  double cand[9];                // rotation Q of the candidate (the model is Q^T), row-major
  double best[9];
  int best_count, cand_count;
  int replace, lo, stop;
  int idx[RR_MAX_SAMPLE];
  int warp_n[RANSAC_WARPS];
};

// ---- thread 0: the rotation of a sample ---------------------------------------------------------------------
// rotation Q (Q b2 ~ b1) of the k sample rows in s.sample, into out (absolute_pose.cuh)
__device__ void rr_rotation(RrShared& s, int k, double* out) {
  pose::rotation_between(k, &s.sample[0][0], &s.sample[0][3], 6, out);
}

// ---- the whole CTA ----------------------------------------------------------------------------------------
// |1 - (Q^T b1) . b2| < t, the model Q^T of rotation Q
struct RrTest {
  double t;
  __device__ __forceinline__ bool operator()(const double* Q, const double* p, const double* q) const {
    const double v0 = Q[0] * p[0] + Q[3] * p[1] + Q[6] * p[2];
    const double v1 = Q[1] * p[0] + Q[4] * p[1] + Q[7] * p[2];
    const double v2 = Q[2] * p[0] + Q[5] * p[1] + Q[8] * p[2];
    return fabs(1.0 - (v0 * q[0] + v1 * q[1] + v2 * q[2])) < t;
  }
};

// inliers of s.cand into s.cand_count
__device__ void rr_count(RrShared& s, const RansacRows& rows, RrTest test) {
  double Q[9];
  for (int k = 0; k < 9; ++k) Q[k] = s.cand[k];
  int c[1] = {0};
  for (int i = threadIdx.x; i < rows.n; i += RANSAC_THREADS) {
    double p[3], q[3];
    rows.get(i, p, q);
    c[0] += test(Q, p, q) ? 1 : 0;
  }
  ransac_sums(c, 1, s.warp_n, &s.cand_count);
}

__global__ void __launch_bounds__(RANSAC_THREADS) rr_ransac(RrArgs a, int staged) {
  __shared__ RrShared s;
  const int pair = a.order[blockIdx.x];
  const long long off = a.pair_start[pair];
  const int n = (int)(a.pair_start[pair + 1] - off);
  const RansacRows rows = ransac_rows(a.bearings, a.bearings, a.row_a + off, a.row_b + off, n, staged);
  int* best_rows = a.best_rows + off;
  const RrTest test{a.ransac_threshold};
  if (threadIdx.x == 0) {
    s.st.reset();
    s.best_count = 0;
    s.stop = 0;
    for (int k = 0; k < 9; ++k) s.best[k] = 0.0;
  }
  __syncthreads();

  for (int it = 0; it < a.iterations; ++it) {
    if (threadIdx.x == 0) {
      stream_sample(s.st, a.src, pair, RR_MIN_SAMPLE, n, s.idx);
      for (int k = 0; k < RR_MIN_SAMPLE; ++k) rows.get(s.idx[k], &s.sample[k][0], &s.sample[k][3]);
      rr_rotation(s, RR_MIN_SAMPLE, s.cand);
    }
    __syncthreads();
    rr_count(s, rows, test);
    // the best model is replaced on ties (std::max(score, best) returns score when they are equal)
    const bool replace = s.cand_count >= s.best_count;
    if (replace) {
      ransac_compact<9>(rows, s.cand, test, s.warp_n, best_rows);
      if (threadIdx.x == 0) {
        s.best_count = s.cand_count;
        for (int k = 0; k < 9; ++k) s.best[k] = s.cand[k];
      }
      __syncthreads();
      if (s.best_count >= RR_MIN_SAMPLE) {
        for (int lo = 0; lo < RR_LO_ITERATIONS; ++lo) {
          if (threadIdx.x == 0) {
            const int m = s.best_count;
            const int size = max(min(RR_MAX_SAMPLE, (int)(m * 0.5)), RR_MIN_SAMPLE);
            stream_sample(s.st, a.src, pair, size, m, s.idx);
            for (int k = 0; k < size; ++k) rows.get(best_rows[s.idx[k]], &s.sample[k][0], &s.sample[k][3]);
            rr_rotation(s, size, s.cand);
          }
          __syncthreads();
          rr_count(s, rows, test);
          if (s.cand_count >= s.best_count) {
            ransac_compact<9>(rows, s.cand, test, s.warp_n, best_rows);
            if (threadIdx.x == 0) {
              s.best_count = s.cand_count;
              for (int k = 0; k < 9; ++k) s.best[k] = s.cand[k];
            }
            __syncthreads();
          }
        }
      }
    }
    if (threadIdx.x == 0) {
      s.stop = ransac_should_stop(s.best_count, n, it);
    }
    __syncthreads();
    if (s.stop) break;
  }

  // chord inliers ||Q b2 - b1|| < threshold of R = lo_model^T = Q
  double Q[9];
  for (int k = 0; k < 9; ++k) Q[k] = s.best[k];
  int c[1] = {0};
  for (int i = threadIdx.x; i < n; i += RANSAC_THREADS) {
    double p[3], q[3];
    rows.get(i, p, q);
    const double d0 = Q[0] * q[0] + Q[1] * q[1] + Q[2] * q[2] - p[0];
    const double d1 = Q[3] * q[0] + Q[4] * q[1] + Q[5] * q[2] - p[1];
    const double d2 = Q[6] * q[0] + Q[7] * q[1] + Q[8] * q[2] - p[2];
    const bool in = sqrt(d0 * d0 + d1 * d1 + d2 * d2) < a.chord_threshold;
    a.chord_mask[off + i] = in ? 1 : 0;
    c[0] += in ? 1 : 0;
  }
  ransac_sums(c, 1, s.warp_n, &s.cand_count);
  if (threadIdx.x == 0) {
    a.chord_inliers[pair] = s.cand_count;
    a.ransac_inliers[pair] = s.best_count;
    for (int r = 0; r < 3; ++r)
      for (int k = 0; k < 3; ++k) a.lo_model[9LL * pair + r * 3 + k] = Q[k * 3 + r];
    stream_record(s.st, a.src, pair);
  }
}

struct RotRansac : DeviceStream<2> {
  RansacBatch batch;
  DevBuf<double> d_bearings, d_lo;
  DevBuf<int> d_ransac, d_chord;
  DevBuf<unsigned char> d_mask;

  explicit RotRansac(int dev) : DeviceStream(dev) {}

  void run(int64_t num_bearings, const double* bearings, int64_t num_pairs, const int64_t* pair_start,
           const int64_t* row_a, const int64_t* row_b, double threshold, int iterations, double* lo_model,
           int32_t* ransac_inliers, int32_t* chord_inliers, uint8_t* chord_mask);
};

void RotRansac::run(int64_t num_bearings, const double* bearings, int64_t num_pairs, const int64_t* pair_start,
                    const int64_t* row_a, const int64_t* row_b, double threshold, int iterations, double* lo_model,
                    int32_t* ransac_inliers, int32_t* chord_inliers, uint8_t* chord_mask) {
  batch.check("rotation RANSAC", "pair", "correspondences", RR_MIN_SAMPLE, num_pairs, pair_start, threshold,
              iterations, {{row_a, bearings, num_bearings, "bearing"}, {row_b, bearings, num_bearings, "bearing"}},
              lo_model && ransac_inliers && chord_inliers && chord_mask);
  if (num_pairs == 0) return;
  batch.plan(stream, num_pairs, pair_start, {row_a, row_b});
  const int64_t R = pair_start[num_pairs];
  upload(d_bearings, bearings, (size_t)num_bearings * 3);
  d_mask.reserve((size_t)R);
  d_lo.reserve((size_t)num_pairs * 9);
  d_ransac.reserve((size_t)num_pairs);
  d_chord.reserve((size_t)num_pairs);

  RrArgs a;
  a.bearings = d_bearings.p;
  a.pair_start = batch.d_start.p;
  a.row_a = batch.d_rows[0].p;
  a.row_b = batch.d_rows[1].p;
  a.chord_threshold = threshold;
  a.ransac_threshold = 1.0 - std::cos(threshold);
  a.iterations = iterations;
  a.src = batch.source();
  a.best_rows = batch.d_best_rows.p;
  a.lo_model = d_lo.p;
  a.ransac_inliers = d_ransac.p;
  a.chord_inliers = d_chord.p;
  a.chord_mask = d_mask.p;

  OSFM_CUDA(cudaEventRecord(ev[0], stream));
  batch.launch(rr_ransac, a, stream);
  OSFM_CUDA(cudaEventRecord(ev[1], stream));
  download(lo_model, d_lo.p, (size_t)num_pairs * 9);
  download(ransac_inliers, d_ransac.p, (size_t)num_pairs);
  download(chord_inliers, d_chord.p, (size_t)num_pairs);
  download(chord_mask, d_mask.p, (size_t)R);
  OSFM_CUDA(cudaStreamSynchronize(stream));
  batch.done = num_pairs;
}

}  // namespace
}  // namespace osfm

struct osfm_rotransac : osfm::Handle<osfm::RotRansac> {
  using Handle::Handle;
  static constexpr const char* null_message = "null rotation RANSAC";
};

extern "C" {

int osfm_rotransac_create(int device, osfm_rotransac** out) { return osfm::create_handle(device, out); }
int osfm_rotransac_destroy(osfm_rotransac* h) { return osfm::destroy_handle(h); }

int osfm_rotransac_run(osfm_rotransac* h, int64_t num_bearings, const double* bearings, int64_t num_pairs,
                       const int64_t* pair_start, const int64_t* row_a, const int64_t* row_b, double threshold,
                       int iterations, double* lo_model, int32_t* ransac_inliers, int32_t* chord_inliers,
                       uint8_t* chord_mask) {
  return osfm::with_handle(h, [&](osfm::RotRansac& K) {
    K.run(num_bearings, bearings, num_pairs, pair_start, row_a, row_b, threshold, iterations, lo_model, ransac_inliers,
          chord_inliers, chord_mask);
  });
}

int osfm_rotransac_set_stream_prefix(osfm_rotransac* h, int64_t length) {
  return osfm::with_handle(h, [&](osfm::RotRansac& K) { K.batch.set_stream_prefix(length); });
}

int osfm_rotransac_set_trace(osfm_rotransac* h, int capacity) {
  return osfm::with_handle(h, [&](osfm::RotRansac& K) { K.batch.set_trace(capacity); });
}

int osfm_rotransac_get_trace(osfm_rotransac* h, int32_t* count, int64_t* stream_used, int32_t* indices) {
  return osfm::with_handle(
      h, [&](osfm::RotRansac& K) { K.batch.get_trace(K.stream, "rotation RANSAC", count, stream_used, indices); });
}

int osfm_rotransac_last_device_ms(osfm_rotransac* h, float* ms) {
  return osfm::with_handle(h, [&](osfm::RotRansac& K) {
    if (!ms) throw osfm::ArgError("null ms");
    *ms = 0.f;
    if (K.batch.done) OSFM_CUDA(cudaEventElapsedTime(ms, K.ev[0], K.ev[1]));
  });
}

}  // extern "C"
