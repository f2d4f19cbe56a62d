// RESECT: absolute-pose RANSAC of many shots at once, for the resection step of the incremental reconstruction.
//
// Replaces, for every candidate image of resect (opensfm/reconstruction.py:695-762), pyrobust's ransac_absolute_pose
// with RANSAC scoring (robust/robust_estimator.h, absolute_pose_model.h), as multiview.absolute_pose_ransac calls it,
// followed by resect's chord-inlier test.  The restatement the results are checked against, and the rules it
// follows, are in oracle/absolute_pose_oracle.py; the solvers (P3P, Lu's iteration) are absolute_pose.cuh.
//
// One CTA per shot (rs_ransac), largest shots first.  Thread 0 draws the sample from the shared mt19937(42) stream
// (ransac_stream.cuh) and solves P3P; the whole CTA then scores the up to 4 models of the sample in one pass over the
// rows (four inlier counts per row read), and the decisions the reference takes model by model (replace the best,
// local optimisation, stop) are replayed in model order from those counts.  A model's inlier rows are listed, in
// ascending order, only when it becomes the best one with at least 3 inliers: local optimisation samples from that
// list, thread 0 fits Lu's iteration to the sample and the CTA counts its inliers.  A shot of at most RANSAC_STAGE_ROWS
// rows is staged in shared memory (bearing and point); a larger one is read through L2 via its row indices.  A last
// pass writes the chord-inlier mask and counts.  The sample stream, the row passes, the launch plan and the argument
// checks are those of ransac_stream.cuh.
#include <cmath>

#include "absolute_pose.cuh"
#include "common.cuh"
#include "ransac_stream.cuh"

namespace osfm {
namespace {

constexpr int RS_MIN_SAMPLE = 3;
constexpr int RS_MAX_SAMPLE = 12;          // local optimisation samples min(12, inliers / 2) rows (at least 3)
constexpr int RS_MAX_MODELS = 4;
constexpr int RS_LO_ITERATIONS = 10;

struct RsArgs {
  const double* bearings;        // 3 per entry, normalised
  const double* points;          // 3 per entry
  const long long* shot_start;
  const long long* row_b;        // bearing of row r
  const long long* row_x;        // point of row r
  const int* order;              // shots of this launch
  double chord_threshold, ransac_threshold;
  int iterations;
  StreamSource src;
  int* best_rows;                // per row: the best model's inlier rows, ascending
  double* lo_model;              // 12 per shot
  int* ransac_inliers;
  int* chord_inliers;
  unsigned char* chord_mask;     // per row
};

struct RsShared {
  StreamState st;
  double b[RS_MAX_SAMPLE * 3], p[RS_MAX_SAMPLE * 3];
  double models[RS_MAX_MODELS][12];
  double cand[12];
  double best[12];
  int idx[RS_MAX_SAMPLE];
  int nm;
  int counts[RS_MAX_MODELS];
  int cand_count, best_count;
  int stop;
  int warp_n[RS_MAX_MODELS][RANSAC_WARPS];
};

// |1 - b . normalize(R X + t)| < t of the pose M = [R | t]
struct RsTest {
  double t;
  __device__ __forceinline__ bool operator()(const double* M, const double* b, const double* x) const {
    const double v0 = M[0] * x[0] + M[1] * x[1] + M[2] * x[2] + M[3];
    const double v1 = M[4] * x[0] + M[5] * x[1] + M[6] * x[2] + M[7];
    const double v2 = M[8] * x[0] + M[9] * x[1] + M[10] * x[2] + M[11];
    const double e = 1.0 - (b[0] * v0 + b[1] * v1 + b[2] * v2) / sqrt(v0 * v0 + v1 * v1 + v2 * v2);
    return fabs(e) < t;
  }
};

// inliers of the nm models at M (12 apart) into counts, in one pass over the rows
template <int NM>
__device__ void rs_count(RsShared& s, const RansacRows& rows, const double* M, RsTest test, int* counts) {
  double m[NM][12];
  for (int j = 0; j < NM; ++j)
    for (int k = 0; k < 12; ++k) m[j][k] = M[12 * j + k];
  int c[NM];
  for (int j = 0; j < NM; ++j) c[j] = 0;
  for (int i = threadIdx.x; i < rows.n; i += RANSAC_THREADS) {
    double b[3], x[3];
    rows.get(i, b, x);
    for (int j = 0; j < NM; ++j) c[j] += test(m[j], b, x) ? 1 : 0;
  }
  ransac_sums(c, NM, &s.warp_n[0][0], counts);
}

// thread 0's solvers, out of line so that their registers do not weigh on the CTA's passes over the rows
__device__ __noinline__ int rs_p3p(const double* b, const double* p, double* models) { return pose::p3p_ke(b, p, models); }
__device__ __noinline__ void rs_lu(int k, const double* b, const double* p, double* out) { pose::lu_pose(k, b, p, out); }

__global__ void __launch_bounds__(RANSAC_THREADS) rs_ransac(RsArgs a, int staged) {
  __shared__ RsShared s;
  const int shot = a.order[blockIdx.x];
  const long long off = a.shot_start[shot];
  const int n = (int)(a.shot_start[shot + 1] - off);
  const RansacRows rows = ransac_rows(a.bearings, a.points, a.row_b + off, a.row_x + off, n, staged);
  int* best_rows = a.best_rows + off;
  const RsTest test{a.ransac_threshold};
  if (threadIdx.x == 0) {
    s.st.reset();
    s.best_count = 0;
    s.stop = 0;
    for (int k = 0; k < 12; ++k) s.best[k] = 0.0;
  }
  __syncthreads();

  for (int it = 0; it < a.iterations; ++it) {
    if (threadIdx.x == 0) {
      stream_sample(s.st, a.src, shot, RS_MIN_SAMPLE, n, s.idx);
      for (int k = 0; k < RS_MIN_SAMPLE; ++k) rows.get(s.idx[k], s.b + 3 * k, s.p + 3 * k);
      s.nm = rs_p3p(s.b, s.p, &s.models[0][0]);
    }
    __syncthreads();
    const int nm = s.nm;
    if (nm == RS_MAX_MODELS) rs_count<RS_MAX_MODELS>(s, rows, &s.models[0][0], test, s.counts);
    // the models in order: std::max(score, best) keeps the new one on ties, then LO, then ShouldStop
    for (int j = 0; j < nm; ++j) {
      const int c = s.counts[j];
      if (c >= s.best_count) {
        __syncthreads();
        if (threadIdx.x == 0) {
          for (int k = 0; k < 12; ++k) s.best[k] = s.models[j][k];
          s.best_count = c;
        }
        if (c >= RS_MIN_SAMPLE) {
          ransac_compact<12>(rows, s.models[j], test, s.warp_n[0], best_rows);
          for (int lo = 0; lo < RS_LO_ITERATIONS; ++lo) {
            if (threadIdx.x == 0) {
              const int m = s.best_count;
              const int size = max(min(RS_MAX_SAMPLE, (int)(m * 0.5)), RS_MIN_SAMPLE);
              stream_sample(s.st, a.src, shot, size, m, s.idx);
              for (int k = 0; k < size; ++k) rows.get(best_rows[s.idx[k]], s.b + 3 * k, s.p + 3 * k);
              rs_lu(size, s.b, s.p, s.cand);
            }
            __syncthreads();
            rs_count<1>(s, rows, s.cand, test, &s.cand_count);
            if (s.cand_count >= s.best_count) {
              ransac_compact<12>(rows, s.cand, test, s.warp_n[0], best_rows);
              if (threadIdx.x == 0) {
                for (int k = 0; k < 12; ++k) s.best[k] = s.cand[k];
                s.best_count = s.cand_count;
              }
            }
            __syncthreads();
          }
        }
        __syncthreads();
      }
      if (threadIdx.x == 0) s.stop = ransac_should_stop(s.best_count, n, it);
      __syncthreads();
      const bool stop = s.stop;
      __syncthreads();
      if (stop) break;
    }
    const bool stop = s.stop;
    __syncthreads();
    if (stop) break;
  }

  // chord inliers ||normalize(R (X - o)) - b|| < threshold, o = -R^T t
  double M[12];
  for (int k = 0; k < 12; ++k) M[k] = s.best[k];
  double o[3];
  for (int c = 0; c < 3; ++c) o[c] = -(M[0 * 4 + c] * M[3] + M[1 * 4 + c] * M[7] + M[2 * 4 + c] * M[11]);
  int cnt[1] = {0};
  for (int i = threadIdx.x; i < n; i += RANSAC_THREADS) {
    double b[3], x[3];
    rows.get(i, b, x);
    const double d0 = x[0] - o[0], d1 = x[1] - o[1], d2 = x[2] - o[2];
    double v0 = M[0] * d0 + M[1] * d1 + M[2] * d2;
    double v1 = M[4] * d0 + M[5] * d1 + M[6] * d2;
    double v2 = M[8] * d0 + M[9] * d1 + M[10] * d2;
    const double r = sqrt(v0 * v0 + v1 * v1 + v2 * v2);
    v0 = v0 / r - b[0];
    v1 = v1 / r - b[1];
    v2 = v2 / r - b[2];
    const bool in = sqrt(v0 * v0 + v1 * v1 + v2 * v2) < a.chord_threshold;
    a.chord_mask[off + i] = in ? 1 : 0;
    cnt[0] += in ? 1 : 0;
  }
  ransac_sums(cnt, 1, &s.warp_n[0][0], &s.cand_count);
  if (threadIdx.x == 0) {
    a.chord_inliers[shot] = s.cand_count;
    a.ransac_inliers[shot] = s.best_count;
    for (int k = 0; k < 12; ++k) a.lo_model[12LL * shot + k] = M[k];
    stream_record(s.st, a.src, shot);
  }
}

struct Resect : DeviceStream<2> {
  RansacBatch batch;
  DevBuf<double> d_bearings, d_points, d_lo;
  DevBuf<int> d_ransac, d_chord;
  DevBuf<unsigned char> d_mask;

  explicit Resect(int dev) : DeviceStream(dev) {}

  void run(int64_t num_bearings, const double* bearings, int64_t num_points, const double* points, int64_t num_shots,
           const int64_t* shot_start, const int64_t* row_bearing, const int64_t* row_point, double threshold,
           int iterations, double* lo_model, int32_t* ransac_inliers, int32_t* chord_inliers, uint8_t* chord_mask);
};

void Resect::run(int64_t num_bearings, const double* bearings, int64_t num_points, const double* points,
                 int64_t num_shots, const int64_t* shot_start, const int64_t* row_bearing, const int64_t* row_point,
                 double threshold, int iterations, double* lo_model, int32_t* ransac_inliers, int32_t* chord_inliers,
                 uint8_t* chord_mask) {
  batch.check("resection", "shot", "rows", RS_MIN_SAMPLE, num_shots, shot_start, threshold, iterations,
              {{row_bearing, bearings, num_bearings, "bearing"}, {row_point, points, num_points, "point"}},
              lo_model && ransac_inliers && chord_inliers && chord_mask);
  if (num_shots == 0) return;
  batch.plan(stream, num_shots, shot_start, {row_bearing, row_point});
  const int64_t R = shot_start[num_shots];
  upload(d_bearings, bearings, (size_t)num_bearings * 3);
  upload(d_points, points, (size_t)num_points * 3);
  d_mask.reserve((size_t)R);
  d_lo.reserve((size_t)num_shots * 12);
  d_ransac.reserve((size_t)num_shots);
  d_chord.reserve((size_t)num_shots);

  RsArgs a;
  a.bearings = d_bearings.p;
  a.points = d_points.p;
  a.shot_start = batch.d_start.p;
  a.row_b = batch.d_rows[0].p;
  a.row_x = batch.d_rows[1].p;
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
  if (num_bearings > 0) {
    ransac_normalize<<<(unsigned)((num_bearings + 255) / 256), 256, 0, stream>>>(d_bearings.p, num_bearings);
    OSFM_LAUNCH_CHECK();
  }
  batch.launch(rs_ransac, a, stream);
  OSFM_CUDA(cudaEventRecord(ev[1], stream));
  download(lo_model, d_lo.p, (size_t)num_shots * 12);
  download(ransac_inliers, d_ransac.p, (size_t)num_shots);
  download(chord_inliers, d_chord.p, (size_t)num_shots);
  download(chord_mask, d_mask.p, (size_t)R);
  OSFM_CUDA(cudaStreamSynchronize(stream));
  batch.done = num_shots;
}

}  // namespace
}  // namespace osfm

struct osfm_resect : osfm::Handle<osfm::Resect> {
  using Handle::Handle;
  static constexpr const char* null_message = "null resection";
};

extern "C" {

int osfm_resect_create(int device, osfm_resect** out) { return osfm::create_handle(device, out); }
int osfm_resect_destroy(osfm_resect* h) { return osfm::destroy_handle(h); }

int osfm_resect_run(osfm_resect* h, int64_t num_bearings, const double* bearings, int64_t num_points,
                    const double* points, int64_t num_shots, const int64_t* shot_start, const int64_t* row_bearing,
                    const int64_t* row_point, double threshold, int iterations, double* lo_model,
                    int32_t* ransac_inliers, int32_t* chord_inliers, uint8_t* chord_mask) {
  return osfm::with_handle(h, [&](osfm::Resect& K) {
    K.run(num_bearings, bearings, num_points, points, num_shots, shot_start, row_bearing, row_point, threshold,
          iterations, lo_model, ransac_inliers, chord_inliers, chord_mask);
  });
}

int osfm_resect_set_stream_prefix(osfm_resect* h, int64_t length) {
  return osfm::with_handle(h, [&](osfm::Resect& K) { K.batch.set_stream_prefix(length); });
}

int osfm_resect_set_trace(osfm_resect* h, int capacity) {
  return osfm::with_handle(h, [&](osfm::Resect& K) { K.batch.set_trace(capacity); });
}

int osfm_resect_get_trace(osfm_resect* h, int32_t* count, int64_t* stream_used, int32_t* indices) {
  return osfm::with_handle(
      h, [&](osfm::Resect& K) { K.batch.get_trace(K.stream, "resection", count, stream_used, indices); });
}

int osfm_resect_last_device_ms(osfm_resect* h, float* ms) {
  return osfm::with_handle(h, [&](osfm::Resect& K) {
    if (!ms) throw osfm::ArgError("null ms");
    *ms = 0.f;
    if (K.batch.done) OSFM_CUDA(cudaEventElapsedTime(ms, K.ev[0], K.ev[1]));
  });
}

}  // extern "C"
