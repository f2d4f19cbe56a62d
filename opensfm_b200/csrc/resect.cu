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
// list, thread 0 fits Lu's iteration to the sample and the CTA counts its inliers.  A shot of at most RS_STAGE_ROWS
// rows is staged in shared memory as fp64 structure-of-arrays (bearing and point, 48 B per row); a larger one is
// read through L2 via its row indices.  A last pass writes the chord-inlier mask and counts.
#include <algorithm>
#include <climits>
#include <cmath>
#include <numeric>
#include <string>
#include <vector>

#include "absolute_pose.cuh"
#include "common.cuh"
#include "ransac_stream.cuh"

namespace osfm {
namespace {

constexpr int RS_THREADS = 128;
constexpr int RS_WARPS = RS_THREADS / 32;
constexpr int RS_STAGE_ROWS = 1024;        // 48 KB of shared memory
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
  StreamSource src;              // trace: trace_cap drawn indices per shot, or null
  int* best_rows;                // per row: the best model's inlier rows, ascending
  double* lo_model;              // 12 per shot
  int* ransac_inliers;
  int* chord_inliers;
  unsigned char* chord_mask;     // per row
  int* trace_count;
  long long* stream_used;
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
  int warp_n[RS_MAX_MODELS][RS_WARPS];
};

struct RsRows {
  const double* sm;              // staged SoA (bx by bz X Y Z, n each) or null
  const double *bearings, *points;
  const long long *rb, *rx;
  int n;
  __device__ __forceinline__ void get(int i, double* b, double* x) const {
    if (sm) {
      b[0] = sm[i]; b[1] = sm[n + i]; b[2] = sm[2 * n + i];
      x[0] = sm[3 * n + i]; x[1] = sm[4 * n + i]; x[2] = sm[5 * n + i];
    } else {
      const double* u = bearings + 3 * rb[i];
      const double* v = points + 3 * rx[i];
      b[0] = __ldg(u); b[1] = __ldg(u + 1); b[2] = __ldg(u + 2);
      x[0] = __ldg(v); x[1] = __ldg(v + 1); x[2] = __ldg(v + 2);
    }
  }
};

// |1 - b . normalize(R X + t)| < t of the pose M = [R | t]
__device__ __forceinline__ bool rs_inlier(const double* M, const double* b, const double* x, double t) {
  const double v0 = M[0] * x[0] + M[1] * x[1] + M[2] * x[2] + M[3];
  const double v1 = M[4] * x[0] + M[5] * x[1] + M[6] * x[2] + M[7];
  const double v2 = M[8] * x[0] + M[9] * x[1] + M[10] * x[2] + M[11];
  const double e = 1.0 - (b[0] * v0 + b[1] * v1 + b[2] * v2) / sqrt(v0 * v0 + v1 * v1 + v2 * v2);
  return fabs(e) < t;
}

// inliers of the nm models at M (12 apart) into counts, in one pass over the rows
template <int NM>
__device__ void rs_count(RsShared& s, const RsRows& rows, const double* M, double t, int* counts) {
  double m[NM][12];
  for (int j = 0; j < NM; ++j)
    for (int k = 0; k < 12; ++k) m[j][k] = M[12 * j + k];
  int c[NM];
  for (int j = 0; j < NM; ++j) c[j] = 0;
  for (int i = threadIdx.x; i < rows.n; i += RS_THREADS) {
    double b[3], x[3];
    rows.get(i, b, x);
    for (int j = 0; j < NM; ++j) c[j] += rs_inlier(m[j], b, x, t) ? 1 : 0;
  }
  for (int j = 0; j < NM; ++j) {
    const int w = __reduce_add_sync(0xffffffffu, c[j]);
    if ((threadIdx.x & 31) == 0) s.warp_n[j][threadIdx.x >> 5] = w;
  }
  __syncthreads();
  if (threadIdx.x < NM) {
    int total = 0;
    for (int w = 0; w < RS_WARPS; ++w) total += s.warp_n[threadIdx.x][w];
    counts[threadIdx.x] = total;
  }
  __syncthreads();
}

// the inlier rows of the pose M, ascending, into out
__device__ void rs_compact(RsShared& s, const RsRows& rows, const double* M, double t, int* out) {
  double m[12];
  for (int k = 0; k < 12; ++k) m[k] = M[k];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int base = 0;
  for (int tile = 0; tile < rows.n; tile += RS_THREADS) {
    const int i = tile + threadIdx.x;
    bool in = false;
    if (i < rows.n) {
      double b[3], x[3];
      rows.get(i, b, x);
      in = rs_inlier(m, b, x, t);
    }
    const unsigned bal = __ballot_sync(0xffffffffu, in);
    if (lane == 0) s.warp_n[0][warp] = __popc(bal);
    __syncthreads();
    int off = base;
    for (int w = 0; w < warp; ++w) off += s.warp_n[0][w];
    if (in) out[off + __popc(bal & ((1u << lane) - 1u))] = i;
    for (int w = warp; w < RS_WARPS; ++w) off += s.warp_n[0][w];
    base = off;
    __syncthreads();
  }
}

// thread 0's solvers, out of line so that their registers do not weigh on the CTA's passes over the rows
__device__ __noinline__ int rs_p3p(const double* b, const double* p, double* models) { return pose::p3p_ke(b, p, models); }
__device__ __noinline__ void rs_lu(int k, const double* b, const double* p, double* out) { pose::lu_pose(k, b, p, out); }

__global__ void rs_normalize(double* bearings, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double* b = bearings + 3 * i;
  const double r = sqrt(b[0] * b[0] + b[1] * b[1] + b[2] * b[2]);
  b[0] /= r;
  b[1] /= r;
  b[2] /= r;
}

extern __shared__ double rs_dyn[];

__global__ void __launch_bounds__(RS_THREADS) rs_ransac(RsArgs a, int staged) {
  __shared__ RsShared s;
  const int shot = a.order[blockIdx.x];
  const long long off = a.shot_start[shot];
  const int n = (int)(a.shot_start[shot + 1] - off);
  RsRows rows{nullptr, a.bearings, a.points, a.row_b + off, a.row_x + off, n};
  if (staged) {
    for (int i = threadIdx.x; i < n; i += RS_THREADS) {
      const double* u = a.bearings + 3 * rows.rb[i];
      const double* v = a.points + 3 * rows.rx[i];
      for (int c = 0; c < 3; ++c) {
        rs_dyn[c * n + i] = u[c];
        rs_dyn[(3 + c) * n + i] = v[c];
      }
    }
    rows.sm = rs_dyn;
  }
  int* best_rows = a.best_rows + off;
  const double t = a.ransac_threshold;
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
    if (nm == RS_MAX_MODELS) rs_count<RS_MAX_MODELS>(s, rows, &s.models[0][0], t, s.counts);
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
          rs_compact(s, rows, s.models[j], t, best_rows);
          for (int lo = 0; lo < RS_LO_ITERATIONS; ++lo) {
            if (threadIdx.x == 0) {
              const int m = s.best_count;
              const int size = max(min(RS_MAX_SAMPLE, (int)(m * 0.5)), RS_MIN_SAMPLE);
              stream_sample(s.st, a.src, shot, size, m, s.idx);
              for (int k = 0; k < size; ++k) rows.get(best_rows[s.idx[k]], s.b + 3 * k, s.p + 3 * k);
              rs_lu(size, s.b, s.p, s.cand);
            }
            __syncthreads();
            rs_count<1>(s, rows, s.cand, t, &s.cand_count);
            if (s.cand_count >= s.best_count) {
              rs_compact(s, rows, s.cand, t, best_rows);
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
  int cnt = 0;
  for (int i = threadIdx.x; i < n; i += RS_THREADS) {
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
    cnt += in ? 1 : 0;
  }
  cnt = __reduce_add_sync(0xffffffffu, cnt);
  if ((threadIdx.x & 31) == 0) s.warp_n[0][threadIdx.x >> 5] = cnt;
  __syncthreads();
  if (threadIdx.x == 0) {
    int total = 0;
    for (int w = 0; w < RS_WARPS; ++w) total += s.warp_n[0][w];
    a.chord_inliers[shot] = total;
    a.ransac_inliers[shot] = s.best_count;
    for (int k = 0; k < 12; ++k) a.lo_model[12LL * shot + k] = M[k];
    if (a.src.trace) {
      a.trace_count[shot] = s.st.trace_n;
      a.stream_used[shot] = s.st.cursor;
    }
  }
}

struct Resect : DeviceStream<2> {
  bool timed = false;
  int trace_cap = 0;
  long long S = 0;

  StreamPrefix prefix;
  SmemOptIn smem_opt_in;
  DevBuf<double> d_bearings, d_points, d_lo;
  DevBuf<long long> d_shot_start, d_row_b, d_row_x, d_stream_used;
  DevBuf<int> d_order, d_best_rows, d_ransac, d_chord, d_trace, d_trace_count;
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
  timed = false;
  S = 0;
  if (num_bearings < 0 || num_points < 0 || num_shots < 0 || num_shots > INT_MAX) throw ArgError("resection: bad sizes");
  if (iterations < 1) throw ArgError("resection: iterations must be at least 1");
  if (!std::isfinite(threshold) || threshold <= 0.0) throw ArgError("resection: threshold must be positive");
  if (!shot_start) throw ArgError("resection: null shot_start");
  if (shot_start[0] != 0) throw ArgError("resection: shot_start[0] must be 0");
  for (int64_t s = 0; s < num_shots; ++s) {
    const int64_t n = shot_start[s + 1] - shot_start[s];
    if (n < RS_MIN_SAMPLE)
      throw ArgError("resection: shot " + std::to_string(s) + " has " + std::to_string(n) +
                     " rows; at least 3 are needed");
    if (n > INT_MAX) throw ArgError("resection: shot " + std::to_string(s) + " has more than 2^31 - 1 rows");
  }
  const int64_t R = shot_start[num_shots];
  if (num_shots > 0 && (!row_bearing || !row_point || !bearings || !points || !lo_model || !ransac_inliers ||
                        !chord_inliers || !chord_mask))
    throw ArgError("resection: null arrays");
  for (int64_t s = 0; s < num_shots; ++s)
    for (int64_t r = shot_start[s]; r < shot_start[s + 1]; ++r) {
      if (row_bearing[r] < 0 || row_bearing[r] >= num_bearings)
        throw ArgError("resection: row " + std::to_string(r - shot_start[s]) + " of shot " + std::to_string(s) +
                       " names a bearing outside [0, " + std::to_string(num_bearings) + ")");
      if (row_point[r] < 0 || row_point[r] >= num_points)
        throw ArgError("resection: row " + std::to_string(r - shot_start[s]) + " of shot " + std::to_string(s) +
                       " names a point outside [0, " + std::to_string(num_points) + ")");
    }
  if (num_shots == 0) return;
  prefix.make(stream);

  // largest shots first; the shots too large for shared memory form their own launch
  std::vector<int> order((size_t)num_shots);
  std::iota(order.begin(), order.end(), 0);
  std::stable_sort(order.begin(), order.end(), [&](int x, int y) {
    return shot_start[x + 1] - shot_start[x] > shot_start[y + 1] - shot_start[y];
  });
  int big = 0;
  while (big < num_shots && shot_start[order[big] + 1] - shot_start[order[big]] > RS_STAGE_ROWS) ++big;
  const int staged_rows = big < num_shots ? (int)(shot_start[order[big] + 1] - shot_start[order[big]]) : 0;

  upload(d_bearings, bearings, (size_t)num_bearings * 3);
  upload(d_points, points, (size_t)num_points * 3);
  upload(d_shot_start, reinterpret_cast<const long long*>(shot_start), (size_t)num_shots + 1);
  upload(d_row_b, reinterpret_cast<const long long*>(row_bearing), (size_t)R);
  upload(d_row_x, reinterpret_cast<const long long*>(row_point), (size_t)R);
  upload(d_order, order.data(), order.size());
  d_best_rows.reserve((size_t)R);
  d_mask.reserve((size_t)R);
  d_lo.reserve((size_t)num_shots * 12);
  d_ransac.reserve((size_t)num_shots);
  d_chord.reserve((size_t)num_shots);
  if (trace_cap > 0) {
    d_trace.reserve((size_t)num_shots * trace_cap);
    d_trace_count.reserve((size_t)num_shots);
    d_stream_used.reserve((size_t)num_shots);
  }

  RsArgs a;
  a.bearings = d_bearings.p;
  a.points = d_points.p;
  a.shot_start = d_shot_start.p;
  a.row_b = d_row_b.p;
  a.row_x = d_row_x.p;
  a.chord_threshold = threshold;
  a.ransac_threshold = 1.0 - std::cos(threshold);
  a.iterations = iterations;
  a.src = prefix.source(trace_cap > 0 ? d_trace.p : nullptr, trace_cap);
  a.best_rows = d_best_rows.p;
  a.lo_model = d_lo.p;
  a.ransac_inliers = d_ransac.p;
  a.chord_inliers = d_chord.p;
  a.chord_mask = d_mask.p;
  a.trace_count = d_trace_count.p;
  a.stream_used = d_stream_used.p;

  OSFM_CUDA(cudaEventRecord(ev[0], stream));
  if (num_bearings > 0) {
    rs_normalize<<<(unsigned)((num_bearings + 255) / 256), 256, 0, stream>>>(d_bearings.p, num_bearings);
    OSFM_LAUNCH_CHECK();
  }
  if (big > 0) {
    a.order = d_order.p;
    rs_ransac<<<big, RS_THREADS, 0, stream>>>(a, 0);
    OSFM_LAUNCH_CHECK();
  }
  if (big < num_shots) {
    const int smem_max = (int)(sizeof(double) * 6 * RS_STAGE_ROWS);
    smem_opt_in(rs_ransac, smem_max);
    const size_t smem = sizeof(double) * 6 * (size_t)staged_rows;
    a.order = d_order.p + big;
    rs_ransac<<<(unsigned)(num_shots - big), RS_THREADS, smem, stream>>>(a, 1);
    OSFM_LAUNCH_CHECK();
  }
  OSFM_CUDA(cudaEventRecord(ev[1], stream));
  download(lo_model, d_lo.p, (size_t)num_shots * 12);
  download(ransac_inliers, d_ransac.p, (size_t)num_shots);
  download(chord_inliers, d_chord.p, (size_t)num_shots);
  download(chord_mask, d_mask.p, (size_t)R);
  OSFM_CUDA(cudaStreamSynchronize(stream));
  S = num_shots;
  timed = true;
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
  return osfm::with_handle(h, [&](osfm::Resect& K) {
    if (length < 1 || length > (1LL << 28)) throw osfm::ArgError("stream prefix length must be in [1, 2^28]");
    K.prefix.want = length;
  });
}

int osfm_resect_set_trace(osfm_resect* h, int capacity) {
  return osfm::with_handle(h, [&](osfm::Resect& K) {
    if (capacity < 0) throw osfm::ArgError("negative trace capacity");
    K.trace_cap = capacity;
  });
}

int osfm_resect_get_trace(osfm_resect* h, int32_t* count, int64_t* stream_used, int32_t* indices) {
  return osfm::with_handle(h, [&](osfm::Resect& K) {
    if (!K.timed || K.trace_cap == 0) throw std::runtime_error("resection: no traced run");
    if (!count || !stream_used || !indices) throw osfm::ArgError("null outputs");
    K.download(count, K.d_trace_count.p, (size_t)K.S);
    K.download(reinterpret_cast<long long*>(stream_used), K.d_stream_used.p, (size_t)K.S);
    K.download(indices, K.d_trace.p, (size_t)K.S * K.trace_cap);
    OSFM_CUDA(cudaStreamSynchronize(K.stream));
  });
}

int osfm_resect_last_device_ms(osfm_resect* h, float* ms) {
  return osfm::with_handle(h, [&](osfm::Resect& K) {
    if (!ms) throw osfm::ArgError("null ms");
    *ms = 0.f;
    if (K.timed) OSFM_CUDA(cudaEventElapsedTime(ms, K.ev[0], K.ev[1]));
  });
}

}  // extern "C"
