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
// A pair of at most RR_STAGE_ROWS rows is staged in shared memory as fp64 structure-of-arrays; a larger one is read
// through L2 via its row indices.  A last pass writes the chord-inlier mask and counts.
//
// The sample stream, its device prefix and the stopping bound are those of ransac_stream.cuh.
#include <algorithm>
#include <cfloat>
#include <climits>
#include <cmath>
#include <memory>
#include <numeric>
#include <vector>

#include "absolute_pose.cuh"
#include "common.cuh"
#include "ransac_stream.cuh"

namespace osfm {
namespace {

constexpr int RR_THREADS = 128;
constexpr int RR_WARPS = RR_THREADS / 32;
constexpr int RR_STAGE_ROWS = 1024;
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
  StreamSource src;              // trace: trace_cap drawn indices per pair, or null
  int* best_rows;                // per row: the best model's inlier rows, ascending
  double* lo_model;              // 9 per pair
  int* ransac_inliers;
  int* chord_inliers;
  unsigned char* chord_mask;     // per row
  int* trace_count;
  long long* stream_used;
};

struct RrShared {
  StreamState st;
  double sample[RR_MAX_SAMPLE][6];
  double cand[9];                // rotation Q of the candidate (the model is Q^T), row-major
  double best[9];
  int best_count, cand_count;
  int replace, lo, stop;
  int idx[RR_MAX_SAMPLE];
  int warp_n[RR_WARPS];
};

struct RrRows {
  const double* sm;              // staged SoA (b1x b1y b1z b2x b2y b2z, n each) or null
  const double* bearings;
  const long long *ra, *rb;
  int n;
  __device__ __forceinline__ void get(int i, double* p, double* q) const {
    if (sm) {
      p[0] = sm[i]; p[1] = sm[n + i]; p[2] = sm[2 * n + i];
      q[0] = sm[3 * n + i]; q[1] = sm[4 * n + i]; q[2] = sm[5 * n + i];
    } else {
      const double* u = bearings + 3 * ra[i];
      const double* v = bearings + 3 * rb[i];
      p[0] = __ldg(u); p[1] = __ldg(u + 1); p[2] = __ldg(u + 2);
      q[0] = __ldg(v); q[1] = __ldg(v + 1); q[2] = __ldg(v + 2);
    }
  }
};

// ---- thread 0: the rotation of a sample ---------------------------------------------------------------------
// rotation Q (Q b2 ~ b1) of the k sample rows in s.sample, into out (absolute_pose.cuh)
__device__ void rr_rotation(RrShared& s, int k, double* out) {
  pose::rotation_between(k, &s.sample[0][0], &s.sample[0][3], 6, out);
}

// ---- the whole CTA ----------------------------------------------------------------------------------------
// |1 - (Q^T b1) . b2| < t, the model Q^T of rotation Q
__device__ __forceinline__ bool rr_inlier(const double* Q, const double* p, const double* q, double t) {
  const double v0 = Q[0] * p[0] + Q[3] * p[1] + Q[6] * p[2];
  const double v1 = Q[1] * p[0] + Q[4] * p[1] + Q[7] * p[2];
  const double v2 = Q[2] * p[0] + Q[5] * p[1] + Q[8] * p[2];
  return fabs(1.0 - (v0 * q[0] + v1 * q[1] + v2 * q[2])) < t;
}

// inliers of s.cand into s.cand_count
__device__ void rr_count(RrShared& s, const RrRows& rows, double t) {
  double Q[9];
  for (int k = 0; k < 9; ++k) Q[k] = s.cand[k];
  int c = 0;
  for (int i = threadIdx.x; i < rows.n; i += RR_THREADS) {
    double p[3], q[3];
    rows.get(i, p, q);
    c += rr_inlier(Q, p, q, t) ? 1 : 0;
  }
  c = __reduce_add_sync(0xffffffffu, c);
  if ((threadIdx.x & 31) == 0) s.warp_n[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    int n = 0;
    for (int w = 0; w < RR_WARPS; ++w) n += s.warp_n[w];
    s.cand_count = n;
  }
  __syncthreads();
}

// s.cand's inlier rows, ascending, into out
__device__ void rr_compact(RrShared& s, const RrRows& rows, double t, int* out) {
  double Q[9];
  for (int k = 0; k < 9; ++k) Q[k] = s.cand[k];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int base = 0;
  for (int tile = 0; tile < rows.n; tile += RR_THREADS) {
    const int i = tile + threadIdx.x;
    bool in = false;
    if (i < rows.n) {
      double p[3], q[3];
      rows.get(i, p, q);
      in = rr_inlier(Q, p, q, t);
    }
    const unsigned bal = __ballot_sync(0xffffffffu, in);
    if (lane == 0) s.warp_n[warp] = __popc(bal);
    __syncthreads();
    int off = base;
    for (int w = 0; w < warp; ++w) off += s.warp_n[w];
    if (in) out[off + __popc(bal & ((1u << lane) - 1u))] = i;
    for (int w = warp; w < RR_WARPS; ++w) off += s.warp_n[w];
    base = off;
    __syncthreads();
  }
}

extern __shared__ double rr_dyn[];

__global__ void __launch_bounds__(RR_THREADS) rr_ransac(RrArgs a, int staged) {
  __shared__ RrShared s;
  const int pair = a.order[blockIdx.x];
  const long long off = a.pair_start[pair];
  const int n = (int)(a.pair_start[pair + 1] - off);
  RrRows rows{nullptr, a.bearings, a.row_a + off, a.row_b + off, n};
  if (staged) {
    for (int i = threadIdx.x; i < n; i += RR_THREADS) {
      const double* u = a.bearings + 3 * rows.ra[i];
      const double* v = a.bearings + 3 * rows.rb[i];
      for (int c = 0; c < 3; ++c) {
        rr_dyn[c * n + i] = u[c];
        rr_dyn[(3 + c) * n + i] = v[c];
      }
    }
    rows.sm = rr_dyn;
  }
  int* best_rows = a.best_rows + off;
  const double t = a.ransac_threshold;
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
    rr_count(s, rows, t);
    // the best model is replaced on ties (std::max(score, best) returns score when they are equal)
    const bool replace = s.cand_count >= s.best_count;
    if (replace) {
      rr_compact(s, rows, t, best_rows);
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
          rr_count(s, rows, t);
          if (s.cand_count >= s.best_count) {
            rr_compact(s, rows, t, best_rows);
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
  int c = 0;
  for (int i = threadIdx.x; i < n; i += RR_THREADS) {
    double p[3], q[3];
    rows.get(i, p, q);
    const double d0 = Q[0] * q[0] + Q[1] * q[1] + Q[2] * q[2] - p[0];
    const double d1 = Q[3] * q[0] + Q[4] * q[1] + Q[5] * q[2] - p[1];
    const double d2 = Q[6] * q[0] + Q[7] * q[1] + Q[8] * q[2] - p[2];
    const bool in = sqrt(d0 * d0 + d1 * d1 + d2 * d2) < a.chord_threshold;
    a.chord_mask[off + i] = in ? 1 : 0;
    c += in ? 1 : 0;
  }
  c = __reduce_add_sync(0xffffffffu, c);
  if ((threadIdx.x & 31) == 0) s.warp_n[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    int total = 0;
    for (int w = 0; w < RR_WARPS; ++w) total += s.warp_n[w];
    a.chord_inliers[pair] = total;
    a.ransac_inliers[pair] = s.best_count;
    for (int r = 0; r < 3; ++r)
      for (int k = 0; k < 3; ++k) a.lo_model[9LL * pair + r * 3 + k] = Q[k * 3 + r];
    if (a.src.trace) {
      a.trace_count[pair] = s.st.trace_n;
      a.stream_used[pair] = s.st.cursor;
    }
  }
}

struct RotRansac : DeviceStream<2> {
  bool timed = false;
  int trace_cap = 0;
  long long P = 0;

  StreamPrefix prefix;
  DevBuf<double> d_bearings, d_lo;
  DevBuf<long long> d_pair_start, d_row_a, d_row_b, d_stream_used;
  DevBuf<int> d_order, d_best_rows, d_ransac, d_chord, d_trace, d_trace_count;
  DevBuf<unsigned char> d_mask;

  explicit RotRansac(int dev) : DeviceStream(dev) {}

  void run(int64_t num_bearings, const double* bearings, int64_t num_pairs, const int64_t* pair_start,
           const int64_t* row_a, const int64_t* row_b, double threshold, int iterations, double* lo_model,
           int32_t* ransac_inliers, int32_t* chord_inliers, uint8_t* chord_mask);
};

void RotRansac::run(int64_t num_bearings, const double* bearings, int64_t num_pairs, const int64_t* pair_start,
                    const int64_t* row_a, const int64_t* row_b, double threshold, int iterations, double* lo_model,
                    int32_t* ransac_inliers, int32_t* chord_inliers, uint8_t* chord_mask) {
  timed = false;
  P = 0;
  if (num_bearings < 0 || num_pairs < 0 || num_pairs > INT_MAX) throw ArgError("rotation RANSAC: bad sizes");
  if (iterations < 1) throw ArgError("rotation RANSAC: iterations must be at least 1");
  if (!std::isfinite(threshold) || threshold <= 0.0) throw ArgError("rotation RANSAC: threshold must be positive");
  if (!pair_start) throw ArgError("rotation RANSAC: null pair_start");
  if (pair_start[0] != 0) throw ArgError("rotation RANSAC: pair_start[0] must be 0");
  for (int64_t p = 0; p < num_pairs; ++p) {
    const int64_t n = pair_start[p + 1] - pair_start[p];
    if (n < RR_MIN_SAMPLE)
      throw ArgError("rotation RANSAC: pair " + std::to_string(p) + " has " + std::to_string(n) +
                     " correspondences; at least 3 are needed");
    if (n > INT_MAX) throw ArgError("rotation RANSAC: pair " + std::to_string(p) + " has more than 2^31 - 1 rows");
  }
  const int64_t R = pair_start[num_pairs];
  if (num_pairs > 0 && (!row_a || !row_b || !bearings || !lo_model || !ransac_inliers || !chord_inliers || !chord_mask))
    throw ArgError("rotation RANSAC: null arrays");
  for (int64_t p = 0; p < num_pairs; ++p)
    for (int64_t r = pair_start[p]; r < pair_start[p + 1]; ++r)
      if (row_a[r] < 0 || row_a[r] >= num_bearings || row_b[r] < 0 || row_b[r] >= num_bearings)
        throw ArgError("rotation RANSAC: row " + std::to_string(r - pair_start[p]) + " of pair " + std::to_string(p) +
                       " names a bearing outside [0, " + std::to_string(num_bearings) + ")");
  if (num_pairs == 0) {
    timed = false;
    return;
  }
  prefix.make(stream);

  // largest pairs first; the pairs too large for shared memory form their own launch
  std::vector<int> order((size_t)num_pairs);
  std::iota(order.begin(), order.end(), 0);
  std::stable_sort(order.begin(), order.end(), [&](int x, int y) {
    return pair_start[x + 1] - pair_start[x] > pair_start[y + 1] - pair_start[y];
  });
  int big = 0;
  while (big < num_pairs && pair_start[order[big] + 1] - pair_start[order[big]] > RR_STAGE_ROWS) ++big;
  const int staged_rows = big < num_pairs ? (int)(pair_start[order[big] + 1] - pair_start[order[big]]) : 0;

  upload(d_bearings, bearings, (size_t)num_bearings * 3);
  upload(d_pair_start, reinterpret_cast<const long long*>(pair_start), (size_t)num_pairs + 1);
  upload(d_row_a, reinterpret_cast<const long long*>(row_a), (size_t)R);
  upload(d_row_b, reinterpret_cast<const long long*>(row_b), (size_t)R);
  upload(d_order, order.data(), order.size());
  d_best_rows.reserve((size_t)R);
  d_mask.reserve((size_t)R);
  d_lo.reserve((size_t)num_pairs * 9);
  d_ransac.reserve((size_t)num_pairs);
  d_chord.reserve((size_t)num_pairs);
  if (trace_cap > 0) {
    d_trace.reserve((size_t)num_pairs * trace_cap);
    d_trace_count.reserve((size_t)num_pairs);
    d_stream_used.reserve((size_t)num_pairs);
  }

  RrArgs a;
  a.bearings = d_bearings.p;
  a.pair_start = d_pair_start.p;
  a.row_a = d_row_a.p;
  a.row_b = d_row_b.p;
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
  if (big > 0) {
    a.order = d_order.p;
    rr_ransac<<<big, RR_THREADS, 0, stream>>>(a, 0);
    OSFM_LAUNCH_CHECK();
  }
  if (big < num_pairs) {
    const size_t smem = sizeof(double) * 6 * (size_t)staged_rows;
    OSFM_CUDA(cudaFuncSetAttribute(rr_ransac, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    a.order = d_order.p + big;
    rr_ransac<<<(unsigned)(num_pairs - big), RR_THREADS, smem, stream>>>(a, 1);
    OSFM_LAUNCH_CHECK();
  }
  OSFM_CUDA(cudaEventRecord(ev[1], stream));
  download(lo_model, d_lo.p, (size_t)num_pairs * 9);
  download(ransac_inliers, d_ransac.p, (size_t)num_pairs);
  download(chord_inliers, d_chord.p, (size_t)num_pairs);
  download(chord_mask, d_mask.p, (size_t)R);
  OSFM_CUDA(cudaStreamSynchronize(stream));
  P = num_pairs;
  timed = true;
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
  return osfm::with_handle(h, [&](osfm::RotRansac& K) {
    if (length < 1 || length > (1LL << 28)) throw osfm::ArgError("stream prefix length must be in [1, 2^28]");
    K.prefix.want = length;
  });
}

int osfm_rotransac_set_trace(osfm_rotransac* h, int capacity) {
  return osfm::with_handle(h, [&](osfm::RotRansac& K) {
    if (capacity < 0) throw osfm::ArgError("negative trace capacity");
    K.trace_cap = capacity;
  });
}

int osfm_rotransac_get_trace(osfm_rotransac* h, int32_t* count, int64_t* stream_used, int32_t* indices) {
  return osfm::with_handle(h, [&](osfm::RotRansac& K) {
    if (!K.timed || K.trace_cap == 0) throw std::runtime_error("rotation RANSAC: no traced run");
    if (!count || !stream_used || !indices) throw osfm::ArgError("null outputs");
    K.download(count, K.d_trace_count.p, (size_t)K.P);
    K.download(reinterpret_cast<long long*>(stream_used), K.d_stream_used.p, (size_t)K.P);
    K.download(indices, K.d_trace.p, (size_t)K.P * K.trace_cap);
    OSFM_CUDA(cudaStreamSynchronize(K.stream));
  });
}

int osfm_rotransac_last_device_ms(osfm_rotransac* h, float* ms) {
  return osfm::with_handle(h, [&](osfm::RotRansac& K) {
    if (!ms) throw osfm::ArgError("null ms");
    *ms = 0.f;
    if (K.timed) OSFM_CUDA(cudaEventElapsedTime(ms, K.ev[0], K.ev[1]));
  });
}

}  // extern "C"
