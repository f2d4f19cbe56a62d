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
// A pair of at most RP_STAGE_ROWS rows is staged in shared memory as fp64 structure-of-arrays (both bearings, 48 B
// per row); a larger one is read through L2 via its row indices.  A last pass writes the inlier mask of the result.
#include <algorithm>
#include <climits>
#include <cmath>
#include <numeric>
#include <string>
#include <vector>

#include "common.cuh"
#include "ransac_stream.cuh"
#include "relative_pose.cuh"

namespace osfm {
namespace {

constexpr int RP_THREADS = 128;
constexpr int RP_WARPS = RP_THREADS / 32;
constexpr int RP_STAGE_ROWS = 1024;        // 48 KB of shared memory
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
  StreamSource src;              // trace: trace_cap drawn indices per pair, or null
  int* best_rows;                // per row: the best model's inlier rows, ascending
  double* lo_model;              // 12 per pair
  int* ransac_inliers;
  unsigned char* mask;           // per row
  int* trace_count;
  long long* stream_used;
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
  int warp_n[RP_MAX_MODELS][RP_WARPS];
};

struct RpRows {
  const double* sm;              // staged SoA (ax ay az bx by bz, n each) or null
  const double* bearings;
  const long long *ra, *rb;
  int n;
  __device__ __forceinline__ void get(int i, double* x, double* y) const {
    if (sm) {
      x[0] = sm[i]; x[1] = sm[n + i]; x[2] = sm[2 * n + i];
      y[0] = sm[3 * n + i]; y[1] = sm[4 * n + i]; y[2] = sm[5 * n + i];
    } else {
      const double* u = bearings + 3 * ra[i];
      const double* v = bearings + 3 * rb[i];
      x[0] = __ldg(u); x[1] = __ldg(u + 1); x[2] = __ldg(u + 2);
      y[0] = __ldg(v); y[1] = __ldg(v + 1); y[2] = __ldg(v + 2);
    }
  }
};

__device__ __forceinline__ bool rp_inlier(const double* M, const double* x, const double* y, double t) {
  return fabs(relpose::evaluate(M, x, y)) < t;
}

// inliers of the nm models at M (12 apart, in shared memory) into counts, in one pass over the rows
__device__ void rp_count(RpShared& s, const RpRows& rows, const double* M, int nm, double t, int* counts) {
  int c[RP_MAX_MODELS];
#pragma unroll
  for (int j = 0; j < RP_MAX_MODELS; ++j) c[j] = 0;
  for (int i = threadIdx.x; i < rows.n; i += RP_THREADS) {
    double x[3], y[3];
    rows.get(i, x, y);
#pragma unroll
    for (int j = 0; j < RP_MAX_MODELS; ++j)
      if (j < nm) c[j] += rp_inlier(M + 12 * j, x, y, t) ? 1 : 0;
  }
#pragma unroll
  for (int j = 0; j < RP_MAX_MODELS; ++j) {
    if (j >= nm) break;
    const int w = __reduce_add_sync(0xffffffffu, c[j]);
    if ((threadIdx.x & 31) == 0) s.warp_n[j][threadIdx.x >> 5] = w;
  }
  __syncthreads();
  if (threadIdx.x < nm) {
    int total = 0;
    for (int w = 0; w < RP_WARPS; ++w) total += s.warp_n[threadIdx.x][w];
    counts[threadIdx.x] = total;
  }
  __syncthreads();
}

// the inlier rows of the pose M, ascending, into out
__device__ void rp_compact(RpShared& s, const RpRows& rows, const double* M, double t, int* out) {
  double m[12];
  for (int k = 0; k < 12; ++k) m[k] = M[k];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int base = 0;
  for (int tile = 0; tile < rows.n; tile += RP_THREADS) {
    const int i = tile + threadIdx.x;
    bool in = false;
    if (i < rows.n) {
      double x[3], y[3];
      rows.get(i, x, y);
      in = rp_inlier(m, x, y, t);
    }
    const unsigned bal = __ballot_sync(0xffffffffu, in);
    if (lane == 0) s.warp_n[0][warp] = __popc(bal);
    __syncthreads();
    int off = base;
    for (int w = 0; w < warp; ++w) off += s.warp_n[0][w];
    if (in) out[off + __popc(bal & ((1u << lane) - 1u))] = i;
    for (int w = warp; w < RP_WARPS; ++w) off += s.warp_n[0][w];
    base = off;
    __syncthreads();
  }
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

__global__ void rp_normalize(double* bearings, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double* b = bearings + 3 * i;
  const double r = sqrt(b[0] * b[0] + b[1] * b[1] + b[2] * b[2]);
  b[0] /= r;
  b[1] /= r;
  b[2] /= r;
}

extern __shared__ double rp_dyn[];

__global__ void __launch_bounds__(RP_THREADS) rp_ransac(RpArgs a, int staged) {
  __shared__ RpShared s;
  const int pair = a.order[blockIdx.x];
  const long long off = a.pair_start[pair];
  const int n = (int)(a.pair_start[pair + 1] - off);
  RpRows rows{nullptr, a.bearings, a.row_a + off, a.row_b + off, n};
  if (staged) {
    for (int i = threadIdx.x; i < n; i += RP_THREADS) {
      const double* u = a.bearings + 3 * rows.ra[i];
      const double* v = a.bearings + 3 * rows.rb[i];
      for (int c = 0; c < 3; ++c) {
        rp_dyn[c * n + i] = u[c];
        rp_dyn[(3 + c) * n + i] = v[c];
      }
    }
    rows.sm = rp_dyn;
  }
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
    if (nm > 0) rp_count(s, rows, &s.models[0][0], nm, t, s.counts);
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
          rp_compact(s, rows, s.models[j], t, best_rows);
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
              rp_count(s, rows, s.cand, 1, t, &s.cand_count);
              if (s.cand_count >= s.best_count) {
                rp_compact(s, rows, s.cand, t, best_rows);
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
  for (int i = threadIdx.x; i < n; i += RP_THREADS) {
    double x[3], y[3];
    rows.get(i, x, y);
    a.mask[off + i] = rp_inlier(M, x, y, t) ? 1 : 0;
  }
  if (threadIdx.x == 0) {
    a.ransac_inliers[pair] = s.best_count;
    for (int k = 0; k < 12; ++k) a.lo_model[12LL * pair + k] = M[k];
    if (a.src.trace) {
      a.trace_count[pair] = s.st.trace_n;
      a.stream_used[pair] = s.st.cursor;
    }
  }
}

struct RelPose : DeviceStream<2> {
  bool timed = false;
  int trace_cap = 0;
  long long P = 0;

  StreamPrefix prefix;
  SmemOptIn smem_opt_in;
  DevBuf<double> d_bearings, d_lo;
  DevBuf<long long> d_pair_start, d_row_a, d_row_b, d_stream_used;
  DevBuf<int> d_order, d_best_rows, d_ransac, d_trace, d_trace_count;
  DevBuf<unsigned char> d_mask;

  explicit RelPose(int dev) : DeviceStream(dev) {}

  void run(int64_t num_bearings, const double* bearings, int64_t num_pairs, const int64_t* pair_start,
           const int64_t* row_a, const int64_t* row_b, double threshold, int iterations, double* lo_model,
           int32_t* ransac_inliers, uint8_t* inlier_mask);
};

void RelPose::run(int64_t num_bearings, const double* bearings, int64_t num_pairs, const int64_t* pair_start,
                  const int64_t* row_a, const int64_t* row_b, double threshold, int iterations, double* lo_model,
                  int32_t* ransac_inliers, uint8_t* inlier_mask) {
  timed = false;
  P = 0;
  if (num_bearings < 0 || num_pairs < 0 || num_pairs > INT_MAX) throw ArgError("relative pose: bad sizes");
  if (iterations < 1) throw ArgError("relative pose: iterations must be at least 1");
  if (!std::isfinite(threshold) || threshold <= 0.0) throw ArgError("relative pose: threshold must be positive");
  if (!pair_start) throw ArgError("relative pose: null pair_start");
  if (pair_start[0] != 0) throw ArgError("relative pose: pair_start[0] must be 0");
  for (int64_t p = 0; p < num_pairs; ++p) {
    const int64_t n = pair_start[p + 1] - pair_start[p];
    if (n < RP_MIN_SAMPLE)
      throw ArgError("relative pose: pair " + std::to_string(p) + " has " + std::to_string(n) +
                     " rows; at least 5 are needed");
    if (n > INT_MAX) throw ArgError("relative pose: pair " + std::to_string(p) + " has more than 2^31 - 1 rows");
  }
  const int64_t R = pair_start[num_pairs];
  if (num_pairs > 0 && (!row_a || !row_b || !bearings || !lo_model || !ransac_inliers || !inlier_mask))
    throw ArgError("relative pose: null arrays");
  for (int64_t p = 0; p < num_pairs; ++p)
    for (int64_t r = pair_start[p]; r < pair_start[p + 1]; ++r)
      if (row_a[r] < 0 || row_a[r] >= num_bearings || row_b[r] < 0 || row_b[r] >= num_bearings)
        throw ArgError("relative pose: row " + std::to_string(r - pair_start[p]) + " of pair " + std::to_string(p) +
                       " names a bearing outside [0, " + std::to_string(num_bearings) + ")");
  if (num_pairs == 0) return;
  prefix.make(stream);

  // largest pairs first; the pairs too large for shared memory form their own launch
  std::vector<int> order((size_t)num_pairs);
  std::iota(order.begin(), order.end(), 0);
  std::stable_sort(order.begin(), order.end(), [&](int x, int y) {
    return pair_start[x + 1] - pair_start[x] > pair_start[y + 1] - pair_start[y];
  });
  int big = 0;
  while (big < num_pairs && pair_start[order[big] + 1] - pair_start[order[big]] > RP_STAGE_ROWS) ++big;
  const int staged_rows = big < num_pairs ? (int)(pair_start[order[big] + 1] - pair_start[order[big]]) : 0;

  upload(d_bearings, bearings, (size_t)num_bearings * 3);
  upload(d_pair_start, reinterpret_cast<const long long*>(pair_start), (size_t)num_pairs + 1);
  upload(d_row_a, reinterpret_cast<const long long*>(row_a), (size_t)R);
  upload(d_row_b, reinterpret_cast<const long long*>(row_b), (size_t)R);
  upload(d_order, order.data(), order.size());
  d_best_rows.reserve((size_t)R);
  d_mask.reserve((size_t)R);
  d_lo.reserve((size_t)num_pairs * 12);
  d_ransac.reserve((size_t)num_pairs);
  if (trace_cap > 0) {
    d_trace.reserve((size_t)num_pairs * trace_cap);
    d_trace_count.reserve((size_t)num_pairs);
    d_stream_used.reserve((size_t)num_pairs);
  }

  RpArgs a;
  a.bearings = d_bearings.p;
  a.pair_start = d_pair_start.p;
  a.row_a = d_row_a.p;
  a.row_b = d_row_b.p;
  a.threshold = 1.0 - std::cos(threshold);
  a.iterations = iterations;
  a.src = prefix.source(trace_cap > 0 ? d_trace.p : nullptr, trace_cap);
  a.best_rows = d_best_rows.p;
  a.lo_model = d_lo.p;
  a.ransac_inliers = d_ransac.p;
  a.mask = d_mask.p;
  a.trace_count = d_trace_count.p;
  a.stream_used = d_stream_used.p;

  OSFM_CUDA(cudaEventRecord(ev[0], stream));
  if (num_bearings > 0) {
    rp_normalize<<<(unsigned)((num_bearings + 255) / 256), 256, 0, stream>>>(d_bearings.p, num_bearings);
    OSFM_LAUNCH_CHECK();
  }
  if (big > 0) {
    a.order = d_order.p;
    rp_ransac<<<big, RP_THREADS, 0, stream>>>(a, 0);
    OSFM_LAUNCH_CHECK();
  }
  if (big < num_pairs) {
    const int smem_max = (int)(sizeof(double) * 6 * RP_STAGE_ROWS);
    smem_opt_in(rp_ransac, smem_max);
    const size_t smem = sizeof(double) * 6 * (size_t)staged_rows;
    a.order = d_order.p + big;
    rp_ransac<<<(unsigned)(num_pairs - big), RP_THREADS, smem, stream>>>(a, 1);
    OSFM_LAUNCH_CHECK();
  }
  OSFM_CUDA(cudaEventRecord(ev[1], stream));
  download(lo_model, d_lo.p, (size_t)num_pairs * 12);
  download(ransac_inliers, d_ransac.p, (size_t)num_pairs);
  download(inlier_mask, d_mask.p, (size_t)R);
  OSFM_CUDA(cudaStreamSynchronize(stream));
  P = num_pairs;
  timed = true;
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

int osfm_relpose_set_stream_prefix(osfm_relpose* h, int64_t length) {
  return osfm::with_handle(h, [&](osfm::RelPose& K) {
    if (length < 1 || length > (1LL << 28)) throw osfm::ArgError("stream prefix length must be in [1, 2^28]");
    K.prefix.want = length;
  });
}

int osfm_relpose_set_trace(osfm_relpose* h, int capacity) {
  return osfm::with_handle(h, [&](osfm::RelPose& K) {
    if (capacity < 0) throw osfm::ArgError("negative trace capacity");
    K.trace_cap = capacity;
  });
}

int osfm_relpose_get_trace(osfm_relpose* h, int32_t* count, int64_t* stream_used, int32_t* indices) {
  return osfm::with_handle(h, [&](osfm::RelPose& K) {
    if (!K.timed || K.trace_cap == 0) throw std::runtime_error("relative pose: no traced run");
    if (!count || !stream_used || !indices) throw osfm::ArgError("null outputs");
    K.download(count, K.d_trace_count.p, (size_t)K.P);
    K.download(reinterpret_cast<long long*>(stream_used), K.d_stream_used.p, (size_t)K.P);
    K.download(indices, K.d_trace.p, (size_t)K.P * K.trace_cap);
    OSFM_CUDA(cudaStreamSynchronize(K.stream));
  });
}

int osfm_relpose_last_device_ms(osfm_relpose* h, float* ms) {
  return osfm::with_handle(h, [&](osfm::RelPose& K) {
    if (!ms) throw osfm::ArgError("null ms");
    *ms = 0.f;
    if (K.timed) OSFM_CUDA(cudaEventElapsedTime(ms, K.ev[0], K.ev[1]));
  });
}

}  // extern "C"
