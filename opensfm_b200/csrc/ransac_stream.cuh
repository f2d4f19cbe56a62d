// What the batched RANSAC estimators (rotransac.cu, resect.cu, relpose.cu) share.  Each runs one CTA of
// RANSAC_THREADS per problem (a pair or a shot), largest problems first, and keeps its own sampling loop, solvers and
// counting loop; the rest is here:
//
// * The sample stream of pyrobust's RANSAC (robust/random_sampler.h, robust_estimator.h): a std::mt19937 seeded with
//   42 and restarted for every problem, indices drawn by libstdc++'s uniform_int_distribution, repeats in a sample
//   drawn again, and the ShouldStop bound.  The restatement these follow is oracle/rotation_ransac_oracle.py.  Every
//   problem consumes the same stream from its start, so a prefix of it is made once per handle and kept on the
//   device (StreamPrefix); a problem that reaches its end continues from the generator state saved after the prefix,
//   in its CTA's shared memory, so the stream stays exact.
// * The block-wide row passes: a problem's rows (two table entries per row, staged in shared memory when the problem
//   has at most RANSAC_STAGE_ROWS rows), the CTA sums of per-thread counts, the ascending list of a model's inlier
//   rows, and the bearing normalisation of resect and relpose.
// * The host side of a batch (RansacBatch): the argument checks, the launch plan and its two launches, and the test
//   hooks (stream prefix length, traces of the drawn indices).
#pragma once

#include <cfloat>
#include <climits>
#include <cmath>
#include <cstdint>
#include <initializer_list>
#include <memory>
#include <numeric>
#include <string>
#include <vector>

#include "common.cuh"

namespace osfm {

constexpr double RANSAC_PROBABILITY = 0.99;   // RobustEstimatorParams::probability; the callers never set it
constexpr long long RANSAC_DEFAULT_PREFIX = 1LL << 16;
constexpr int RANSAC_THREADS = 128;
constexpr int RANSAC_WARPS = RANSAC_THREADS / 32;
constexpr int RANSAC_STAGE_ROWS = 1024;       // 48 KB of shared memory at 48 B per row

// std::mt19937: the 32-bit Mersenne twister with its standard seeding.
struct Mt {
  static constexpr int N = 624, M = 397;
  uint32_t s[N];
  int i;
  __host__ __device__ void seed(uint32_t x) {
    s[0] = x;
    for (int k = 1; k < N; ++k) s[k] = 1812433253u * (s[k - 1] ^ (s[k - 1] >> 30)) + (uint32_t)k;
    i = N;
  }
  __host__ __device__ void twist() {
    for (int k = 0; k < N; ++k) {
      const uint32_t y = (s[k] & 0x80000000u) | (s[(k + 1) % N] & 0x7fffffffu);
      s[k] = s[(k + M) % N] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
    }
    i = 0;
  }
  __host__ __device__ uint32_t next() {
    if (i >= N) twist();
    uint32_t y = s[i++];
    y ^= y >> 11;
    y ^= (y << 7) & 0x9d2c5680u;
    y ^= (y << 15) & 0xefc60000u;
    y ^= y >> 18;
    return y;
  }
};

// Where a launch reads the stream from, and where it records the drawn indices (trace, trace_cap per problem), how
// many were drawn and how many generator outputs each problem used.
struct StreamSource {
  const uint32_t* prefix;
  long long prefix_len;
  const Mt* saved;               // the generator after prefix_len outputs
  int* trace;                    // or null
  int trace_cap;
  int* trace_count;
  long long* stream_used;
};

// One problem's position in the stream; lives in shared memory and is touched by one thread.
struct StreamState {
  Mt mt;                         // live once the problem has used the whole prefix
  long long cursor;
  int mt_live;
  int trace_n;
  __device__ void reset() {
    cursor = 0;
    mt_live = 0;
    trace_n = 0;
  }
};

__device__ inline uint32_t stream_next(StreamState& s, const StreamSource& a) {
  if (s.cursor < a.prefix_len) return __ldg(a.prefix + s.cursor++);
  if (!s.mt_live) {
    s.mt = *a.saved;
    s.mt_live = 1;
  }
  ++s.cursor;
  return s.mt.next();
}

// uniform_int_distribution<unsigned long>(0, n - 1) over a 32-bit generator, libstdc++ 13: Lemire's 64-bit product,
// rejecting low words below 2^32 mod n
__device__ inline int stream_draw(StreamState& s, const StreamSource& a, uint32_t n) {
  unsigned long long prod = (unsigned long long)stream_next(s, a) * n;
  uint32_t low = (uint32_t)prod;
  if (low < n) {
    const uint32_t thr = (0u - n) % n;
    while (low < thr) {
      prod = (unsigned long long)stream_next(s, a) * n;
      low = (uint32_t)prod;
    }
  }
  return (int)(prod >> 32);
}

// `size` distinct indices in [0, n) into idx, redrawing repeats; recorded in problem `item`'s trace
__device__ inline void stream_sample(StreamState& s, const StreamSource& a, int item, int size, int n, int* idx) {
  for (int k = 0; k < size; ++k) {
    int v;
    bool dup;
    do {
      v = stream_draw(s, a, (uint32_t)n);
      dup = false;
      for (int j = 0; j < k; ++j) dup |= idx[j] == v;
    } while (dup);
    idx[k] = v;
    if (a.trace) {
      if (s.trace_n < a.trace_cap) a.trace[(long long)item * a.trace_cap + s.trace_n] = v;
      ++s.trace_n;
    }
  }
}

// thread 0, when problem `item` is done: how many indices it drew and how many generator outputs it used
__device__ inline void stream_record(const StreamState& s, const StreamSource& a, int item) {
  if (a.trace) {
    a.trace_count[item] = s.trace_n;
    a.stream_used[item] = s.cursor;
  }
}

// ShouldStop with `minimal`-row samples: stop once log(1 - p) / log(min(1 - eps, 1 - ratio^minimal)) < iteration
__device__ inline bool ransac_should_stop(int best_inliers, int n, int iteration, int minimal = 3) {
  const double ratio = (double)best_inliers / n;
  const double p1 = fmin(1.0 - DBL_EPSILON, 1.0 - pow(ratio, (double)minimal));
  return log(1.0 - RANSAC_PROBABILITY) / log(p1) < (double)iteration;
}

// ---- the whole CTA: a problem's rows ----------------------------------------------------------------------------
// Row i of a problem is entry ia[i] of table ta and entry ib[i] of table tb (3 doubles each; for pairs both tables
// are the bearing table).  A problem of at most RANSAC_STAGE_ROWS rows is staged in shared memory as fp64
// structure-of-arrays (a's x y z, then b's x y z, n each); a larger one is read through L2.
struct RansacRows {
  const double* sm;              // the staged rows, or null
  const double *ta, *tb;
  const long long *ia, *ib;
  int n;
  __device__ __forceinline__ void get(int i, double* x, double* y) const {
    if (sm) {
      x[0] = sm[i]; x[1] = sm[n + i]; x[2] = sm[2 * n + i];
      y[0] = sm[3 * n + i]; y[1] = sm[4 * n + i]; y[2] = sm[5 * n + i];
    } else {
      const double* u = ta + 3 * ia[i];
      const double* v = tb + 3 * ib[i];
      x[0] = __ldg(u); x[1] = __ldg(u + 1); x[2] = __ldg(u + 2);
      y[0] = __ldg(v); y[1] = __ldg(v + 1); y[2] = __ldg(v + 2);
    }
  }
};

extern __shared__ double ransac_dyn[];

// A problem's n rows, staged into the dynamic shared array when `staged`; the caller's next barrier publishes them.
__device__ __forceinline__ RansacRows ransac_rows(const double* ta, const double* tb, const long long* ia,
                                                  const long long* ib, int n, int staged) {
  RansacRows rows{nullptr, ta, tb, ia, ib, n};
  if (staged) {
    for (int i = threadIdx.x; i < n; i += RANSAC_THREADS) {
      const double* u = ta + 3 * ia[i];
      const double* v = tb + 3 * ib[i];
      for (int c = 0; c < 3; ++c) {
        ransac_dyn[c * n + i] = u[c];
        ransac_dyn[(3 + c) * n + i] = v[c];
      }
    }
    rows.sm = ransac_dyn;
  }
  return rows;
}

// counts[j] = the CTA's sum of every thread's c[j], for j < nm <= NC.  warp_n is NC x RANSAC_WARPS ints of shared
// scratch; ends with a barrier, so every thread may read counts.
template <int NC>
__device__ __forceinline__ void ransac_sums(const int (&c)[NC], int nm, int* warp_n, int* counts) {
#pragma unroll
  for (int j = 0; j < NC; ++j) {
    if (j >= nm) break;
    const int w = __reduce_add_sync(0xffffffffu, c[j]);
    if ((threadIdx.x & 31) == 0) warp_n[j * RANSAC_WARPS + (threadIdx.x >> 5)] = w;
  }
  __syncthreads();
  if (threadIdx.x < nm) {
    int total = 0;
    for (int w = 0; w < RANSAC_WARPS; ++w) total += warp_n[threadIdx.x * RANSAC_WARPS + w];
    counts[threadIdx.x] = total;
  }
  __syncthreads();
}

// The rows on which the model M (NM doubles) passes test(M, x, y), ascending, into out; returns how many there are.
// warp_n is RANSAC_WARPS ints of shared scratch.
template <int NM, class Test>
__device__ int ransac_compact(const RansacRows& rows, const double* M, Test test, int* warp_n, int* out) {
  double m[NM];
  for (int k = 0; k < NM; ++k) m[k] = M[k];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int base = 0;
  for (int tile = 0; tile < rows.n; tile += RANSAC_THREADS) {
    const int i = tile + threadIdx.x;
    bool in = false;
    if (i < rows.n) {
      double x[3], y[3];
      rows.get(i, x, y);
      in = test(m, x, y);
    }
    const unsigned bal = __ballot_sync(0xffffffffu, in);
    if (lane == 0) warp_n[warp] = __popc(bal);
    __syncthreads();
    int off = base;
    for (int w = 0; w < warp; ++w) off += warp_n[w];
    if (in) out[off + __popc(bal & ((1u << lane) - 1u))] = i;
    for (int w = warp; w < RANSAC_WARPS; ++w) off += warp_n[w];
    base = off;
    __syncthreads();
  }
  return base;
}

// The n bearings (3 each) scaled to unit length, in place.  A template, so that only the sources that launch it
// (resect.cu, relpose.cu) compile it.
namespace {
template <class T>
__global__ void ransac_normalize(T* bearings, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  T* b = bearings + 3 * i;
  const T r = sqrt(b[0] * b[0] + b[1] * b[1] + b[2] * b[2]);
  b[0] /= r;
  b[1] /= r;
  b[2] /= r;
}
}  // namespace

// ---- the host ------------------------------------------------------------------------------------------------
// The first `want` outputs of mt19937(42) on the device and the generator after them, remade when `want` changes.
struct StreamPrefix {
  long long len = 0, want = RANSAC_DEFAULT_PREFIX;
  DevBuf<uint32_t> d_prefix;
  DevBuf<Mt> d_saved;

  void make(cudaStream_t stream) {
    if (len == want) return;
    auto mt = std::make_unique<Mt>();
    mt->seed(42u);
    std::vector<uint32_t> h((size_t)want);
    for (auto& v : h) v = mt->next();
    upload(d_prefix, h.data(), h.size(), stream);
    upload(d_saved, mt.get(), 1, stream);
    OSFM_CUDA(cudaStreamSynchronize(stream));
    len = want;
  }
};

// One of a problem's row index arrays, as RansacBatch::check sees it: row r names entry rows[r] of a table of `size`
// entries, called `noun` in the error message.
struct RowIndex {
  const int64_t* rows;
  const void* table;
  int64_t size;
  const char* noun;
};

// A batch of RANSAC problems on one engine's stream: the stream prefix, the problems' row layout on the device, the
// launch plan and the traces of the last run.  Problem p owns rows [start[p], start[p + 1]).
struct RansacBatch {
  StreamPrefix prefix;
  SmemOptIn smem_opt_in;
  int trace_cap = 0;
  long long done = 0;            // problems of the last run that completed, 0 after a failed or empty one
  int big = 0;                   // the problems above RANSAC_STAGE_ROWS rows, first in d_order
  int staged_rows = 0;           // the rows of the largest of the others
  long long num = 0;
  DevBuf<long long> d_start, d_rows[2], d_stream_used;
  DevBuf<int> d_order, d_best_rows, d_trace, d_trace_count;

  // The argument checks of a run, in order; every message starts with `what` and names a problem as `item`.  Row
  // r's index arrays are checked one after the other, row by row.  `outputs` is whether the caller's output arrays
  // are all non-null.
  void check(const std::string& what, const char* item, const char* row_noun, int min_rows, int64_t num_problems,
             const int64_t* start, double threshold, int iterations, std::initializer_list<RowIndex> index,
             bool outputs) {
    done = 0;
    bool sizes = num_problems >= 0 && num_problems <= INT_MAX;
    for (const RowIndex& x : index) sizes = sizes && x.size >= 0;
    if (!sizes) throw ArgError(what + ": bad sizes");
    if (iterations < 1) throw ArgError(what + ": iterations must be at least 1");
    if (!std::isfinite(threshold) || threshold <= 0.0) throw ArgError(what + ": threshold must be positive");
    if (!start) throw ArgError(what + ": null " + item + "_start");
    if (start[0] != 0) throw ArgError(what + ": " + item + "_start[0] must be 0");
    for (int64_t p = 0; p < num_problems; ++p) {
      const int64_t n = start[p + 1] - start[p];
      if (n < min_rows)
        throw ArgError(what + ": " + item + " " + std::to_string(p) + " has " + std::to_string(n) + " " + row_noun +
                       "; at least " + std::to_string(min_rows) + " are needed");
      if (n > INT_MAX) throw ArgError(what + ": " + item + " " + std::to_string(p) + " has more than 2^31 - 1 rows");
    }
    bool arrays = outputs;
    for (const RowIndex& x : index) arrays = arrays && x.rows && x.table;
    if (num_problems > 0 && !arrays) throw ArgError(what + ": null arrays");
    for (int64_t p = 0; p < num_problems; ++p)
      for (int64_t r = start[p]; r < start[p + 1]; ++r)
        for (const RowIndex& x : index)
          if (x.rows[r] < 0 || x.rows[r] >= x.size)
            throw ArgError(what + ": row " + std::to_string(r - start[p]) + " of " + item + " " + std::to_string(p) +
                           " names a " + x.noun + " outside [0, " + std::to_string(x.size) + ")");
  }

  // Largest problems first (a stable order); the problems too large for shared memory form their own launch.
  // Makes the stream prefix, uploads the row layout (one or two row index arrays) and reserves the workspaces.
  void plan(cudaStream_t stream, int64_t num_problems, const int64_t* start,
            std::initializer_list<const int64_t*> rows) {
    num = num_problems;
    prefix.make(stream);
    std::vector<int> order((size_t)num);
    std::iota(order.begin(), order.end(), 0);
    std::stable_sort(order.begin(), order.end(),
                     [&](int x, int y) { return start[x + 1] - start[x] > start[y + 1] - start[y]; });
    big = 0;
    while (big < num && start[order[big] + 1] - start[order[big]] > RANSAC_STAGE_ROWS) ++big;
    staged_rows = big < num ? (int)(start[order[big] + 1] - start[order[big]]) : 0;

    const size_t R = (size_t)start[num];
    upload(d_start, reinterpret_cast<const long long*>(start), (size_t)num + 1, stream);
    int k = 0;
    for (const int64_t* r : rows) upload(d_rows[k++], reinterpret_cast<const long long*>(r), R, stream);
    upload(d_order, order.data(), order.size(), stream);
    d_best_rows.reserve(R);
    if (trace_cap > 0) {
      d_trace.reserve((size_t)num * trace_cap);
      d_trace_count.reserve((size_t)num);
      d_stream_used.reserve((size_t)num);
    }
  }

  StreamSource source() const {
    return StreamSource{prefix.d_prefix.p, prefix.len,      prefix.d_saved.p,   trace_cap > 0 ? d_trace.p : nullptr,
                        trace_cap,         d_trace_count.p, d_stream_used.p};
  }

  // kernel(a, staged) over the plan: the large problems reading their rows through L2, then the others staged.
  template <class Args>
  void launch(void (*kernel)(Args, int), Args a, cudaStream_t stream) {
    if (big > 0) {
      a.order = d_order.p;
      kernel<<<big, RANSAC_THREADS, 0, stream>>>(a, 0);
      OSFM_LAUNCH_CHECK();
    }
    if (big < num) {
      smem_opt_in(kernel, (int)(sizeof(double) * 6 * RANSAC_STAGE_ROWS));
      a.order = d_order.p + big;
      kernel<<<(unsigned)(num - big), RANSAC_THREADS, sizeof(double) * 6 * (size_t)staged_rows, stream>>>(a, 1);
      OSFM_LAUNCH_CHECK();
    }
  }

  void set_stream_prefix(int64_t length) {
    if (length < 1 || length > (1LL << 28)) throw ArgError("stream prefix length must be in [1, 2^28]");
    prefix.want = length;
  }

  void set_trace(int capacity) {
    if (capacity < 0) throw ArgError("negative trace capacity");
    trace_cap = capacity;
  }

  // the traces of the last run: per problem, how many indices it drew, the generator outputs it used and the first
  // trace_cap indices
  void get_trace(cudaStream_t stream, const std::string& what, int32_t* count, int64_t* stream_used, int32_t* indices) {
    if (!done || trace_cap == 0) throw std::runtime_error(what + ": no traced run");
    if (!count || !stream_used || !indices) throw ArgError("null outputs");
    download(count, d_trace_count.p, (size_t)done, stream);
    download(reinterpret_cast<long long*>(stream_used), d_stream_used.p, (size_t)done, stream);
    download(indices, d_trace.p, (size_t)done * trace_cap, stream);
    OSFM_CUDA(cudaStreamSynchronize(stream));
  }
};

}  // namespace osfm
