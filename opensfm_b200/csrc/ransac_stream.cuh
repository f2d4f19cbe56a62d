// The sample stream of pyrobust's RANSAC (robust/random_sampler.h, robust_estimator.h), shared by the batched
// estimators (rotransac.cu, resect.cu, relpose.cu): a std::mt19937 seeded with 42 and restarted for every problem,
// indices drawn by libstdc++'s uniform_int_distribution, repeats in a sample drawn again, and the ShouldStop bound.
// The restatement these follow is oracle/rotation_ransac_oracle.py.
//
// Every problem consumes the same stream from its start, so a prefix of it is made once per handle and kept on the
// device (StreamPrefix); a problem that reaches its end continues from the generator state saved after the prefix,
// in its CTA's shared memory, so the stream stays exact.
#pragma once

#include <cfloat>
#include <cmath>
#include <cstdint>
#include <memory>
#include <vector>

#include "common.cuh"

namespace osfm {

constexpr double RANSAC_PROBABILITY = 0.99;   // RobustEstimatorParams::probability; the callers never set it
constexpr long long RANSAC_DEFAULT_PREFIX = 1LL << 16;

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

// Where a launch reads the stream from, and where it records the drawn indices (trace, trace_cap per problem).
struct StreamSource {
  const uint32_t* prefix;
  long long prefix_len;
  const Mt* saved;               // the generator after prefix_len outputs
  int* trace;                    // or null
  int trace_cap;
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

// ShouldStop with `minimal`-row samples: stop once log(1 - p) / log(min(1 - eps, 1 - ratio^minimal)) < iteration
__device__ inline bool ransac_should_stop(int best_inliers, int n, int iteration, int minimal = 3) {
  const double ratio = (double)best_inliers / n;
  const double p1 = fmin(1.0 - DBL_EPSILON, 1.0 - pow(ratio, (double)minimal));
  return log(1.0 - RANSAC_PROBABILITY) / log(p1) < (double)iteration;
}

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
  StreamSource source(int* trace, int trace_cap) const { return StreamSource{d_prefix.p, len, d_saved.p, trace, trace_cap}; }
};

}  // namespace osfm
