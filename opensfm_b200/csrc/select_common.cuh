// Per-image neighbour selection over a block of all-pairs distances, shared by the VLAD (vlad.cu) and BoW (bow.cu)
// pair selectors: construct_pairs / pairs_from_neighbors (opensfm/pairs_selection.py:471-490, 764-795).
#pragma once
#include <cub/cub.cuh>

#include "common.cuh"

namespace osfm {
namespace {

constexpr int VS_THREADS = 256;          // selection: one CTA per reference row

// Order-preserving key of a distance: ascending for numbers, every NaN after them (np.argsort's order).
__device__ __forceinline__ unsigned long long dist_key(double d) {
  if (isnan(d)) return ~0ull;
  const unsigned long long b = (unsigned long long)__double_as_longlong(d);
  return (b >> 63) ? ~b : (b | (1ull << 63));
}

// One CTA per reference row of the block: the k smallest eligible candidates by (distance, column) -- the order a
// stable argsort over the candidate list gives -- per camera group.  With camera labels there are two groups, the
// candidates of the reference's camera and the others (pairs_from_neighbors), otherwise one.
// order: NULL, or nref x ncand ints: the position of candidate j in reference r's own candidate list (-1: not in
// it), which then replaces the column as the tie-break and decides eligibility with the mask.
// Selection: radix select of the k-th key over eight 8-bit digits; without `order`, one pass in column order that
// keeps every key below it and the first `need` keys equal to it; with `order`, a second radix select over the
// positions of the keys equal to it.  Output: the selected columns in ascending order.
__global__ void __launch_bounds__(VS_THREADS)
    neighbor_select_kernel(const double* __restrict__ dist, int ncand, int row0, int nref, const int* __restrict__ ref_ids,
                           const int* __restrict__ cand_ids, const uint32_t* __restrict__ mask, int mask_words,
                           const int* __restrict__ order, const int* __restrict__ labels, int k, int stride,
                           int* __restrict__ out_count, int* __restrict__ out_cols, double* __restrict__ out_dist) {
  using Scan = cub::BlockScan<int, VS_THREADS>;
  __shared__ typename Scan::TempStorage scan_tmp;
  __shared__ int hist[256];
  __shared__ unsigned long long s_prefix;
  __shared__ int s_need;
  const int row = row0 + blockIdx.x;
  const double* d = dist + (size_t)blockIdx.x * ncand;
  const int* pos = order ? order + (size_t)row * ncand : nullptr;
  const int self = ref_ids[row];
  const int ngroups = labels ? 2 : 1;
  const size_t base = (size_t)row * stride;
  // the want-th smallest of key(j) over the columns j with in(j), digits top .. 0: the key -> s_prefix, how many
  // keys equal to it to keep -> s_need
  auto radix_select = [&](auto in, auto key, int top, int want) {
    __syncthreads();   // every thread has read the previous result
    if (threadIdx.x == 0) { s_prefix = 0ull; s_need = want; }
    for (int shift = top; shift >= 0; shift -= 8) {
      for (int b = threadIdx.x; b < 256; b += VS_THREADS) hist[b] = 0;
      __syncthreads();
      const unsigned long long prefix = s_prefix;
      const unsigned long long hi = shift == top ? 0ull : (~0ull << (shift + 8));
      for (int j = threadIdx.x; j < ncand; j += VS_THREADS) {
        if (!in(j)) continue;
        const unsigned long long kj = key(j);
        if ((kj & hi) == (prefix & hi)) atomicAdd(&hist[(kj >> shift) & 255], 1);
      }
      __syncthreads();
      if (threadIdx.x == 0) {
        int cum = 0, w = s_need, b = 0;
        for (; b < 255 && cum + hist[b] < w; ++b) cum += hist[b];
        s_need = w - cum;
        s_prefix = prefix | ((unsigned long long)b << shift);
      }
      __syncthreads();
    }
  };
  int written = 0;
  for (int g = 0; g < ngroups; ++g) {
    auto eligible = [&](int j) {
      if (cand_ids[j] == self) return false;
      if (mask && !((mask[(size_t)row * mask_words + (j >> 5)] >> (j & 31)) & 1u)) return false;
      if (pos && pos[j] < 0) return false;
      if (labels && ((labels[nref + j] == labels[row]) != (g == 0))) return false;
      return true;
    };
    auto key = [&](int j) { return dist_key(d[j]); };
    int cnt = 0;
    for (int j = threadIdx.x; j < ncand; j += VS_THREADS) cnt += eligible(j);
    int total_elig;
    Scan(scan_tmp).ExclusiveSum(cnt, cnt, total_elig);
    __syncthreads();
    const bool take_all = total_elig <= k;
    unsigned long long thr = ~0ull;
    int need = 0;
    unsigned long long pthr = 0ull;   // with `order`: the last position kept among the keys equal to thr
    if (!take_all) {
      radix_select(eligible, key, 56, k);
      thr = s_prefix;
      need = s_need;   // keys equal to thr to keep, lowest columns (or positions) first
      if (pos) {
        radix_select([&](int j) { return eligible(j) && key(j) == thr; },
                     [&](int j) { return (unsigned long long)(unsigned)pos[j]; }, 24, need);
        pthr = s_prefix;   // positions are distinct: exactly `need` of them are <= pthr
      }
    }
    int eq_before = 0;
    for (int j0 = 0; j0 < ncand; j0 += VS_THREADS) {
      const int j = j0 + threadIdx.x;
      bool lt = false, eq = false;
      double dj = 0.0;
      if (j < ncand && eligible(j)) {
        dj = d[j];
        if (take_all) lt = true;
        else {
          const unsigned long long kj = dist_key(dj);
          lt = kj < thr;
          eq = kj == thr;
        }
      }
      bool take;
      if (pos) {
        take = lt || (eq && (unsigned long long)(unsigned)pos[j] <= pthr);
      } else {
        int eq_rank, eq_total;
        Scan(scan_tmp).ExclusiveSum((int)eq, eq_rank, eq_total);
        __syncthreads();
        take = lt || (eq && eq_before + eq_rank < need);
        eq_before += eq_total;
      }
      int p, ntake;
      Scan(scan_tmp).ExclusiveSum((int)take, p, ntake);
      __syncthreads();
      if (take) {
        out_cols[base + written + p] = j;
        out_dist[base + written + p] = dj;
      }
      written += ntake;
    }
  }
  if (threadIdx.x == 0) out_count[row] = written;
}

}  // namespace
}  // namespace osfm
