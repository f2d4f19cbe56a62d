// Per-image neighbour selection over a block of all-pairs distances, shared by the VLAD (vlad.cu) and BoW (bow.cu)
// pair selectors: construct_pairs / pairs_from_neighbors (opensfm/pairs_selection.py:471-490, 764-795).
#pragma once
#include <cub/cub.cuh>

#include <algorithm>
#include <vector>

#include "common.cuh"
#include "match_common.cuh"

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

// A kind of pair selection (VladRows in vlad.cu, BowRows in bow.cu) supplies its row type, its distance kernel's tile
// height, the lookup of a set's resident array (`of`) and the row in it, and its own device tables (BoW: the pairwise
// plan).  The calls come in this order: table_bytes(len) for rows of length len, upload() into the table, then
// distances(), which launches one block of distances.

// Host side of the selection: the rows of the listed sets, one device table, the reference rows in blocks (the
// distance block stays under 256 MB as a multiple of the tile height, and the distance grid's y dimension within
// 65535) of distances + neighbor_select_kernel, and the selected columns compacted into out_offsets / out_cols /
// out_dist.
// VLAD passes mask_bits, BoW passes order.
template <class Kind>
void select_neighbors(Matcher& M, Kind& kind, int nref, const int* ref_ids, int ncand, const int* cand_ids,
                      const uint32_t* mask_bits, const int32_t* order, const int* labels, int k, int64_t* out_offsets,
                      int32_t* out_cols, double* out_dist) {
  using Row = typename Kind::Row;
  if ((nref > 0 && (!ref_ids || !out_offsets)) || (ncand > 0 && !cand_ids)) throw ArgError("null arrays");
  if (nref == 0) return;
  out_offsets[0] = 0;
  const int ngroups = labels ? 2 : 1;
  const int stride = ngroups * std::min(k, ncand);
  if (ncand == 0 || stride == 0) {
    for (int r = 0; r < nref; ++r) out_offsets[r + 1] = 0;
    return;
  }
  if (!out_cols || !out_dist) throw ArgError("null output arrays");
  const size_t nrows = (size_t)nref + ncand;
  std::vector<int> ids(nrows);
  std::copy(ref_ids, ref_ids + nref, ids.begin());
  std::copy(cand_ids, cand_ids + ncand, ids.begin() + nref);
  int L = -1;
  std::vector<const Row*> rows(nrows);
  for (size_t i = 0; i < nrows; ++i) {
    const auto& a = Kind::of(M, ids[i], L);
    L = a.len;
    rows[i] = Kind::row(a);
  }
  const int mask_words = (ncand + 31) / 32;
  const size_t mask_bytes = mask_bits ? sizeof(uint32_t) * (size_t)nref * mask_words : 0;
  const size_t order_bytes = order ? sizeof(int) * (size_t)nref * ncand : 0;
  // device table: row pointers | ids | labels | mask | order | the kind's tables | counts | columns | distances
  TableLayout t;
  t.add(sizeof(Row*) * nrows);
  const size_t o_ids = t.add(sizeof(int) * nrows);
  const size_t o_lab = t.add(labels ? sizeof(int) * nrows : 0);
  const size_t o_mask = t.add(mask_bytes), o_ord = t.add(order_bytes), o_kind = t.add(kind.table_bytes(L));
  const size_t o_cnt = t.add(sizeof(int) * (size_t)nref);
  const size_t o_cols = t.add(sizeof(int) * (size_t)nref * stride);
  const size_t o_dist = t.add(sizeof(double) * (size_t)nref * stride);
  M.d_tab.reserve(t.size);
  uint8_t* base = M.d_tab.p;
  auto upload = [&](size_t off, const void* src, size_t bytes) {
    if (src) OSFM_CUDA(cudaMemcpyAsync(base + off, src, bytes, cudaMemcpyHostToDevice, M.stream));
  };
  upload(0, rows.data(), sizeof(Row*) * nrows);
  upload(o_ids, ids.data(), sizeof(int) * nrows);
  upload(o_lab, labels, sizeof(int) * nrows);
  upload(o_mask, mask_bits, mask_bytes);
  upload(o_ord, order, order_bytes);
  kind.upload(M, base + o_kind);
  const Row* const* d_rows = reinterpret_cast<const Row* const*>(base);
  const int* d_ids = reinterpret_cast<const int*>(base + o_ids);
  int* d_cnt = reinterpret_cast<int*>(base + o_cnt);
  int* d_cols = reinterpret_cast<int*>(base + o_cols);
  double* d_dist = reinterpret_cast<double*>(base + o_dist);
  const long long budget = (256ll << 20) / (long long)(sizeof(double) * ncand);
  const long long cap = std::min<long long>(budget / Kind::TILE_M * Kind::TILE_M, 65535ll * Kind::TILE_M);
  const int block = (int)std::max<long long>(Kind::TILE_M, std::min<long long>(nref, cap));
  M.d_dist.reserve((size_t)block * ncand);
  for (int r0 = 0; r0 < nref; r0 += block) {
    const int nb = std::min(block, nref - r0);
    kind.distances(M, base + o_kind, d_rows + r0, nb, d_rows + nref, ncand, L, M.d_dist.p, ncand);
    neighbor_select_kernel<<<nb, VS_THREADS, 0, M.stream>>>(
        M.d_dist.p, ncand, r0, nref, d_ids, d_ids + nref,
        mask_bits ? reinterpret_cast<const uint32_t*>(base + o_mask) : nullptr, mask_words,
        order ? reinterpret_cast<const int*>(base + o_ord) : nullptr,
        labels ? reinterpret_cast<const int*>(base + o_lab) : nullptr, k, stride, d_cnt, d_cols, d_dist);
    OSFM_LAUNCH_CHECK();
  }
  std::vector<int> cnt(nref);
  std::vector<int> cols((size_t)nref * stride);
  std::vector<double> dist((size_t)nref * stride);
  OSFM_CUDA(cudaMemcpyAsync(cnt.data(), d_cnt, sizeof(int) * nref, cudaMemcpyDeviceToHost, M.stream));
  OSFM_CUDA(cudaMemcpyAsync(cols.data(), d_cols, sizeof(int) * cols.size(), cudaMemcpyDeviceToHost, M.stream));
  OSFM_CUDA(cudaMemcpyAsync(dist.data(), d_dist, sizeof(double) * dist.size(), cudaMemcpyDeviceToHost, M.stream));
  OSFM_CUDA(cudaStreamSynchronize(M.stream));
  int64_t o = 0;
  for (int r = 0; r < nref; ++r) {
    std::copy(cols.begin() + (size_t)r * stride, cols.begin() + (size_t)r * stride + cnt[r], out_cols + o);
    std::copy(dist.begin() + (size_t)r * stride, dist.begin() + (size_t)r * stride + cnt[r], out_dist + o);
    o += cnt[r];
    out_offsets[r + 1] = o;
  }
}

// The distances of host row `query` to all n host rows of len elements (osfm_vlad_distances, osfm_bow_distances):
// the rows, their pointers and the kind's tables go to the staging buffer, one 1 x n block runs.
template <class Kind>
void distances_to_row(Matcher& M, Kind& kind, const typename Kind::Row* host, int n, int len, int query, double* out_n) {
  using Row = typename Kind::Row;
  TableLayout t;
  t.add(sizeof(Row) * (size_t)n * len);
  const size_t o_ptr = t.add(sizeof(Row*) * (size_t)n), o_out = t.add(sizeof(double) * (size_t)n);
  const size_t o_kind = t.add(kind.table_bytes(len));
  M.staging.reserve(t.size);
  Row* d_v = reinterpret_cast<Row*>(M.staging.p);
  const Row** d_p = reinterpret_cast<const Row**>(M.staging.p + o_ptr);
  double* d_out = reinterpret_cast<double*>(M.staging.p + o_out);
  std::vector<const Row*> rows(n);
  for (int i = 0; i < n; ++i) rows[i] = d_v + (size_t)i * len;
  OSFM_CUDA(cudaMemcpyAsync(d_v, host, sizeof(Row) * (size_t)n * len, cudaMemcpyHostToDevice, M.stream));
  OSFM_CUDA(cudaMemcpyAsync(d_p, rows.data(), sizeof(Row*) * (size_t)n, cudaMemcpyHostToDevice, M.stream));
  kind.upload(M, M.staging.p + o_kind);
  kind.distances(M, M.staging.p + o_kind, d_p + query, 1, d_p, n, len, d_out, n);
  OSFM_CUDA(cudaMemcpyAsync(out_n, d_out, sizeof(double) * (size_t)n, cudaMemcpyDeviceToHost, M.stream));
  OSFM_CUDA(cudaStreamSynchronize(M.stream));
}

}  // namespace
}  // namespace osfm
