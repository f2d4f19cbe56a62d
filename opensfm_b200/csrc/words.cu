// WORDS matcher on the device (SURVEY.md §8f.3); the VLAD kernels are in vlad.cu.
//
// Replaces features::match_using_words (opensfm/src/features/src/matching.cc:24-88, bound as
// pyfeatures.match_using_words, called by opensfm/matching.py:636-656).
//
// match_using_words: the features of image 2 are indexed by their nearest visual word (a multimap word ->
// feature, equal words in insertion order); every feature i of image 1 walks its k nearest words, scores the
// features of image 2 filed under each word with the L2 distance (float32, summed in dimension order, sqrt),
// keeps the best and the second best distance (strict `<`: the first of equal candidates wins), stops after the
// word during which `max_checks` candidates have been scored, and is matched when
// best < lowes_ratio * second (float32; a single candidate passes because second = +inf).
// Here the index is a CSR built on the host by a stable counting sort (same candidate order as the multimap),
// and one thread walks the candidates of one feature with the same sequence of float32 operations (separate
// multiply and add, no FMA contraction, like the reference's x86-64 baseline build).
#include <algorithm>
#include <vector>

#include "common.cuh"
#include "match_common.cuh"

namespace osfm {

__global__ void __launch_bounds__(128)
    words_match_kernel(const float* __restrict__ f1, int n1, const int* __restrict__ w1, int k, const float* __restrict__ f2,
                       const int* __restrict__ wstart, const int* __restrict__ worder, int nwords, int dim, float ratio,
                       int max_checks, int* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n1) return;
  const float* pa = f1 + (size_t)i * dim;
  float best = __builtin_huge_valf(), second = __builtin_huge_valf();
  int best_match = -1, checks = 0;
  for (int j = 0; j < k; ++j) {
    const int word = w1[(size_t)i * k + j];
    if (word >= 0 && word < nwords) {
      for (int c = wstart[word]; c < wstart[word + 1]; ++c) {
        const int match = worder[c];
        const float* pb = f2 + (size_t)match * dim;
        float d = 0.f;
        for (int e = 0; e < dim; ++e) {
          const float t = __fsub_rn(pa[e], pb[e]);
          d = __fadd_rn(d, __fmul_rn(t, t));
        }
        d = __fsqrt_rn(d);
        if (d < best) { second = best; best = d; best_match = match; }
        else if (d < second) second = d;
        ++checks;
      }
    }
    if (checks >= max_checks) break;
  }
  out[i] = (best < __fmul_rn(ratio, second)) ? best_match : -1;
}

}  // namespace osfm

extern "C" {

int osfm_match_words(osfm_matcher* m, const float* f1, int n1, const int32_t* words1, int words_per_feature,
                     const float* f2, int n2, const int32_t* words2, int dim, float lowes_ratio, int max_checks,
                     int32_t* out_match) {
  return osfm::with_handle(m, [&](osfm::Matcher& M) {
    if (n1 < 0 || n2 < 0 || dim <= 0 || words_per_feature <= 0) throw osfm::ArgError("bad sizes");
    if ((n1 > 0 && (!f1 || !words1 || !out_match)) || (n2 > 0 && (!f2 || !words2))) throw osfm::ArgError("null arrays");
    if (n1 == 0) return;
    // CSR of image 2's features by word: stable counting sort = the multimap's order among equal words
    int nwords = 0;
    for (int i = 0; i < n2; ++i) nwords = std::max(nwords, words2[i] + 1);
    std::vector<int> start((size_t)nwords + 1, 0), order((size_t)std::max(n2, 1));
    for (int i = 0; i < n2; ++i) if (words2[i] >= 0) ++start[words2[i] + 1];
    for (int w = 0; w < nwords; ++w) start[w + 1] += start[w];
    {
      std::vector<int> fill(start.begin(), start.end() - 1);
      for (int i = 0; i < n2; ++i) if (words2[i] >= 0) order[fill[words2[i]]++] = i;
    }
    const size_t b_f1 = sizeof(float) * (size_t)n1 * dim, b_f2 = sizeof(float) * (size_t)std::max(n2, 1) * dim;
    const size_t b_w1 = sizeof(int) * (size_t)n1 * words_per_feature;
    osfm::TableLayout tab;
    tab.add(b_f1);
    const size_t o_f2 = tab.add(b_f2), o_w1 = tab.add(b_w1), o_st = tab.add(sizeof(int) * start.size());
    const size_t o_or = tab.add(sizeof(int) * order.size()), o_out = tab.add(sizeof(int) * (size_t)n1);
    M.staging.reserve(tab.size);
    uint8_t* base = M.staging.p;
    OSFM_CUDA(cudaMemcpyAsync(base, f1, b_f1, cudaMemcpyHostToDevice, M.stream));
    if (n2 > 0) OSFM_CUDA(cudaMemcpyAsync(base + o_f2, f2, sizeof(float) * (size_t)n2 * dim, cudaMemcpyHostToDevice, M.stream));
    OSFM_CUDA(cudaMemcpyAsync(base + o_w1, words1, b_w1, cudaMemcpyHostToDevice, M.stream));
    OSFM_CUDA(cudaMemcpyAsync(base + o_st, start.data(), sizeof(int) * start.size(), cudaMemcpyHostToDevice, M.stream));
    OSFM_CUDA(cudaMemcpyAsync(base + o_or, order.data(), sizeof(int) * order.size(), cudaMemcpyHostToDevice, M.stream));
    osfm::words_match_kernel<<<(n1 + 127) / 128, 128, 0, M.stream>>>(
        reinterpret_cast<const float*>(base), n1, reinterpret_cast<const int*>(base + o_w1), words_per_feature,
        reinterpret_cast<const float*>(base + o_f2), reinterpret_cast<const int*>(base + o_st),
        reinterpret_cast<const int*>(base + o_or), nwords, dim, lowes_ratio, max_checks, reinterpret_cast<int*>(base + o_out));
    OSFM_LAUNCH_CHECK();
    OSFM_CUDA(cudaMemcpyAsync(out_match, base + o_out, sizeof(int) * (size_t)n1, cudaMemcpyDeviceToHost, M.stream));
    OSFM_CUDA(cudaStreamSynchronize(M.stream));   // start / order go out of scope
  });
}

}  // extern "C"
