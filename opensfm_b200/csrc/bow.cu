// Bag-of-words pair selection on the device (SURVEY.md §8f.3): visual words of resident descriptor sets, their
// weighted word histograms, all-pairs L1 distances and the per-image neighbour selection of
// pairs_selection.match_candidates_with_bow.
//
// Replaces bow.BagOfWords.map_to_words (opensfm/bow.py; cv2 BruteForce knnMatch against the vocabulary),
// BagOfWords.histogram, pairs_selection.bow_distances (pairs_selection.py:690-708) and construct_pairs /
// pairs_from_neighbors (pairs_selection.py:471-490, 764-795).
//
// Words: the k nearest vocabulary words of every row in cv2's ranking -- sqrt of the float32 squared distance
// summed in cv2's order (cv_tile_d2, match_common.cuh), ties to the lower word index -- so the indices are the ones
// knnMatch returns, in the same order.
// Histograms and distances: float64 arithmetic in the order numpy runs it.  h = bincount * weights (one rounded
// multiply per word), h / h.sum(), and np.fabs(h - h2).sum(), where every sum follows numpy's pairwise summation
// of a contiguous vector: leaves of at most 128 elements, each summed by 8 stride-8 accumulators combined as
// ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)) plus its n % 8 tail in order, and the leaves combined by the split tree
// n2 = n/2 - (n/2) % 8.  The host writes that order down once per length (pairwise_plan) and the kernels follow it,
// so histograms and distances are the reference's bit for bit.
#include <cfloat>
#include <cmath>
#include <vector>

#include "common.cuh"
#include "match_common.cuh"
#include "select_common.cuh"

namespace osfm {

namespace {

constexpr int BW_TS = 64;               // word assignment: queries per CTA and words per tile (4 x 4 per thread)
constexpr int BW_LD = BW_TS + 4;        // floats per element row of a shared tile
constexpr int BW_KEY_LD = BW_TS + 1;    // floats per query row of the distance-key tile
constexpr int BW_KMAX = 64;             // longest word list per row
constexpr int BW_MAX_D = 320;           // padded floats per row: 2 x 320 x 68 x 4 B + the lists fit in shared memory
constexpr int PW_LEAF = 128;            // numpy's pairwise-summation block
constexpr int BD_TM = 16, BD_TN = 32;   // distance tile: reference rows x candidate rows, 1 x 2 per thread
constexpr int BOW_MAX_DEPTH = 32;       // partial sums of the pairwise tree alive at once (~log2(n / 64) + 1)
constexpr size_t BOW_BATCH_BYTES = (size_t)256 << 20;   // per-chunk lists + words of one batch of sets

struct BowJob {
  const float* f;    // the set's zero-padded float32 rows, D floats each
  int* first;        // resident nearest word of every row
  long long row0;    // first row of the set in the batch
  int n;
};

struct HistJob {
  const int* words;  // nearest word of every row
  double* h;         // the histogram, nwords doubles
  int n;
};

// (key, index) before (key', index'): the order of cv2's stable insertion; index -1 (empty) is last
__device__ __forceinline__ bool kv_less(float s, unsigned i, float s2, unsigned i2) {
  return s < s2 || (s == s2 && i < i2);
}

// One CTA per (64 rows of a set, chunk of the vocabulary): the k nearest words of the chunk for each row.
// Per 64 x 64 tile: cv2-order distances (cv_tile_d2), their float32 square roots into shared memory, then warp w
// updates the sorted lists of rows 8w .. 8w+7: a row's candidates that beat its k-th entry (after the first few
// hundred words almost none) are inserted one at a time, in word order, by a warp-wide shift.
// Lists: 64 entries per row in shared memory, lane l holding positions l and l + 32 while it inserts.
// Output: each row's sorted list of the chunk, k (key, word) entries, word -1 where the chunk has fewer than k.
// flags |= 1 when a row has a non-finite element.
__global__ void __launch_bounds__(256)
    bow_words_kernel(const BowJob* __restrict__ jobs, const int* __restrict__ tile_prefix, int njobs,
                     const float* __restrict__ vocab, int nwords, int D, int nblk, int k, int nchunks, int chunk_len,
                     float* __restrict__ pkey, int* __restrict__ pidx, int* __restrict__ flags) {
  extern __shared__ __align__(16) float bw_smem[];
  int lo = 0, hi = njobs - 1;
  const int cta = blockIdx.x;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (tile_prefix[mid] <= cta) lo = mid; else hi = mid - 1;
  }
  const BowJob job = jobs[lo];
  const int local = cta - tile_prefix[lo];
  const int qtile = local / nchunks, chunk = local % nchunks;
  const int q0 = qtile * BW_TS;
  const int t_begin = chunk * chunk_len, t_end = min(nwords, t_begin + chunk_len);
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15, lane = tid & 31, warp = tid >> 5;
  float* As = bw_smem;
  float* Bs = As + (size_t)D * BW_LD;                                   // vocabulary tile, then the key tile
  float* lkey = Bs + max(D * BW_LD, BW_TS * BW_KEY_LD);
  int* lidx = reinterpret_cast<int*>(lkey + BW_TS * BW_KMAX);

  cv_load_tile<BW_TS, BW_LD>(As, job.f, q0, job.n, D);
  for (int e = tid; e < BW_TS * BW_KMAX; e += 256) { lkey[e] = __builtin_huge_valf(); lidx[e] = -1; }
  __syncthreads();
  if (chunk == 0) {
    bool finite = true;
    for (int e = tid; e < D * BW_TS; e += 256) finite &= isfinite(As[(e / BW_TS) * BW_LD + e % BW_TS]);
    if (!finite) atomicOr(flags, 1);
  }
  constexpr unsigned FULL = 0xffffffffu;
  for (int t0 = t_begin; t0 < t_end; t0 += BW_TS) {
    __syncthreads();   // the previous key tile has been read
    cv_load_tile<BW_TS, BW_LD>(Bs, vocab, t0, t_end, D);
    __syncthreads();
    float d2[4][4];
    cv_tile_d2<4, BW_LD>(As, Bs, D, nblk, ty, tx, d2);
    __syncthreads();   // the vocabulary tile has been read: its space takes the keys
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) Bs[(ty * 4 + i) * BW_KEY_LD + tx * 4 + j] = __fsqrt_rn(d2[i][j]);
    __syncthreads();
    for (int qq = 0; qq < BW_TS / 8; ++qq) {
      const int q = warp * (BW_TS / 8) + qq;
      if (q0 + q >= job.n) break;
      float* lk = lkey + q * BW_KMAX;
      int* li = lidx + q * BW_KMAX;
      const float s0 = Bs[q * BW_KEY_LD + lane], s1 = Bs[q * BW_KEY_LD + lane + 32];
      const unsigned w0 = t0 + lane, w1 = t0 + lane + 32;
      const float ks = lk[k - 1];
      const unsigned ki = (unsigned)li[k - 1];
      unsigned m0 = __ballot_sync(FULL, (int)w0 < t_end && kv_less(s0, w0, ks, ki));
      unsigned m1 = __ballot_sync(FULL, (int)w1 < t_end && kv_less(s1, w1, ks, ki));
      if ((m0 | m1) == 0) continue;
      float e0k = lk[lane], e1k = lk[lane + 32];
      unsigned e0i = (unsigned)li[lane], e1i = (unsigned)li[lane + 32];
      while (m0 | m1) {
        float s;
        unsigned wi;
        if (m0) {
          const int src = __ffs(m0) - 1;
          m0 &= m0 - 1;
          s = __shfl_sync(FULL, s0, src);
          wi = t0 + src;
        } else {
          const int src = __ffs(m1) - 1;
          m1 &= m1 - 1;
          s = __shfl_sync(FULL, s1, src);
          wi = t0 + 32 + src;
        }
        const int p = __popc(__ballot_sync(FULL, kv_less(e0k, e0i, s, wi))) +
                      __popc(__ballot_sync(FULL, kv_less(e1k, e1i, s, wi)));
        if (p >= k) continue;   // no longer among the k nearest after the candidates inserted before it
        const float u0k = __shfl_up_sync(FULL, e0k, 1), u1k = __shfl_up_sync(FULL, e1k, 1);
        const unsigned u0i = __shfl_up_sync(FULL, e0i, 1), u1i = __shfl_up_sync(FULL, e1i, 1);
        const float l0k = __shfl_sync(FULL, e0k, 31);
        const unsigned l0i = __shfl_sync(FULL, e0i, 31);
        if (lane + 32 == p) { e1k = s; e1i = wi; }
        else if (lane + 32 > p) { e1k = lane ? u1k : l0k; e1i = lane ? u1i : l0i; }
        if (lane == p) { e0k = s; e0i = wi; }
        else if (lane > p) { e0k = u0k; e0i = u0i; }
      }
      lk[lane] = e0k;
      lk[lane + 32] = e1k;
      li[lane] = (int)e0i;
      li[lane + 32] = (int)e1i;
      __syncwarp();
    }
  }
  __syncthreads();
  for (int e = tid; e < BW_TS * k; e += 256) {
    const int q = e / k, p = e % k;
    if (q0 + q >= job.n) continue;
    const size_t o = ((size_t)(job.row0 + q0 + q) * nchunks + chunk) * k + p;
    pkey[o] = lkey[q * BW_KMAX + p];
    pidx[o] = lidx[q * BW_KMAX + p];
  }
}

// Merge the chunk lists of every row (grid = (entries / 256, jobs)): one thread per list entry, whose rank in the
// row is its position in its own list plus the entries of the other lists before it (binary search; (key, word)
// pairs are distinct).  Ranks below kout go to words[row][rank]; rank 0 is also the set's resident first word.
__global__ void bow_merge_kernel(const BowJob* __restrict__ jobs, const float* __restrict__ pkey,
                                 const int* __restrict__ pidx, int nchunks, int k, int kout, int* __restrict__ words) {
  const BowJob job = jobs[blockIdx.y];
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long long)job.n * nchunks * k) return;
  const long long row = e / ((long long)nchunks * k);
  const int c = (int)(e / k % nchunks), p = (int)(e % k);
  const size_t base = (size_t)(job.row0 + row) * nchunks * k;
  const float s = pkey[base + (size_t)c * k + p];
  const int w = pidx[base + (size_t)c * k + p];
  if (w < 0) return;
  int rank = p;
  for (int c2 = 0; c2 < nchunks; ++c2) {
    if (c2 == c) continue;
    const float* ck = pkey + base + (size_t)c2 * k;
    const int* ci = pidx + base + (size_t)c2 * k;
    int a = 0, b = k;   // entries of list c2 before (s, w)
    while (a < b) {
      const int mid = (a + b) >> 1;
      if (kv_less(ck[mid], (unsigned)ci[mid], s, (unsigned)w)) a = mid + 1; else b = mid;
    }
    rank += a;
  }
  if (rank >= kout) return;
  words[(size_t)(job.row0 + row) * kout + rank] = w;
  if (rank == 0) job.first[row] = w;
}

// numpy's pairwise sum of the leaf x(0 .. len-1) for NO vectors at once: x(e, o) is element e of vector o
template <int NO, class F>
__device__ __forceinline__ void pairwise_leaf(F x, int len, double (&res)[NO]) {
  if (len < 8) {
#pragma unroll
    for (int o = 0; o < NO; ++o) res[o] = 0.0;
    for (int e = 0; e < len; ++e)
#pragma unroll
      for (int o = 0; o < NO; ++o) res[o] = __dadd_rn(res[o], x(e, o));
    return;
  }
  double r[NO][8];
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int o = 0; o < NO; ++o) r[o][j] = x(j, o);
  int i = 8;
  for (; i < len - len % 8; i += 8)
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int o = 0; o < NO; ++o) r[o][j] = __dadd_rn(r[o][j], x(i + j, o));
#pragma unroll
  for (int o = 0; o < NO; ++o)
    res[o] = __dadd_rn(__dadd_rn(__dadd_rn(r[o][0], r[o][1]), __dadd_rn(r[o][2], r[o][3])),
                       __dadd_rn(__dadd_rn(r[o][4], r[o][5]), __dadd_rn(r[o][6], r[o][7])));
  for (; i < len; ++i)
#pragma unroll
    for (int o = 0; o < NO; ++o) res[o] = __dadd_rn(res[o], x(i, o));
}

// One CTA per set: word counts (exact in float64 whatever the order of the atomics), h = count * weight,
// the pairwise sum (leaf sums in parallel, the tree by one thread), h / sum.
__global__ void __launch_bounds__(256)
    bow_histogram_kernel(const HistJob* __restrict__ jobs, const double* __restrict__ weights, int nwords,
                         const int2* __restrict__ leaves, int nleaves, const int* __restrict__ prog, int nprog) {
  extern __shared__ double leaf_sum[];
  __shared__ double s_total;
  const HistJob job = jobs[blockIdx.x];
  double* h = job.h;
  for (int i = threadIdx.x; i < nwords; i += blockDim.x) h[i] = 0.0;
  __syncthreads();
  for (int i = threadIdx.x; i < job.n; i += blockDim.x) atomicAdd(h + job.words[i], 1.0);
  __syncthreads();
  for (int i = threadIdx.x; i < nwords; i += blockDim.x) h[i] = __dmul_rn(h[i], weights[i]);
  __syncthreads();
  for (int l = threadIdx.x; l < nleaves; l += blockDim.x) {
    const int2 lf = leaves[l];
    double r[1];
    pairwise_leaf<1>([&](int e, int) { return h[lf.x + e]; }, lf.y, r);
    leaf_sum[l] = r[0];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double st[BOW_MAX_DEPTH];
    int sp = 0;
    for (int t = 0; t < nprog; ++t) {
      if (prog[t] >= 0) st[sp++] = leaf_sum[prog[t]];
      else { st[sp - 2] = __dadd_rn(st[sp - 2], st[sp - 1]); --sp; }
    }
    s_total = st[0];
  }
  __syncthreads();
  const double total = s_total;
  for (int i = threadIdx.x; i < nwords; i += blockDim.x) h[i] = __ddiv_rn(h[i], total);
}

// out[i * ldo + j] = sum_e |a_i[e] - b_j[e]| in numpy's pairwise order (|x - y| is symmetric, so d(a, b) == d(b, a)
// bit for bit).  CTA tile BD_TM x BD_TN, each thread one reference row x two candidate rows.  The plan's leaves are
// staged through shared memory one at a time; each output's pending partial sums of the tree live in a shared
// stack (depth entries per output), pushed by a leaf and combined by an add, uniformly across the CTA.
__global__ void __launch_bounds__(256)
    bow_distance_kernel(const double* const* __restrict__ arows, int na, const double* const* __restrict__ brows,
                        int nb, const int2* __restrict__ leaves, const int* __restrict__ prog, int nprog,
                        double* __restrict__ out, long long ldo) {
  extern __shared__ double bd_smem[];
  double* As = bd_smem;                     // [PW_LEAF][BD_TM]
  double* Bs = As + PW_LEAF * BD_TM;        // [PW_LEAF][BD_TN]
  double* st = Bs + PW_LEAF * BD_TN;        // [depth][256][2]
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const int a0 = blockIdx.y * BD_TM, b0 = blockIdx.x * BD_TN;
  int sp = 0;
  for (int t = 0; t < nprog; ++t) {
    const int op = prog[t];
    if (op < 0) {
#pragma unroll
      for (int o = 0; o < 2; ++o) {
        double* lo = st + ((size_t)(sp - 2) * 256 + tid) * 2 + o;
        *lo = __dadd_rn(*lo, lo[512]);
      }
      --sp;
      continue;
    }
    const int2 lf = leaves[op];
    __syncthreads();   // the previous leaf has been read
    for (int idx = tid; idx < BD_TM * lf.y; idx += 256) {
      const int r = idx / lf.y, e = idx % lf.y;
      As[e * BD_TM + r] = a0 + r < na ? __ldg(arows[a0 + r] + lf.x + e) : 0.0;
    }
    for (int idx = tid; idx < BD_TN * lf.y; idx += 256) {
      const int r = idx / lf.y, e = idx % lf.y;
      Bs[e * BD_TN + r] = b0 + r < nb ? __ldg(brows[b0 + r] + lf.x + e) : 0.0;
    }
    __syncthreads();
    double r[2];
    pairwise_leaf<2>([&](int e, int o) { return fabs(__dsub_rn(As[e * BD_TM + ty], Bs[e * BD_TN + tx + 16 * o])); },
                     lf.y, r);
    st[((size_t)sp * 256 + tid) * 2 + 0] = r[0];
    st[((size_t)sp * 256 + tid) * 2 + 1] = r[1];
    ++sp;
  }
#pragma unroll
  for (int o = 0; o < 2; ++o) {
    const int ia = a0 + ty, jb = b0 + tx + 16 * o;
    if (ia < na && jb < nb) out[(size_t)ia * ldo + jb] = st[tid * 2 + o];
  }
}

// numpy's pairwise order for a vector of length n: leaves (start, length) left to right and the post-order program
// (i >= 0: push leaf i's sum, -1: add the two partial sums on top); depth = most partial sums alive at once.
// On the device: leaves | program, `bytes` in all.
struct PairwisePlan {
  std::vector<int2> leaves;
  std::vector<int> prog;
  int depth = 0;
  size_t o_prog = 0, bytes = 0;
};

PairwisePlan pairwise_plan(long long n) {
  PairwisePlan P;
  int sp = 0;
  auto rec = [&](auto&& self, long long start, long long m) -> void {
    if (m <= PW_LEAF) {
      P.prog.push_back((int)P.leaves.size());
      P.leaves.push_back(make_int2((int)start, (int)m));
      P.depth = std::max(P.depth, ++sp);
      return;
    }
    long long m2 = m / 2;
    m2 -= m2 % 8;
    self(self, start, m2);
    self(self, start + m2, m - m2);
    P.prog.push_back(-1);
    --sp;
  };
  rec(rec, 0, n);
  if (P.depth > BOW_MAX_DEPTH) throw ArgError("BoW vector too long");
  P.o_prog = align256(sizeof(int2) * P.leaves.size());
  P.bytes = P.o_prog + align256(sizeof(int) * P.prog.size());
  return P;
}

void upload_plan(Matcher& M, const PairwisePlan& P, uint8_t* dst) {
  OSFM_CUDA(cudaMemcpyAsync(dst, P.leaves.data(), sizeof(int2) * P.leaves.size(), cudaMemcpyHostToDevice, M.stream));
  OSFM_CUDA(cudaMemcpyAsync(dst + P.o_prog, P.prog.data(), sizeof(int) * P.prog.size(), cudaMemcpyHostToDevice, M.stream));
}

// BoW rows for select_neighbors / distances_to_row (select_common.cuh): the histograms, with the pairwise plan of
// their length in the table.
struct BowRows {
  using Row = double;
  static constexpr int TILE_M = BD_TM;
  PairwisePlan P;
  static const SlabArray<double>& of(Matcher& M, int id, int len) {
    return M.resident(id, &DescSet::bow_hist, len, "descriptor set has no BoW histogram (osfm_matcher_bow_histograms)",
                      "BoW histograms of different lengths");
  }
  static const double* row(const SlabArray<double>& h) { return h.p; }
  size_t table_bytes(int len) {
    P = pairwise_plan(len);
    return P.bytes;
  }
  void upload(Matcher& M, uint8_t* plan) { upload_plan(M, P, plan); }
  void distances(Matcher& M, const uint8_t* plan, const double* const* arows, int na, const double* const* brows,
                 int nb, int, double* out, long long ldo) {
    const size_t smem = sizeof(double) * ((size_t)PW_LEAF * (BD_TM + BD_TN) + (size_t)P.depth * 512);
    OSFM_CUDA(cudaFuncSetAttribute(bow_distance_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid((unsigned)((nb + BD_TN - 1) / BD_TN), (unsigned)((na + BD_TM - 1) / BD_TM));
    bow_distance_kernel<<<grid, 256, smem, M.stream>>>(arows, na, brows, nb, reinterpret_cast<const int2*>(plan),
                                                        reinterpret_cast<const int*>(plan + P.o_prog),
                                                        (int)P.prog.size(), out, ldo);
    OSFM_LAUNCH_CHECK();
  }
};

}  // namespace

static int padded_floats(int dim) { return (int)(((size_t)dim * 4 + 63) / 64 * 64 / 4); }   // match.cu add_async

// The k nearest words of every row of the listed sets (the caller holds the matcher's lock and has checked the
// arguments).  Valid sets (float32 / uint8-stored L2 of dimension dim) get their first words resident and all
// min(k, nwords) words in out_words, rows of set i from out_offsets[i]; the others get no rows.
static void bow_words_run(Matcher& M, int count, const int* set_ids, const float* vocab, int nwords, int dim, int k,
                          int64_t* out_offsets, int32_t* out_words, int* out_valid) {
  for (int i = 0; i < count; ++i)
    if (!M.sets.count(set_ids[i])) throw ArgError("unknown descriptor set id");
  OSFM_CUDA(cudaStreamSynchronize(M.stream));   // earlier work may still read state released below
  const int kout = std::min(k, nwords);
  std::vector<int> job_set;
  std::vector<int64_t> job_out;
  long long total_qtiles = 0;
  int64_t rows = 0;
  out_offsets[0] = 0;
  for (int i = 0; i < count; ++i) {
    DescSet& s = M.sets[set_ids[i]];
    const bool valid = !s.u8 && s.dim == dim;
    out_valid[i] = valid;
    M.release(s.bow_words);
    M.release(s.bow_hist);
    if (valid) {
      M.slab_new(s.bow_words, sizeof(int) * (size_t)std::max(s.n, 1), nwords);
      if (s.n > 0) {
        job_set.push_back(set_ids[i]);
        job_out.push_back(rows);
        total_qtiles += (s.n + BW_TS - 1) / BW_TS;
      }
      rows += s.n;
    }
    out_offsets[i + 1] = rows;
  }
  if (job_set.empty()) return;
  const int D = padded_floats(dim), nblk = dim / 16;
  // vocabulary chunks: enough CTAs to fill the card when the sets are few
  const int wtiles = (nwords + BW_TS - 1) / BW_TS;
  int nchunks = (int)std::min<long long>(std::max<long long>(1, (4ll * M.num_sms + total_qtiles - 1) / total_qtiles),
                                         std::min(wtiles, 16));
  const int chunk_len = (wtiles + nchunks - 1) / nchunks * BW_TS;
  nchunks = (nwords + chunk_len - 1) / chunk_len;
  std::vector<float> hv((size_t)nwords * D, 0.0f);
  for (int w = 0; w < nwords; ++w) std::copy(vocab + (size_t)w * dim, vocab + (size_t)(w + 1) * dim, hv.begin() + (size_t)w * D);
  M.d_bow_vocab.reserve(hv.size());
  M.d_bow_flags.reserve(1);
  OSFM_CUDA(cudaMemcpyAsync(M.d_bow_vocab.p, hv.data(), sizeof(float) * hv.size(), cudaMemcpyHostToDevice, M.stream));
  OSFM_CUDA(cudaMemsetAsync(M.d_bow_flags.p, 0, sizeof(int), M.stream));
  const size_t smem = sizeof(float) * ((size_t)D * BW_LD + std::max(D * BW_LD, BW_TS * BW_KEY_LD) + 2 * BW_TS * BW_KMAX);
  OSFM_CUDA(cudaFuncSetAttribute(bow_words_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  // batches of sets whose lists and words fit the batch budget (a set larger than it goes alone)
  const size_t row_bytes = (size_t)nchunks * k * (sizeof(float) + sizeof(int)) + (size_t)kout * sizeof(int);
  const long long max_rows = std::max<long long>(1, (long long)(BOW_BATCH_BYTES / row_bytes));
  size_t j0 = 0;
  while (j0 < job_set.size()) {
    std::vector<BowJob> jobs;
    std::vector<int> prefix;
    long long brows = 0;
    int ctas = 0, max_n = 0;
    size_t j1 = j0;
    for (; j1 < job_set.size() && jobs.size() < 65535; ++j1) {
      const DescSet& s = M.sets[job_set[j1]];
      if (j1 > j0 && brows + s.n > max_rows) break;
      BowJob b;
      b.f = reinterpret_cast<const float*>(s.rows.p);   // float32 zero-padded rows for every non-Hamming set
      b.first = s.bow_words.p;
      b.row0 = brows;
      b.n = s.n;
      jobs.push_back(b);
      prefix.push_back(ctas);
      ctas += (s.n + BW_TS - 1) / BW_TS * nchunks;
      brows += s.n;
      max_n = std::max(max_n, s.n);
    }
    const size_t o_pre = align256(sizeof(BowJob) * jobs.size());
    M.d_tab.reserve(o_pre + sizeof(int) * prefix.size());
    const size_t nl = (size_t)brows * nchunks * k;
    TableLayout work;
    work.add(sizeof(float) * nl);
    const size_t o_idx = work.add(sizeof(int) * nl), o_w = work.add(sizeof(int) * (size_t)brows * kout);
    M.d_bow_work.reserve(work.size);
    const BowJob* d_jobs = reinterpret_cast<const BowJob*>(M.d_tab.p);
    const int* d_pre = reinterpret_cast<const int*>(M.d_tab.p + o_pre);
    float* d_key = reinterpret_cast<float*>(M.d_bow_work.p);
    int* d_idx = reinterpret_cast<int*>(M.d_bow_work.p + o_idx);
    int* d_words = reinterpret_cast<int*>(M.d_bow_work.p + o_w);
    OSFM_CUDA(cudaMemcpyAsync(M.d_tab.p, jobs.data(), sizeof(BowJob) * jobs.size(), cudaMemcpyHostToDevice, M.stream));
    OSFM_CUDA(cudaMemcpyAsync(M.d_tab.p + o_pre, prefix.data(), sizeof(int) * prefix.size(), cudaMemcpyHostToDevice,
                              M.stream));
    bow_words_kernel<<<(unsigned)ctas, 256, smem, M.stream>>>(d_jobs, d_pre, (int)jobs.size(), M.d_bow_vocab.p, nwords, D,
                                                              nblk, k, nchunks, chunk_len, d_key, d_idx, M.d_bow_flags.p);
    OSFM_LAUNCH_CHECK();
    dim3 mgrid((unsigned)(((long long)max_n * nchunks * k + 255) / 256), (unsigned)jobs.size());
    bow_merge_kernel<<<mgrid, 256, 0, M.stream>>>(d_jobs, d_key, d_idx, nchunks, k, kout, d_words);
    OSFM_LAUNCH_CHECK();
    if (out_words)
      OSFM_CUDA(cudaMemcpyAsync(out_words + job_out[j0] * kout, d_words, sizeof(int) * (size_t)brows * kout,
                                cudaMemcpyDeviceToHost, M.stream));
    OSFM_CUDA(cudaStreamSynchronize(M.stream));   // the tables and the work buffer serve the next batch
    j0 = j1;
  }
  int flags = 0;
  OSFM_CUDA(cudaMemcpy(&flags, M.d_bow_flags.p, sizeof(int), cudaMemcpyDeviceToHost));
  if (flags) {
    for (int id : job_set) {
      M.release(M.sets[id].bow_words);
      M.release(M.sets[id].bow_hist);
    }
    throw ArgError("non-finite descriptor element in a BoW input set");
  }
}

static void check_word_args(const float* vocab, int nwords, int dim, int k) {
  if (nwords <= 0 || dim <= 0 || k <= 0) throw ArgError("bad BoW word sizes");
  if (k > BW_KMAX) throw ArgError("BoW word assignment supports k <= 64");
  if (padded_floats(dim) > BW_MAX_D) throw ArgError("BoW word assignment supports descriptors of at most 320 floats");
  if (!vocab) throw ArgError("null vocabulary");
  for (size_t e = 0; e < (size_t)nwords * dim; ++e)
    if (!std::isfinite(vocab[e])) throw ArgError("non-finite BoW vocabulary element");
}

// device tables (weights | plan | jobs) and one CTA per histogram
static void launch_bow_histograms(Matcher& M, const std::vector<HistJob>& jobs, const double* weights, int nwords,
                                  const PairwisePlan& P) {
  TableLayout tab;
  tab.add(sizeof(double) * (size_t)nwords);
  const size_t o_plan = tab.add(P.bytes), o_jobs = tab.add(sizeof(HistJob) * jobs.size());
  M.d_tab.reserve(tab.size);
  uint8_t* base = M.d_tab.p;
  OSFM_CUDA(cudaMemcpyAsync(base, weights, sizeof(double) * (size_t)nwords, cudaMemcpyHostToDevice, M.stream));
  upload_plan(M, P, base + o_plan);
  OSFM_CUDA(cudaMemcpyAsync(base + o_jobs, jobs.data(), sizeof(HistJob) * jobs.size(), cudaMemcpyHostToDevice, M.stream));
  const size_t smem = sizeof(double) * P.leaves.size();
  OSFM_CUDA(cudaFuncSetAttribute(bow_histogram_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  bow_histogram_kernel<<<(unsigned)jobs.size(), 256, smem, M.stream>>>(
      reinterpret_cast<const HistJob*>(base + o_jobs), reinterpret_cast<const double*>(base), nwords,
      reinterpret_cast<const int2*>(base + o_plan), (int)P.leaves.size(),
      reinterpret_cast<const int*>(base + o_plan + P.o_prog), (int)P.prog.size());
  OSFM_LAUNCH_CHECK();
}
}  // namespace osfm

extern "C" {

int osfm_matcher_bow_words(osfm_matcher* m, int count, const int* set_ids, const float* vocab, int nwords, int dim,
                           int k, int64_t* out_offsets, int32_t* out_words, int* out_valid) {
  using namespace osfm;
  return with_handle(m, [&](Matcher& M) {
    if (count < 0) throw ArgError("bad BoW set count");
    if (!out_offsets || (count > 0 && (!set_ids || !out_valid))) throw ArgError("null arrays");
    check_word_args(vocab, nwords, dim, k);
    bow_words_run(M, count, set_ids, vocab, nwords, dim, k, out_offsets, out_words, out_valid);
  });
}

int osfm_bow_map_to_words(osfm_matcher* m, const float* desc, int n, int dim, const float* vocab, int nwords, int k,
                          int32_t* out) {
  using namespace osfm;
  return with_handle(m, [&](Matcher& M) {
    if (n < 0 || (n > 0 && (!desc || !out))) throw ArgError("bad descriptor arguments");
    check_word_args(vocab, nwords, dim, k);
    const int id = M.add(desc, n, dim, false);
    try {
      int64_t offs[2];
      int valid = 0;
      bow_words_run(M, 1, &id, vocab, nwords, dim, k, offs, out, &valid);
    } catch (...) {
      M.remove(id);
      throw;
    }
    M.remove(id);
  });
}

int osfm_matcher_bow_histograms(osfm_matcher* m, int count, const int* set_ids, const double* weights, int nwords,
                                int* out_valid) {
  using namespace osfm;
  return with_handle(m, [&](Matcher& M) {
    if (count < 0 || nwords <= 0) throw ArgError("bad BoW histogram sizes");
    if (!weights || (count > 0 && (!set_ids || !out_valid))) throw ArgError("null arrays");
    const PairwisePlan P = pairwise_plan(nwords);
    for (int i = 0; i < count; ++i)
      if (!M.sets.count(set_ids[i])) throw ArgError("unknown descriptor set id");
    OSFM_CUDA(cudaStreamSynchronize(M.stream));   // earlier work may still read histograms released below
    // load_histograms: a set needs more than 8 words (pairs_selection.py:712-727)
    std::vector<HistJob> jobs;
    for (int i = 0; i < count; ++i) {
      DescSet& s = M.sets[set_ids[i]];
      M.release(s.bow_hist);
      const bool valid = s.bow_words.p && s.bow_words.len == nwords && s.n > 8;
      out_valid[i] = valid;
      if (!valid) continue;
      M.slab_new(s.bow_hist, sizeof(double) * (size_t)nwords, nwords);
      jobs.push_back(HistJob{s.bow_words.p, s.bow_hist.p, s.n});
    }
    if (jobs.empty()) return;
    launch_bow_histograms(M, jobs, weights, nwords, P);
    OSFM_CUDA(cudaStreamSynchronize(M.stream));
  });
}

int osfm_bow_histogram(osfm_matcher* m, const int32_t* words, int n, const double* weights, int nwords, double* out) {
  using namespace osfm;
  return with_handle(m, [&](Matcher& M) {
    if (n < 0 || nwords <= 0 || !weights || !out || (n > 0 && !words)) throw ArgError("bad BoW histogram arguments");
    for (int i = 0; i < n; ++i)
      if (words[i] < 0 || words[i] >= nwords) throw ArgError("word index out of range");
    const PairwisePlan P = pairwise_plan(nwords);
    const size_t o_h = align256(sizeof(int) * (size_t)std::max(n, 1));
    M.staging.reserve(o_h + sizeof(double) * (size_t)nwords);
    int* d_w = reinterpret_cast<int*>(M.staging.p);
    double* d_h = reinterpret_cast<double*>(M.staging.p + o_h);
    if (n > 0) OSFM_CUDA(cudaMemcpyAsync(d_w, words, sizeof(int) * (size_t)n, cudaMemcpyHostToDevice, M.stream));
    launch_bow_histograms(M, {HistJob{d_w, d_h, n}}, weights, nwords, P);
    OSFM_CUDA(cudaMemcpyAsync(out, d_h, sizeof(double) * (size_t)nwords, cudaMemcpyDeviceToHost, M.stream));
    OSFM_CUDA(cudaStreamSynchronize(M.stream));
  });
}

int osfm_matcher_bow_get(osfm_matcher* m, int set_id, double* out) {
  using namespace osfm;
  return with_handle(m, [&](Matcher& M) {
    if (!out) throw ArgError("null arguments");
    const SlabArray<double>& h = BowRows::of(M, set_id, -1);
    OSFM_CUDA(cudaMemcpyAsync(out, h.p, sizeof(double) * (size_t)h.len, cudaMemcpyDeviceToHost, M.stream));
    OSFM_CUDA(cudaStreamSynchronize(M.stream));
  });
}

int osfm_matcher_bow_select(osfm_matcher* m, int nref, const int* ref_ids, int ncand, const int* cand_ids,
                            const int32_t* cand_order, const int* camera_labels, int k, int64_t* out_offsets,
                            int32_t* out_cols, double* out_dist) {
  using namespace osfm;
  return with_handle(m, [&](Matcher& M) {
    if (nref < 0 || ncand < 0 || k < 0) throw ArgError("bad BoW selection sizes");
    BowRows kind;
    select_neighbors(M, kind, nref, ref_ids, ncand, cand_ids, nullptr, cand_order, camera_labels, k, out_offsets,
                     out_cols, out_dist);
  });
}

int osfm_bow_distances(osfm_matcher* m, const double* hist, int n, int len, int query, double* out_n) {
  using namespace osfm;
  return with_handle(m, [&](Matcher& M) {
    if (n <= 0 || len <= 0 || query < 0 || query >= n || !hist || !out_n) throw ArgError("bad BoW distance arguments");
    BowRows kind;
    distances_to_row(M, kind, hist, n, len, query, out_n);
  });
}

}  // extern "C"
