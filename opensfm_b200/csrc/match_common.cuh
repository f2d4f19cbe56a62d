// Types shared by the SIMT and tensor-core (wgmma) matching kernels.
#pragma once
#include <cuda_bf16.h>

#include <map>
#include <vector>

#include "common.cuh"

namespace osfm {

// Running two-nearest list of one query, in cv2's ranking space:
// s = sqrt(float32 d^2) for L2, bit count for Hamming; i = train index or -1.
struct Top2 {
  float s1;
  int i1;
  float s2;
  int i2;
};

__host__ __device__ inline Top2 top2_empty() {
  Top2 t;
  t.s1 = __builtin_huge_valf();
  t.s2 = __builtin_huge_valf();
  t.i1 = -1;
  t.i2 = -1;
  return t;
}

// Insert candidate (s, i); order is lexicographic (distance, index), which is
// what cv2's stable insertion with a strict `<` produces when trains are
// visited in increasing index order.
__host__ __device__ inline void top2_insert(Top2& t, float s, int i) {
  if (s < t.s1 || (s == t.s1 && (unsigned)i < (unsigned)t.i1)) {
    t.s2 = t.s1; t.i2 = t.i1;
    t.s1 = s; t.i1 = i;
  } else if (s < t.s2 || (s == t.s2 && (unsigned)i < (unsigned)t.i2)) {
    t.s2 = s; t.i2 = i;
  }
}

__host__ __device__ inline void top2_merge(Top2& t, const Top2& o) {
  if (o.i1 >= 0) top2_insert(t, o.s1, o.i1);
  if (o.i2 >= 0) top2_insert(t, o.s2, o.i2);
}

// cv2's float32 L2 distances of one tile: the shared-memory halves and the arithmetic of bf_top2_f32_cv
// (match.cu), also used by the word assignment of bow.cu.
//
// cv2::batchDistance -> normL2Sqr_(const float*, const float*, int) (OpenCV core, the x86-64 baseline
// build of the opencv-python wheels: 4-lane universal intrinsics, no FMA) accumulates
//     acc[a][l] += t*t   for element e = 16*blk + 4*a + l   (four 4-lane accumulators, mul then add),
// combines  v[l] = ((acc[0][l] + acc[1][l]) + acc[2][l]) + acc[3][l],
// reduces   d = (v[0] + v[2]) + (v[1] + v[3]),
// and adds the dim % 16 tail sequentially, d += t*t.  (Probed against live cv2 4.13 in
// tests/test_match_oracle.py::test_cv2_float_sum_order; integer-valued descriptors are exact in any order.)
// Every accumulator receives one term per 16-element block, so the tile walks the 16 (a, l) slots in
// the outer loop and the blocks in the inner loop: one live accumulator per pair instead of sixteen.
// Both operand tiles hold whole rows in shared memory ([element][row], 128-bit conflict-free reads).
// MT = micro-tile edge per thread of a 256-thread CTA (TS = 16 MT rows per tile side), LD = floats per element row.

// rows r0 .. min(r0 + TS, rend) of src (D floats per row) -> dst[e * LD + row], zero rows beyond rend
template <int TS, int LD>
__device__ __forceinline__ void cv_load_tile(float* dst, const float* __restrict__ src, int r0, int rend, int D) {
  const int nvec = D >> 2;
  for (int idx = threadIdx.x; idx < TS * nvec; idx += 256) {
    const int row = idx % TS, v = idx / TS;
    float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
    if (r0 + row < rend) x = *reinterpret_cast<const float4*>(src + (size_t)(r0 + row) * D + v * 4);
    dst[(v * 4 + 0) * LD + row] = x.x;
    dst[(v * 4 + 1) * LD + row] = x.y;
    dst[(v * 4 + 2) * LD + row] = x.z;
    dst[(v * 4 + 3) * LD + row] = x.w;
  }
}

// d2[i][j] = squared distance of tile rows (As row ty * MT + i, Bs row tx * MT + j) over D padded elements,
// nblk = full 16-element blocks of the true dimension
template <int MT, int LD>
__device__ __forceinline__ void cv_tile_d2(const float* As, const float* Bs, int D, int nblk, int ty, int tx,
                                           float (&d2)[MT][MT]) {
  float u[MT][MT], w[MT][MT];
#pragma unroll
  for (int li = 0; li < 4; ++li) {
    const int l = (li == 0) ? 0 : (li == 1) ? 2 : (li == 2) ? 1 : 3;  // lanes 0, 2 feed u; 1, 3 feed w
    float s[MT][MT];
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      float acc[MT][MT];
#pragma unroll
      for (int i = 0; i < MT; ++i)
#pragma unroll
        for (int j = 0; j < MT; ++j) acc[i][j] = 0.f;
      const float* pa = As + (size_t)(4 * a + l) * LD + ty * MT;
      const float* pb = Bs + (size_t)(4 * a + l) * LD + tx * MT;
      for (int blk = 0; blk < nblk; ++blk) {
        float av[MT], bv[MT];
        if constexpr (MT == 4) {
          const float4 a4 = *reinterpret_cast<const float4*>(pa);
          const float4 b4 = *reinterpret_cast<const float4*>(pb);
          av[0] = a4.x; av[1] = a4.y; av[2] = a4.z; av[3] = a4.w;
          bv[0] = b4.x; bv[1] = b4.y; bv[2] = b4.z; bv[3] = b4.w;
        } else {
          const float2 a2 = *reinterpret_cast<const float2*>(pa);
          const float2 b2 = *reinterpret_cast<const float2*>(pb);
          av[0] = a2.x; av[1] = a2.y; bv[0] = b2.x; bv[1] = b2.y;
        }
#pragma unroll
        for (int i = 0; i < MT; ++i)
#pragma unroll
          for (int j = 0; j < MT; ++j) {
            const float t = __fsub_rn(av[i], bv[j]);
            acc[i][j] = __fadd_rn(acc[i][j], __fmul_rn(t, t));   // mul, then add: no FMA contraction
          }
        pa += 16 * LD;
        pb += 16 * LD;
      }
#pragma unroll
      for (int i = 0; i < MT; ++i)
#pragma unroll
        for (int j = 0; j < MT; ++j) s[i][j] = a == 0 ? acc[i][j] : __fadd_rn(s[i][j], acc[i][j]);
    }
#pragma unroll
    for (int i = 0; i < MT; ++i)
#pragma unroll
      for (int j = 0; j < MT; ++j) {
        if (li == 0) u[i][j] = s[i][j];
        else if (li == 1) u[i][j] = __fadd_rn(u[i][j], s[i][j]);
        else if (li == 2) w[i][j] = s[i][j];
        else w[i][j] = __fadd_rn(w[i][j], s[i][j]);
      }
  }
#pragma unroll
  for (int i = 0; i < MT; ++i)
#pragma unroll
    for (int j = 0; j < MT; ++j) d2[i][j] = __fadd_rn(u[i][j], w[i][j]);
  // scalar tail of the true dimension (zero padding beyond it adds +0)
  for (int e = nblk * 16; e < D; ++e) {
    float av[MT], bv[MT];
#pragma unroll
    for (int i = 0; i < MT; ++i) { av[i] = As[(size_t)e * LD + ty * MT + i]; bv[i] = Bs[(size_t)e * LD + tx * MT + i]; }
#pragma unroll
    for (int i = 0; i < MT; ++i)
#pragma unroll
      for (int j = 0; j < MT; ++j) {
        const float t = __fsub_rn(av[i], bv[j]);
        d2[i][j] = __fadd_rn(d2[i][j], __fmul_rn(t, t));
      }
  }
}

// One direction of one image pair.
struct MatchJob {
  const void* q;  // queries, padded rows (float32 or packed uint8 words)
  const void* t;  // trains
  const __nv_bfloat16* q_tc;  // tensor-core operand copies (blocked core-matrix layout), or null
  const __nv_bfloat16* t_tc;
  const float* q_norm;        // |q_i|^2 (tensor-core path)
  const float* t_norm;
  int nq, nt;
  int dim, dim_padded;  // dim_padded: 4-byte elements per padded row
  int qtiles;
  int nchunks, chunk_len;
  long long partial_off;  // Top2 partial[partial_off + chunk * nq + q]
  long long match_off;    // int32 match[match_off + q]
  const uint8_t* mask;
  long long mask_sq, mask_st;
  // guided matching: one bit per (query, train), row-major over the queries, mask_words 32-bit words per row
  const uint32_t* mask_bits;
  int mask_words;
};
__device__ __forceinline__ bool job_allows(const MatchJob& job, int gq, int gt) {
  if (job.mask && job.mask[(size_t)gq * job.mask_sq + (size_t)gt * job.mask_st] == 0) return false;
  if (job.mask_bits && !((job.mask_bits[(size_t)gq * job.mask_words + (gt >> 5)] >> (gt & 31)) & 1u)) return false;
  return true;
}

// Tile `tile` of a submission: queries q0 .. q0 + M - 1 of `job` against its trains t_begin .. t_end - 1 (chunk
// `chunk`).  A job's tiles are its query tiles times its chunks, chunk fastest; tile_prefix[i] is job i's first tile.
struct MatchTile {
  MatchJob job;
  int q0, t_begin, t_end, chunk;
};
template <int M>
__device__ __forceinline__ MatchTile decode_tile(const MatchJob* __restrict__ jobs, const int* __restrict__ tile_prefix,
                                                 int njobs, int tile) {
  int lo = 0, hi = njobs - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (tile_prefix[mid] <= tile) lo = mid; else hi = mid - 1;
  }
  MatchTile t;
  t.job = jobs[lo];
  const int local = tile - tile_prefix[lo];
  t.q0 = local / t.job.nchunks * M;
  t.chunk = local % t.job.nchunks;
  t.t_begin = t.chunk * t.job.chunk_len;
  t.t_end = min(t.job.nt, t.t_begin + t.job.chunk_len);
  return t;
}

// Offsets of arrays packed into one device table, each on a 256-byte boundary.
inline size_t align256(size_t bytes) { return (bytes + 255) / 256 * 256; }
struct TableLayout {
  size_t size = 0;
  size_t add(size_t bytes) {
    const size_t o = size;
    size += align256(bytes);
    return o;
  }
};

// An array in the matcher's slabs (Matcher::slab_new / Matcher::release); null until allocated.
template <class T>
struct SlabArray {
  T* p = nullptr;
  int slab = -1;
  size_t bytes = 0;
  int len = 0;   // the length its owner records with it
};

struct DescSet {
  // one allocation: the zero-padded rows (n x row_bytes), then the tensor-core operands of a set that has them
  SlabArray<char> rows;
  int n = 0, dim = 0, dim_padded = 0, row_bytes = 0;
  bool u8 = false;
  // tensor-core operands (float32 sets with integer values in [0,255] and dim <= 128, Hamming sets of <= 63 bytes):
  // L2 [A-role | B-role | norms], Hamming [A-role | B-role]
  char* tc_data() const { return rows.p + align256((size_t)std::max(n, 1) * row_bytes); }
  const __nv_bfloat16* tc_q = nullptr;
  const __nv_bfloat16* tc_t = nullptr;
  const float* tc_norm = nullptr;
  bool tc_ok = false;
  float tc_max_norm = 0.0f;  // max_i |x_i|^2
  int rows_padded = 0;
  // device memory comes from the matcher's slabs; the exactness flag / max norm of a freshly added set
  // live in d_info[slot] until refresh_info() reads them back (no host sync per add)
  int slot = -1;
  bool info_pending = false;
  // unit bearing vectors of the features (n x 3 float32), for guided matching
  SlabArray<float> bearings;
  // VLAD descriptor of the set (vlad.cu): [unnormalised | normalised], len floats each
  SlabArray<float> vlad;
  // BoW state (bow.cu): the nearest visual word of every row (n ints, words of a len-word vocabulary) and
  // the weighted, normalised word histogram (len doubles)
  SlabArray<int> bow_words;
  SlabArray<double> bow_hist;
};

// The two layouts of one pair's epipolar bitmask in the last guided submission (the test hook reads them back).
struct EpiMasks {
  const uint32_t *F, *T;   // F: n1 rows of w2 words (over n2), T: n2 rows of w1 words (over n1)
  int n1, n2, w1, w2;
};

struct Slab {
  char* base = nullptr;
  size_t cap = 0, used = 0;   // bump pointer
  int live = 0;
  // ranges below `used` that were released while neighbours stayed live: (offset, bytes), sorted, coalesced.
  // A long-lived matcher that replaces descriptor sets key by key reuses them instead of growing.
  std::vector<std::pair<size_t, size_t>> free_ranges;
};

// Its methods expect the device to be current; the C entry points make it so (with_handle).
struct Matcher : DeviceStream<4> {
  int num_sms = 132;
  int next_id = 1;
  int kernel_choice = 0;
  int last_kernel = 0;
  long long last_total_results = 0;
  int last_npairs = 0;
  bool results_in_match_buf = true;
  SmemOptIn opt_in_smem;
  std::map<int, DescSet> sets;
  std::vector<MatchJob> h_jobs;
  std::vector<int> h_prefix;
  std::vector<long long> h_out_off;
  DevBuf<MatchJob> d_jobs;
  DevBuf<int> d_prefix;
  DevBuf<long long> d_out_off;
  DevBuf<Top2> d_partial;
  DevBuf<int32_t> d_match, d_out;
  DevBuf<uint8_t> staging, mask_buf;
  DevBuf<int> d_flags;
  DevBuf<uint32_t> d_mask_bits;
  DevBuf<int> d_pair_counts;
  DevBuf<long long> d_pair_off;
  DevBuf<int32_t> d_pairs;
  DevBuf<double> d_epi_vec, d_epi_pose;
  std::vector<EpiMasks> last_masks;   // empty unless the last submission was guided
  PinnedBuf<double> p_epi_pose;
  PinnedBuf<MatchJob> p_jobs;
  PinnedBuf<int> p_prefix;
  PinnedBuf<long long> p_out_off;
  // VLAD workspaces (vlad.cu): centres, per-feature nearest centre, error flags
  DevBuf<float> d_vlad_centers;
  DevBuf<int> d_vlad_assign, d_vlad_flags;
  // BoW workspaces (bow.cu): padded vocabulary, per-chunk top-k lists + words of a batch, error flags
  DevBuf<float> d_bow_vocab;
  DevBuf<uint8_t> d_bow_work;
  DevBuf<int> d_bow_flags;
  // VLAD and BoW: job / plan / selection tables and the selection's distance block.  Every call that uses them
  // synchronises the stream before it returns.
  DevBuf<uint8_t> d_tab;
  DevBuf<double> d_dist;

  explicit Matcher(int dev);
  ~Matcher();

  std::vector<Slab> slabs;
  DevBuf<int> d_info;                 // [MAX_SLOTS][2]: not-exact flag, max |x|^2 (float bits)
  std::vector<int> h_info;
  std::vector<int> free_slots, pending;
  int next_slot = 0;
  static constexpr int MAX_SLOTS = 1 << 16;
  void* slab_alloc(size_t bytes, int* slab_idx);
  void slab_release(int idx, void* ptr, size_t bytes);
  template <class T>
  void slab_new(SlabArray<T>& a, size_t bytes, int len) {
    a.p = static_cast<T*>(slab_alloc(bytes, &a.slab));
    a.bytes = bytes;
    a.len = len;
  }
  // callers synchronise the stream first; slab_release counts a release even of a null pointer, so only what was
  // allocated goes back
  template <class T>
  void release(SlabArray<T>& a) {
    if (a.p) slab_release(a.slab, a.p, a.bytes);
    a = SlabArray<T>();
  }
  // the array `field` of set `id`, whose len must equal `len` when len >= 0
  template <class T>
  const SlabArray<T>& resident(int id, SlabArray<T> DescSet::*field, int len, const char* missing, const char* mismatch) {
    auto it = sets.find(id);
    if (it == sets.end()) throw ArgError("unknown descriptor set id");
    const SlabArray<T>& a = it->second.*field;
    if (!a.p) throw ArgError(missing);
    if (len >= 0 && a.len != len) throw ArgError(mismatch);
    return a;
  }
  void refresh_info();
  // u8: Hamming descriptors.  u8_as_l2: uint8 storage of an L2 descriptor (widened to float32 on the device).
  int add_async(const void* host, int n, int dim, bool u8, bool u8_as_l2 = false);  // no host sync; the host buffer must stay valid
  int add(const void* host, int n, int dim, bool u8, bool u8_as_l2 = false);
  void remove(int id);
  void clear();
  void free_set(DescSet& s);
  // guided: pose12 = npairs x 12 doubles [R cam2->cam1 row-major | origin of camera 2 in camera 1] and the angle
  // threshold; the epipolar mask is built on the device as a bitmask (matching.py:847-868)
  void match_pairs_async(int npairs, const int* ids_a, const int* ids_b, double ratio, bool symmetric,
                         const uint8_t* dmask, const double* pose12 = nullptr, double epi_threshold = 0.0);
  void set_bearings(int id, const float* host_n_by_3);
  void get_epipolar_masks(int pair, uint32_t* F, uint32_t* T);
  void fetch(int32_t* out, int64_t capacity);
  long long fetch_pairs(long long* offsets_out, int32_t* pairs_out, long long capacity_rows);
  void last_ms(float* total, float* kernel);
  void one_shot(const void* f1, int n1, const void* f2, int n2, int dim, bool u8, double ratio,
                const uint8_t* mask, bool symmetric, int32_t* out);
  // match_tc.cu
  void prepare_tc(DescSet& s, const void* src, bool src_u8, float* padded_dst);
  void prepare_h8(DescSet& s, const uint8_t* src, int src_stride);   // +-1 fp8 operands of a Hamming set
};

// The distance kernel of a submission; the values are those osfm_matcher_last_kernel returns.
enum class DistKernel : int {
  SIMT = 1,         // bf_top2_simt (Hamming), bf_top2_f32_cv (float32)
  TC_L2 = 2,        // bf_top2_wg<KIND_L2> (match_tc.cu)
  TC_HAMMING = 3,   // bf_top2_wg<KIND_HAMMING>
};

// What the distance kernel fixes in a submission's plan.
struct KernelPlan {
  int tile_m;        // query rows per tile
  int chunk_unit;    // train chunks are whole multiples of this many rows
  int ctas_per_sm;   // the trains are split into chunks until the tiles reach this many per SM
  bool squared;      // the partials hold d^2, which bf_top2_finalize takes the square root of
  int smem;          // dynamic shared memory of a CTA
  void (*launch)(Matcher& m, int njobs, int ntiles, int smem);
};

// match_tc.cu
bool tc_available();
KernelPlan tc_plan(DistKernel kernel, bool masked);   // kernel: TC_L2 or TC_HAMMING; masked: guided L2
int tc_rows_padded(int n);
size_t tc_operand_bytes(int rows_padded);
bool tc_capable(int dim, bool u8);
// tensor-core Hamming (match_tc.cu)
size_t h8_operand_bytes(int rows_padded);
bool h8_capable(int nbytes);

}  // namespace osfm

struct osfm_matcher : osfm::Handle<osfm::Matcher> {
  using Handle::Handle;
  static constexpr const char* null_message = "null matcher";
};
