// VLAD pair selection on the device (SURVEY.md §8f.3): descriptors of resident descriptor sets, all-pairs
// distances and the per-image neighbour selection of pairs_selection.match_candidates_with_vlad.
//
// Replaces features::compute_vlad_descriptor and features::compute_vlad_distances
// (opensfm/src/features/src/matching.cc:90-145), vlad.signed_square_root_normalize (opensfm/vlad.py) and
// construct_pairs / pairs_from_neighbors (opensfm/pairs_selection.py:471-490, 764-795).
//
// compute_vlad_descriptor: every feature goes to the first centre of smallest squared distance below FLT_MAX, the
// distance summed in dimension order with separate float32 subtract, multiply and add (Eigen reduces the strided
// row of a column-major MatXf sequentially; no FMA contraction, like the reference's x86-64 baseline build), and its
// residual f - c is added to the centre's segment, feature after feature.  Both steps here do the same float32
// operations in the same order, so the unnormalised vector is bit for bit the reference's.
#include <cfloat>
#include <cmath>
#include <vector>

#include "common.cuh"
#include "match_common.cuh"
#include "select_common.cuh"

namespace osfm {

namespace {

constexpr int VA_THREADS = 128;          // word assignment: one thread per feature
constexpr int VA_CH = 32;                // centres whose distance chains one thread interleaves
constexpr int VN_THREADS_MAX = 256;      // accumulation + normalisation: one CTA per set
constexpr int VD_TM = 32, VD_TN = 64, VD_TK = 32;   // distance tile: reference rows x candidate rows x elements
constexpr size_t VLAD_SMEM_MAX = 200 * 1024;

struct VladJob {
  const float* f;    // float32 rows, stride ld (the set's zero-padded copy)
  float* v;          // [unnormalised | normalised], 2 x L floats
  long long aoff;    // first entry of the set in the assignment buffer
  int n, ld;
};

// Nearest centre of every feature.  ct: the centres transposed, [dim][ncp] with ncp = ncenters rounded up to VA_CH
// and the padding centres at +inf (their distance is +inf, never below FLT_MAX).  flags |= 1 for a non-finite
// descriptor element, |= 2 for a feature with no centre below FLT_MAX (the reference indexes segment(-D) there).
__global__ void __launch_bounds__(VA_THREADS)
    vlad_assign_kernel(const VladJob* __restrict__ jobs, const float* __restrict__ ct, int ncp, int dim,
                       int* __restrict__ assign, int* __restrict__ flags) {
  extern __shared__ float4 smem4[];
  float* sc = reinterpret_cast<float*>(smem4);
  for (int e = threadIdx.x; e < dim * ncp; e += blockDim.x) sc[e] = ct[e];
  __syncthreads();
  const VladJob job = jobs[blockIdx.y];
  const int i = blockIdx.x * VA_THREADS + threadIdx.x;
  if (i >= job.n) return;
  const float* f = job.f + (size_t)i * job.ld;
  float best = FLT_MAX;
  int best_c = -1;
  bool finite = true;
  for (int c0 = 0; c0 < ncp; c0 += VA_CH) {
    float s[VA_CH];
#pragma unroll
    for (int j = 0; j < VA_CH; ++j) s[j] = 0.0f;   // 0 + (f0 - c0)^2 == (f0 - c0)^2 exactly
    for (int k4 = 0; k4 < dim; k4 += 4) {
      const float4 x4 = __ldg(reinterpret_cast<const float4*>(f + k4));   // rows are 64-byte aligned, zero-padded
      const float xs[4] = {x4.x, x4.y, x4.z, x4.w};
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int k = k4 + u;
        if (k >= dim) break;
        const float x = xs[u];
        if (c0 == 0) finite &= isfinite(x);
        const float4* cr = reinterpret_cast<const float4*>(sc + (size_t)k * ncp + c0);
#pragma unroll
        for (int q = 0; q < VA_CH / 4; ++q) {
          const float4 c = cr[q];
          float t;
          t = __fsub_rn(x, c.x); s[4 * q + 0] = __fadd_rn(s[4 * q + 0], __fmul_rn(t, t));
          t = __fsub_rn(x, c.y); s[4 * q + 1] = __fadd_rn(s[4 * q + 1], __fmul_rn(t, t));
          t = __fsub_rn(x, c.z); s[4 * q + 2] = __fadd_rn(s[4 * q + 2], __fmul_rn(t, t));
          t = __fsub_rn(x, c.w); s[4 * q + 3] = __fadd_rn(s[4 * q + 3], __fmul_rn(t, t));
        }
      }
    }
#pragma unroll
    for (int j = 0; j < VA_CH; ++j)
      if (s[j] < best) { best = s[j]; best_c = c0 + j; }
  }
  if (!finite) atomicOr(flags, 1);
  else if (best_c < 0) atomicOr(flags, 2);
  assign[job.aoff + i] = best_c;
}

// numpy's sign(v) * sqrt(|v|) in float32
__device__ __forceinline__ float signed_sqrt(float v) {
  return v > 0.0f ? __fsqrt_rn(v) : v < 0.0f ? -__fsqrt_rn(-v) : (v == 0.0f ? 0.0f : v);
}

// One CTA per set: v[c][k] += f[k] - c[k] feature after feature (thread k owns column k of every segment, so each
// element's sum runs in feature order), then the unnormalised vector, its signed square root and the division by
// the norm (sum of squares in fp64, rounded to float32, float32 square root; a zero vector becomes 0/0 = NaN).
// Every feature without a centre (assignment -1) has raised a flag in vlad_assign_kernel, earlier on this stream;
// then the call fails and nothing is accumulated, so no assignment below is negative.
__global__ void __launch_bounds__(VN_THREADS_MAX)
    vlad_accumulate_kernel(const VladJob* __restrict__ jobs, const float* __restrict__ centers, int nc, int dim,
                           const int* __restrict__ assign, const int* __restrict__ flags) {
  if (*flags) return;
  extern __shared__ float4 smem4[];
  float* v = reinterpret_cast<float*>(smem4);
  __shared__ double warp_sum[VN_THREADS_MAX / 32];
  __shared__ float s_norm;
  const VladJob job = jobs[blockIdx.x];
  const int L = nc * dim;
  for (int e = threadIdx.x; e < L; e += blockDim.x) v[e] = 0.0f;
  __syncthreads();
  const int* a = assign + job.aoff;
  for (int k = threadIdx.x; k < dim; k += blockDim.x) {
    constexpr int B = 8;   // loads of the next B features are issued before their ordered updates
    int i = 0;
    for (; i + B <= job.n; i += B) {
      int c[B];
      float r[B];
#pragma unroll
      for (int u = 0; u < B; ++u) c[u] = __ldg(a + i + u);
#pragma unroll
      for (int u = 0; u < B; ++u)
        r[u] = __fsub_rn(__ldg(job.f + (size_t)(i + u) * job.ld + k), __ldg(centers + (size_t)c[u] * dim + k));
#pragma unroll
      for (int u = 0; u < B; ++u) v[c[u] * dim + k] = __fadd_rn(v[c[u] * dim + k], r[u]);
    }
    for (; i < job.n; ++i) {
      const int c = __ldg(a + i);
      v[c * dim + k] = __fadd_rn(v[c * dim + k], __fsub_rn(__ldg(job.f + (size_t)i * job.ld + k), __ldg(centers + (size_t)c * dim + k)));
    }
  }
  __syncthreads();
  double part = 0.0;
  for (int e = threadIdx.x; e < L; e += blockDim.x) {
    const float x = v[e];
    job.v[e] = x;
    const float w = signed_sqrt(x);
    v[e] = w;
    part += (double)w * (double)w;
  }
  for (int o = 16; o; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
  if ((threadIdx.x & 31) == 0) warp_sum[threadIdx.x >> 5] = part;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += warp_sum[w];
    s_norm = __fsqrt_rn(__double2float_rn(t));
  }
  __syncthreads();
  const float nrm = s_norm;
  for (int e = threadIdx.x; e < L; e += blockDim.x) job.v[L + e] = __fdiv_rn(v[e], nrm);
}

// out[i * ldo + j] = sqrt(sum_e (double(a_i[e]) - double(b_j[e]))^2), e ascending in one chain per output, so
// d(a, b) == d(b, a) bit for bit.  Direct differences, not |a|^2 + |b|^2 - 2ab, which cancels for near-duplicates.
// Register tile: each thread 2 reference rows x 4 candidate rows; operands staged through shared memory as fp64.
__global__ void __launch_bounds__(256)
    vlad_distance_kernel(const float* const* __restrict__ arows, int na, const float* const* __restrict__ brows, int nb,
                         int L, double* __restrict__ out, long long ldo) {
  __shared__ double As[VD_TK][VD_TM + 1];
  __shared__ double Bs[VD_TK][VD_TN + 1];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int a0 = blockIdx.y * VD_TM, b0 = blockIdx.x * VD_TN;
  const int kk = threadIdx.x & (VD_TK - 1), r0 = threadIdx.x / VD_TK;   // staging: element kk of rows r0 + 8 r
  const float* ap[VD_TM / 8];
  const float* bp[VD_TN / 8];
#pragma unroll
  for (int r = 0; r < VD_TM / 8; ++r) ap[r] = a0 + r0 + 8 * r < na ? arows[a0 + r0 + 8 * r] : nullptr;
#pragma unroll
  for (int r = 0; r < VD_TN / 8; ++r) bp[r] = b0 + r0 + 8 * r < nb ? brows[b0 + r0 + 8 * r] : nullptr;
  double acc[2][4];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.0;
  for (int k0 = 0; k0 < L; k0 += VD_TK) {
    const int k = k0 + kk;
#pragma unroll
    for (int r = 0; r < VD_TM / 8; ++r) As[kk][r0 + 8 * r] = (ap[r] && k < L) ? (double)__ldg(ap[r] + k) : 0.0;
#pragma unroll
    for (int r = 0; r < VD_TN / 8; ++r) Bs[kk][r0 + 8 * r] = (bp[r] && k < L) ? (double)__ldg(bp[r] + k) : 0.0;
    __syncthreads();
#pragma unroll 4
    for (int e = 0; e < VD_TK; ++e) {
      double x[2], y[4];
#pragma unroll
      for (int i = 0; i < 2; ++i) x[i] = As[e][ty + 16 * i];
#pragma unroll
      for (int j = 0; j < 4; ++j) y[j] = Bs[e][tx + 16 * j];
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const double t = x[i] - y[j];
          acc[i][j] = fma(t, t, acc[i][j]);   // zero padding adds fma(0, 0, s) = s
        }
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int ia = a0 + ty + 16 * i, jb = b0 + tx + 16 * j;
      if (ia < na && jb < nb) out[(size_t)ia * ldo + jb] = sqrt(acc[i][j]);
    }
}

// VLAD rows for select_neighbors / distances_to_row (select_common.cuh): the normalised half of each descriptor.
struct VladRows {
  using Row = float;
  static constexpr int TILE_M = VD_TM;
  static const SlabArray<float>& of(Matcher& M, int id, int len) {
    return M.resident(id, &DescSet::vlad, len, "descriptor set has no VLAD descriptor (osfm_matcher_vlad_compute)",
                      "VLAD descriptors of different lengths");
  }
  static const float* row(const SlabArray<float>& v) { return v.p + v.len; }
  size_t table_bytes(int) { return 0; }
  void upload(Matcher&, uint8_t*) {}
  void distances(Matcher& M, const uint8_t*, const float* const* arows, int na, const float* const* brows, int nb,
                 int L, double* out, long long ldo) {
    dim3 grid((unsigned)((nb + VD_TN - 1) / VD_TN), (unsigned)((na + VD_TM - 1) / VD_TM));
    vlad_distance_kernel<<<grid, 256, 0, M.stream>>>(arows, na, brows, nb, L, out, ldo);
    OSFM_LAUNCH_CHECK();
  }
};

}  // namespace
}  // namespace osfm

extern "C" {

int osfm_matcher_vlad_compute(osfm_matcher* m, int count, const int* set_ids, const float* centers, int ncenters, int dim,
                              int* out_valid) {
  using namespace osfm;
  return with_handle(m, [&](Matcher& M) {
    if (count < 0 || ncenters <= 0 || dim <= 0) throw ArgError("bad VLAD sizes");
    if ((count > 0 && (!set_ids || !out_valid)) || !centers) throw ArgError("null arrays");
    const int ncp = (ncenters + VA_CH - 1) / VA_CH * VA_CH;
    const size_t L = (size_t)ncenters * dim;
    if ((size_t)dim * ncp * sizeof(float) > VLAD_SMEM_MAX || L * sizeof(float) > VLAD_SMEM_MAX)
      throw ArgError("VLAD vocabulary too large: ncenters x dim float32 must fit in 200 KB of shared memory");
    for (size_t e = 0; e < L; ++e)
      if (!std::isfinite(centers[e])) throw ArgError("non-finite VLAD centre");
    for (int i = 0; i < count; ++i)
      if (!M.sets.count(set_ids[i])) throw ArgError("unknown descriptor set id");
    OSFM_CUDA(cudaStreamSynchronize(M.stream));   // earlier work may still read VLADs released below
    // one descriptor per set; Hamming sets and sets of another dimension have none (unnormalized_vlad -> None)
    std::vector<VladJob> jobs;
    std::vector<int> job_set;
    long long nfeat = 0;
    int max_n = 0;
    for (int i = 0; i < count; ++i) {
      DescSet& s = M.sets[set_ids[i]];
      const bool valid = !s.u8 && s.dim == dim;
      out_valid[i] = valid;
      if (!valid || (size_t)s.vlad.len != L) M.release(s.vlad);
      if (!valid) continue;
      if (!s.vlad.p) M.slab_new(s.vlad, 2 * L * sizeof(float), (int)L);
      VladJob j;
      j.f = reinterpret_cast<const float*>(s.rows.p);   // float32 zero-padded rows for every non-Hamming set (match.cu add_async)
      j.v = s.vlad.p;
      j.aoff = nfeat;
      j.n = s.n;
      j.ld = s.dim_padded;
      jobs.push_back(j);
      job_set.push_back(set_ids[i]);
      nfeat += s.n;
      max_n = std::max(max_n, s.n);
    }
    if (jobs.empty()) return;
    // centres: row-major for the residuals, transposed and padded with +inf for the assignment
    std::vector<float> hc(L + (size_t)dim * ncp, __builtin_huge_valf());
    std::copy(centers, centers + L, hc.begin());
    for (int c = 0; c < ncenters; ++c)
      for (int k = 0; k < dim; ++k) hc[L + (size_t)k * ncp + c] = centers[(size_t)c * dim + k];
    M.d_vlad_centers.reserve(hc.size());
    M.d_vlad_assign.reserve((size_t)std::max<long long>(nfeat, 1));
    M.d_vlad_flags.reserve(1);
    M.d_tab.reserve(sizeof(VladJob) * jobs.size());
    OSFM_CUDA(cudaMemcpyAsync(M.d_vlad_centers.p, hc.data(), sizeof(float) * hc.size(), cudaMemcpyHostToDevice, M.stream));
    OSFM_CUDA(cudaMemcpyAsync(M.d_tab.p, jobs.data(), sizeof(VladJob) * jobs.size(), cudaMemcpyHostToDevice, M.stream));
    OSFM_CUDA(cudaMemsetAsync(M.d_vlad_flags.p, 0, sizeof(int), M.stream));
    const VladJob* d_jobs = reinterpret_cast<const VladJob*>(M.d_tab.p);
    const size_t smem_a = (size_t)dim * ncp * sizeof(float), smem_n = L * sizeof(float);
    OSFM_CUDA(cudaFuncSetAttribute(vlad_assign_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_a));
    OSFM_CUDA(cudaFuncSetAttribute(vlad_accumulate_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_n));
    const int nthreads = std::min(VN_THREADS_MAX, std::max(32, (dim + 31) / 32 * 32));
    for (size_t j0 = 0; j0 < jobs.size(); j0 += 32768) {   // gridDim.y <= 65535
      const int nj = (int)std::min<size_t>(32768, jobs.size() - j0);
      if (max_n > 0) {
        dim3 grid((unsigned)((max_n + VA_THREADS - 1) / VA_THREADS), (unsigned)nj);
        vlad_assign_kernel<<<grid, VA_THREADS, smem_a, M.stream>>>(d_jobs + j0, M.d_vlad_centers.p + L, ncp, dim,
                                                                   M.d_vlad_assign.p, M.d_vlad_flags.p);
        OSFM_LAUNCH_CHECK();
      }
      vlad_accumulate_kernel<<<nj, nthreads, smem_n, M.stream>>>(d_jobs + j0, M.d_vlad_centers.p, ncenters, dim,
                                                                M.d_vlad_assign.p, M.d_vlad_flags.p);
      OSFM_LAUNCH_CHECK();
    }
    int flags = 0;
    OSFM_CUDA(cudaMemcpyAsync(&flags, M.d_vlad_flags.p, sizeof(int), cudaMemcpyDeviceToHost, M.stream));
    OSFM_CUDA(cudaStreamSynchronize(M.stream));
    if (flags) {
      for (int id : job_set) M.release(M.sets[id].vlad);
      throw ArgError(flags & 1 ? "non-finite descriptor element in a VLAD input set"
                               : "a feature's squared distance to every VLAD centre overflows float32");
    }
  });
}

int osfm_matcher_vlad_get(osfm_matcher* m, int set_id, int unnormalized, float* out) {
  using namespace osfm;
  return with_handle(m, [&](Matcher& M) {
    if (!out) throw ArgError("null arguments");
    const SlabArray<float>& v = VladRows::of(M, set_id, -1);
    OSFM_CUDA(cudaMemcpyAsync(out, v.p + (unnormalized ? 0 : v.len), sizeof(float) * (size_t)v.len,
                              cudaMemcpyDeviceToHost, M.stream));
    OSFM_CUDA(cudaStreamSynchronize(M.stream));
  });
}

int osfm_matcher_vlad_select(osfm_matcher* m, int nref, const int* ref_ids, int ncand, const int* cand_ids,
                             const uint32_t* cand_mask_bits, const int* camera_labels, int k, int64_t* out_offsets,
                             int32_t* out_cols, double* out_dist) {
  using namespace osfm;
  return with_handle(m, [&](Matcher& M) {
    if (nref < 0 || ncand < 0 || k < 0) throw ArgError("bad VLAD selection sizes");
    VladRows kind;
    select_neighbors(M, kind, nref, ref_ids, ncand, cand_ids, cand_mask_bits, nullptr, camera_labels, k, out_offsets,
                     out_cols, out_dist);
  });
}

int osfm_vlad_distances(osfm_matcher* m, const float* vlad, int n, int dim, int query, double* out_n) {
  using namespace osfm;
  return with_handle(m, [&](Matcher& M) {
    if (n <= 0 || dim <= 0 || query < 0 || query >= n || !vlad || !out_n) throw ArgError("bad VLAD arguments");
    VladRows kind;
    distances_to_row(M, kind, vlad, n, dim, query, out_n);
  });
}

}  // extern "C"
