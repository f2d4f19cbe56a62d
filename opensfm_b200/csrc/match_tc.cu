// Tensor-core distance kernels for brute-force matching on H100 (sm_90a): warpgroup MMA (wgmma) with register
// accumulators, operands staged by the bulk-copy (TMA) engine through an mbarrier pipeline.
//
// L2 ("BruteForce"): the N x M x 128 contraction of opensfm/matching.py:742-747 (cv2 knnMatch)
// is a dense GEMM: d2(i,j) = |a_i|^2 + |b_j|^2 - 2 a_i.b_j.  For descriptors
// whose values are integers in [0,255] (HAHOG / SIFT as OpenSfM stores them,
// opensfm/features.py:526-534, and the synthetic scenes) every product and
// partial sum is an integer below 2^24, so bf16 operands with fp32 accumulation
// reproduce the float32 sum of squared differences of cv2 bit for bit.
//
// Operand layout (built once per descriptor set by prepare_tc):
//   K = 144 = 128 descriptor dims + 16 augmentation columns.
//   A role (queries):  [ a_i            | 1, 1, 1, 0 ... ]
//   B role (trains):   [ -2 b_j         | hi, mid, lo of |b_j|^2, 0 ... ]
//   => accumulator(i,j) = |b_j|^2 - 2 a_i.b_j = d2(i,j) - |a_i|^2   (exact)
//   so the epilogue needs no per-column add: ranking within a query row is
//   the ranking of the accumulator itself.
// Rows are stored in HBM already in the canonical K-major no-swizzle ("interleave") core-matrix order of wgmma:
// [row/8][k/8][row%8][k%8] bf16, 128 bytes per core matrix, so one tile is a single contiguous range and is
// staged with one cp.async.bulk per operand tile; LBO = 128 B (K-adjacent core matrices), SBO = 18*128 B
// (8-row groups).
//
// Kernel (bf_top2_wg, both the L2 and the Hamming kind): persistent, 1 CTA / SM, 3 warpgroups:
//   warps 0-3, 4-7  two consumer warpgroups.  Each owns MB x 64 rows of the task's query tile and, for every
//           128-row train tile, issues wgmma.mma_async (m64 n128, one per 64-row block) into registers, waits,
//           hands the shared-memory stage back and keeps a running top-2 per row over its accumulator fragment:
//           group-of-8 min filter against the row's current second best, exact updates only inside a group that
//           beats it.  While one warpgroup runs its epilogue the other one's MMAs keep the tensor cores busy.
//   warps 8-11  producer warpgroup: one thread issues the bulk copies (query tile buffers, train tiles in STAGES
//           stages); the warpgroup hands most of its registers to the consumers (setmaxnreg).
// A thread of the m64 accumulator fragment holds two rows (lane/4 and lane/4 + 8 of its warp's 16) and, of each,
// the columns 8j + 2 (lane%4) + {0, 1}: the four threads of a quad merge their partial top-2 lists at the end of
// a task (lexicographic (value, index), i.e. cv2's insertion order).
#include <cuda_bf16.h>

#include "async_copy.cuh"
#include "common.cuh"
#include "match_common.cuh"

namespace osfm {

constexpr int TC_KD = 128;               // descriptor dims carried
constexpr int TC_KP = 144;               // padded K (9 x 16)
constexpr int TC_KCH = TC_KP / 8;        // 16-byte K chunks per row
constexpr int TC_ROW_BYTES = TC_KP * 2;  // 288
constexpr int TC_LBO = 128;              // bytes between K-adjacent core matrices
constexpr int H8_ROW_BYTES = 512;
constexpr int H8_KCH = H8_ROW_BYTES / 16;   // 16-byte K chunks per row
constexpr int WG_N = 128;                   // train rows per tile (wgmma N)
constexpr int WG_CONSUMERS = 2;             // consumer warpgroups per CTA
constexpr int WG_THREADS = 128 * (WG_CONSUMERS + 1);   // + one producer warpgroup
// Registers: the producer warpgroup releases down to 40 a thread, the consumers take 232 (64 512 of the 65 536).
constexpr int WG_PRODUCER_REGS = 40, WG_CONSUMER_REGS = 232;
static_assert(128 * (WG_PRODUCER_REGS + WG_CONSUMERS * WG_CONSUMER_REGS) <= 65536, "register file of an SM");

enum { KIND_L2 = 0, KIND_HAMMING = 1 };
template <int KIND>
struct WgCfg;
// L2: 256 query rows per task (128 per warpgroup, two m64 blocks = 128 accumulator registers a thread): every train
// tile brought into shared memory feeds 256 rows, which keeps the L2 -> SM traffic at 1.1 bytes per distance.
// Two query buffers let the next task's queries load under the current task.  2 x 72 + 2 x 36 KB = 216 KB.
template <>
struct WgCfg<KIND_L2> {
  static constexpr int ROW_BYTES = TC_ROW_BYTES, MB = 2, QBUF = 2, STAGES = 2;
};
// Hamming: 512 fp8 per row; 128 query rows per task (64 per warpgroup), one query buffer: 64 + 2 x 64 KB = 192 KB.
template <>
struct WgCfg<KIND_HAMMING> {
  static constexpr int ROW_BYTES = H8_ROW_BYTES, MB = 1, QBUF = 1, STAGES = 2;
};
template <int KIND>
struct WgGeom {
  using C = WgCfg<KIND>;
  static constexpr int M = WG_CONSUMERS * C::MB * 64;   // query rows per task
  static constexpr int Q_BYTES = M * C::ROW_BYTES;
  static constexpr int T_BYTES = WG_N * C::ROW_BYTES;
  static constexpr int SBO = C::ROW_BYTES / 16 * 128;   // bytes between 8-row groups
  static constexpr int KSTEPS = C::ROW_BYTES / 32;      // one wgmma K step = 32 bytes of K (k16 bf16 / k32 e4m3)
  static constexpr int SMEM = C::QBUF * Q_BYTES + C::STAGES * T_BYTES;
};
static_assert(WgGeom<KIND_L2>::SMEM <= 227 * 1024 - 1024, "L2 kernel exceeds the H100 shared memory of a block");
static_assert(WgGeom<KIND_HAMMING>::SMEM <= 227 * 1024 - 1024, "Hamming kernel exceeds the H100 shared memory of a block");
static_assert(WgGeom<KIND_L2>::M == 256, "tc_rows_padded pads sets to whole L2 query tiles");

// The library is built for sm_90a only, so this is the H100 class (compute capability 9.0) it can run on.
bool tc_available() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return false;
  int major = 0, minor = 0;
  cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
  cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev);
  return major == 9 && minor == 0;
}

// ---------------------------------------------------------------------------
// Operand preparation
// ---------------------------------------------------------------------------
// One warp per padded row, one pass over the uploaded float32 matrix: exactness check (integers in
// [0,255]), |x|^2, max |x|^2, the zero-padded float32 row of the SIMT kernel (when it is not the
// upload itself) and both bf16 operand roles in the wgmma core-matrix order.
// info[0] |= 1 if any value is not bf16-exact; info[1] = max |x|^2 as float bits.
// SrcT = float (the reference's in-memory form, features.py:169-170) or uint8_t (the on-disk form of HAHOG / SIFT
// descriptors, uploaded as bytes and widened here: a quarter of the host->device traffic).
template <class SrcT>
__global__ void __launch_bounds__(256)
    tc_prepare_set(const SrcT* __restrict__ src, int n, int dim, int rows_padded, float* __restrict__ padded, int dim_padded,
                   float* __restrict__ norm, __nv_bfloat16* __restrict__ qa, __nv_bfloat16* __restrict__ tb,
                   int* __restrict__ info) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows_padded) return;
  float v[4] = {0.f, 0.f, 0.f, 0.f};
  bool bad = false;
  if (row < n) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int k = lane * 4 + e;
      if (k < dim) {
        v[e] = (float)src[(size_t)row * dim + k];
        bad |= !(v[e] >= 0.0f && v[e] <= 255.0f && v[e] == floorf(v[e]));
      }
    }
    if (padded) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int k = lane * 4 + e;
        if (k < dim_padded) padded[(size_t)row * dim_padded + k] = v[e];
      }
    }
  }
  float s = fmaf(v[0], v[0], fmaf(v[1], v[1], fmaf(v[2], v[2], v[3] * v[3])));
#pragma unroll
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  bad = __any_sync(0xffffffffu, bad);
  if (lane == 0) {
    norm[row] = s;
    if (bad) atomicOr(&info[0], 1);
    if (row < n) atomicMax(reinterpret_cast<unsigned*>(&info[1]), __float_as_uint(s));
  }
  // data chunks: lanes 2c and 2c+1 hold the two halves of 16-byte chunk c
  {
    const int c = lane >> 1;
    const size_t off = ((size_t)(row >> 3) * TC_KCH + c) * 64 + (row & 7) * 8 + (lane & 1) * 4;
    __align__(8) __nv_bfloat16 a[4], b[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      a[e] = __float2bfloat16(v[e]);
      b[e] = __float2bfloat16(-2.0f * v[e]);
    }
    *reinterpret_cast<uint2*>(qa + off) = *reinterpret_cast<const uint2*>(a);
    *reinterpret_cast<uint2*>(tb + off) = *reinterpret_cast<const uint2*>(b);
  }
  // augmentation chunk (lane 0) and the zero chunk that pads K to 144 (lane 1)
  if (lane < TC_KCH - TC_KD / 8) {
    const int c = TC_KD / 8 + lane;
    const size_t off = ((size_t)(row >> 3) * TC_KCH + c) * 64 + (row & 7) * 8;
    __align__(16) __nv_bfloat16 a[8], b[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      a[e] = __float2bfloat16(0.0f);
      b[e] = __float2bfloat16(0.0f);
    }
    if (lane == 0) {
      if (row < n) {
        a[0] = a[1] = a[2] = __float2bfloat16(1.0f);
        const __nv_bfloat16 hi = __float2bfloat16(s);
        const float r1 = s - __bfloat162float(hi);
        const __nv_bfloat16 mid = __float2bfloat16(r1);
        const float r2 = r1 - __bfloat162float(mid);
        b[0] = hi; b[1] = mid; b[2] = __float2bfloat16(r2);
      } else {
        // padding trains can never be selected: accumulator = +inf for real queries
        b[0] = __float2bfloat16(__builtin_huge_valf());
      }
    }
    *reinterpret_cast<uint4*>(qa + off) = *reinterpret_cast<const uint4*>(a);
    *reinterpret_cast<uint4*>(tb + off) = *reinterpret_cast<const uint4*>(b);
  }
}

// src: the dense n x dim float32 upload on this stream; padded_dst: the SIMT kernel's zero-padded copy
// to fill as well, or null when the upload already is that copy.  Asynchronous: s.tc_ok is decided by
// Matcher::refresh_info() from d_info[s.slot].
void Matcher::prepare_tc(DescSet& s, const void* src, bool src_u8, float* padded_dst) {
  const int rows_padded = s.rows_padded;
  const size_t op_bytes = (size_t)rows_padded * TC_ROW_BYTES;
  __nv_bfloat16* qa = reinterpret_cast<__nv_bfloat16*>(s.tc_data());
  __nv_bfloat16* tb = reinterpret_cast<__nv_bfloat16*>(s.tc_data() + op_bytes);
  float* norm = reinterpret_cast<float*>(s.tc_data() + 2 * op_bytes);
  if (src_u8)
    tc_prepare_set<uint8_t><<<(rows_padded + 7) / 8, 256, 0, stream>>>(static_cast<const uint8_t*>(src), s.n, s.dim, rows_padded,
                                                                      padded_dst, s.dim_padded, norm, qa, tb, d_info.p + 2 * s.slot);
  else
    tc_prepare_set<float><<<(rows_padded + 7) / 8, 256, 0, stream>>>(static_cast<const float*>(src), s.n, s.dim, rows_padded,
                                                                    padded_dst, s.dim_padded, norm, qa, tb, d_info.p + 2 * s.slot);
  OSFM_LAUNCH_CHECK();
  s.tc_q = qa;
  s.tc_t = tb;
  s.tc_norm = norm;
  s.info_pending = true;
}
int tc_rows_padded(int n) {   // whole query tiles (and whole train tiles) of both kernels
  constexpr int M = WgGeom<KIND_L2>::M;
  return (n + M - 1) / M * M;
}
size_t tc_operand_bytes(int rows_padded) { return 2 * (size_t)rows_padded * TC_ROW_BYTES + (size_t)rows_padded * sizeof(float); }
bool tc_capable(int dim, bool u8) { return !u8 && dim <= TC_KD && tc_available(); }

// ---------------------------------------------------------------------------
// wgmma PTX wrappers (mbarrier and bulk copy: async_copy.cuh)
// ---------------------------------------------------------------------------
// wgmma shared-memory descriptor, K-major without swizzle: start >> 4 @0, LBO >> 4 @16 (K-adjacent core
// matrices), SBO >> 4 @32 (8-row groups), base offset 0 @49, layout type 0 (interleave) @62
template <int SBO>
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr) {
  return (uint64_t)((saddr >> 4) & 0x3fff) | ((uint64_t)((TC_LBO >> 4) & 0x3fff) << 16) |
         ((uint64_t)((SBO >> 4) & 0x3fff) << 32);
}

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// Pins the accumulator registers at this point of the program: the compiler may not move their reads above the
// wait of the asynchronous MMA that writes them, nor their last uses below the next MMA issue.
__device__ __forceinline__ void wg_fence_operands(float (&d)[64]) {
#pragma unroll
  for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

#define OSFM_WG_D8(d, i) \
  "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
#define OSFM_WG_D64(d)                                                                                       \
  OSFM_WG_D8(d, 0), OSFM_WG_D8(d, 8), OSFM_WG_D8(d, 16), OSFM_WG_D8(d, 24), OSFM_WG_D8(d, 32), OSFM_WG_D8(d, 40), \
      OSFM_WG_D8(d, 48), OSFM_WG_D8(d, 56)
#define OSFM_WG_REGS64                                                                                   \
  "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, " \
  "%22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, "  \
  "%42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, "  \
  "%62, %63}"

// D(64 x 128, fp32) (+)= A(64 x K step) * B(K step x 128); accumulate = 0 overwrites D
template <int KIND>
__device__ __forceinline__ void wg_mma(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate);
template <>
__device__ __forceinline__ void wg_mma<KIND_L2>(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n.reg .pred p;\n"
      "setp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 " OSFM_WG_REGS64 ", %64, %65, p, 1, 1, 0, 0;\n}\n"
      : OSFM_WG_D64(d)
      : "l"(adesc), "l"(bdesc), "r"(accumulate)
      : "memory");
}
template <>
__device__ __forceinline__ void wg_mma<KIND_HAMMING>(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n.reg .pred p;\n"
      "setp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k32.f32.e4m3.e4m3 " OSFM_WG_REGS64 ", %64, %65, p, 1, 1;\n}\n"
      : OSFM_WG_D64(d)
      : "l"(adesc), "l"(bdesc), "r"(accumulate)
      : "memory");
}

// Epilogue state of one query row: the two smallest accumulator values (L2: d^2 - |a|^2; Hamming: 2 H - nbits;
// exact integers either way) with their train indices.  For L2, ranking in d^2 is the ranking cv2 uses (sqrt'd
// float32 distance, ties -> lowest index) as long as float32 sqrt is injective on the integers involved, i.e.
// d^2 < 2^22; the host only selects this kernel for descriptor sets whose norms guarantee that bound
// (choose_kernel, match.cu), everything else goes to the exact SIMT kernel.
struct RowState {
  float q1, q2;
  int i1, i2;
};

__device__ __forceinline__ void row_update(RowState& st, float x, int idx) {
  const bool lt1 = x < st.q1;
  const bool lt2 = x < st.q2;
  st.q2 = lt1 ? st.q1 : (lt2 ? x : st.q2);
  st.i2 = lt1 ? st.i1 : (lt2 ? idx : st.i2);
  st.q1 = lt1 ? x : st.q1;
  st.i1 = lt1 ? idx : st.i1;
}

// The 32 values of one row (H = 0: fragment row lane/4, H = 1: lane/4 + 8) in one 64 x 128 accumulator, in
// increasing column order: col0 + 8 j + e for fragment element 4 j + 2 H + e.  Four groups of 8, one min test
// against the row's second best each, exact (predicated) updates only inside a group that beats it.  MASKED
// (guided matching): mw[g] holds the row's mask bits of columns 32 g .. 32 g + 31 shifted to this thread's
// columns; a clear bit reads as +inf and can never enter the row's two best.
template <int H, bool MASKED>
__device__ __forceinline__ void row_consume(RowState& st, const float (&d)[64], int col0, const uint32_t (&mw)[4]) {
#pragma unroll
  for (int g = 0; g < 4; ++g) {
    if (MASKED && (mw[g] & 0x03030303u) == 0u) continue;
    float x[8];
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const float v = d[4 * (4 * g + jj) + 2 * H + e];
        x[2 * jj + e] = (!MASKED || ((mw[g] >> (8 * jj + e)) & 1u)) ? v : __builtin_huge_valf();
      }
    }
    const float m = fminf(fminf(fminf(x[0], x[1]), fminf(x[2], x[3])), fminf(fminf(x[4], x[5]), fminf(x[6], x[7])));
    if (m < st.q2) {
#pragma unroll
      for (int k = 0; k < 8; ++k)
        if (x[k] < st.q2) row_update(st, x[k], col0 + 32 * g + 8 * (k >> 1) + (k & 1));
    }
  }
}

template <int KIND, bool MASKED>
__global__ void __launch_bounds__(WG_THREADS, 1)
    bf_top2_wg(const MatchJob* __restrict__ jobs, const int* __restrict__ tile_prefix, int njobs, int ntasks,
               Top2* __restrict__ partial, int* __restrict__ err_flag) {
  using C = WgCfg<KIND>;
  using G = WgGeom<KIND>;
  constexpr int MB = C::MB, QBUF = C::QBUF, STAGES = C::STAGES;
  constexpr int CONSUMER_WARPS = 4 * WG_CONSUMERS;
  extern __shared__ __align__(1024) uint8_t smem[];
  __shared__ __align__(8) uint64_t bar_qfull[QBUF], bar_qempty[QBUF], bar_full[STAGES], bar_empty[STAGES];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int i = 0; i < QBUF; ++i) {
      mbar_init(&bar_qfull[i], 1);
      mbar_init(&bar_qempty[i], CONSUMER_WARPS);   // one arrival per consumer warp
    }
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&bar_full[i], 1);
      mbar_init(&bar_empty[i], CONSUMER_WARPS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp >= CONSUMER_WARPS) {
    // ===== bulk-copy producer =====
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(WG_PRODUCER_REGS));
    if (warp == CONSUMER_WARPS && lane == 0) {
      int stage = 0, ph = 0, n = 0;
      for (int task = blockIdx.x; task < ntasks; task += gridDim.x, ++n) {
        const MatchTile t = decode_tile<G::M>(jobs, tile_prefix, njobs, task);
        const int ntiles = (t.t_end - t.t_begin + WG_N - 1) / WG_N;
        const int b = n % QBUF, qph = (n / QBUF) & 1;
        mbar_wait(&bar_qempty[b], qph ^ 1, err_flag);
        // the last query tile of a job may hold no rows for the second warpgroup: only the first half is loaded
        const uint32_t qbytes = (t.job.nq - t.q0 > G::M / 2) ? G::Q_BYTES : G::Q_BYTES / 2;
        mbar_expect_tx(&bar_qfull[b], qbytes);
        bulk_copy_g2s(smem + b * G::Q_BYTES, reinterpret_cast<const uint8_t*>(t.job.q_tc) + (size_t)t.q0 * C::ROW_BYTES,
                      qbytes, &bar_qfull[b]);
        for (int i = 0; i < ntiles; ++i) {
          mbar_wait(&bar_empty[stage], ph ^ 1, err_flag);
          mbar_expect_tx(&bar_full[stage], G::T_BYTES);
          bulk_copy_g2s(smem + QBUF * G::Q_BYTES + stage * G::T_BYTES,
                        reinterpret_cast<const uint8_t*>(t.job.t_tc) + (size_t)(t.t_begin + i * WG_N) * C::ROW_BYTES,
                        G::T_BYTES, &bar_full[stage]);
          if (++stage == STAGES) { stage = 0; ph ^= 1; }
        }
      }
    }
    return;
  }

  // ===== consumer warpgroups =====
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(WG_CONSUMER_REGS));
  const int wg = warp >> 2, w = warp & 3, quad = lane & 3;
  const int wg_row0 = wg * MB * 64;   // first query row of this warpgroup in the task's tile
  float acc[MB][64];
#pragma unroll
  for (int mb = 0; mb < MB; ++mb)
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[mb][i] = 0.0f;
  int stage = 0, ph = 0, n = 0;
  for (int task = blockIdx.x; task < ntasks; task += gridDim.x, ++n) {
    const MatchTile t = decode_tile<G::M>(jobs, tile_prefix, njobs, task);
    const int ntiles = (t.t_end - t.t_begin + WG_N - 1) / WG_N;
    const int b = n % QBUF, qph = (n / QBUF) & 1;
    const bool active = t.job.nq - t.q0 > wg_row0;
    RowState st[2 * MB];
#pragma unroll
    for (int r = 0; r < 2 * MB; ++r) {
      st[r].q1 = st[r].q2 = __builtin_huge_valf();
      st[r].i1 = st[r].i2 = -1;
    }
    mbar_wait(&bar_qfull[b], qph, err_flag);
    const uint32_t q_addr = smem_u32(smem + b * G::Q_BYTES) + (wg_row0 / 8) * G::SBO;
    for (int i = 0; i < ntiles; ++i) {
      mbar_wait(&bar_full[stage], ph, err_flag);
      if (active) {
        const uint32_t t_addr = smem_u32(smem + QBUF * G::Q_BYTES + stage * G::T_BYTES);
#pragma unroll
        for (int mb = 0; mb < MB; ++mb) wg_fence_operands(acc[mb]);
        wg_fence();
#pragma unroll
        for (int k = 0; k < G::KSTEPS; ++k) {
          // one K step = 32 bytes of K = two core matrices = 256 bytes further in both operands
          const uint64_t koff = (uint64_t)((k * 2 * TC_LBO) >> 4);
          const uint64_t bdesc = gmma_desc<G::SBO>(t_addr) + koff;
#pragma unroll
          for (int mb = 0; mb < MB; ++mb)
            wg_mma<KIND>(acc[mb], gmma_desc<G::SBO>(q_addr + mb * 8 * G::SBO) + koff, bdesc, k > 0 ? 1u : 0u);
        }
        wg_commit();
        wg_wait_all();
#pragma unroll
        for (int mb = 0; mb < MB; ++mb) wg_fence_operands(acc[mb]);
      }
      // the stage's operands have been read by this warp's MMAs: hand it back before the epilogue
      __syncwarp();
      if (lane == 0) mbar_arrive(&bar_empty[stage]);
      if (++stage == STAGES) { stage = 0; ph ^= 1; }
      if (active) {
        const int col_base = t.t_begin + i * WG_N;
#pragma unroll
        for (int mb = 0; mb < MB; ++mb) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            uint32_t mw[4] = {0u, 0u, 0u, 0u};
            if (MASKED) {
              const int gq = t.q0 + wg_row0 + mb * 64 + 16 * w + (lane >> 2) + 8 * h;
              if (gq < t.job.nq) {
                const uint32_t* mrow = t.job.mask_bits + (size_t)gq * t.job.mask_words;
                const int w0 = col_base >> 5;
#pragma unroll
                for (int q = 0; q < 4; ++q)
                  if (w0 + q < t.job.mask_words) mw[q] = mrow[w0 + q] >> (2 * quad);
              }
            }
            if (h == 0) row_consume<0, MASKED>(st[2 * mb], acc[mb], col_base + 2 * quad, mw);
            else row_consume<1, MASKED>(st[2 * mb + 1], acc[mb], col_base + 2 * quad, mw);
          }
        }
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&bar_qempty[b]);
    if (!active) continue;
#pragma unroll
    for (int r = 0; r < 2 * MB; ++r) {
      Top2 a;
      a.s1 = st[r].q1; a.i1 = st[r].i1; a.s2 = st[r].q2; a.i2 = st[r].i2;
#pragma unroll
      for (int off = 1; off <= 2; off <<= 1) {   // the quad's four column subsets of the row
        Top2 o;
        o.s1 = __shfl_xor_sync(0xffffffffu, a.s1, off);
        o.i1 = __shfl_xor_sync(0xffffffffu, a.i1, off);
        o.s2 = __shfl_xor_sync(0xffffffffu, a.s2, off);
        o.i2 = __shfl_xor_sync(0xffffffffu, a.i2, off);
        top2_merge(a, o);
      }
      // padding trains (index >= nt) lose to every real one but still enter the list of a query with fewer than
      // two real candidates (Hamming scores them finite): a train set of one row must give no match, as in cv2
      if (a.i2 >= t.job.nt) a.i2 = -1;
      if (a.i1 >= t.job.nt) a.i1 = -1;
      const int gq = t.q0 + wg_row0 + (r >> 1) * 64 + 16 * w + (lane >> 2) + 8 * (r & 1);
      if (quad == 0 && gq < t.job.nq) {
        Top2 out;
        if (KIND == KIND_L2) {   // squared distances (exact integers in fp32)
          const float na = t.job.q_norm[gq];
          out.s1 = a.i1 >= 0 ? fmaxf(a.s1 + na, 0.0f) : __builtin_huge_valf();
          out.s2 = a.i2 >= 0 ? fmaxf(a.s2 + na, 0.0f) : __builtin_huge_valf();
        } else {                 // accumulator = 2 H - nbits  ->  the Hamming distance cv2 reports
          const float nbits = (float)(t.job.dim * 8);
          out.s1 = a.i1 >= 0 ? (a.s1 + nbits) * 0.5f : __builtin_huge_valf();
          out.s2 = a.i2 >= 0 ? (a.s2 + nbits) * 0.5f : __builtin_huge_valf();
        }
        out.i1 = a.i1;
        out.i2 = a.i2;
        partial[t.job.partial_off + (size_t)t.chunk * t.job.nq + gq] = out;
      }
    }
  }
}

// ===========================================================================================================
// Hamming distance on the tensor cores ("BruteForce-Hamming": AKAZE MLDB 61 bytes, ORB 32 bytes).
//
// Bits become +-1 in fp8 (E4M3: +1 = 0x38, -1 = 0xB8, both exact): for two descriptors a, b of nbits bits
//     sum_i a_i b_i = (#equal bits) - (#different bits) = nbits - 2 H(a, b),
// so with the train operand negated the fp32 accumulator is 2 H - nbits, an exact integer (|value| <= 512, well
// inside the precision the fp8 MMA keeps), and its ranking inside a query row is cv2's ranking by Hamming distance
// (ties -> lowest index through the same epilogue as the L2 kernel).  K = 512 fp8 per row; positions beyond nbits
// are 0 in real rows of both roles (they add nothing), +1 in every query row and +448 in the *padding* rows of a
// train set, so a padding train scores >= 8 * 448 - nbits > any real one and never ranks above it (needs >= 8 spare
// positions: nbytes <= 63); the epilogue drops the padding trains a query with fewer than two real ones keeps.  wgmma m64 n128 k32 e4m3, operands in the same no-swizzle K-major core-matrix order as
// the bf16 kernel (a core matrix row is 16 bytes = 16 fp8), 512 B per row.
// ===========================================================================================================
size_t h8_operand_bytes(int rows_padded) { return 2 * (size_t)rows_padded * H8_ROW_BYTES; }
bool h8_capable(int nbytes) { return nbytes >= 1 && nbytes <= 63 && tc_available(); }

// one thread per (row, 16-byte K chunk): 16 bits of the source row -> 16 fp8 values in both roles
__global__ void __launch_bounds__(256)
    h8_prepare_set(const uint8_t* __restrict__ src, int n, int nbytes, int src_stride, int rows_padded, uint8_t* __restrict__ qa,
                   uint8_t* __restrict__ tb) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (size_t)rows_padded * H8_KCH) return;
  const int row = (int)(idx / H8_KCH), c = (int)(idx % H8_KCH);
  const int nbits = nbytes * 8;
  __align__(16) uint8_t a[16], b[16];
#pragma unroll
  for (int e = 0; e < 16; ++e) {
    const int bit = c * 16 + e;
    uint8_t va = 0, vb = 0;
    if (row < n) {
      if (bit < nbits) {
        const int on = (src[(size_t)row * src_stride + (bit >> 3)] >> (bit & 7)) & 1;
        va = on ? 0x38 : 0xB8;   // +1 / -1
        vb = on ? 0xB8 : 0x38;   // negated
      } else {
        va = 0x38;               // +1 against the padding trains' markers
      }
    } else if (bit >= nbits) {
      vb = 0x7E;                 // +448: a padding train can never win
    }
    a[e] = va; b[e] = vb;
  }
  const size_t off = ((size_t)(row >> 3) * H8_KCH + c) * 128 + (row & 7) * 16;
  *reinterpret_cast<uint4*>(qa + off) = *reinterpret_cast<const uint4*>(a);
  *reinterpret_cast<uint4*>(tb + off) = *reinterpret_cast<const uint4*>(b);
}

void Matcher::prepare_h8(DescSet& s, const uint8_t* src, int src_stride) {
  const size_t op_bytes = (size_t)s.rows_padded * H8_ROW_BYTES;
  uint8_t* qa = reinterpret_cast<uint8_t*>(s.tc_data());
  uint8_t* tb = qa + op_bytes;
  const size_t total = (size_t)s.rows_padded * H8_KCH;
  h8_prepare_set<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(src, s.n, s.dim, src_stride, s.rows_padded, qa, tb);
  OSFM_LAUNCH_CHECK();
  s.tc_q = reinterpret_cast<const __nv_bfloat16*>(qa);
  s.tc_t = reinterpret_cast<const __nv_bfloat16*>(tb);
  s.tc_norm = nullptr;
  s.tc_ok = true;
}

template <int KIND, bool MASKED>
static void launch_wg(Matcher& m, int njobs, int ntasks, int smem) {
  m.opt_in_smem(bf_top2_wg<KIND, MASKED>, smem);
  m.d_flags.reserve(4);
  OSFM_CUDA(cudaMemsetAsync(m.d_flags.p + 1, 0, sizeof(int), m.stream));
  const int grid = std::min(ntasks, m.num_sms);
  bf_top2_wg<KIND, MASKED><<<grid, WG_THREADS, smem, m.stream>>>(m.d_jobs.p, m.d_prefix.p, njobs, ntasks, m.d_partial.p,
                                                                 m.d_flags.p + 1);
  OSFM_LAUNCH_CHECK();
}

// Persistent CTAs over WG_N-row train tiles; the trains are split until there are two tasks per SM.
KernelPlan tc_plan(DistKernel kernel, bool masked) {
  if (kernel == DistKernel::TC_HAMMING)
    return {WgGeom<KIND_HAMMING>::M, WG_N, 2, false, WgGeom<KIND_HAMMING>::SMEM, launch_wg<KIND_HAMMING, false>};
  return {WgGeom<KIND_L2>::M, WG_N, 2, true, WgGeom<KIND_L2>::SMEM,
          masked ? launch_wg<KIND_L2, true> : launch_wg<KIND_L2, false>};
}

}  // namespace osfm
