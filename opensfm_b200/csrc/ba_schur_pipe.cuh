// Segment Schur complement, persistent and warp-specialised (included by ba.cu after ba_reduced.cuh).
//
// Same mathematics and the same per-segment tables as ba_schur_mma (ba_reduced.cuh): per chunk of SM_PCH points of a
// segment the operands Yt = -(W V^-1)^T, Wt = W^T, Jt = Js^T are built in shared memory and the upper 8x8 tiles of
// sum_p (U_p - Y_p W_p^T) are accumulated with mma.m8n8k4.f64, flushed once per segment with fp64 atomics.
// What changes is the schedule.  ba_schur_mma runs one CTA per segment, and its phases (tables, loads, rows, mma,
// flush) are separated by CTA barriers: 40k clocks per segment of which the tensor pipe is busy ~4k (OSFM_BA_TRACE).
// Here one CTA per SM walks a contiguous range of chunks (ranges cut at segment boundaries, balanced by chunk count):
//   * 8 producer warps (two threads per observation of the chunk, each half of the camera-side columns): cp.async the
//     residual / Jacobian plane values, the point blocks and the column scales of chunk n + 1 into a staging buffer
//     while they build the operands of chunk n from the other staging buffer into one of two operand buffers
//     (mbarrier full / empty ring);
//   * two consumer groups of 6 warps each: a group owns every other segment (segment index parity), multiplies the
//     chunks of its segment out of the operand ring and then flushes its accumulators; while one group flushes the
//     other one keeps the tensor pipe busy.  A warp owns the tile rows (p, nt - 1 - p) of the upper triangle (nt + 1
//     tiles for every p): the A fragment of a row is loaded once per k-step and reused by all its tiles (1.2
//     shared-memory loads per DMMA instead of 2).
//   * The flush is a table lookup.  Decoding where an accumulator element goes (shot pair -> parameter-block pair ->
//     block offset, transposed / diagonal / shared-block cases) takes ~50 instructions per element, 4455 elements per
//     segment: 40 % of all instructions of ba_schur_mma, and 20k clocks per segment for the 6 warps of a group here.
//     The destinations depend only on the structure, so sp_flush_tables writes them once per run(): one int per
//     (segment, warp, tile slot, fragment element, lane) = (offset << 2 | add-U flag | double flag) or -1
//     (20 KB per segment, 430 MB at C4).  A warp prefetches its 3.3 KB with cp.async at the start of a segment.
//     (scattered fp64 RED into L2 are several times slower than a warp's RED to 32 consecutive elements, and a C4
//     launch issues 87M of them.)
// Eligible: wc == 9, nres == 2 (a 3-parameter camera and a pose per shot), the camera side of the chunk list;
// everything else keeps ba_schur_mma.  OSFM_BA_FALLBACK_CTA_PER_SEGMENT_SCHUR switches back for A/B runs.
#pragma once

#include "async_copy.cuh"

namespace osfm {

constexpr int SP_PROD_WARPS = 8;
constexpr int SP_CONS_WARPS = 6;                    // per consumer group: one per pair of tile rows
constexpr int SP_PROD_THREADS = 32 * SP_PROD_WARPS;
constexpr int SP_CONS_THREADS = 32 * SP_CONS_WARPS;
constexpr int SP_THREADS = SP_PROD_THREADS + 2 * SP_CONS_THREADS;   // 640
constexpr int SP_ROWS = 26;                         // staged plane rows: r (nres) + Jp (3 nres) + Jc (wc nres)
static_assert(SP_ROWS == 2 * (1 + 3 + 9), "the plane rows of an observation with wc == 9, nres == 2");
constexpr int SP_OBS = SM_PCH * SEG_KMAX;           // 128 observations per chunk at most
constexpr int SP_SLOTS = SM_NT + 1;                 // tiles of a row pair (p, nt - 1 - p): nt + 1
constexpr int SP_NPAIR9 = 9 * (SEG_KMAX * (SEG_KMAX + 1) / 2);
static_assert(2 * SP_OBS == SP_PROD_THREADS, "two producer threads per observation of a chunk");
static_assert(2 * SP_CONS_WARPS >= SM_NT, "a consumer warp per pair of tile rows");

struct SchurChunk {      // 48 bytes, read with three 16-byte loads
  long long ibase;       // first observation of the chunk (sorted order)
  long long tab_off;     // per-segment tables of its segment (offset into tab, ints)
  int p0, pf0;           // first local point; its free-point offset (-1: the segment's points are constant)
  int seg, seg_chunk0;   // segment, first chunk of that segment
  int seg_nch, np;       // chunks of the segment, points in this chunk
  int k, pad;
};
static_assert(sizeof(SchurChunk) == 48, "three int4");

__global__ void sp_chunk_counts(BAView v, const int* __restrict__ seg_start, int nseg, int* __restrict__ nch) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s > nseg) return;
  nch[s] = s == nseg ? 0 : (seg_start[s + 1] - seg_start[s] + SM_PCH - 1) / SM_PCH;
}
// one warp per segment
__global__ void sp_fill_chunks(BAView v, const int* __restrict__ seg_start, int nseg, const int* __restrict__ chunk0,
                               const long long* __restrict__ tab_off, SchurChunk* __restrict__ out) {
  const int s = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (s >= nseg) return;
  const int p_begin = seg_start[s], p_end = seg_start[s + 1];
  const long long o0 = v.pt_start[p_begin];
  const int k = (int)(v.pt_start[p_begin + 1] - o0);
  const int c0 = chunk0[s], nch = chunk0[s + 1] - c0;
  const int pf_first = v.pt_poff[p_begin];
  for (int c = threadIdx.x & 31; c < nch; c += 32) {
    SchurChunk e;
    e.p0 = p_begin + c * SM_PCH;
    e.np = min(SM_PCH, p_end - e.p0);
    e.ibase = o0 + (long long)c * SM_PCH * k;
    e.tab_off = tab_off[s];
    e.pf0 = pf_first >= 0 ? pf_first + c * SM_PCH : -1;
    e.seg = s; e.seg_chunk0 = c0; e.seg_nch = nch; e.k = k; e.pad = 0;
    out[c0 + c] = e;
  }
}

struct SpOperand {
  double Yt[SM_KC][SM_LD];
  double Wt[SM_KC][SM_LD];
  double Jt[SM_KC][SM_LD];
  double G[SM_PCH][SEG_NA];
};
static_assert(sizeof(SpOperand) >= sizeof(double) * (SEG_NA * SEG_NA + SEG_NA * SEG_WCMAX) / 2, "the flush tile of a segment fits");
struct SpStage {
  double pl[SP_ROWS][SP_OBS];
  double ptd[SM_PCH][12];   // V^-1 (6), V^-1 g_p (3), Jacobi scale of the point (3)
  double scol[SEG_NA];
};
constexpr int SP_FT_WARP = SP_SLOTS * 2 * 32;                   // flush-table ints of one warp
constexpr int SP_FT_SEG = SP_CONS_WARPS * SP_FT_WARP;            // ... of one segment
struct SpFlush {      // per consumer group: the flush table of its current segment + gcol
  int t[SP_CONS_WARPS][SP_FT_WARP];
  int gcol[SEG_NA];
};
struct SpSmem {
  SpOperand op[2];
  SpStage st[2];
  SpFlush ft[2];
  // full[group][buffer]: a group waits only for the chunks it owns, so it has to see every phase of the barrier it
  // waits on (mbarrier parity waits cannot tell phase u + 1 from phase u - 1) -> one "full" barrier per (group, buffer);
  // empty[buffer] is waited on by the producers alone, once per use.
  uint64_t full[2][2], empty[2];
};

__device__ __forceinline__ void sp_cp8(void* dst, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void sp_cp4(void* dst, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void sp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void sp_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void sp_bar(int id, int count) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory"); }
__device__ __forceinline__ SchurChunk sp_load_chunk(const SchurChunk* chunks, int n) {
  const int4* p = reinterpret_cast<const int4*>(chunks + n);
  union { int4 q[3]; SchurChunk e; } u;
  u.q[0] = __ldg(p); u.q[1] = __ldg(p + 1); u.q[2] = __ldg(p + 2);
  return u.e;
}

// Flush destinations of every (segment, consumer warp, tile slot, fragment element, lane): the same decoding as the
// flush of ba_schur_mma, done once per run() (grid = segments, block = SP_CONS_THREADS).
__global__ void __launch_bounds__(SP_CONS_THREADS)
    sp_flush_tables(BAView v, const int* __restrict__ seg_start, const long long* __restrict__ tab_off,
                    const int* __restrict__ tab, int* __restrict__ ftab) {
  const int s = blockIdx.x;
  const int cw = threadIdx.x >> 5, lane = threadIdx.x & 31, fr = lane >> 2, fk = lane & 3;
  const int wc = v.wc;
  const int p0 = seg_start[s];
  const int k = (int)(v.pt_start[p0 + 1] - v.pt_start[p0]);
  const int ncols = k * wc, nt = (ncols + 7) >> 3;
  const int* T = tab + tab_off[s];
  const int* meta = T + ncols;
  const int* offt = T + 2 * ncols;
  const bool active = cw < ((nt + 1) >> 1);
  const int rowA = active ? cw : 0, rowB = active ? nt - 1 - cw : 0;
  const int nA = active ? nt - rowA : 0, nB = (active && rowB > rowA) ? nt - rowB : 0;
  int* out = ftab + (size_t)s * SP_FT_SEG + cw * SP_FT_WARP + lane;
  for (int j = 0; j < SP_SLOTS; ++j) {
    const bool isA = j < nA;
    const int jj = isA ? j : j - nA;
    const int ti = isA ? rowA : rowB, tj = ti + jj;
    const int row = 8 * ti + fr;
    for (int el = 0; el < 2; ++el) {
      int code = -1;
      const int col = 8 * tj + 2 * fk + el;
      if (j < nA + nB && row < ncols && col < ncols) {
        const int m1 = meta[row], m2 = meta[col];
        const int a = row / wc, bb = col / wc;
        if (m1 >= 0 && m2 >= 0 && a <= bb) {
          const int B1 = m1 >> 12, s1 = (m1 >> 10) & 3, sz1 = (m1 >> 5) & 31, r1 = m1 & 31;
          const int B2 = m2 >> 12, s2 = (m2 >> 10) & 3, sz2 = (m2 >> 5) & 31, r2 = m2 & 31;
          int pos = -1, dbl = 0;
          if (B1 < B2) {
            pos = r1 * sz2 + r2;
          } else if (B1 > B2) {
            if (a != bb) pos = r2 * sz1 + r1;
          } else if (a == bb) {
            if (r2 >= r1) pos = r1 * sz1 + r2;
          } else {
            dbl = r1 == r2;
            pos = min(r1, r2) * sz1 + max(r1, r2);
          }
          if (pos >= 0)
            code = ((offt[seg_pair_index(a, bb, k) * 9 + s1 * 3 + s2] + pos) << 2) | ((a == bb && jj < 2) ? 1 : 0) | (dbl ? 2 : 0);
        }
      }
      out[(j * 2 + el) * 32] = code;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------
// Camera-side gradient and squared column norms over the chunk list (wc == 9, nres == 2): a warp owns a contiguous
// range of chunks (cut at segment starts), reads one 48-byte entry per chunk (the entry of chunk n + 1 is in registers
// while chunk n is reduced; walking seg_start / pt_start instead costs three dependent loads per chunk before the next
// copy can be issued) and takes the global columns from the per-segment table.  Staging: one bulk copy (TMA engine)
// per plane row and chunk, two stages per warp, one mbarrier each.
// ---------------------------------------------------------------------------------------------------------
constexpr int CC_WARPS = 5;
constexpr int CC_ROWS = 20;                       // r[2] + Jc[2 * 9]
constexpr int CC_STAGE_DOUBLES = CC_ROWS * SP_OBS;
constexpr int CC_SMEM = CC_WARPS * 2 * CC_STAGE_DOUBLES * (int)sizeof(double);   // 204,800 bytes

__global__ void __launch_bounds__(32 * CC_WARPS, 1)
    ba_colnorm_grad_chunks(BAView v, const SchurChunk* __restrict__ chunks, int nchunks, const int* __restrict__ tab,
                           double* colnorm2, double* grad) {
  extern __shared__ __align__(128) double cc_tiles[];
  __shared__ __align__(8) uint64_t bars[CC_WARPS][2];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int w = 0; w < CC_WARPS; ++w)
      for (int st = 0; st < 2; ++st) mbar_init(&bars[w][st], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  double* tile[2] = {cc_tiles + (size_t)(warp * 2) * CC_STAGE_DOUBLES, cc_tiles + (size_t)(warp * 2 + 1) * CC_STAGE_DOUBLES};
  const size_t N = (size_t)v.N;
  const int gw = blockIdx.x * CC_WARPS + warp, nw = gridDim.x * CC_WARPS;
  auto cut = [&](int b) -> int {
    if (b <= 0) return 0;
    const long long c = (long long)b * nchunks / nw;
    if (c >= nchunks) return nchunks;
    const SchurChunk e = sp_load_chunk(chunks, (int)c);
    return e.seg_chunk0 == (int)c ? (int)c : e.seg_chunk0 + e.seg_nch;
  };
  const int c_lo = cut(gw), c_hi = cut(gw + 1);
  if (c_lo >= c_hi) return;

  // returns whether the bulk-copy path was used (every plane run 16-byte aligned)
  auto stage = [&](int st, const SchurChunk& e) -> bool {
    const int run = e.np * e.k;
    const bool aligned = ((e.ibase | (long long)run | (long long)N) & 1LL) == 0;
    if (aligned) {
      if (lane == 0) {
        const uint32_t bytes = (uint32_t)run * 8u;
        mbar_expect_tx(&bars[warp][st], bytes * CC_ROWS);
        for (int row = 0; row < CC_ROWS; ++row) {
          const double* src = (row < 2 ? v.r + (size_t)row * N : v.Jc + (size_t)(row - 2) * N) + e.ibase;
          bulk_copy_g2s(tile[st] + row * SP_OBS, src, bytes, &bars[warp][st]);
        }
      }
    } else {
      for (int idx = lane; idx < CC_ROWS * run; idx += 32) {
        const int row = idx / run, el = idx - row * run;
        tile[st][row * SP_OBS + el] = (row < 2 ? v.r + (size_t)row * N : v.Jc + (size_t)(row - 2) * N)[e.ibase + el];
      }
    }
    return aligned;
  };

  SchurChunk e = sp_load_chunk(chunks, c_lo);
  bool cur_tma = stage(0, e);
  unsigned phase0 = 0u, phase1 = 0u;
  double n2[3] = {0.0, 0.0, 0.0}, gr[3] = {0.0, 0.0, 0.0};
  int col[3] = {-1, -1, -1};
  for (int n = c_lo; n < c_hi; ++n) {
    const int st = (n - c_lo) & 1;
    SchurChunk en = e;
    bool next_tma = false;
    if (n + 1 < c_hi) {
      en = sp_load_chunk(chunks, n + 1);
      next_tma = stage(st ^ 1, en);
    }
    const int k = e.k, np = e.np, nacc = k * 9;
    if (n == e.seg_chunk0) {
#pragma unroll
      for (int u = 0; u < 3; ++u) {
        const int a = lane + 32 * u;
        col[u] = a < nacc ? __ldg(tab + e.tab_off + a) : -1;
        n2[u] = 0.0; gr[u] = 0.0;
      }
    }
    if (cur_tma) {
      mbar_wait(&bars[warp][st], st ? phase1 : phase0);
      if (st) phase1 ^= 1u; else phase0 ^= 1u;
    } else {
      __syncwarp();
    }
    const double* T = tile[st];
#pragma unroll
    for (int u = 0; u < 3; ++u) {
      const int a = lane + 32 * u;
      if (a < nacc) {
        const int c = a / 9, j = a - c * 9;
        for (int pi = 0; pi < np; ++pi) {
          const int el = pi * k + c;
          const double j0 = T[(2 + j) * SP_OBS + el], j1 = T[(2 + 9 + j) * SP_OBS + el];
          n2[u] += j0 * j0 + j1 * j1;
          gr[u] += j0 * T[el] + j1 * T[SP_OBS + el];
        }
      }
    }
    __syncwarp();   // the tile may be overwritten by the copy issued in the next iteration
    if (n == e.seg_chunk0 + e.seg_nch - 1) {
#pragma unroll
      for (int u = 0; u < 3; ++u)
        if (col[u] >= 0) { atomicAdd(&colnorm2[col[u]], n2[u]); atomicAdd(&grad[col[u]], gr[u]); }
    }
    e = en;
    cur_tma = next_tma;
  }
}

// ---------------------------------------------------------------------------------------------------------
// Linearisation over the chunk list, with the reductions that otherwise re-read the planes it writes (every camera
// perspective, no rig cameras: wc == 9, nres == 2).  Every thread evaluates one observation as ba_linearize<1, NB, TYPE> does and writes the
// same planes; it also puts the 27 products its observation adds to the sums into shared memory:
//   camera side  Jc_j^2 and Jc_j r (9 columns each, summed over the two residual rows),
//   point side   the upper triangle of Jp^T Jp (6) and Jp^T r (3).
// CTA b owns the chunks that start in the observation window [b W, (b + 1) W) of the segment observations: whole
// chunks, so whole points, fewer than W + SP_OBS observations, handled in passes of FL_THREADS.  After a pass
//   * the first thread of every point (of its part in the pass) sums the point's products in observation order and,
//     once the point is complete, stores its column norms and gradient into colnorm2 / grad and the nine sums into
//     ptsum[9][npf] (ba_point_blocks_sums) with plain stores: no other CTA sees the point;
//   * thread (segment piece, shot slot c, column j) sums the piece's products of that column, and issues one fp64
//     atomic per column into colnorm2 / grad when the piece ends (destinations from the per-segment table, -1 for
//     constant blocks).
// A point or a piece that crosses the pass boundary carries its partial sums in shared memory.  CTAs past the last
// window linearise the observations outside the segments ([n_fast, N)) without reductions.
// ---------------------------------------------------------------------------------------------------------
constexpr int FL_THREADS = 128;             // observations per pass
constexpr int FL_WIN = 128;                 // observation window of a CTA's chunk starts
constexpr int FL_MAXCH = FL_WIN;            // chunk starts in one window (a chunk has at least one observation)
constexpr int FL_NV = 27;                   // products per observation: 9 + 9 camera side, 6 + 3 point side
static_assert(FL_WIN + SP_OBS <= 2 * FL_THREADS, "a CTA's observations take at most two passes");

struct FlSmem {
  double st[FL_NV][FL_THREADS];             // products of the pass's observations
  double cost[FL_THREADS];                  // per thread, over the passes
  double pcarry[9];                         // the point that crosses the pass boundary
  double ccarry[2][SEG_KMAX * 9];           // the segment piece that crosses it
  long long pc_tab[FL_MAXCH];               // per piece: its segment's table (offset into tab)
  int ch_lo[FL_MAXCH + 1];                  // per chunk: first observation, relative to the CTA's first; [nch] = end
  int ch_k[FL_MAXCH], ch_pf[FL_MAXCH], ch_seg[FL_MAXCH];
  int pc_lo[FL_MAXCH + 1], pc_k[FL_MAXCH], pc_item0[FL_MAXCH + 1];   // pieces (runs of one segment's chunks)
  int nch, npc;
  long long base;
};

// last index q in [lo, hi) with a[q] <= x (a ascending, a[lo] <= x)
__device__ __forceinline__ int fl_find(const int* a, int lo, int hi, int x) {
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (a[mid] <= x) lo = mid; else hi = mid;
  }
  return lo;
}

// One observation, as the uniform-type branch of ba_linearize<1>: writes r, Jc, Jp and returns the cost.  With PROD
// also its FL_NV products, st[q * FL_THREADS] (formed column by column, so that the weighted values need not stay
// live together).
template <int TYPE, bool PROD>
__device__ __forceinline__ double fl_eval(const BAView& v, const Params& p, long long i, double* st) {
  const int shot = v.obs_shot[i];
  const int cam = v.shot_cam[shot];
  constexpr int C = 3;
  const int pt = v.obs_point[i];
  double camp[MAX_CAM_PARAMS], ri[6], rc[6], X[3];
#pragma unroll
  for (int j = 0; j < C; ++j) camp[j] = p.cam[v.cam_off[cam] + j];
#pragma unroll
  for (int j = 0; j < 6; ++j) ri[j] = p.inst[6 * (size_t)v.shot_inst[shot] + j];
#pragma unroll
  for (int j = 0; j < 3; ++j) X[j] = p.pts[3 * (size_t)pt + j];
  double r[3], jc[3 * MAX_CAM_PARAMS], jri[18], jrc[18], jp[9];
  observation_eval(TYPE, camp, ri, rc, false, X, v.obs_x[i], v.obs_y[i], v.obs_isig[i], r, jc, jri, jrc, jp);
  const double s = r[0] * r[0] + r[1] * r[1];
  double w;
  double cost = 0.5 * robust_loss(v.loss, v.loss_a, s, &w);
  const bool pfree = v.pt_poff[pt] >= 0;
  if (!pfree && v.cam_poff[cam] < 0 && v.inst_poff[v.shot_inst[shot]] < 0) cost = 0.0;   // see ba_linearize
  const size_t N = (size_t)v.N;
  const double r0 = w * r[0], r1 = w * r[1];
  v.r[i] = r0;
  v.r[N + i] = r1;
#pragma unroll
  for (int j = 0; j < 9; ++j) {
    const double a0 = w * (j < C ? jc[j] : jri[j - C]), a1 = w * (j < C ? jc[C + j] : jri[6 + j - C]);
    v.Jc[(size_t)j * N + i] = a0;
    v.Jc[(size_t)(9 + j) * N + i] = a1;
    if (PROD) {
      st[j * FL_THREADS] = a0 * a0 + a1 * a1;
      st[(9 + j) * FL_THREADS] = a0 * r0 + a1 * r1;
    }
  }
  double x[2][3];
#pragma unroll
  for (int k = 0; k < 2; ++k)
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      x[k][j] = pfree ? w * jp[k * 3 + j] : 0.0;
      v.Jp[((size_t)k * 3 + j) * N + i] = x[k][j];
    }
  if (PROD) {
    st[18 * FL_THREADS] = x[0][0] * x[0][0] + x[1][0] * x[1][0];
    st[19 * FL_THREADS] = x[0][0] * x[0][1] + x[1][0] * x[1][1];
    st[20 * FL_THREADS] = x[0][0] * x[0][2] + x[1][0] * x[1][2];
    st[21 * FL_THREADS] = x[0][1] * x[0][1] + x[1][1] * x[1][1];
    st[22 * FL_THREADS] = x[0][1] * x[0][2] + x[1][1] * x[1][2];
    st[23 * FL_THREADS] = x[0][2] * x[0][2] + x[1][2] * x[1][2];
    st[24 * FL_THREADS] = x[0][0] * r0 + x[1][0] * r1;
    st[25 * FL_THREADS] = x[0][1] * r0 + x[1][1] * r1;
    st[26 * FL_THREADS] = x[0][2] * r0 + x[1][2] * r1;
  }
  return cost;
}

template <int TYPE>
__global__ void __launch_bounds__(FL_THREADS, 5)
    ba_linearize_fused(BAView v, Params p, Scalars* sc, const SchurChunk* __restrict__ chunks, int nchunks,
                       long long n_fast, const int* __restrict__ tab, double* __restrict__ colnorm2,
                       double* __restrict__ grad, double* __restrict__ ptsum) {
  static_assert(TYPE == PT_PERSPECTIVE, "3 camera parameters + 6 pose parameters = 9 columns; the fisheye model does "
                                       "not fit the 5-CTA register bound without spills");
  __shared__ FlSmem sm;
  const int t = threadIdx.x;
  const long long nwin = (n_fast + FL_WIN - 1) / FL_WIN;
  double cost = 0.0;
  if (blockIdx.x >= nwin) {   // observations outside the segments: planes and cost only
    const long long i = n_fast + (blockIdx.x - nwin) * (long long)FL_THREADS + t;
    if (i < v.N) cost = fl_eval<TYPE, false>(v, p, i, nullptr);
  } else {
    // ---- chunks of the window, and their runs by segment ("pieces") ----
    if (t == 0) {
      const long long w0 = (long long)blockIdx.x * FL_WIN, w1 = min(w0 + FL_WIN, n_fast);
      auto first_at = [&](long long x) {   // first chunk with ibase >= x
        int lo = 0, hi = nchunks;
        while (lo < hi) {
          const int mid = (lo + hi) >> 1;
          if (__ldg(&chunks[mid].ibase) < x) lo = mid + 1; else hi = mid;
        }
        return lo;
      };
      const int c_lo = first_at(w0), c_hi = first_at(w1);
      sm.nch = c_hi - c_lo;
      sm.ch_seg[0] = c_lo;   // passed on to the loaders below
      sm.base = c_lo < nchunks ? __ldg(&chunks[c_lo].ibase) : n_fast;
      sm.ch_lo[sm.nch] = (int)((c_hi < nchunks ? __ldg(&chunks[c_hi].ibase) : n_fast) - sm.base);
    }
    __syncthreads();
    const int nch = sm.nch, c_lo = sm.ch_seg[0];
    const long long base = sm.base;
    __syncthreads();   // ch_seg[0] is overwritten below
    if (nch > 0) {   // (uniform over the CTA)
      for (int q = t; q < nch; q += FL_THREADS) {
        const SchurChunk e = sp_load_chunk(chunks, c_lo + q);
        sm.ch_lo[q] = (int)(e.ibase - base);
        sm.ch_k[q] = e.k;
        sm.ch_pf[q] = e.pf0;
        sm.ch_seg[q] = e.seg;
        if (q == 0 || e.seg_chunk0 == c_lo + q) sm.pc_tab[q] = e.tab_off;   // a piece starts here
      }
      __syncthreads();
      if (t == 0) {
        int npc = 0, item = 0;
        for (int q = 0; q < nch; ++q) {
          if (q == 0 || sm.ch_seg[q] != sm.ch_seg[q - 1]) {
            sm.pc_lo[npc] = sm.ch_lo[q];
            sm.pc_k[npc] = sm.ch_k[q];
            sm.pc_tab[npc] = sm.pc_tab[q];   // npc <= q: written before it is read again
            sm.pc_item0[npc] = item;
            item += 9 * sm.ch_k[q];
            ++npc;
          }
        }
        sm.pc_lo[npc] = sm.ch_lo[nch];
        sm.pc_item0[npc] = item;
        sm.npc = npc;
      }
      sm.cost[t] = 0.0;
      __syncthreads();
      // the loop state is re-read from shared memory after every barrier: nothing but p0 and the cost stays live
      // across the evaluation, which needs every register the 5-CTA bound leaves
      for (int p0 = 0; p0 < sm.ch_lo[sm.nch]; p0 += FL_THREADS) {
        if (p0 + t < sm.ch_lo[sm.nch]) sm.cost[t] += fl_eval<TYPE, true>(v, p, sm.base + p0 + t, &sm.st[0][t]);
        __syncthreads();
        const int nch = sm.nch, npc = sm.npc;
        const int p1 = min(sm.ch_lo[nch], p0 + FL_THREADS);
        const int e = p0 + t;
        int ch = 0, k = 1, c = 0, pi = 0;   // chunk of observation e, point in the chunk, shot slot
        if (e < p1) {
          ch = fl_find(sm.ch_lo, 0, nch, e);
          k = sm.ch_k[ch];
          const int rel = e - sm.ch_lo[ch];
          pi = rel / k;
          c = rel - pi * k;
        }
        // point side: the first thread of every point's part in this pass
        if (e < p1 && (c == 0 || e == p0)) {
          const int run = min(k - c, p1 - e);
          double s[9];
#pragma unroll
          for (int q = 0; q < 9; ++q) s[q] = c != 0 ? sm.pcarry[q] : 0.0;
          for (int u = 0; u < run; ++u) {
#pragma unroll
            for (int q = 0; q < 9; ++q) s[q] += sm.st[18 + q][t + u];
          }
          if (c + run == k) {
            const int pf0 = sm.ch_pf[ch];
            if (pf0 >= 0) {
              const int pf = pf0 + pi;
              const size_t NP = (size_t)v.npf;
              const size_t col = (size_t)v.nc + 3 * (size_t)pf;
              colnorm2[col] = s[0]; colnorm2[col + 1] = s[3]; colnorm2[col + 2] = s[5];
              grad[col] = s[6]; grad[col + 1] = s[7]; grad[col + 2] = s[8];
#pragma unroll
              for (int q = 0; q < 9; ++q) ptsum[q * NP + pf] = s[q];
            }
          } else {   // continues in the next pass (read there by its thread 0, after two barriers)
#pragma unroll
            for (int q = 0; q < 9; ++q) sm.pcarry[q] = s[q];
          }
        }
        // camera side: items (piece, c, j) of the pieces that overlap this pass
        const int qa = fl_find(sm.pc_lo, 0, npc, p0), qb = fl_find(sm.pc_lo, 0, npc, p1 - 1) + 1;
        const int i0 = sm.pc_item0[qa], i1 = sm.pc_item0[qb];
        for (int it = i0 + t; it < i1; it += FL_THREADS) {
          const int q = fl_find(sm.pc_item0, qa, qb, it);
          const int a = it - sm.pc_item0[q];
          const int kq = sm.pc_k[q], cq = a / 9, j = a - cq * 9;
          const int lo = sm.pc_lo[q], hi = sm.pc_lo[q + 1];
          int e0 = lo + cq;   // first observation of slot cq at or after p0
          if (e0 < p0) e0 += (p0 - e0 + kq - 1) / kq * kq;
          double n2 = 0.0, gr = 0.0;
          if (lo < p0) { n2 = sm.ccarry[0][a]; gr = sm.ccarry[1][a]; }
          for (int ee = e0; ee < min(hi, p1); ee += kq) {
            n2 += sm.st[j][ee - p0];
            gr += sm.st[9 + j][ee - p0];
          }
          if (hi > p1) {
            sm.ccarry[0][a] = n2; sm.ccarry[1][a] = gr;
          } else {
            const int col = __ldg(tab + sm.pc_tab[q] + a);
            if (col >= 0) { atomicAdd(&colnorm2[col], n2); atomicAdd(&grad[col], gr); }
          }
        }
        __syncthreads();   // the products of the next pass overwrite st
      }
      cost = sm.cost[t];
    }
  }
  const double tot = block_reduce_sum(cost);
  if (threadIdx.x == 0 && tot != 0.0) atomicAdd(&sc->cost, tot);
}

// V^-1, g_p, V^-1 g_p of the points [0, p_count) from the unscaled sums of ba_linearize_fused (ptsum[9][npf]:
// Jp^T Jp upper triangle xx xy xz yy yz zz, then Jp^T r): V_s = s_i s_j V_ij, g_s = s_i g_i; then as ba_point_blocks.
__global__ void __launch_bounds__(PB_THREADS)
    ba_point_blocks_sums(BAView v, int p_count, const double* __restrict__ ptsum, const double* __restrict__ scale,
                         const double* __restrict__ diag, double inv_radius, double* __restrict__ Vinv,
                         double* __restrict__ gpo, double* __restrict__ Vig, int* __restrict__ rank_flag) {
  const int p = blockIdx.x * PB_THREADS + threadIdx.x;
  if (p >= p_count) return;
  const int pf = v.pt_poff[p];
  if (pf < 0) return;
  const size_t NP = (size_t)v.npf;
  const int nc = v.nc;
  const double s0 = scale[nc + 3 * pf], s1 = scale[nc + 3 * pf + 1], s2 = scale[nc + 3 * pf + 2];
  double V[9];
  V[0] = ptsum[0 * NP + pf] * s0 * s0; V[1] = ptsum[1 * NP + pf] * s0 * s1; V[2] = ptsum[2 * NP + pf] * s0 * s2;
  V[3] = ptsum[3 * NP + pf] * s1 * s1; V[4] = ptsum[4 * NP + pf] * s1 * s2; V[5] = ptsum[5 * NP + pf] * s2 * s2;
  V[6] = ptsum[6 * NP + pf] * s0; V[7] = ptsum[7 * NP + pf] * s1; V[8] = ptsum[8 * NP + pf] * s2;
  point_block_finish(v, pf, V, diag, inv_radius, Vinv, gpo, Vig, rank_flag);
}

template <bool PROF>
__global__ void __launch_bounds__(SP_THREADS, 1)
    ba_schur_pipe(BAView v, const SchurChunk* __restrict__ chunks, int nchunks, const int* __restrict__ tab,
                  const double* __restrict__ scale, const double* __restrict__ Vinv, const double* __restrict__ Vig,
                  const int* __restrict__ ftab, double* __restrict__ Sval, double* __restrict__ rhs, unsigned long long* prof) {
  // prof != null (OSFM_BA_TRACE): clock64 totals of one thread per role, summed over the CTAs:
  //   [0..3] producer: copy wait + barrier, wait for a free operand buffer, build, chunks
  //   [4..8] consumer group 0 / [9..13] group 1: (unused), wait for operands, mma, flush, segments
  extern __shared__ __align__(16) unsigned char sp_raw[];
  SpSmem& sm = *reinterpret_cast<SpSmem*>(sp_raw);
  constexpr int wc = 9;
  const int nres = v.nres;
  const int tid = threadIdx.x;

  // chunk range of this CTA: [b C / G, (b + 1) C / G) moved up to the next segment start
  auto cut = [&](int b) -> int {
    if (b <= 0) return 0;
    const long long c = (long long)b * nchunks / gridDim.x;
    if (c >= nchunks) return nchunks;
    const SchurChunk e = sp_load_chunk(chunks, (int)c);
    return e.seg_chunk0 == (int)c ? (int)c : e.seg_chunk0 + e.seg_nch;
  };
  const int c_lo = cut(blockIdx.x), c_hi = cut(blockIdx.x + 1);

  if (tid == 0) {
    for (int i = 0; i < 2; ++i) {
      mbar_init(&sm.full[0][i], SP_PROD_THREADS);
      mbar_init(&sm.full[1][i], SP_PROD_THREADS);
      mbar_init(&sm.empty[i], SP_CONS_WARPS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (c_lo >= c_hi) return;

  // register split (launch allocation 96 / thread): the producers give up what the accumulators of the consumers need
  if (tid < SP_PROD_THREADS) {
    // =============================== producers ===============================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 72;");
    const int t = tid & (SP_OBS - 1);          // observation of the chunk
    const int half = tid >> 7;                 // which half of the camera-side columns
    const int c2_lo = half ? (wc + 1) / 2 : 0, c2_hi = half ? wc : (wc + 1) / 2;
    const size_t N = (size_t)v.N, NP = (size_t)v.npf;
    auto issue = [&](int n) {
      const SchurChunk e = sp_load_chunk(chunks, n);
      SpStage& S = sm.st[(n - c_lo) & 1];
      const int run = e.np * e.k;
      if (t < run) {
        const size_t i = (size_t)e.ibase + t;
        for (int q = 0; q < nres; ++q) {
          if (half == 0) {
            sp_cp8(&S.pl[q][t], &v.r[q * N + i]);
#pragma unroll
            for (int j = 0; j < 3; ++j) sp_cp8(&S.pl[nres + q * 3 + j][t], &v.Jp[((size_t)q * 3 + j) * N + i]);
          }
#pragma unroll
          for (int c2 = 0; c2 < wc; ++c2)
            if (c2 >= c2_lo && c2 < c2_hi) sp_cp8(&S.pl[nres * 4 + q * wc + c2][t], &v.Jc[((size_t)q * wc + c2) * N + i]);
        }
      }
      const int ncols = e.k * wc;
      const int* T = tab + e.tab_off;
      long long nints = 2LL * ncols + 9LL * (e.k * (e.k + 1) / 2);
      if (half == 1) {
        if (t < SM_PCH * 12 && e.pf0 >= 0) {
          const int lp = t / 12, ee = t - lp * 12;
          if (lp < e.np) {
            const size_t pf = (size_t)e.pf0 + lp;
            const double* src = ee < 6 ? &Vinv[ee * NP + pf] : ee < 9 ? &Vig[(ee - 6) * NP + pf] : &scale[v.nc + 3 * pf + (ee - 9)];
            sp_cp8(&S.ptd[lp][ee], src);
          }
        }
        if (t < ncols) sp_cp8(&S.scol[t], reinterpret_cast<const double*>(T + nints + (nints & 1)) + t);
      }
      sp_commit();
    };
    issue(c_lo);
    long long pk[3] = {0, 0, 0}, tk = PROF ? clock64() : 0;
    auto pmark = [&](int slot) {
      if (PROF) { const long long now = clock64(); pk[slot] += now - tk; tk = now; }
    };
    for (int n = c_lo; n < c_hi; ++n) {
      const int r = n - c_lo, buf = r & 1, use = r >> 1;
      sp_wait_all();                              // my copies of chunk n have landed
      sp_bar(1, SP_PROD_THREADS);                 // everybody's have; and everybody is done reading the other stage
      pmark(0);
      if (n + 1 < c_hi) issue(n + 1);
      const SchurChunk e = sp_load_chunk(chunks, n);
      const SpStage& S = sm.st[r & 1];
      SpOperand& O = sm.op[buf];
      const int np = e.np, k = e.k, run = np * k, ncols = k * wc;
      const bool pfree = e.pf0 >= 0;
      mbar_wait(&sm.empty[buf], (use & 1) ^ 1);   // the consumers released this operand buffer
      pmark(1);
      // rows [3 np, 4 ksteps) and the padding columns [ncols, 8 nt) must read as zero
      {
        const int nt8 = ((ncols + 7) >> 3) << 3;
        const int k0 = 3 * np, k1 = ((3 * np + 3) >> 2) << 2;
        for (int idx = tid; idx < (k1 - k0) * nt8; idx += SP_PROD_THREADS) {
          const int kk = k0 + idx / nt8, cc = idx % nt8;
          O.Yt[kk][cc] = 0.0; O.Wt[kk][cc] = 0.0; O.Jt[kk][cc] = 0.0;
        }
        const int padc = nt8 - ncols;
        for (int idx = tid; idx < k0 * padc; idx += SP_PROD_THREADS) {
          const int kk = idx / padc, cc = ncols + idx % padc;
          O.Yt[kk][cc] = 0.0; O.Wt[kk][cc] = 0.0; O.Jt[kk][cc] = 0.0;
        }
      }
      if (t < run) {
        const int lp = t / k, bb = t - lp * k;
        const double* pd = S.ptd[lp];
        double rr[3] = {0.0, 0.0, 0.0}, jp[3][3];
#pragma unroll
        for (int q = 0; q < 3; ++q) {
          const bool on = q < nres;
          if (on) rr[q] = S.pl[q][t];
#pragma unroll
          for (int j = 0; j < 3; ++j) jp[q][j] = (on && pfree) ? S.pl[nres + q * 3 + j][t] * pd[9 + j] : 0.0;
        }
        double v6[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0}, vg[3] = {0.0, 0.0, 0.0};
        if (pfree) {
#pragma unroll
          for (int e6 = 0; e6 < 6; ++e6) v6[e6] = pd[e6];
#pragma unroll
          for (int e3 = 0; e3 < 3; ++e3) vg[e3] = pd[6 + e3];
        }
#pragma unroll
        for (int cc = 0; cc < (wc + 1) / 2; ++cc) {
          const int c2 = c2_lo + cc;
          if (c2 >= c2_hi) break;
          const int col = bb * wc + c2;
          const double sc = S.scol[col];
          double js[3], w[3] = {0.0, 0.0, 0.0}, gr = 0.0;
#pragma unroll
          for (int q = 0; q < 3; ++q) {
            js[q] = q < nres ? S.pl[nres * 4 + q * wc + c2][t] * sc : 0.0;
            gr += js[q] * rr[q];
#pragma unroll
            for (int j = 0; j < 3; ++j) w[j] += js[q] * jp[q][j];
          }
          const double y0 = w[0] * v6[0] + w[1] * v6[1] + w[2] * v6[2];
          const double y1 = w[0] * v6[1] + w[1] * v6[3] + w[2] * v6[4];
          const double y2 = w[0] * v6[2] + w[1] * v6[4] + w[2] * v6[5];
          gr -= w[0] * vg[0] + w[1] * vg[1] + w[2] * vg[2];
          O.Jt[3 * lp + 0][col] = js[0]; O.Jt[3 * lp + 1][col] = js[1]; O.Jt[3 * lp + 2][col] = js[2];
          O.Wt[3 * lp + 0][col] = w[0];  O.Wt[3 * lp + 1][col] = w[1];  O.Wt[3 * lp + 2][col] = w[2];
          O.Yt[3 * lp + 0][col] = -y0;   O.Yt[3 * lp + 1][col] = -y1;   O.Yt[3 * lp + 2][col] = -y2;
          O.G[lp][col] = gr;
        }
      }
      mbar_arrive(&sm.full[e.seg & 1][buf]);
      pmark(2);
    }
    if (PROF && tid == 0) {
      for (int i = 0; i < 3; ++i) atomicAdd(&prof[i], (unsigned long long)pk[i]);
      atomicAdd(&prof[3], (unsigned long long)(c_hi - c_lo));
    }
    return;
  }

  // =============================== consumers ===============================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 112;");
  const int g = (tid - SP_PROD_THREADS) / SP_CONS_THREADS;         // group 0 / 1: segments of that parity
  const int gt = (tid - SP_PROD_THREADS) - g * SP_CONS_THREADS;    // thread in the group
  const int cw = gt >> 5, lane = gt & 31;
  const int fr = lane >> 2, fk = lane & 3;
  // accumulators: c[j] = tile slot j of the row pair, dA / dB = Js^T Js of the (t, t) and (t, t + 1) tiles of each row
  double c[SP_SLOTS][2], dA[2][2], dB[2][2];
  double racc = 0.0;
  int ncols = 0, kseg = 0, nt = 0, rowA = 0, rowB = 0, nA = 0, nB = 0;
  int uses0 = 0, uses1 = 0;   // chunks of this group that went through each operand buffer so far
  int nsegs = 0;
  SpFlush& FT = sm.ft[g];
  long long ck[4] = {0, 0, 0, 0}, tk = PROF ? clock64() : 0;
  auto cmark = [&](int slot) {
    if (PROF) { const long long now = clock64(); ck[slot] += now - tk; tk = now; }
  };
  // tile column of slot j (the caller guarantees j < nA + nB for a meaningful answer; otherwise tile 0)
  auto slot_tj = [&](int j) -> int { return j < nA ? rowA + j : (j - nA < nB ? rowB + (j - nA) : 0); };

  for (int n = c_lo; n < c_hi; ++n) {
    const SchurChunk e = sp_load_chunk(chunks, n);
    if ((e.seg & 1) != g) continue;
    const int buf = (n - c_lo) & 1;
    if (n == e.seg_chunk0) {
      // ---- new segment: zero accumulators, my pair of tile rows ----
      kseg = e.k;
      ncols = kseg * wc;
      nt = (ncols + 7) >> 3;
      racc = 0.0;
      const bool active = cw < ((nt + 1) >> 1);
      rowA = active ? cw : 0;
      rowB = active ? nt - 1 - cw : 0;
      nA = active ? nt - rowA : 0;
      nB = (active && rowB > rowA) ? nt - rowB : 0;
#pragma unroll
      for (int j = 0; j < SP_SLOTS; ++j) { c[j][0] = 0.0; c[j][1] = 0.0; }
#pragma unroll
      for (int j = 0; j < 2; ++j) { dA[j][0] = 0.0; dA[j][1] = 0.0; dB[j][0] = 0.0; dB[j][1] = 0.0; }
      ++nsegs;
      // my share of the segment's flush table (and gcol): needed after the last chunk, in flight during the products.
      // Every lane copies exactly what it reads back itself, and the previous flush of this warp is over.
      {
        const int* src = ftab + (size_t)e.seg * SP_FT_SEG + cw * SP_FT_WARP + lane;
#pragma unroll
        for (int q = 0; q < SP_SLOTS * 2; ++q) sp_cp4(&FT.t[cw][q * 32 + lane], src + q * 32);
        if (gt < ncols) sp_cp4(&FT.gcol[gt], tab + e.tab_off + gt);
        sp_commit();
      }
    }
    mbar_wait(&sm.full[g][buf], (buf ? uses1++ : uses0++) & 1);
    cmark(1);
    {
      const SpOperand& O = sm.op[buf];
      const int np = e.np;
      const int ksteps = (3 * np + 3) >> 2;
      const bool pfree = e.pf0 >= 0;
      const double* Y0 = &O.Yt[0][0] + fk * SM_LD + fr;
      const double* W0 = &O.Wt[0][0] + fk * SM_LD + fr;
      const double* J0 = &O.Jt[0][0] + fk * SM_LD + fr;
      const int a1 = min(rowA + 1, nt - 1), b1 = min(rowB + 1, nt - 1);   // clamped: the (t, t + 1) tile of the last row does not exist
      if (nA > 0) {
        for (int ks = 0; ks < ksteps; ++ks) {
          const int ko = ks * 4 * SM_LD;
          if (pfree) {
            const double aA = Y0[ko + 8 * rowA], aB = Y0[ko + 8 * rowB];
#pragma unroll
            for (int j = 0; j < SP_SLOTS; ++j) dmma884(c[j][0], c[j][1], j < nA ? aA : aB, W0[ko + 8 * slot_tj(j)]);
          }
          const double jA = J0[ko + 8 * rowA], jA1 = J0[ko + 8 * a1], jB = J0[ko + 8 * rowB], jB1 = J0[ko + 8 * b1];
          dmma884(dA[0][0], dA[0][1], jA, jA);
          dmma884(dA[1][0], dA[1][1], jA, jA1);
          dmma884(dB[0][0], dB[0][1], jB, jB);
          dmma884(dB[1][0], dB[1][1], jB, jB1);
        }
      }
      if (gt < ncols)
        for (int lp = 0; lp < np; ++lp) racc += O.G[lp][gt];
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&sm.empty[buf]);
    cmark(2);
    if (n == e.seg_chunk0 + e.seg_nch - 1) {
      // ---- flush the segment: destinations from the table, values straight from the fragments ----
      sp_wait_all();
      if (gt < ncols && FT.gcol[gt] >= 0) atomicAdd(&rhs[FT.gcol[gt]], racc);
#pragma unroll
      for (int j = 0; j < SP_SLOTS; ++j) {
        const bool isA = j < nA;
        const int jj = isA ? j : j - nA;
#pragma unroll
        for (int el = 0; el < 2; ++el) {
          const int code = FT.t[cw][(j * 2 + el) * 32 + lane];
          if (code < 0) continue;
          double val = c[j][el];
          if (code & 1) val += isA ? dA[jj & 1][el] : dB[jj & 1][el];
          if (code & 2) val *= 2.0;
          atomicAdd(&Sval[code >> 2], val);
        }
      }
      cmark(3);
    }
  }
  if (PROF && gt == 0) {
    for (int i = 0; i < 4; ++i) atomicAdd(&prof[4 + 5 * g + i], (unsigned long long)ck[i]);
    atomicAdd(&prof[8 + 5 * g], (unsigned long long)nsegs);
  }
}

}  // namespace osfm
