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
// Eligible: nres * (wc + 4) <= SP_ROWS plane rows per observation (2-D residuals with wc <= 9); everything else
// keeps ba_schur_mma.  OSFM_BA_SCHUR_PIPE=0 switches back for A/B runs.
#pragma once

namespace osfm {

constexpr int SP_PROD_WARPS = 8;
constexpr int SP_CONS_WARPS = 6;                    // per consumer group: one per pair of tile rows
constexpr int SP_PROD_THREADS = 32 * SP_PROD_WARPS;
constexpr int SP_CONS_THREADS = 32 * SP_CONS_WARPS;
constexpr int SP_THREADS = SP_PROD_THREADS + 2 * SP_CONS_THREADS;   // 640
constexpr int SP_ROWS = 26;                         // staged plane rows: r (nres) + Jp (3 nres) + Jc (wc nres)
constexpr int SP_OBS = SM_PCH * SEG_KMAX;           // 128 observations per chunk at most
constexpr int SP_SLOTS = SM_NT + 1;                 // tiles of a row pair (p, nt - 1 - p): nt + 1
constexpr int SP_NPAIR9 = 9 * (SEG_KMAX * (SEG_KMAX + 1) / 2);
static_assert(2 * SP_OBS == SP_PROD_THREADS, "two producer threads per observation of a chunk");
static_assert(2 * SP_CONS_WARPS >= SM_NT, "a consumer warp per pair of tile rows");
static_assert((SP_ROWS / 2) - 4 <= 9, "same-shot blocks are only accumulated in the tiles (t, t) and (t, t + 1): wc <= 9");

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
  unsigned long long full[2][2], empty[2];
};

__device__ __forceinline__ uint32_t sp_saddr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void sp_cp8(void* dst, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(sp_saddr(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void sp_cp4(void* dst, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(sp_saddr(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void sp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void sp_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void sp_bar(int id, int count) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory"); }
__device__ __forceinline__ void sp_mbar_init(unsigned long long* b, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(sp_saddr(b)), "r"(count) : "memory");
}
__device__ __forceinline__ void sp_mbar_arrive(unsigned long long* b) {
  asm volatile("{\n.reg .b64 st;\nmbarrier.arrive.shared::cta.b64 st, [%0];\n}" ::"r"(sp_saddr(b)) : "memory");
}
__device__ __forceinline__ void sp_mbar_wait(unsigned long long* b, int parity) {
  const uint32_t a = sp_saddr(b);
  uint32_t done = 0;
  long long t0 = 0;
  int spins = 0;
  while (true) {
    asm volatile(
        "{\n.reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n}"
        : "=r"(done)
        : "r"(a), "r"(parity)
        : "memory");
    if (done) break;
    if ((++spins & 1023) == 0) {   // a protocol bug must not hang the GPU
      if (t0 == 0) t0 = clock64();
      else if (clock64() - t0 > 8000000000LL) __trap();
    }
  }
}
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
// Camera-side gradient and squared column norms over the chunk list (wc == 9, nres == 2): ba_colnorm_grad_tma
// (ba.cu) walks seg_start / pt_start with three dependent loads per chunk before it can issue the next copy; here a
// warp owns a contiguous range of chunks (cut at segment starts), reads one 48-byte entry per chunk (the entry of
// chunk n + 1 is in registers while chunk n is reduced) and takes the global columns from the per-segment table.
// Staging as there: one bulk copy (TMA engine) per plane row and chunk, two stages per warp, one mbarrier each.
// ---------------------------------------------------------------------------------------------------------
constexpr int CC_WARPS = 5;
constexpr int CC_ROWS = 20;                       // r[2] + Jc[2 * 9]
constexpr int CC_STAGE_DOUBLES = CC_ROWS * SP_OBS;
constexpr int CC_SMEM = CC_WARPS * 2 * CC_STAGE_DOUBLES * (int)sizeof(double);   // 204,800 bytes

__global__ void __launch_bounds__(32 * CC_WARPS, 1)
    ba_colnorm_grad_chunks(BAView v, const SchurChunk* __restrict__ chunks, int nchunks, const int* __restrict__ tab,
                           double* colnorm2, double* grad) {
  extern __shared__ __align__(128) double cc_tiles[];
  __shared__ __align__(8) unsigned long long bars[CC_WARPS][2];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int w = 0; w < CC_WARPS; ++w)
      for (int st = 0; st < 2; ++st) sp_mbar_init(&bars[w][st], 1);
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
        const uint32_t bar = sp_saddr(&bars[warp][st]);
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes * CC_ROWS) : "memory");
        for (int row = 0; row < CC_ROWS; ++row) {
          const double* src = (row < 2 ? v.r + (size_t)row * N : v.Jc + (size_t)(row - 2) * N) + e.ibase;
          asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                           sp_saddr(tile[st] + row * SP_OBS)),
                       "l"(src), "r"(bytes), "r"(bar)
                       : "memory");
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
      sp_mbar_wait(&bars[warp][st], st ? phase1 : phase0);
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

template <int WC, bool PROF>
__global__ void __launch_bounds__(SP_THREADS, 1)
    ba_schur_pipe(BAView v, const SchurChunk* __restrict__ chunks, int nchunks, const int* __restrict__ tab,
                  const double* __restrict__ scale, const double* __restrict__ Vinv, const double* __restrict__ Vig,
                  const int* __restrict__ ftab, double* __restrict__ Sval, double* __restrict__ rhs, unsigned long long* prof) {
  // prof != null (OSFM_BA_TRACE): clock64 totals of one thread per role, summed over the CTAs:
  //   [0..3] producer: copy wait + barrier, wait for a free operand buffer, build, chunks
  //   [4..8] consumer group 0 / [9..13] group 1: (unused), wait for operands, mma, flush, segments
  extern __shared__ __align__(16) unsigned char sp_raw[];
  SpSmem& sm = *reinterpret_cast<SpSmem*>(sp_raw);
  const int wc = WC ? WC : v.wc;
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
      sp_mbar_init(&sm.full[0][i], SP_PROD_THREADS);
      sp_mbar_init(&sm.full[1][i], SP_PROD_THREADS);
      sp_mbar_init(&sm.empty[i], SP_CONS_WARPS);
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
          for (int c2 = 0; c2 < (WC ? WC : SEG_WCMAX); ++c2)
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
      sp_mbar_wait(&sm.empty[buf], (use & 1) ^ 1);   // the consumers released this operand buffer
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
        for (int cc = 0; cc < ((WC ? WC : SEG_WCMAX) + 1) / 2; ++cc) {
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
      sp_mbar_arrive(&sm.full[e.seg & 1][buf]);
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
    sp_mbar_wait(&sm.full[g][buf], (buf ? uses1++ : uses0++) & 1);
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
    if (lane == 0) sp_mbar_arrive(&sm.empty[buf]);
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
