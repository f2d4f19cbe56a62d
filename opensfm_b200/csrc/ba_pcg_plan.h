// Shared-memory plan of the pipelined PCG (pcg_pipelined in ba_reduced.cuh): which preconditioner groups every CTA
// owns and where its slices live in dynamic shared memory.  Plain host C++ (no CUDA), so that the plan of a given
// problem structure can be checked by a CPU test.
//
// A CTA keeps, for its own groups: the rows of S (8 B per stored entry), a packed copy of the mat-vec input m per
// column list (8 B per column), the column lists themselves (uint16), the groups' inverted diagonal blocks at n x n,
// a few per-row vectors and tables, and the deflation rows and barrier buffers.  The S slice dominates, and it is
// also what the CTA's mat-vec streams on every iteration, so one cut balances both the footprint and the work.
#pragma once
#include <algorithm>
#include <vector>

namespace osfm {

constexpr int PCG_THREADS = 512;   // threads of both persistent PCG kernels; one thread owns one row in pcg_pipelined
constexpr int PCG_ND = 7;   // deflation vectors: the similarity gauge of the rig instances (3 translations, 3 rotations, scale)
constexpr int PCG_NW = 10;  // doubles per CTA on the wide barrier: gamma, delta, |r|^2, PCG_ND projections

// What a set of groups occupies as one CTA's share
struct PcgPipeLoad {
  long long ent = 0, cols = 0, minv = 0;   // stored S entries, packed columns, doubles of the packed group inverses
  int rows = 0, groups = 0;
  void add(const PcgPipeLoad& o) {
    ent += o.ent; cols += o.cols; minv += o.minv; rows += o.rows; groups += o.groups;
  }
  void max_with(const PcgPipeLoad& o) {
    ent = std::max(ent, o.ent); cols = std::max(cols, o.cols); minv = std::max(minv, o.minv);
    rows = std::max(rows, o.rows); groups = std::max(groups, o.groups);
  }
};

struct PcgPipePlan {
  bool fits = false;
  std::vector<int> grp_lo;   // [G + 1] first group of every CTA
  PcgPipeLoad max;           // per-component maxima over the CTAs: the layout is sized by them
  // byte offsets into dynamic shared memory (the packed m at 0) and its size
  long long off_S = 0, off_Minv = 0, off_vec = 0, off_cols = 0, off_rows = 0, off_defl = 0, total = 0;
  long long available = 0;   // dynamic shared memory one CTA may use
};

inline long long pcg_up16(long long x) { return (x + 15) / 16 * 16; }

// Lays the kernel's dynamic shared memory out for a CTA with load `m` on a grid of G CTAs; returns the bytes.
inline long long pcg_pipe_layout(const PcgPipeLoad& m, int G, PcgPipePlan* p = nullptr) {
  const long long off_S = pcg_up16(8 * m.cols), off_Minv = off_S + pcg_up16(8 * m.ent);
  const long long off_vec = off_Minv + pcg_up16(8 * m.minv), off_cols = off_vec + pcg_up16(24LL * m.rows);
  const long long off_rows = off_cols + pcg_up16(2 * m.cols);
  // row tables (9 ints per row) and, per group, its first row and the offset of its inverse
  const long long off_defl = pcg_up16(off_rows + 36LL * m.rows + 8LL * (m.groups + 1));
  // own rows of the deflation vectors W and of S W, then the gather buffer of the wide barrier
  const long long total = off_defl + 2LL * PCG_ND * 8 * m.rows + 8LL * PCG_NW * G + 8LL * PCG_NW * m.rows;
  if (p) {
    p->off_S = off_S; p->off_Minv = off_Minv; p->off_vec = off_vec; p->off_cols = off_cols; p->off_rows = off_rows;
    p->off_defl = off_defl; p->total = total;
  }
  return total;
}

// Whether block rows b1 and b2 of a CSR block structure (columns sorted within a row) store the same block columns:
// then their ELL rows have the same column list and a CTA keeps one copy of it (and of the packed m) for both.
inline bool pcg_rows_share_columns(const std::vector<int>& row_ptr, const std::vector<int>& row_col, int b1, int b2) {
  if (b1 < 0 || b2 < 0) return false;
  const int n1 = row_ptr[b1 + 1] - row_ptr[b1];
  if (row_ptr[b2 + 1] - row_ptr[b2] != n1) return false;
  return std::equal(row_col.begin() + row_ptr[b1], row_col.begin() + row_ptr[b1] + n1, row_col.begin() + row_ptr[b2]);
}

// The plan for groups (grp_b1[g], grp_b2[g] or -1) of blocks with blk_sz[b] rows and row_M[b] stored columns;
// shared[g] = 1 when the two block rows of group g share one column list.  Contiguous group ranges, one per CTA,
// chosen to minimise the largest CTA footprint: binary search on the bound, every CTA filled greedily up to it (and
// never so far that a later CTA is left without a group).  `available` is the CTA's opt-in limit less the kernel's
// static shared memory and a reserve.
inline PcgPipePlan plan_pcg_pipelined(const std::vector<int>& grp_b1, const std::vector<int>& grp_b2,
                                      const std::vector<int>& blk_sz, const std::vector<int>& row_M,
                                      const std::vector<char>& shared, int G, long long available) {
  const int n = (int)grp_b1.size();
  std::vector<PcgPipeLoad> load(n);
  for (int g = 0; g < n; ++g) {
    PcgPipeLoad& l = load[g];
    for (int k = 0; k < 2; ++k) {
      const int b = k ? grp_b2[g] : grp_b1[g];
      if (b < 0) continue;
      l.ent += (long long)blk_sz[b] * row_M[b];
      if (!(k && shared[g])) l.cols += row_M[b];
      l.rows += blk_sz[b];
    }
    l.minv = (long long)l.rows * l.rows;
    l.groups = 1;
  }
  // greedy fill under `bound`; false when some CTA cannot take its next group
  auto fill = [&](long long bound, std::vector<int>& lo) {
    lo.assign(G + 1, n);
    int g = 0;
    for (int c = 0; c < G; ++c) {
      lo[c] = g;
      PcgPipeLoad acc;
      while (g < n && n - g > G - 1 - c) {
        PcgPipeLoad next = acc;
        next.add(load[g]);
        if (next.rows > PCG_THREADS || pcg_pipe_layout(next, G) > bound) break;
        acc = next;
        ++g;
      }
      if (acc.groups == 0 && g < n && n - g > G - 1 - c) return false;
    }
    return g == n;
  };
  PcgPipePlan p;
  p.available = available;
  PcgPipeLoad all;
  for (int g = 0; g < n; ++g) all.add(load[g]);
  std::vector<int>& lo = p.grp_lo;
  long long lo_b = 0, hi_b = pcg_pipe_layout(all, G);
  if (!fill(hi_b, lo)) {   // more rows than the grid has threads: no plan
    p.max = all;
    pcg_pipe_layout(p.max, G, &p);
    return p;
  }
  while (hi_b - lo_b > 1) {   // fill(hi_b) holds, fill(lo_b) does not
    const long long mid = lo_b + (hi_b - lo_b) / 2;
    if (fill(mid, lo)) hi_b = mid; else lo_b = mid;
  }
  fill(hi_b, lo);
  for (int c = 0; c < G; ++c) {
    PcgPipeLoad cta;
    for (int g = lo[c]; g < lo[c + 1]; ++g) cta.add(load[g]);
    p.max.max_with(cta);
  }
  pcg_pipe_layout(p.max, G, &p);
  p.fits = p.max.rows <= PCG_THREADS && p.max.ent < (1LL << 30) && p.total <= available;
  return p;
}

}  // namespace osfm
