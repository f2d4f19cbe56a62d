// Host build of the pipelined PCG's shared-memory plan (opensfm_b200/csrc/ba_pcg_plan.h) behind a C ABI for
// tests/test_ba_pcg_plan_cpu.py.  g++ -O2 -fPIC -shared -std=c++17.
#include "../../opensfm_b200/csrc/ba_pcg_plan.h"

extern "C" {

// The plan of groups (b1[g], b2[g] or -1) on a CSR block structure (row_ptr [nblk + 1], sorted row_col) with blocks
// of blk_sz rows, as BA::plan_pcg makes it.  Writes grp_lo [G + 1], shared [ngroups] and
// out = {fits, total bytes, worst CTA's entries, columns, inverse doubles, rows, groups}.
void hp_plan(int ngroups, const int* b1, const int* b2, int nblk, const int* blk_sz, const int* row_ptr,
             const int* row_col, int G, long long available, int* grp_lo, char* shared, long long* out) {
  const std::vector<int> vb1(b1, b1 + ngroups), vb2(b2, b2 + ngroups), vsz(blk_sz, blk_sz + nblk);
  const std::vector<int> vptr(row_ptr, row_ptr + nblk + 1), vcol(row_col, row_col + row_ptr[nblk]);
  std::vector<int> row_M(nblk, 0);   // as pcg_row_sizes
  for (int b = 0; b < nblk; ++b)
    for (int e = vptr[b]; e < vptr[b + 1]; ++e) row_M[b] += vsz[vcol[e]];
  std::vector<char> sh(ngroups);
  for (int g = 0; g < ngroups; ++g) sh[g] = shared[g] = osfm::pcg_rows_share_columns(vptr, vcol, vb1[g], vb2[g]);
  const osfm::PcgPipePlan p = osfm::plan_pcg_pipelined(vb1, vb2, vsz, row_M, sh, G, available);
  for (int c = 0; c <= G; ++c) grp_lo[c] = p.grp_lo[c];
  const long long o[7] = {p.fits, p.total, p.max.ent, p.max.cols, p.max.minv, p.max.rows, p.max.groups};
  for (int i = 0; i < 7; ++i) out[i] = o[i];
}

}
