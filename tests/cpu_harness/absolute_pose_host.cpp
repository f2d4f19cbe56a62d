// Test-only: compiles the product's __host__ __device__ absolute-pose solvers (P3P, the quartic, Lu's iteration)
// with g++ so tests can compare them against oracle/absolute_pose_oracle.py without a GPU.
#include "../../opensfm_b200/csrc/absolute_pose.cuh"
extern "C" {
int hd_p3p(const double* b, const double* p, double* models) { return osfm::pose::p3p_ke(b, p, models); }
int hd_lu(int k, const double* b, const double* p, double* out) { return osfm::pose::lu_pose(k, b, p, out); }
int hd_solve_quartic(const double* coef, double* roots) {
  if (!osfm::pose::solve_quartic(coef, roots)) return 0;
  for (int m = 0; m < 4; ++m) roots[m] = osfm::pose::refine_quartic_root(coef, roots[m]);
  return 4;
}
}
