// Test-only: compiles the product's __host__ __device__ relative-pose solvers (five points, N points, the
// decomposition of an essential, the model's error, the Hessenberg QR) with g++ so tests can compare them against
// oracle/relative_pose_oracle.py and numpy without a GPU.
#include "../../opensfm_b200/csrc/relative_pose.cuh"
extern "C" {
int hd_five_point(const double* x1, const double* x2, double* Es, double* margin) {
  return osfm::relpose::five_point(x1, x2, Es, margin);
}
int hd_n_points(int k, const double* x1, const double* x2, double* E, double* margin) {
  return osfm::relpose::n_points(k, x1, x2, E, margin);
}
void hd_pose_from_essential(const double* E, int k, const double* x1, const double* x2, double* out, double* margin) {
  osfm::relpose::pose_from_essential(E, k, x1, x2, out, margin);
}
double hd_evaluate(const double* M, const double* x, const double* y) { return osfm::relpose::evaluate(M, x, y); }
int hd_eigenvalues(double* a, int n, double* wr, double* wi) { return osfm::relpose::eigenvalues(a, n, wr, wi); }
}
