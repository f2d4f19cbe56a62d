// Relative-pose solvers of pyrobust's RelativePose model (geometry/essential.h, geometry/relative_pose.h,
// robust/relative_pose_model.h), fp64, for the device and, compiled by g++, for the host tests
// (tests/cpu_harness/relative_pose_host.cpp):
//
//   five_point         Stewenius' five-point solver: the nullspace of the 5 epipolar rows, the 10 x 20 constraint
//                      matrix, the reference's Gauss-Jordan without pivoting, the real eigenvalues of the 10 x 10
//                      action matrix (Hessenberg form and Francis' double-shift QR) and their eigenvectors; up to 10
//                      essentials, in ascending order of their eigenvalue
//   n_points           EssentialNPoints: the smallest right singular vector of 9 to 12 epipolar rows, kept when
//                      sigma_8 / sigma_9 > 4, projected onto singular values ((a + b) / 2, (a + b) / 2, 0)
//   pose_from_essential RelativePoseFromEssential: the 4 decompositions scored on the rows given
//   evaluate           RelativePose::Evaluate: 1 - (px . x + py . y) / 2 of the midpoint triangulation
//
// The restatement, and the reasons for its deliberate differences (the canonical order of the essentials, the rule
// for a real eigenvalue, the eigen-decompositions in place of Eigen's JacobiSVD), are in
// oracle/relative_pose_oracle.py.  Matrices are row-major; a pose is the 3 x 4 [R | t] with x2 = R x1 + t.
#pragma once

#include <cmath>

#ifdef __CUDACC__
#define OSFM_HD __host__ __device__ inline
#else
#define OSFM_HD inline
#endif

namespace osfm {
namespace relpose {

constexpr int MAX_MODELS = 10;
constexpr double MIDPOINT_DET_EPS = 1e-10;     // TriangulateTwoBearingsMidpointSolve's only validity test
constexpr double REAL_TOLERANCE = 1e-6;        // an eigenvalue is real when |Im| <= this * (1 + |Re|)
constexpr double NULLSPACE_RATIO = 4.0;        // SolveAX0: sigma_8 / sigma_9 above this
constexpr int JACOBI_SWEEPS = 30;
constexpr int HQR_ITERATIONS = 30;             // per eigenvalue

OSFM_HD bool finite(double x) {
#ifdef __CUDA_ARCH__
  return isfinite(x);
#else
  return std::isfinite(x);
#endif
}

OSFM_HD double dot3(const double* a, const double* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

OSFM_HD void cross3(const double* a, const double* b, double* c) {
  c[0] = a[1] * b[2] - a[2] * b[1];
  c[1] = a[2] * b[0] - a[0] * b[2];
  c[2] = a[0] * b[1] - a[1] * b[0];
}

OSFM_HD void normalize3(double* a) {
  const double r = sqrt(dot3(a, a));
  a[0] /= r;
  a[1] /= r;
  a[2] /= r;
}

// ---------------------------------------------------------------------------------------------------------------
// Triangulation and the model's error
// ---------------------------------------------------------------------------------------------------------------

// The midpoint of the rays 0 + l0 b0 and c1 + l1 b1; false when |det| < 1e-10.
OSFM_HD bool midpoint(const double* c1, const double* b0, const double* b1, double* X) {
  const double r0 = dot3(c1, b0), r1 = dot3(c1, b1);
  const double a00 = dot3(b0, b0), a10 = dot3(b0, b1), a01 = -a10, a11 = -dot3(b1, b1);
  const double det = a00 * a11 - a01 * a10;
  if (-MIDPOINT_DET_EPS < det && det < MIDPOINT_DET_EPS) return false;
  const double l0 = (a11 * r0 - a01 * r1) / det;
  const double l1 = (a00 * r1 - a10 * r0) / det;
  for (int c = 0; c < 3; ++c) X[c] = 0.5 * (l0 * b0[c] + (c1[c] + l1 * b1[c]));
  return true;
}

// (px . x + py . y) / 2 of the pose M for the row (x, y), and whether the row triangulates
OSFM_HD bool agreement(const double* M, const double* x, const double* y, double* out) {
  double c1[3], by[3], X[3];
  for (int c = 0; c < 3; ++c) {
    c1[c] = -(M[0 * 4 + c] * M[3] + M[1 * 4 + c] * M[7] + M[2 * 4 + c] * M[11]);
    by[c] = M[0 * 4 + c] * y[0] + M[1 * 4 + c] * y[1] + M[2 * 4 + c] * y[2];
  }
  if (!midpoint(c1, x, by, X)) return false;
  double px[3] = {X[0], X[1], X[2]};
  normalize3(px);
  double py[3];
  for (int r = 0; r < 3; ++r) py[r] = M[r * 4] * X[0] + M[r * 4 + 1] * X[1] + M[r * 4 + 2] * X[2] + M[r * 4 + 3];
  normalize3(py);
  *out = (dot3(px, x) + dot3(py, y)) * 0.5;
  return true;
}

// RelativePose::Evaluate for unit x, y: 1 - agreement, or 1 when the row does not triangulate
OSFM_HD double evaluate(const double* M, const double* x, const double* y) {
  double a;
  return agreement(M, x, y, &a) ? 1.0 - a : 1.0;
}

// ---------------------------------------------------------------------------------------------------------------
// Symmetric eigen-decomposition (cyclic Jacobi), n <= 9
// ---------------------------------------------------------------------------------------------------------------

// S (n x n, destroyed) = V diag(w) V^T with w descending; V's columns are the eigenvectors.
OSFM_HD void sym_eig(double* S, int n, double* V, double* w) {
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < n; ++j) V[i * n + j] = i == j ? 1.0 : 0.0;
  for (int sweep = 0; sweep < JACOBI_SWEEPS; ++sweep) {
    double off = 0.0, all = 0.0;
    for (int i = 0; i < n; ++i)
      for (int j = 0; j < n; ++j) {
        const double v = S[i * n + j] * S[i * n + j];
        all += v;
        if (i != j) off += v;
      }
    if (!(off > 1e-32 * all)) break;
    for (int p = 0; p < n - 1; ++p)
      for (int q = p + 1; q < n; ++q) {
        const double apq = S[p * n + q];
        if (apq == 0.0) continue;
        const double theta = (S[q * n + q] - S[p * n + p]) / (2.0 * apq);
        const double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < n; ++k) {
          const double kp = S[k * n + p], kq = S[k * n + q];
          S[k * n + p] = c * kp - s * kq;
          S[k * n + q] = s * kp + c * kq;
        }
        for (int k = 0; k < n; ++k) {
          const double pk = S[p * n + k], qk = S[q * n + k];
          S[p * n + k] = c * pk - s * qk;
          S[q * n + k] = s * pk + c * qk;
        }
        for (int k = 0; k < n; ++k) {
          const double kp = V[k * n + p], kq = V[k * n + q];
          V[k * n + p] = c * kp - s * kq;
          V[k * n + q] = s * kp + c * kq;
        }
      }
  }
  for (int i = 0; i < n; ++i) w[i] = S[i * n + i];
  // selection sort, descending, moving the columns of V along
  for (int i = 0; i < n - 1; ++i) {
    int m = i;
    for (int j = i + 1; j < n; ++j)
      if (w[j] > w[m]) m = j;
    if (m == i) continue;
    const double tw = w[i];
    w[i] = w[m];
    w[m] = tw;
    for (int k = 0; k < n; ++k) {
      const double tv = V[k * n + i];
      V[k * n + i] = V[k * n + m];
      V[k * n + m] = tv;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// RelativePoseFromEssential
// ---------------------------------------------------------------------------------------------------------------

// The left and right singular vectors of E for its two largest singular values (u0, u1, v0, v1), u2 = u0 x u1 and
// v2 = v0 x v1 (so that det U = det V = 1), and the singular values s.
OSFM_HD void essential_svd(const double* E, double* U, double* V, double* s) {
  double S[9], w[3];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) S[i * 3 + j] = E[i] * E[j] + E[3 + i] * E[3 + j] + E[6 + i] * E[6 + j];
  sym_eig(S, 3, V, w);
  double u[2][3];
  for (int k = 0; k < 2; ++k) {
    for (int r = 0; r < 3; ++r) u[k][r] = E[r * 3] * V[k] + E[r * 3 + 1] * V[3 + k] + E[r * 3 + 2] * V[6 + k];
  }
  normalize3(u[0]);
  const double d = dot3(u[0], u[1]);
  for (int r = 0; r < 3; ++r) u[1][r] -= d * u[0][r];
  normalize3(u[1]);
  double u2[3], v0[3] = {V[0], V[3], V[6]}, v1[3] = {V[1], V[4], V[7]}, v2[3];
  cross3(u[0], u[1], u2);
  cross3(v0, v1, v2);
  for (int r = 0; r < 3; ++r) {
    U[r * 3] = u[0][r];
    U[r * 3 + 1] = u[1][r];
    U[r * 3 + 2] = u2[r];
    V[r * 3 + 2] = v2[r];
  }
  for (int k = 0; k < 3; ++k) s[k] = sqrt(w[k] > 0.0 ? w[k] : 0.0);
}

// The pose [R | t] of the 4 decompositions of E (t = +-u2, R = U W V^T or U W^T V^T) with the largest score on the
// k rows (x1, x2), scored as the reference does: the sum of agreement over the rows that triangulate; a pose only
// replaces the best one when its score is larger, starting from 0 (all zeros when none beats 0).  margin: the
// smallest gap between the winning score and another candidate's (or 0).
OSFM_HD void pose_from_essential(const double* E, int k, const double* x1, const double* x2, double* out,
                                 double* margin) {
  double U[9], V[9], s[3];
  essential_svd(E, U, V, s);
  double scores[5];
  scores[4] = 0.0;
  double best = 0.0;
  int win = 4;
  for (int c = 0; c < 12; ++c) out[c] = 0.0;
  for (int i = 0; i < 2; ++i) {
    double t[3];
    for (int r = 0; r < 3; ++r) t[r] = i == 0 ? U[r * 3 + 2] : -U[r * 3 + 2];
    normalize3(t);
    for (int j = 0; j < 2; ++j) {
      // U W V^T = -u0 v1^T + u1 v0^T + u2 v2^T; U W^T V^T flips the first two terms
      const double sg = j == 0 ? 1.0 : -1.0;
      double M[12];
      for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c)
          M[r * 4 + c] = sg * (U[r * 3 + 1] * V[c * 3] - U[r * 3] * V[c * 3 + 1]) + U[r * 3 + 2] * V[c * 3 + 2];
        M[r * 4 + 3] = t[r];
      }
      double score = 0.0;
      for (int q = 0; q < k; ++q) {
        double a;
        if (agreement(M, x1 + 3 * q, x2 + 3 * q, &a)) score += a;
      }
      scores[2 * i + j] = score;
      if (score > best) {
        best = score;
        win = 2 * i + j;
        for (int c = 0; c < 12; ++c) out[c] = M[c];
      }
    }
  }
  double m = INFINITY;
  for (int c = 0; c < 5; ++c)
    if (c != win) m = fmin(m, fabs(best - scores[c]));
  *margin = m;
}

// ---------------------------------------------------------------------------------------------------------------
// EssentialNPoints
// ---------------------------------------------------------------------------------------------------------------

// row q of the epipolar system x2^T E x1 = 0 in E's row-major entries
OSFM_HD void epipolar_row(const double* x1, const double* x2, double* a) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) a[3 * i + j] = x2[i] * x1[j];
}

// EssentialNPoints of k rows: none below 9 rows; otherwise 1 essential into E or 0 (a nullspace of more than one dimension).  The
// singular values of the k x 9 system are the square roots of the eigenvalues of A^T A.  ratio_margin:
// |sigma_8 / sigma_9 - 4|.
OSFM_HD int n_points(int k, const double* x1, const double* x2, double* E, double* ratio_margin) {
  *ratio_margin = INFINITY;
  if (k < 9) return 0;   // SolveAX0 refuses an under-determined system
  double AtA[81], V[81], w[9];
  for (int i = 0; i < 81; ++i) AtA[i] = 0.0;
  for (int q = 0; q < k; ++q) {
    double a[9];
    epipolar_row(x1 + 3 * q, x2 + 3 * q, a);
    for (int i = 0; i < 9; ++i)
      for (int j = 0; j < 9; ++j) AtA[i * 9 + j] += a[i] * a[j];
  }
  sym_eig(AtA, 9, V, w);
  const double s7 = sqrt(w[7] > 0.0 ? w[7] : 0.0), s8 = sqrt(w[8] > 0.0 ? w[8] : 0.0);
  const double ratio = s7 / s8;
  *ratio_margin = fabs(ratio - NULLSPACE_RATIO);
  if (!(ratio > NULLSPACE_RATIO)) return 0;
  double E0[9];
  for (int i = 0; i < 9; ++i) E0[i] = V[i * 9 + 8];
  // the closest essential: singular values ((a + b) / 2, (a + b) / 2, 0)
  double U[9], VE[9], s[3];
  essential_svd(E0, U, VE, s);
  const double m = 0.5 * (s[0] + s[1]);
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) E[r * 3 + c] = m * (U[r * 3] * VE[c * 3] + U[r * 3 + 1] * VE[c * 3 + 1]);
  return 1;
}

// ---------------------------------------------------------------------------------------------------------------
// EssentialFivePoints
// ---------------------------------------------------------------------------------------------------------------

// Monomials of degree <= 3 in x, y, z, in the reference's order: by degree descending, then by the power of z,
// then by the power of y (xxx xxy xyy yyy xxz xyz yyz xzz yzz zzz xx xy yy xz yz zz x y z 1).
OSFM_HD int mono_index(int py, int pz, int d) {
  const int offset = d == 3 ? 0 : d == 2 ? 10 : d == 1 ? 16 : 19;
  int before = 0;
  for (int e = 0; e < pz; ++e) before += d - e + 1;
  return offset + before + py;
}

// exponents (y, z, degree) of monomial k
OSFM_HD void mono_exponents(int k, int* py, int* pz, int* d) {
  int idx = 0;
  for (int deg = 3; deg >= 0; --deg)
    for (int ez = 0; ez <= deg; ++ez)
      for (int ey = 0; ey <= deg - ez; ++ey, ++idx)
        if (idx == k) {
          *py = ey;
          *pz = ez;
          *d = deg;
          return;
        }
}

// out += a * b for polynomials a of degree <= da and b of degree <= db (da + db <= 3), 20 coefficients each
OSFM_HD void poly_mul_add(const double* a, int da, const double* b, int db, double sign, double* out) {
  const int first_a = da == 1 ? 16 : 10, first_b = db == 1 ? 16 : 10;
  for (int i = first_a; i < 20; ++i) {
    if (a[i] == 0.0) continue;
    int ya = 0, za = 0, dga = 0;
    mono_exponents(i, &ya, &za, &dga);
    for (int j = first_b; j < 20; ++j) {
      int yb = 0, zb = 0, dgb = 0;
      mono_exponents(j, &yb, &zb, &dgb);
      out[mono_index(ya + yb, za + zb, dga + dgb)] += sign * a[i] * b[j];
    }
  }
}

// The reference's Gauss-Jordan of the 10 x 20 constraint matrix, without pivoting: false on a zero diagonal.
OSFM_HD bool gauss_jordan(double* M) {
  for (int i = 0; i < 10; ++i) {
    const double dg = M[i * 20 + i];
    if (dg == 0.0) return false;
    for (int c = 0; c < 20; ++c) M[i * 20 + c] /= dg;
    for (int j = i + 1; j < 10; ++j) {
      const double e = M[j * 20 + i];
      if (e == 0.0) continue;
      for (int c = 0; c < 20; ++c) M[j * 20 + c] = M[j * 20 + c] / e - M[i * 20 + c];
    }
  }
  for (int i = 9; i >= 0; --i)
    for (int j = 0; j < i; ++j) {
      const double f = M[j * 20 + i];
      for (int c = 0; c < 20; ++c) M[j * 20 + c] -= f * M[i * 20 + c];
    }
  return true;
}

// The 4-dimensional nullspace of the 5 x 9 epipolar system: the last 4 columns of Q of the Householder QR of A^T.
OSFM_HD void nullspace5(const double* x1, const double* x2, double* N /* 9 x 4 */) {
  double W[9][5], v[5][9];
  for (int q = 0; q < 5; ++q) {
    double a[9];
    epipolar_row(x1 + 3 * q, x2 + 3 * q, a);
    for (int i = 0; i < 9; ++i) W[i][q] = a[i];
  }
  double beta[5];
  for (int j = 0; j < 5; ++j) {
    double nx = 0.0;
    for (int i = j; i < 9; ++i) nx += W[i][j] * W[i][j];
    nx = sqrt(nx);
    const double alpha = W[j][j] >= 0.0 ? -nx : nx;
    for (int i = 0; i < 9; ++i) v[j][i] = i < j ? 0.0 : W[i][j];
    v[j][j] -= alpha;
    double b = 0.0;
    for (int i = j; i < 9; ++i) b += v[j][i] * v[j][i];
    beta[j] = b;
    if (b == 0.0) continue;
    for (int c = j; c < 5; ++c) {
      double p = 0.0;
      for (int i = j; i < 9; ++i) p += v[j][i] * W[i][c];
      p = 2.0 * p / b;
      for (int i = j; i < 9; ++i) W[i][c] -= p * v[j][i];
    }
  }
  // Q e_c = H_0 H_1 ... H_4 e_c for c = 5 .. 8
  for (int c = 0; c < 4; ++c) {
    double e[9];
    for (int i = 0; i < 9; ++i) e[i] = i == 5 + c ? 1.0 : 0.0;
    for (int j = 4; j >= 0; --j) {
      if (beta[j] == 0.0) continue;
      double p = 0.0;
      for (int i = j; i < 9; ++i) p += v[j][i] * e[i];
      p = 2.0 * p / beta[j];
      for (int i = j; i < 9; ++i) e[i] -= p * v[j][i];
    }
    for (int i = 0; i < 9; ++i) N[i * 4 + c] = e[i];
  }
}

// The action matrix of multiplication by x, from the eliminated constraint matrix M (Stewenius' construction)
OSFM_HD void action_matrix(const double* M, double* A /* 10 x 10 */) {
  const int rows[6] = {0, 1, 2, 4, 5, 7};
  for (int i = 0; i < 100; ++i) A[i] = 0.0;
  for (int r = 0; r < 6; ++r)
    for (int c = 0; c < 10; ++c) A[r * 10 + c] = -M[rows[r] * 20 + 10 + c];
  A[6 * 10 + 0] = 1.0;
  A[7 * 10 + 1] = 1.0;
  A[8 * 10 + 3] = 1.0;
  A[9 * 10 + 6] = 1.0;
}

// Eigenvalues (wr, wi) of the n x n matrix a (destroyed): reduction to upper Hessenberg form by stabilised
// elementary similarity transforms, then Francis' double-shift QR with EISPACK's exceptional shifts; false when an
// eigenvalue takes more than HQR_ITERATIONS steps.
OSFM_HD bool eigenvalues(double* a, int n, double* wr, double* wi) {
#define A_(i, j) a[(i) * n + (j)]
  for (int m = 1; m < n - 1; ++m) {
    double x = 0.0;
    int i = m;
    for (int j = m; j < n; ++j)
      if (fabs(A_(j, m - 1)) > fabs(x)) {
        x = A_(j, m - 1);
        i = j;
      }
    if (i != m) {
      for (int j = m - 1; j < n; ++j) {
        const double t = A_(i, j);
        A_(i, j) = A_(m, j);
        A_(m, j) = t;
      }
      for (int j = 0; j < n; ++j) {
        const double t = A_(j, i);
        A_(j, i) = A_(j, m);
        A_(j, m) = t;
      }
    }
    if (x != 0.0)
      for (i = m + 1; i < n; ++i) {
        double y = A_(i, m - 1);
        if (y != 0.0) {
          y /= x;
          A_(i, m - 1) = y;
          for (int j = m; j < n; ++j) A_(i, j) -= y * A_(m, j);
          for (int j = 0; j < n; ++j) A_(j, m) += y * A_(j, i);
        }
      }
  }
  for (int i = 2; i < n; ++i)
    for (int j = 0; j < i - 1; ++j) A_(i, j) = 0.0;

  double anorm = 0.0;
  for (int i = 0; i < n; ++i)
    for (int j = i > 0 ? i - 1 : 0; j < n; ++j) anorm += fabs(A_(i, j));
  int nn = n - 1;
  double t = 0.0;
  double p = 0.0, q = 0.0, r = 0.0, s, w, x, y, z;
  while (nn >= 0) {
    int its = 0, l;
    do {
      for (l = nn; l >= 1; --l) {
        s = fabs(A_(l - 1, l - 1)) + fabs(A_(l, l));
        if (s == 0.0) s = anorm;
        if (fabs(A_(l, l - 1)) + s == s) {
          A_(l, l - 1) = 0.0;
          break;
        }
      }
      x = A_(nn, nn);
      if (l == nn) {
        wr[nn] = x + t;
        wi[nn--] = 0.0;
      } else {
        y = A_(nn - 1, nn - 1);
        w = A_(nn, nn - 1) * A_(nn - 1, nn);
        if (l == nn - 1) {
          p = 0.5 * (y - x);
          q = p * p + w;
          z = sqrt(fabs(q));
          x += t;
          if (q >= 0.0) {
            z = p + (p >= 0.0 ? fabs(z) : -fabs(z));
            wr[nn - 1] = wr[nn] = x + z;
            if (z != 0.0) wr[nn] = x - w / z;
            wi[nn - 1] = wi[nn] = 0.0;
          } else {
            wr[nn - 1] = wr[nn] = x + p;
            wi[nn - 1] = -(wi[nn] = z);
          }
          nn -= 2;
        } else {
          if (its == HQR_ITERATIONS) return false;
          if (its == 10 || its == 20) {
            t += x;
            for (int i = 0; i <= nn; ++i) A_(i, i) -= x;
            s = fabs(A_(nn, nn - 1)) + fabs(A_(nn - 1, nn - 2));
            y = x = 0.75 * s;
            w = -0.4375 * s * s;
          }
          ++its;
          int m;
          for (m = nn - 2; m >= l; --m) {
            z = A_(m, m);
            r = x - z;
            s = y - z;
            p = (r * s - w) / A_(m + 1, m) + A_(m, m + 1);
            q = A_(m + 1, m + 1) - z - r - s;
            r = A_(m + 2, m + 1);
            s = fabs(p) + fabs(q) + fabs(r);
            p /= s;
            q /= s;
            r /= s;
            if (m == l) break;
            const double u = fabs(A_(m, m - 1)) * (fabs(q) + fabs(r));
            const double v = fabs(p) * (fabs(A_(m - 1, m - 1)) + fabs(z) + fabs(A_(m + 1, m + 1)));
            if (u + v == v) break;
          }
          for (int i = m + 2; i <= nn; ++i) {
            A_(i, i - 2) = 0.0;
            if (i != m + 2) A_(i, i - 3) = 0.0;
          }
          for (int k = m; k <= nn - 1; ++k) {
            if (k != m) {
              p = A_(k, k - 1);
              q = A_(k + 1, k - 1);
              r = 0.0;
              if (k != nn - 1) r = A_(k + 2, k - 1);
              if ((x = fabs(p) + fabs(q) + fabs(r)) != 0.0) {
                p /= x;
                q /= x;
                r /= x;
              }
            }
            const double nrm = sqrt(p * p + q * q + r * r);
            if ((s = p >= 0.0 ? nrm : -nrm) != 0.0) {
              if (k == m) {
                if (l != m) A_(k, k - 1) = -A_(k, k - 1);
              } else {
                A_(k, k - 1) = -s * x;
              }
              p += s;
              x = p / s;
              y = q / s;
              z = r / s;
              q /= p;
              r /= p;
              for (int j = k; j <= nn; ++j) {
                p = A_(k, j) + q * A_(k + 1, j);
                if (k != nn - 1) {
                  p += r * A_(k + 2, j);
                  A_(k + 2, j) -= p * z;
                }
                A_(k + 1, j) -= p * y;
                A_(k, j) -= p * x;
              }
              const int mmin = nn < k + 3 ? nn : k + 3;
              for (int i = l; i <= mmin; ++i) {
                p = x * A_(i, k) + y * A_(i, k + 1);
                if (k != nn - 1) {
                  p += z * A_(i, k + 2);
                  A_(i, k + 2) -= p * r;
                }
                A_(i, k + 1) -= p * q;
                A_(i, k) -= p;
              }
            }
          }
        }
      }
    } while (l < nn - 1);
  }
#undef A_
  return true;
}

// A null vector of the 10 x 10 matrix B (destroyed) by Gaussian elimination with complete pivoting; the last
// unknown is set to 1 and a zero pivot's unknown to 0.
OSFM_HD void null_vector10(double* B, double* v) {
  int col[10];
  for (int j = 0; j < 10; ++j) col[j] = j;
  for (int k = 0; k < 9; ++k) {
    int pi = k, pj = k;
    double big = -1.0;
    for (int i = k; i < 10; ++i)
      for (int j = k; j < 10; ++j)
        if (fabs(B[i * 10 + j]) > big) {
          big = fabs(B[i * 10 + j]);
          pi = i;
          pj = j;
        }
    if (pi != k)
      for (int j = 0; j < 10; ++j) {
        const double t = B[k * 10 + j];
        B[k * 10 + j] = B[pi * 10 + j];
        B[pi * 10 + j] = t;
      }
    if (pj != k) {
      for (int i = 0; i < 10; ++i) {
        const double t = B[i * 10 + k];
        B[i * 10 + k] = B[i * 10 + pj];
        B[i * 10 + pj] = t;
      }
      const int t = col[k];
      col[k] = col[pj];
      col[pj] = t;
    }
    const double d = B[k * 10 + k];
    if (d == 0.0) continue;
    for (int i = k + 1; i < 10; ++i) {
      const double f = B[i * 10 + k] / d;
      for (int j = k; j < 10; ++j) B[i * 10 + j] -= f * B[k * 10 + j];
    }
  }
  double y[10];
  y[9] = 1.0;
  for (int k = 8; k >= 0; --k) {
    double s = 0.0;
    for (int j = k + 1; j < 10; ++j) s += B[k * 10 + j] * y[j];
    y[k] = B[k * 10 + k] == 0.0 ? 0.0 : -s / B[k * 10 + k];
  }
  for (int j = 0; j < 10; ++j) v[col[j]] = y[j];
}

// The constraint matrix of the nullspace basis N (9 x 4; E = x N0 + y N1 + z N2 + N3): det(E) = 0 and
// 2 E E^T E - trace(E E^T) E = 0.
OSFM_HD void constraints(const double* N, double* M /* 10 x 20 */) {
  double E[9][20];
  for (int e = 0; e < 9; ++e) {
    for (int c = 0; c < 20; ++c) E[e][c] = 0.0;
    E[e][16] = N[e * 4];
    E[e][17] = N[e * 4 + 1];
    E[e][18] = N[e * 4 + 2];
    E[e][19] = N[e * 4 + 3];
  }
  for (int i = 0; i < 200; ++i) M[i] = 0.0;
  // det(E) by the first row's cofactors, each a 2 x 2 minor of rows 1, 2
  for (int j = 0; j < 3; ++j) {
    const int j1 = (j + 1) % 3, j2 = (j + 2) % 3;
    double minor[20];
    for (int c = 0; c < 20; ++c) minor[c] = 0.0;
    poly_mul_add(E[3 + j1], 1, E[6 + j2], 1, 1.0, minor);
    poly_mul_add(E[3 + j2], 1, E[6 + j1], 1, -1.0, minor);
    poly_mul_add(minor, 2, E[j], 1, 1.0, M);
  }
  // L = E E^T - trace(E E^T) / 2 I, then the rows of L E
  double L[9][20];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      for (int c = 0; c < 20; ++c) L[i * 3 + j][c] = 0.0;
      if (j < i) {
        for (int c = 0; c < 20; ++c) L[i * 3 + j][c] = L[j * 3 + i][c];
        continue;
      }
      for (int k = 0; k < 3; ++k) poly_mul_add(E[i * 3 + k], 1, E[j * 3 + k], 1, 1.0, L[i * 3 + j]);
    }
  double half_trace[20];
  for (int c = 0; c < 20; ++c) half_trace[c] = 0.5 * (L[0][c] + L[4][c] + L[8][c]);
  for (int i = 0; i < 3; ++i)
    for (int c = 0; c < 20; ++c) L[i * 4][c] -= half_trace[c];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j)
      for (int k = 0; k < 3; ++k) poly_mul_add(L[i * 3 + k], 2, E[k * 3 + j], 1, 1.0, M + (1 + i * 3 + j) * 20);
}

// EssentialFivePoints of 5 rows: the number of essentials written to Es (9 each, unit Frobenius norm), in ascending
// order of their eigenvalue.  class_margin: the smallest | |Im| - REAL_TOLERANCE (1 + |Re|) | / (1 + |Re|) of the
// action matrix's eigenvalues with a nonzero imaginary part.
OSFM_HD int five_point(const double* x1, const double* x2, double* Es, double* class_margin) {
  double N[36], M[200], A[100], B[100], wr[10], wi[10];
  *class_margin = INFINITY;
  nullspace5(x1, x2, N);
  constraints(N, M);
  if (!gauss_jordan(M)) return 0;
  action_matrix(M, A);
  for (int i = 0; i < 100; ++i)
    if (!finite(A[i])) return 0;
  for (int i = 0; i < 100; ++i) B[i] = A[i];
  if (!eigenvalues(B, 10, wr, wi)) return 0;
  double roots[10];
  int nr = 0;
  for (int i = 0; i < 10; ++i) {
    const double scale = 1.0 + fabs(wr[i]);
    if (wi[i] != 0.0) *class_margin = fmin(*class_margin, fabs(fabs(wi[i]) - REAL_TOLERANCE * scale) / scale);
    if (fabs(wi[i]) <= REAL_TOLERANCE * scale) roots[nr++] = wr[i];
  }
  // ascending (insertion sort)
  for (int i = 1; i < nr; ++i)
    for (int j = i; j > 0 && roots[j] < roots[j - 1]; --j) {
      const double t = roots[j];
      roots[j] = roots[j - 1];
      roots[j - 1] = t;
    }
  for (int s = 0; s < nr; ++s) {
    double v[10];
    for (int i = 0; i < 100; ++i) B[i] = A[i] - (i % 11 == 0 ? roots[s] : 0.0);
    null_vector10(B, v);
    const double x = v[6] / v[9], y = v[7] / v[9], z = v[8] / v[9];
    double* E = Es + 9 * s;
    double nrm = 0.0;
    for (int e = 0; e < 9; ++e) {
      E[e] = x * N[e * 4] + y * N[e * 4 + 1] + z * N[e * 4 + 2] + N[e * 4 + 3];
      nrm += E[e] * E[e];
    }
    nrm = sqrt(nrm);
    for (int e = 0; e < 9; ++e) E[e] /= nrm;
  }
  return nr;
}

}  // namespace relpose
}  // namespace osfm
