// Absolute-pose solvers of pyrobust's AbsolutePose model (geometry/absolute_pose.h), fp64, for the device and, compiled
// by g++, for the host tests (tests/cpu_harness/absolute_pose_host.cpp):
//
//   p3p_ke           Ke and Roumeliotis' P3P: the quartic in cos(theta1) by the closed form of foundation::SolveQuartic
//                    (complex pow, principal branches), each root refined by 5 Newton steps, up to 4 models
//   lu_pose          Lu, Hager and Mjolsness' orthogonal iteration (AbsolutePoseNPoints) from a scaled Horn start
//   rotation_between RotationBetweenPoints: the polar factor of the centred cross-covariance, negated if improper,
//                    with the proper (Kabsch) completion for exactly 3 rows
//
// The restatement and the reasons for its one deliberate difference (the 3-row completion) are in
// oracle/absolute_pose_oracle.py and oracle/rotation_ransac_oracle.py.  Matrices are row-major; a pose is the 3 x 4
// [R | t] with x_camera = R X + t.
#pragma once

#include <cmath>

#ifdef __CUDACC__
#define OSFM_HD __host__ __device__ inline
#else
#define OSFM_HD inline
#endif

namespace osfm {
namespace pose {

constexpr int POLAR_MAX_ITERATIONS = 50;
constexpr double POLAR_UNSCALED_BELOW = 1e-2;  // Frobenius step below which the Newton iteration stops scaling
constexpr double POLAR_TOLERANCE = 1e-14;      // Frobenius step below which it stops
constexpr int QUARTIC_NEWTON_STEPS = 5;
constexpr double QUARTIC_NEWTON_TOLERANCE = 1e-20;
constexpr int LU_MAX_ITERATIONS = 100;
constexpr double LU_TOLERANCE = 1e-7;

OSFM_HD bool finite(double x) {
#ifdef __CUDA_ARCH__
  return isfinite(x);
#else
  return std::isfinite(x);
#endif
}

// ---- 3 x 3 algebra ------------------------------------------------------------------------------------------
// cof(X) has columns c1 x c2, c2 x c0, c0 x c1 (c_j the columns of X), so X^-T = cof(X) / det(X)
OSFM_HD void cofactor(const double* X, double* C) {
  for (int j = 0; j < 3; ++j) {
    const int a = (j + 1) % 3, b = (j + 2) % 3;
    C[0 * 3 + j] = X[1 * 3 + a] * X[2 * 3 + b] - X[2 * 3 + a] * X[1 * 3 + b];
    C[1 * 3 + j] = X[2 * 3 + a] * X[0 * 3 + b] - X[0 * 3 + a] * X[2 * 3 + b];
    C[2 * 3 + j] = X[0 * 3 + a] * X[1 * 3 + b] - X[1 * 3 + a] * X[0 * 3 + b];
  }
}

OSFM_HD double frobenius(const double* X) {
  double s = 0.0;
  for (int k = 0; k < 9; ++k) s += X[k] * X[k];
  return sqrt(s);
}

// orthogonal polar factor by scaled Newton (Higham), in place; false if X is singular or not finite
OSFM_HD bool polar(double* X) {
  const double nx = frobenius(X);
  if (!finite(nx) || nx == 0.0) return false;
  for (int k = 0; k < 9; ++k) X[k] /= nx;
  bool scaled = true;
  for (int it = 0; it < POLAR_MAX_ITERATIONS; ++it) {
    double C[9];
    cofactor(X, C);
    const double d = X[0] * C[0] + X[3] * C[3] + X[6] * C[6];
    if (d == 0.0 || !finite(d)) return false;
    for (int k = 0; k < 9; ++k) C[k] /= d;
    const double z = scaled ? sqrt(frobenius(C) / frobenius(X)) : 1.0;
    double step = 0.0;
    for (int k = 0; k < 9; ++k) {
      const double xn = scaled ? 0.5 * (z * X[k] + C[k] / z) : 0.5 * (X[k] + C[k]);
      step += (xn - X[k]) * (xn - X[k]);
      X[k] = xn;
    }
    step = sqrt(step);
    if (step < POLAR_UNSCALED_BELOW) scaled = false;
    if (step <= POLAR_TOLERANCE) break;
  }
  for (int k = 0; k < 9; ++k)
    if (!finite(X[k])) return false;
  return true;
}

OSFM_HD double det3(const double* X) {
  double C[9];
  cofactor(X, C);
  return X[0] * C[0] + X[3] * C[3] + X[6] * C[6];
}

// ClosestRotationMatrix: the polar factor, negated if improper; false if there is none
OSFM_HD bool closest_rotation(double* X) {
  if (!polar(X)) return false;
  if (det3(X) < 0.0)
    for (int q = 0; q < 9; ++q) X[q] = -X[q];
  return true;
}

// The rotation Q with Q b_i ~ a_i of k rows (a_i at a + i * stride, b_i at b + i * stride), into out: the polar
// factor of the centred cross-covariance sum (a_i - mean a)(b_i - mean b)^T, negated if improper; for k = 3 (rank 2)
// the polar factor of M + (|M| / |cof M|) cof M, the proper completion.  The identity if M is singular.
OSFM_HD void rotation_between(int k, const double* a, const double* b, int stride, double* out) {
  double m1[3], m2[3];
  for (int c = 0; c < 3; ++c) {
    m1[c] = a[c];
    m2[c] = b[c];
  }
  for (int i = 1; i < k; ++i)
    for (int c = 0; c < 3; ++c) {
      m1[c] += a[i * stride + c];
      m2[c] += b[i * stride + c];
    }
  for (int c = 0; c < 3; ++c) {
    m1[c] /= k;
    m2[c] /= k;
  }
  double X[9];
  for (int q = 0; q < 9; ++q) X[q] = 0.0;
  for (int i = 0; i < k; ++i) {
    double dp[3], dq[3];
    for (int c = 0; c < 3; ++c) {
      dp[c] = a[i * stride + c] - m1[c];
      dq[c] = b[i * stride + c] - m2[c];
    }
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) X[r * 3 + c] += dp[r] * dq[c];
  }
  if (k == 3) {
    double C[9];
    cofactor(X, C);
    const double nc = frobenius(C);
    if (nc > 0.0) {
      const double w = frobenius(X) / nc;
      for (int q = 0; q < 9; ++q) X[q] = X[q] + w * C[q];
    }
  }
  if (!polar(X)) {
    for (int q = 0; q < 9; ++q) out[q] = (q % 4 == 0) ? 1.0 : 0.0;
    return;
  }
  const double sgn = det3(X) < 0.0 ? -1.0 : 1.0;
  for (int q = 0; q < 9; ++q) out[q] = sgn * X[q];
}

OSFM_HD void matmul3(const double* A, const double* B, double* C) {
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) C[r * 3 + c] = A[r * 3] * B[c] + A[r * 3 + 1] * B[3 + c] + A[r * 3 + 2] * B[6 + c];
}

OSFM_HD void matvec3(const double* A, const double* x, double* y) {
  for (int r = 0; r < 3; ++r) y[r] = A[r * 3] * x[0] + A[r * 3 + 1] * x[1] + A[r * 3 + 2] * x[2];
}

OSFM_HD void cross3(const double* u, const double* v, double* w) {
  w[0] = u[1] * v[2] - u[2] * v[1];
  w[1] = u[2] * v[0] - u[0] * v[2];
  w[2] = u[0] * v[1] - u[1] * v[0];
}

OSFM_HD double dot3(const double* u, const double* v) { return u[0] * v[0] + u[1] * v[1] + u[2] * v[2]; }
OSFM_HD double norm3(const double* u) { return sqrt(dot3(u, u)); }

// ---- the quartic of foundation::SolveQuartic ------------------------------------------------------------------
struct Cx {
  double re, im;
};
OSFM_HD Cx cx(double re) { return Cx{re, 0.0}; }
OSFM_HD Cx operator+(Cx a, Cx b) { return Cx{a.re + b.re, a.im + b.im}; }
OSFM_HD Cx operator-(Cx a, Cx b) { return Cx{a.re - b.re, a.im - b.im}; }
OSFM_HD Cx operator*(double s, Cx a) { return Cx{s * a.re, s * a.im}; }
OSFM_HD Cx operator/(Cx a, double s) { return Cx{a.re / s, a.im / s}; }
OSFM_HD Cx operator/(Cx a, Cx b) {
  const double d = b.re * b.re + b.im * b.im;
  return Cx{(a.re * b.re + a.im * b.im) / d, (a.im * b.re - a.re * b.im) / d};
}
// std::pow(complex, real): the real pow for a positive real z, else polar(exp(y log|z|), y arg z)
OSFM_HD Cx cx_pow(Cx z, double y) {
  if (z.im == 0.0 && z.re > 0.0) return Cx{pow(z.re, y), 0.0};
  const double lr = log(hypot(z.re, z.im)), th = atan2(z.im, z.re);
  const double rho = exp(y * lr), phi = y * th;
  return Cx{rho * cos(phi), rho * sin(phi)};
}

// coefficients c[0] + c[1] x + ... + c[4] x^4; false when the closed form is degenerate (all of Q1..Q4 below eps)
OSFM_HD bool solve_quartic(const double* coef, double* roots) {
  const double eps = 2.220446049250313e-16;
  const double a = fabs(coef[4]) > eps ? coef[4] : eps;
  const double b = coef[3] / a, c = coef[2] / a, d = coef[1] / a, e = coef[0] / a;
  const double Q1 = c * c - 3. * b * d + 12. * e;
  const double Q2 = 2. * c * c * c - 9. * b * c * d + 27. * d * d + 27. * b * b * e - 72. * c * e;
  const double Q3 = 8. * b * c - 16. * d - 2. * b * b * b;
  const double Q4 = 3. * b * b - 8. * c;
  if (fabs(Q1) < eps && fabs(Q2) < eps && fabs(Q3) < eps && fabs(Q4) < eps) return false;
  const Cx Q5 = cx_pow(cx(Q2 / 2.) + cx_pow(cx(Q2 * Q2 / 4. - Q1 * Q1 * Q1), 1. / 2.), 1. / 3.);
  const Cx Q6 = (cx(Q1) / Q5 + Q5) / 3.;
  const Cx Q7 = 2. * cx_pow(cx(Q4 / 12.) + Q6, 1. / 2.);
  const Cx Q3Q7 = cx(Q3) / Q7;
  const Cx base = cx(4. * Q4 / 6.) - 4. * Q6;
  const Cx s1 = cx_pow(base - Q3Q7, 1. / 2.), s2 = cx_pow(base + Q3Q7, 1. / 2.);
  roots[0] = (cx(-b) - Q7 - s1).re / 4.;
  roots[1] = (cx(-b) - Q7 + s1).re / 4.;
  roots[2] = (cx(-b) + Q7 - s2).re / 4.;
  roots[3] = (cx(-b) + Q7 + s2).re / 4.;
  return true;
}

// RefineQuarticRoots: 5 Newton steps per root, stopping when the step is below 1e-20 (or the derivative is 0)
OSFM_HD double refine_quartic_root(const double* coef, double x) {
  for (int i = 0; i < QUARTIC_NEWTON_STEPS; ++i) {
    const double f = (((coef[4] * x + coef[3]) * x + coef[2]) * x + coef[1]) * x + coef[0];
    const double x2 = x * x, x3 = x2 * x;
    const double df = 4.0 * coef[4] * x3 + 3.0 * coef[3] * x2 + 2.0 * coef[2] * x + coef[1];
    const double decr = df == 0.0 ? 0.0 : f / df;
    if (fabs(decr) < QUARTIC_NEWTON_TOLERANCE) break;
    x -= decr;
  }
  return x;
}

// RotationMatrixAroundAxis(cos, sin, v), row-major
OSFM_HD void rotation_around_axis(double c, double s, const double* v, double* R) {
  const double omc = 1.0 - c;
  R[0] = c + v[0] * v[0] * omc;
  R[3] = -v[2] * s + v[0] * v[1] * omc;
  R[6] = v[1] * s + v[0] * v[2] * omc;
  R[1] = v[2] * s + v[0] * v[1] * omc;
  R[4] = c + v[1] * v[1] * omc;
  R[7] = -v[0] * s + v[1] * v[2] * omc;
  R[2] = -v[1] * s + v[0] * v[2] * omc;
  R[5] = v[0] * s + v[1] * v[2] * omc;
  R[8] = c + v[2] * v[2] * omc;
}

// AbsolutePoseThreePoints: bearings b (3 x 3, one row per point) and world points p; writes 4 poses (row-major
// 3 x 4 [R | t], world to camera) into models and returns 4, or returns 0 when sigma = 0, k3 . b3 = 0 or the
// quartic is degenerate.  A root with |cos| > 1 gives a NaN pose.
OSFM_HD int p3p_ke(const double* b, const double* p, double* models) {
  const double *b1 = b, *b2 = b + 3, *b3 = b + 6, *p1 = p, *p2 = p + 3, *p3 = p + 6;
  double k1[3], k3[3], u1[3], u2[3], v1[3], v2[3], u1_k1[3], k3s[3];
  for (int c = 0; c < 3; ++c) {
    k1[c] = p1[c] - p2[c];
    u1[c] = p1[c] - p3[c];
    u2[c] = p2[c] - p3[c];
  }
  const double nk1 = norm3(k1);
  for (int c = 0; c < 3; ++c) k1[c] /= nk1;
  cross3(b1, b2, k3);
  const double b1_b2 = norm3(k3);
  for (int c = 0; c < 3; ++c) k3[c] /= b1_b2;
  cross3(b1, b3, v1);
  cross3(b2, b3, v2);
  cross3(u1, k1, u1_k1);
  const double sigma = norm3(u1_k1);
  if (sigma == 0.0) return 0;
  for (int c = 0; c < 3; ++c) k3s[c] = u1_k1[c] / sigma;
  const double k3_b3 = dot3(k3, b3);
  if (k3_b3 == 0.0) return 0;
  const double b1b2 = dot3(b1, b2);
  const double f11 = sigma * k3_b3;
  const double f21 = sigma * b1b2 * k3_b3;
  const double f22 = sigma * k3_b3 * b1_b2;
  const double f13 = sigma * dot3(v1, k3);
  const double f23 = sigma * dot3(v2, k3);
  const double f24 = dot3(u2, k1) * k3_b3 * b1_b2;
  const double f15 = -dot3(u1, k1) * k3_b3;
  const double f25 = -dot3(u2, k1) * b1b2 * k3_b3;
  const double g1 = f13 * f22;
  const double g2 = f13 * f25 - f15 * f23;
  const double g3 = f11 * f23 - f13 * f21;
  const double g4 = -f13 * f24;
  const double g5 = f11 * f22;
  const double g6 = f11 * f25 - f15 * f21;
  const double g7 = -f15 * f24;
  double coef[5];
  coef[4] = g5 * g5 + g1 * g1 + g3 * g3;
  coef[3] = 2.0 * (g5 * g6 + g1 * g2 + g3 * g4);
  coef[2] = g6 * g6 + 2.0 * g5 * g7 + g2 * g2 + g4 * g4 - g1 * g1 - g3 * g3;
  coef[1] = 2.0 * (g6 * g7 - g1 * g2 - g3 * g4);
  coef[0] = g7 * g7 - g2 * g2 - g4 * g4;
  double roots[4];
  if (!solve_quartic(coef, roots)) return 0;

  // c_barre = [k1 | k3'' | k1 x k3''] (columns), c_barre_barre = [b1; k3; b1 x k3] (rows)
  double cb[9], cbb[9], w[3];
  cross3(k1, k3s, w);
  for (int r = 0; r < 3; ++r) {
    cb[r * 3 + 0] = k1[r];
    cb[r * 3 + 1] = k3s[r];
    cb[r * 3 + 2] = w[r];
  }
  cross3(b1, k3, w);
  for (int c = 0; c < 3; ++c) {
    cbb[0 * 3 + c] = b1[c];
    cbb[1 * 3 + c] = k3[c];
    cbb[2 * 3 + c] = w[c];
  }
  const double e1[3] = {1.0, 0.0, 0.0}, e2[3] = {0.0, 1.0, 0.0};
  const double sgn = k3_b3 < 0.0 ? -1.0 : 1.0;
  for (int m = 0; m < 4; ++m) {
    const double cos1 = refine_quartic_root(coef, roots[m]);
    const double sin1 = sgn * sqrt(1.0 - cos1 * cos1);
    const double t = sin1 / (g5 * cos1 * cos1 + g6 * cos1 + g7);
    const double cos3 = t * (g1 * cos1 + g2);
    const double sin3 = t * (g3 * cos1 + g4);
    double c1[9], c2[9], A[9], B[9], R[9];
    rotation_around_axis(cos1, sin1, e1, c1);
    rotation_around_axis(cos3, sin3, e2, c2);
    matmul3(cb, c1, A);
    matmul3(A, c2, B);
    matmul3(B, cbb, R);
    double* M = models + 12 * m;
    if (!closest_rotation(R)) {
      for (int q = 0; q < 12; ++q) M[q] = NAN;
      continue;
    }
    // translation = p3 - (sigma sin1 / k3_b3) R b3; the pose is [R^T | -R^T translation]
    double Rb3[3], tr[3];
    matvec3(R, b3, Rb3);
    const double f = (sigma * sin1) / k3_b3;
    for (int c = 0; c < 3; ++c) tr[c] = p3[c] - f * Rb3[c];
    for (int r = 0; r < 3; ++r) {
      for (int c = 0; c < 3; ++c) M[r * 4 + c] = R[c * 3 + r];
      M[r * 4 + 3] = -(R[0 * 3 + r] * tr[0] + R[1 * 3 + r] * tr[1] + R[2 * 3 + r] * tr[2]);
    }
  }
  return 4;
}

// ---- AbsolutePoseNPoints ------------------------------------------------------------------------------------
// Lu's orthogonal iteration on k rows (bearings b, world points p, k x 3 each; k <= 12) into the pose out (3 x 4).
// Returns the number of iterations run; *margin, when given, is lowered to the smallest |relative change - 1e-7|.
OSFM_HD int lu_pose(int k, const double* b, const double* p, double* out, double* margin = nullptr) {
  double qbar[3] = {0.0, 0.0, 0.0}, pbar[3] = {0.0, 0.0, 0.0};
  for (int i = 0; i < k; ++i)
    for (int c = 0; c < 3; ++c) {
      qbar[c] += b[3 * i + c];
      pbar[c] += p[3 * i + c];
    }
  for (int c = 0; c < 3; ++c) {
    qbar[c] /= k;
    pbar[c] /= k;
  }
  double s_num = 0.0, s_den = 0.0;
  for (int i = 0; i < k; ++i) {
    double dq[3], dp[3];
    for (int c = 0; c < 3; ++c) {
      dq[c] = b[3 * i + c] - qbar[c];
      dp[c] = p[3 * i + c] - pbar[c];
    }
    const double np = norm3(dp), nq = norm3(dq);
    s_num += np * np;
    s_den += nq * nq;
  }
  const double scale = sqrt(s_num / s_den);
  double R[9], t[3], Rp[3];
  rotation_between(k, b, p, 3, R);
  matvec3(R, pbar, Rp);
  for (int c = 0; c < 3; ++c) t[c] = scale * qbar[c] - Rp[c];

  double q[12 * 3];
  int it = 0;
  while (it < LU_MAX_ITERATIONS) {
    ++it;
    for (int i = 0; i < k; ++i) {
      const double* v = b + 3 * i;
      const double vv = dot3(v, v);
      double x[3];
      matvec3(R, p + 3 * i, x);
      for (int c = 0; c < 3; ++c) x[c] += t[c];
      // F x with F = v v^T / (v . v)
      for (int r = 0; r < 3; ++r) q[3 * i + r] = (v[r] * v[0] / vv) * x[0] + (v[r] * v[1] / vv) * x[1] + (v[r] * v[2] / vv) * x[2];
    }
    rotation_between(k, q, p, 3, R);
    // TranslationBetweenPoints: (I - mean F)^-1 mean (F - I) R p
    double F1[9], F2[3] = {0.0, 0.0, 0.0};
    for (int e = 0; e < 9; ++e) F1[e] = 0.0;
    for (int i = 0; i < k; ++i) {
      const double* v = b + 3 * i;
      const double vv = dot3(v, v);
      double F[9], x[3];
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) F[r * 3 + c] = v[r] * v[c] / vv;
      for (int e = 0; e < 9; ++e) F1[e] += F[e];
      matvec3(R, p + 3 * i, x);
      for (int r = 0; r < 3; ++r)
        F2[r] += (F[r * 3] - (r == 0)) * x[0] + (F[r * 3 + 1] - (r == 1)) * x[1] + (F[r * 3 + 2] - (r == 2)) * x[2];
    }
    double A[9], C[9], nt[3];
    for (int r = 0; r < 3; ++r) F2[r] /= k;
    for (int e = 0; e < 9; ++e) A[e] = (e % 4 == 0 ? 1.0 : 0.0) - F1[e] / k;
    cofactor(A, C);
    const double det = A[0] * C[0] + A[3] * C[3] + A[6] * C[6];
    // A^-1 = cof(A)^T / det(A)
    for (int r = 0; r < 3; ++r) nt[r] = (C[0 * 3 + r] * F2[0] + C[1 * 3 + r] * F2[1] + C[2 * 3 + r] * F2[2]) / det;
    double d[3] = {nt[0] - t[0], nt[1] - t[1], nt[2] - t[2]};
    const double rel = norm3(d) / norm3(t);
    if (margin) *margin = fmin(*margin, fabs(rel - LU_TOLERANCE));
    if (rel < LU_TOLERANCE) break;
    for (int c = 0; c < 3; ++c) t[c] = nt[c];
  }
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) out[r * 4 + c] = R[r * 3 + c];
    out[r * 4 + 3] = t[r];
  }
  return it;
}

}  // namespace pose
}  // namespace osfm
