// TRIANGULATE: 3-D points of many tracks at once, from the observations a tracks handle keeps on the device.
//
// Replaces, for every track triangulate_shot_features / retriangulate hand to it (opensfm/reconstruction.py:
// 1143-1226), TrackTriangulator.triangulate (:1032-1073): TriangulateBearingsMidpoint (geometry/src/triangulation.cc:
// 137-177, its closed-form solve geometry/triangulation.h:58-82) and PointRefinement (triangulation.cc:221-233, a
// Ceres TinySolver over the bearing residuals normalize(X - c_i) - b_i).  The restatement the results are checked
// against, and the TinySolver rules it follows, are in oracle/triangulation_oracle.py.
//
// One thread per track (tri_tracks).  A track's observations are read straight from the handle's (track, image)
// sorted arrays on every pass, rotated into the world frame on the fly from the per-image R^T, so a track of any
// length runs in the same registers; the per-image arrays are small enough to stay in L1.  Passes: count the
// observations in reconstructed images, angle test over pairs (stops at the first pair that passes), midpoint
// sums, reprojection and depth tests, then at most `iterations` Levenberg-Marquardt steps of two passes each.
#include <math_constants.h>

#include <cmath>

#include "triangulate.cuh"

namespace osfm {
namespace {

constexpr int TRI_THREADS = 128;
constexpr double TRI_PI = 3.14159265358979323846;   // M_PI
// TinySolver's default options (the reference sets only max_num_iterations)
constexpr double TRI_GRADIENT_TOLERANCE = 1e-10;
constexpr double TRI_PARAMETER_TOLERANCE = 1e-8;
constexpr double TRI_COST_THRESHOLD = 2.220446049250313e-16;   // std::numeric_limits<double>::epsilon()
constexpr double TRI_INITIAL_TRUST_REGION = 1e4;
constexpr double TRI_MIN_DIAGONAL = 1e-6;
constexpr double TRI_MAX_DIAGONAL = 1e32;

struct TriArgs {
  int T;
  const int* obs_image;
  const long long* track_start;
  const double* rt;              // R^T of every image, row-major
  const double* origin;          // 3 per image
  const unsigned char* in;       // image is in the reconstruction
  const double* bearings;        // 3 per observation, camera frame
  const unsigned char* selected;
  double threshold, min_angle, min_depth;
  int iterations;
  int8_t* status;
  double* X;
};

__device__ __forceinline__ double tri_dot(const double* u, const double* v) {
  return u[0] * v[0] + u[1] * v[1] + u[2] * v[2];
}

// geometry::AngleBetweenVectors: 0 when |cos| >= 1, and NaN (which passes no comparison) for a zero vector
__device__ __forceinline__ double tri_angle(const double* u, const double* v) {
  const double c = tri_dot(u, v) / sqrt(tri_dot(u, u) * tri_dot(v, v));
  return fabs(c) >= 1.0 ? 0.0 : acos(c);
}

// observation r of image im: its world-frame bearing R^T b and its camera's origin
__device__ __forceinline__ void tri_ray(const TriArgs& a, int r, int im, double* w, double* c) {
  const double* R = a.rt + 9LL * im;
  const double* bp = a.bearings + 3LL * r;
  const double b0 = __ldg(bp), b1 = __ldg(bp + 1), b2 = __ldg(bp + 2);
  for (int k = 0; k < 3; ++k) {
    w[k] = __ldg(R + 3 * k) * b0 + __ldg(R + 3 * k + 1) * b1 + __ldg(R + 3 * k + 2) * b2;
    c[k] = __ldg(a.origin + 3 * im + k);
  }
}

__device__ __forceinline__ bool tri_kept(const TriArgs& a, int r, int* im) {
  *im = __ldg(a.obs_image + r);
  return __ldg(a.in + *im) != 0;
}

// cofactor (i, j) of a row-major 3x3, as Eigen's 3x3 inverse takes it
__device__ __forceinline__ double tri_cof(const double* m, int i, int j) {
  const int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
  return m[i1 * 3 + j1] * m[i2 * 3 + j2] - m[i1 * 3 + j2] * m[i2 * 3 + j1];
}

// Bearing cost at x: cost = |f|^2 / 2 of f_i = normalize(x - c_i) - w_i; with lin, also J^T J (upper triangle,
// xx xy xz yy yz zz) and J^T (-f) of the unscaled Jacobian (Normalize::ForwardDerivatives, symmetric)
__device__ __forceinline__ double tri_cost(const TriArgs& a, int b, int e, const double* x, bool lin, double* jtj,
                           double* jte) {
  double cost = 0.0;
  if (lin) {
    for (int k = 0; k < 6; ++k) jtj[k] = 0.0;
    for (int k = 0; k < 3; ++k) jte[k] = 0.0;
  }
  for (int r = b; r < e; ++r) {
    int im;
    if (!tri_kept(a, r, &im)) continue;
    double w[3], c[3];
    tri_ray(a, r, im, w, c);
    const double p0 = x[0] - c[0], p1 = x[1] - c[1], p2 = x[2] - c[2];
    const double x2 = p0 * p0, y2 = p1 * p1, z2 = p2 * p2;
    const double n2 = x2 + y2 + z2;
    const double inv = 1.0 / sqrt(n2);
    const double f0 = p0 * inv - w[0], f1 = p1 * inv - w[1], f2 = p2 * inv - w[2];
    cost += f0 * f0 + f1 * f1 + f2 * f2;
    if (!lin) continue;
    const double i3 = 1.0 / (sqrt(n2) * n2);
    const double jxx = (y2 + z2) * i3, jyy = (x2 + z2) * i3, jzz = (x2 + y2) * i3;
    const double jxy = -p0 * p1 * i3, jxz = -p0 * p2 * i3, jyz = -p1 * p2 * i3;
    jtj[0] += jxx * jxx + jxy * jxy + jxz * jxz;
    jtj[1] += jxx * jxy + jxy * jyy + jxz * jyz;
    jtj[2] += jxx * jxz + jxy * jyz + jxz * jzz;
    jtj[3] += jxy * jxy + jyy * jyy + jyz * jyz;
    jtj[4] += jxy * jxz + jyy * jyz + jyz * jzz;
    jtj[5] += jxz * jxz + jyz * jyz + jzz * jzz;
    jte[0] -= jxx * f0 + jxy * f1 + jxz * f2;
    jte[1] -= jxy * f0 + jyy * f1 + jyz * f2;
    jte[2] -= jxz * f0 + jyz * f1 + jzz * f2;
  }
  return 0.5 * cost;
}

// Solve (A) y = g for a symmetric positive definite 3x3 given by its upper triangle, by Cholesky
__device__ __forceinline__ void tri_solve(const double* A, const double* g, double* y) {
  const double l00 = sqrt(A[0]);
  const double l10 = A[1] / l00, l20 = A[2] / l00;
  const double l11 = sqrt(A[3] - l10 * l10);
  const double l21 = (A[4] - l20 * l10) / l11;
  const double l22 = sqrt(A[5] - l20 * l20 - l21 * l21);
  const double z0 = g[0] / l00;
  const double z1 = (g[1] - l10 * z0) / l11;
  const double z2 = (g[2] - l20 * z0 - l21 * z1) / l22;
  y[2] = z2 / l22;
  y[1] = (z1 - l21 * y[2]) / l11;
  y[0] = (z0 - l10 * y[1] - l20 * y[2]) / l00;
}

// The Jacobi-scaled normal equations of TinySolver's Update from the unscaled sums A = J^T J, je = J^T (-f):
// jtj = S A S, g = S je, S = diag(s)
__device__ __forceinline__ void tri_scale(const double* A, const double* je, const double* s, double* jtj, double* g, double* gmax) {
  jtj[0] = s[0] * A[0] * s[0];
  jtj[1] = s[0] * A[1] * s[1];
  jtj[2] = s[0] * A[2] * s[2];
  jtj[3] = s[1] * A[3] * s[1];
  jtj[4] = s[1] * A[4] * s[2];
  jtj[5] = s[2] * A[5] * s[2];
  *gmax = 0.0;
  for (int k = 0; k < 3; ++k) {
    g[k] = s[k] * je[k];
    *gmax = fmax(*gmax, fabs(g[k]));
  }
}

// PointRefinement: TinySolver from x for at most `iterations` iterations (oracle/triangulation_oracle.py)
__device__ __forceinline__ void tri_refine(const TriArgs& a, int b, int e, double* x) {
  double A[6], je[3], s[3], jtj[6], g[3], gmax;
  double cost = tri_cost(a, b, e, x, true, A, je);
  // the Jacobi scaling 1 / (1 + column norms of J) is fixed at the first evaluation
  s[0] = 1.0 / (1.0 + sqrt(A[0]));
  s[1] = 1.0 / (1.0 + sqrt(A[3]));
  s[2] = 1.0 / (1.0 + sqrt(A[5]));
  tri_scale(A, je, s, jtj, g, &gmax);
  if (gmax < TRI_GRADIENT_TOLERANCE) return;
  double u = 1.0 / TRI_INITIAL_TRUST_REGION, v = 2.0;
  for (int it = 1; it < a.iterations; ++it) {
    double reg[6] = {jtj[0], jtj[1], jtj[2], jtj[3], jtj[4], jtj[5]};
    reg[0] += u * fmin(fmax(jtj[0], TRI_MIN_DIAGONAL), TRI_MAX_DIAGONAL);
    reg[3] += u * fmin(fmax(jtj[3], TRI_MIN_DIAGONAL), TRI_MAX_DIAGONAL);
    reg[5] += u * fmin(fmax(jtj[5], TRI_MIN_DIAGONAL), TRI_MAX_DIAGONAL);
    double step[3];
    tri_solve(reg, g, step);
    const double dx[3] = {s[0] * step[0], s[1] * step[1], s[2] * step[2]};
    const double xn = sqrt(tri_dot(x, x));
    if (sqrt(tri_dot(dx, dx)) < TRI_PARAMETER_TOLERANCE * (xn + TRI_PARAMETER_TOLERANCE)) break;
    const double xnew[3] = {x[0] + dx[0], x[1] + dx[1], x[2] + dx[2]};
    const double cost_change = 2.0 * cost - 2.0 * tri_cost(a, b, e, xnew, false, nullptr, nullptr);
    // step . (2 g - jtj step)
    const double h0 = jtj[0] * step[0] + jtj[1] * step[1] + jtj[2] * step[2];
    const double h1 = jtj[1] * step[0] + jtj[3] * step[1] + jtj[4] * step[2];
    const double h2 = jtj[2] * step[0] + jtj[4] * step[1] + jtj[5] * step[2];
    const double model_change =
        step[0] * (2.0 * g[0] - h0) + step[1] * (2.0 * g[1] - h1) + step[2] * (2.0 * g[2] - h2);
    const double rho = cost_change / model_change;
    if (rho > 0.0) {
      for (int k = 0; k < 3; ++k) x[k] = xnew[k];
      cost = tri_cost(a, b, e, x, true, A, je);
      tri_scale(A, je, s, jtj, g, &gmax);
      if (gmax < TRI_GRADIENT_TOLERANCE || cost < TRI_COST_THRESHOLD) break;
      const double t = 2.0 * rho - 1.0;
      u *= fmax(1.0 / 3.0, 1.0 - t * t * t);
      v = 2.0;
    } else {
      u *= v;
      v *= 2.0;
    }
  }
}

// TrackTriangulator.triangulate of the observations [b, e); x receives the point when the result is TRI_OK
__device__ __forceinline__ int8_t tri_track(const TriArgs& a, int b, int e, double* x) {
  int n = 0, im;
  for (int r = b; r < e; ++r) n += tri_kept(a, r, &im) ? 1 : 0;
  if (n < 2) return TRI_TOO_FEW;

  bool angle_ok = false;
  for (int i = b; i < e && !angle_ok; ++i) {
    int ii;
    if (!tri_kept(a, i, &ii)) continue;
    double wi[3], ci[3];
    tri_ray(a, i, ii, wi, ci);
    for (int j = b; j < i && !angle_ok; ++j) {
      int jj;
      if (!tri_kept(a, j, &jj)) continue;
      double wj[3], cj[3];
      tri_ray(a, j, jj, wj, cj);
      const double angle = tri_angle(wi, wj);
      angle_ok = angle >= a.min_angle && angle <= TRI_PI - a.min_angle;
    }
  }
  if (!angle_ok) return TRI_BAD_ANGLE;

  // X = (I + BBt Cinv) A / n - Cinv BBtA, Cinv = (n I - BBt)^-1
  double S[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, SA[3] = {0, 0, 0}, A[3] = {0, 0, 0};
  for (int r = b; r < e; ++r) {
    if (!tri_kept(a, r, &im)) continue;
    double w[3], c[3];
    tri_ray(a, r, im, w, c);
    for (int k = 0; k < 3; ++k) {
      for (int l = 0; l < 3; ++l) S[3 * k + l] += w[k] * w[l];
      SA[k] += (w[k] * w[0]) * c[0] + (w[k] * w[1]) * c[1] + (w[k] * w[2]) * c[2];
      A[k] += c[k];
    }
  }
  const double dn = (double)n;
  double C[9], Ci[9];
  for (int k = 0; k < 9; ++k) C[k] = (k % 4 == 0 ? dn : 0.0) - S[k];
  const double c00 = tri_cof(C, 0, 0), c10 = tri_cof(C, 1, 0), c20 = tri_cof(C, 2, 0);
  const double invdet = 1.0 / (c00 * C[0] + c10 * C[3] + c20 * C[6]);
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) Ci[3 * r + c] = tri_cof(C, c, r) * invdet;
  for (int k = 0; k < 3; ++k) {
    double mA = A[k];   // row k of (I + S Ci) times A
    for (int l = 0; l < 3; ++l) {
      const double m = S[3 * k] * Ci[l] + S[3 * k + 1] * Ci[3 + l] + S[3 * k + 2] * Ci[6 + l];
      mA += m * A[l];
    }
    x[k] = mA / dn - (Ci[3 * k] * SA[0] + Ci[3 * k + 1] * SA[1] + Ci[3 * k + 2] * SA[2]);
  }

  for (int r = b; r < e; ++r) {
    if (!tri_kept(a, r, &im)) continue;
    double w[3], c[3];
    tri_ray(a, r, im, w, c);
    const double p[3] = {x[0] - c[0], x[1] - c[1], x[2] - c[2]};
    if (tri_angle(p, w) > a.threshold || tri_dot(p, w) < a.min_depth) return TRI_BAD_REPROJECTION;
  }
  tri_refine(a, b, e, x);
  return TRI_OK;
}

__global__ void __launch_bounds__(TRI_THREADS) tri_tracks(TriArgs a) {
  const int t = blockIdx.x * TRI_THREADS + threadIdx.x;
  if (t >= a.T) return;
  double x[3] = {CUDART_NAN, CUDART_NAN, CUDART_NAN};
  int8_t st = TRI_NOT_SELECTED;
  if (__ldg(a.selected + t)) {
    st = tri_track(a, (int)__ldg(a.track_start + t), (int)__ldg(a.track_start + t + 1), x);
    if (st != TRI_OK) x[0] = x[1] = x[2] = CUDART_NAN;
  }
  a.status[t] = st;
  for (int k = 0; k < 3; ++k) a.X[3LL * t + k] = x[k];
}

}  // namespace

void triangulate_tracks(TriWorkspace& w, cudaStream_t stream, cudaEvent_t ev_start, cudaEvent_t ev_end,
                        const TriTopology& topo, const double* image_rt, const double* image_origin,
                        const uint8_t* image_in, const double* bearings, const uint8_t* selected, double threshold,
                        double min_ray_angle, double min_depth, int iterations, int8_t* status, double* X) {
  w.timed = false;
  if (iterations < 1) throw ArgError("triangulate: iterations must be at least 1");
  if (!std::isfinite(threshold) || !std::isfinite(min_ray_angle) || !std::isfinite(min_depth))
    throw ArgError("triangulate: threshold, min_ray_angle and min_depth must be finite");
  if (topo.T > 0 && (!selected || !status || !X)) throw ArgError("triangulate: null per-track arrays");
  if (topo.I > 0 && (!image_rt || !image_origin || !image_in)) throw ArgError("triangulate: null per-image arrays");
  if (topo.nobs > 0 && !bearings) throw ArgError("triangulate: null bearings");
  upload(w.image_rt, image_rt, (size_t)topo.I * 9, stream);
  upload(w.image_origin, image_origin, (size_t)topo.I * 3, stream);
  upload(w.image_in, image_in, (size_t)topo.I, stream);
  upload(w.bearings, bearings, (size_t)topo.nobs * 3, stream);
  upload(w.selected, selected, (size_t)topo.T, stream);
  w.status.reserve(std::max(topo.T, 1));
  w.X.reserve(std::max<size_t>((size_t)topo.T * 3, 1));

  TriArgs a;
  a.T = topo.T;
  a.obs_image = topo.obs_image;
  a.track_start = topo.track_start;
  a.rt = w.image_rt.p;
  a.origin = w.image_origin.p;
  a.in = w.image_in.p;
  a.bearings = w.bearings.p;
  a.selected = w.selected.p;
  a.threshold = threshold;
  a.min_angle = min_ray_angle;
  a.min_depth = min_depth;
  a.iterations = iterations;
  a.status = w.status.p;
  a.X = w.X.p;
  OSFM_CUDA(cudaEventRecord(ev_start, stream));
  if (topo.T > 0) {
    tri_tracks<<<(unsigned)((topo.T + TRI_THREADS - 1) / TRI_THREADS), TRI_THREADS, 0, stream>>>(a);
    OSFM_LAUNCH_CHECK();
  }
  OSFM_CUDA(cudaEventRecord(ev_end, stream));
  download(status, w.status.p, (size_t)topo.T, stream);
  download(X, w.X.p, (size_t)topo.T * 3, stream);
  OSFM_CUDA(cudaStreamSynchronize(stream));
  w.timed = true;
}

}  // namespace osfm
