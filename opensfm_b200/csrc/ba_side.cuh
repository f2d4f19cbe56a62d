// Side terms of the bundle adjustment: the O(#shots) residual blocks that share the reduced camera
// system with the point projections (SURVEY.md §8a "secondary residuals").
//
// The reference builds them as ceres autodiff cost functions (opensfm/src/bundle/src/bundle_adjuster.cc:
// 745-778 position prior with bias + scale group, 817-856 relative motion, 858-900 relative rotation,
// 902-944 common position, 956-1022 up vector / pan / tilt / roll, 1024-1084 linear motion, 1086-1101
// gauge-fix translation prior, 610-625 DUAL transition barrier, 727-736 std-deviation regulariser;
// functors in bundle/error/absolute_motion_errors.h, relative_motion_errors.h, motion_prior_errors.h,
// parameters_errors.h, position_functors.h, data/bias.h).  Here every term is a small record; its
// residual function is written once over a scalar type T and differentiated on the device with
// single-direction dual numbers: thread j of a term's CTA evaluates the residual with the seed on
// parameter j, which yields column j of the Jacobian -- the same "exact derivative of the same
// formula" the reference gets from ceres::Jet, without a 36-wide gradient in registers.
// The rotation helpers restate ceres/rotation.h (AngleAxisToQuaternion, QuaternionProduct,
// QuaternionToAngleAxis, AngleAxisRotatePoint: Ceres Solver 2.1/2.2, pinned by conda.yml:10 /
// Dockerfile.ubuntu24:12), including their small-angle branches.
//
// Terms live on the camera side only (cameras, rig instances, rig cameras, "ext" blocks = biases,
// reconstruction scales, std-deviation scales); point priors are diagonal and handled in ba.cu.
// Included by ba.cu after ba_reduced.cuh.
#pragma once

namespace osfm {

// ---- single-direction dual number ---------------------------------------------------------
struct Dual1 {
  double v, d;
  OSFM_HD Dual1() : v(0.0), d(0.0) {}
  OSFM_HD Dual1(double x) : v(x), d(0.0) {}
  OSFM_HD Dual1(double x, double dx) : v(x), d(dx) {}
};
OSFM_HD Dual1 operator+(Dual1 a, Dual1 b) { return Dual1(a.v + b.v, a.d + b.d); }
OSFM_HD Dual1 operator-(Dual1 a, Dual1 b) { return Dual1(a.v - b.v, a.d - b.d); }
OSFM_HD Dual1 operator-(Dual1 a) { return Dual1(-a.v, -a.d); }
OSFM_HD Dual1 operator*(Dual1 a, Dual1 b) { return Dual1(a.v * b.v, a.d * b.v + a.v * b.d); }
OSFM_HD Dual1 operator/(Dual1 a, Dual1 b) {
  const double inv = 1.0 / b.v, q = a.v * inv;
  return Dual1(q, (a.d - q * b.d) * inv);
}
OSFM_HD bool operator<(Dual1 a, Dual1 b) { return a.v < b.v; }
OSFM_HD bool operator>(Dual1 a, Dual1 b) { return a.v > b.v; }
OSFM_HD bool operator<=(Dual1 a, Dual1 b) { return a.v <= b.v; }
OSFM_HD bool operator==(Dual1 a, Dual1 b) { return a.v == b.v; }

OSFM_HD double sd_val(double x) { return x; }
OSFM_HD double sd_val(Dual1 x) { return x.v; }
OSFM_HD double sd_sqrt(double x) { return sqrt(x); }
OSFM_HD Dual1 sd_sqrt(Dual1 x) { const double s = sqrt(x.v); return Dual1(s, x.d / (2.0 * s)); }
OSFM_HD double sd_sin(double x) { return sin(x); }
OSFM_HD Dual1 sd_sin(Dual1 x) { return Dual1(sin(x.v), cos(x.v) * x.d); }
OSFM_HD double sd_cos(double x) { return cos(x); }
OSFM_HD Dual1 sd_cos(Dual1 x) { return Dual1(cos(x.v), -sin(x.v) * x.d); }
OSFM_HD double sd_atan2(double y, double x) { return atan2(y, x); }
OSFM_HD Dual1 sd_atan2(Dual1 y, Dual1 x) {
  const double n = x.v * x.v + y.v * y.v;
  return Dual1(atan2(y.v, x.v), (x.v * y.d - y.v * x.d) / n);
}
OSFM_HD double sd_asin(double x) { return asin(x); }
OSFM_HD Dual1 sd_asin(Dual1 x) { return Dual1(asin(x.v), x.d / sqrt(1.0 - x.v * x.v)); }
OSFM_HD double sd_log(double x) { return log(x); }
OSFM_HD Dual1 sd_log(Dual1 x) { return Dual1(log(x.v), x.d / x.v); }
OSFM_HD double sd_abs(double x) { return fabs(x); }
OSFM_HD Dual1 sd_abs(Dual1 x) { return x.v < 0.0 ? -x : x; }   // ceres::abs(Jet): sign(a) * derivative

// ---- ceres/rotation.h restated ---------------------------------------------------------------
template <class T>
OSFM_HD void aa_to_quat(const T* a, T* q) {
  const T th2 = a[0] * a[0] + a[1] * a[1] + a[2] * a[2];
  if (sd_val(th2) > 0.0) {
    const T th = sd_sqrt(th2);
    const T half = th * T(0.5);
    const T k = sd_sin(half) / th;
    q[0] = sd_cos(half); q[1] = a[0] * k; q[2] = a[1] * k; q[3] = a[2] * k;
  } else {
    // first-order Taylor at zero: keeps the derivative of the seed direction (ceres does the same for Jets)
    const T k(0.5);
    q[0] = T(1.0); q[1] = a[0] * k; q[2] = a[1] * k; q[3] = a[2] * k;
  }
}
template <class T>
OSFM_HD void quat_product(const T* z, const T* w, T* zw) {
  zw[0] = z[0] * w[0] - z[1] * w[1] - z[2] * w[2] - z[3] * w[3];
  zw[1] = z[0] * w[1] + z[1] * w[0] + z[2] * w[3] - z[3] * w[2];
  zw[2] = z[0] * w[2] - z[1] * w[3] + z[2] * w[0] + z[3] * w[1];
  zw[3] = z[0] * w[3] + z[1] * w[2] - z[2] * w[1] + z[3] * w[0];
}
template <class T>
OSFM_HD void quat_to_aa(const T* q, T* a) {
  const T s2 = q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
  if (sd_val(s2) > 0.0) {
    const T s = sd_sqrt(s2);
    const T c = q[0];
    // atan2(-s, -c) when cos < 0 keeps the angle in (-pi, pi]
    const T two_theta = T(2.0) * (sd_val(c) < 0.0 ? sd_atan2(-s, -c) : sd_atan2(s, c));
    const T k = two_theta / s;
    a[0] = q[1] * k; a[1] = q[2] * k; a[2] = q[3] * k;
  } else {
    const T k(2.0);
    a[0] = q[1] * k; a[1] = q[2] * k; a[2] = q[3] * k;
  }
}
template <class T>
OSFM_HD void aa_rotate_point(const T* aa, const T* pt, T* out) {
  const T th2 = aa[0] * aa[0] + aa[1] * aa[1] + aa[2] * aa[2];
  if (sd_val(th2) > DBL_EPSILON) {
    const T th = sd_sqrt(th2);
    const T c = sd_cos(th), s = sd_sin(th);
    const T w[3] = {aa[0] / th, aa[1] / th, aa[2] / th};
    const T wx[3] = {w[1] * pt[2] - w[2] * pt[1], w[2] * pt[0] - w[0] * pt[2], w[0] * pt[1] - w[1] * pt[0]};
    const T tmp = (w[0] * pt[0] + w[1] * pt[1] + w[2] * pt[2]) * (T(1.0) - c);
    out[0] = pt[0] * c + wx[0] * s + w[0] * tmp;
    out[1] = pt[1] * c + wx[1] * s + w[1] * tmp;
    out[2] = pt[2] * c + wx[2] * s + w[2] * tmp;
  } else {
    const T wx[3] = {aa[1] * pt[2] - aa[2] * pt[1], aa[2] * pt[0] - aa[0] * pt[2], aa[0] * pt[1] - aa[1] * pt[0]};
    out[0] = pt[0] + wx[0]; out[1] = pt[1] + wx[1]; out[2] = pt[2] + wx[2];
  }
}
// error_utils.h:14-41
template <class T>
OSFM_HD void mult_rotations(const T* R1, const T* R2, T* out) {
  T q1[4], q2[4], q[4];
  aa_to_quat(R1, q1); aa_to_quat(R2, q2);
  quat_product(q1, q2, q);
  quat_to_aa(q, out);
}
template <class T>
OSFM_HD void mult_rotations3(const T* R1, const T* R2, const T* R3, T* out) {
  T q1[4], q2[4], q3[4], q12[4], q[4];
  aa_to_quat(R1, q1); aa_to_quat(R2, q2); aa_to_quat(R3, q3);
  quat_product(q1, q2, q12);
  quat_product(q12, q3, q);
  quat_to_aa(q, out);
}
// position_functors.h:14-66 (rig_camera == nullptr <=> FUNCTOR_NOT_SET)
template <class T>
OSFM_HD void shot_rotation(const T* inst, const T* rc, T* R) {
  if (rc) mult_rotations(inst, rc, R);
  else { R[0] = inst[0]; R[1] = inst[1]; R[2] = inst[2]; }
}
template <class T>
OSFM_HD void shot_position(const T* inst, const T* rc, T* t) {
  t[0] = inst[3]; t[1] = inst[4]; t[2] = inst[5];
  if (rc) {
    T c[3];
    aa_rotate_point(inst, rc + 3, c);
    t[0] = t[0] + c[0]; t[1] = t[1] + c[1]; t[2] = t[2] + c[2];
  }
}
// error_utils.h:87-97
template <class T>
OSFM_HD T diff_between_angles(const T& a, double b) {
  const T d = a - T(b);
  if (sd_val(d) > M_PI) return d - T(2.0 * M_PI);
  if (sd_val(d) < -M_PI) return d + T(2.0 * M_PI);
  return d;
}

// reconstruction_alignment.h:224-234: point of the world frame -> frame of a reconstruction [R | t | scale]
template <class T>
OSFM_HD void ra_transform_point(const T* rec, const double* point, T* out) {
  const T p[3] = {(T(point[0]) - rec[3]) / rec[6], (T(point[1]) - rec[4]) / rec[6], (T(point[2]) - rec[5]) / rec[6]};
  const T Rt[3] = {-rec[0], -rec[1], -rec[2]};
  aa_rotate_point(Rt, p, out);
}
// optical centre -R^t t of a constant shot [R | t] (world-to-camera parametrisation of RAShot)
OSFM_HD void ra_shot_centre(const double* shot, double* c) {
  const double Rt[3] = {-shot[0], -shot[1], -shot[2]};
  double v[3];
  aa_rotate_point<double>(Rt, shot + 3, v);
  c[0] = -v[0]; c[1] = -v[1]; c[2] = -v[2];
}

// ---- term records ----------------------------------------------------------------------------
constexpr int SIDE_MAX_BLOCKS = 6;
constexpr int SIDE_MAX_RES = 7;
constexpr int SIDE_MAX_PARAMS = 40;   // linear motion: 3 instances + 3 rig cameras = 36
constexpr int SIDE_THREADS = 64;

// block kinds
enum { SB_CAM = 0, SB_INST = 1, SB_RIGCAM = 2, SB_EXT = 3 };

// One term = the C ABI's record (include/opensfm_b200.h): type, nres, nblocks, kind[6], idx[6], loss (-1 = no
// loss function, i.e. nullptr in the reference), loss_a, cofs (first constant), aux[4] (type-specific integers).
using SideTerm = osfm_side_term;

struct SideView {
  int n;
  const SideTerm* terms;
  const double* consts;
  const int* jofs;      // [n + 1] offsets into J (nres * nparams doubles per term)
  const int* rofs;      // [n + 1] offsets into r
  double* J;
  double* r;
  // ext blocks
  const int *ext_off, *ext_np, *ext_poff;
  const int* ext_blk;
};

struct SideBlock {
  const double* p;   // parameters
  int np;            // count
  int col;           // first reduced column or -1 (constant)
  int blk;           // parameter-block id or -1
};
__device__ __forceinline__ SideBlock side_block(const BAView& v, const BlkMaps& bm, const SideView& sv, const Params& p,
                                                int kind, int idx) {
  SideBlock b;
  if (kind == SB_CAM) { b.p = p.cam + v.cam_off[idx]; b.np = v.cam_np[idx]; b.col = v.cam_poff[idx]; b.blk = bm.cam_blk[idx]; }
  else if (kind == SB_INST) { b.p = p.inst + 6 * (size_t)idx; b.np = 6; b.col = v.inst_poff[idx]; b.blk = bm.inst_blk[idx]; }
  else if (kind == SB_RIGCAM) { b.p = p.rc + 6 * (size_t)idx; b.np = 6; b.col = v.rc_poff[idx]; b.blk = bm.rc_blk[idx]; }
  else { b.p = p.ext + sv.ext_off[idx]; b.np = sv.ext_np[idx]; b.col = sv.ext_poff[idx]; b.blk = sv.ext_blk[idx]; }
  return b;
}

// Tukey's biweight (ceres::TukeyLoss, used by the common-position term, bundle_adjuster.cc:905): rho'' <= 0.
OSFM_HD double side_loss(int loss, double a, double s, double* w) {
  if (loss < 0) { *w = 1.0; return s; }
  if (loss == OSFM_LOSS_TUKEY) {
    const double a2 = a * a;
    if (s <= a2) {
      const double v = 1.0 - s / a2, v2 = v * v;
      *w = sqrt(fmax(DBL_MIN, v2));   // rho' = (1 - s/a^2)^2
      return a2 / 3.0 * (1.0 - v2 * v);
    }
    *w = 0.0;
    return a2 / 3.0;
  }
  return robust_loss(loss, a, s, w);
}

// ---- the residual functions ------------------------------------------------------------------
// x[b] = parameters of block b as T; c = constants of the term.  Returns false when the residual cannot be
// evaluated (relative motion with a zero scale: the reference's functor returns false).
template <class T>
__device__ bool side_eval(const SideTerm& t, const double* __restrict__ c, T* const* x, T* r) {
  switch (t.type) {
    case OSFM_SIDE_UP_VECTOR: {          // absolute_motion_errors.h:12-39; c = acceleration (unit), scale
      T R[3], z[3];
      shot_rotation<T>(x[0], x[1], R);
      const T acc[3] = {T(c[0]), T(c[1]), T(c[2])};
      aa_rotate_point(R, acc, z);
      r[0] = T(c[3]) * z[0]; r[1] = T(c[3]) * z[1]; r[2] = T(c[3]) * (z[2] - T(1.0));
      return true;
    }
    case OSFM_SIDE_PAN: {                // :41-65; c = angle, scale
      T R[3], z[3];
      shot_rotation<T>(x[0], x[1], R);
      const T ez[3] = {T(0.0), T(0.0), T(1.0)};
      aa_rotate_point(R, ez, z);
      if (fabs(sd_val(z[0])) < 1e-8 && fabs(sd_val(z[1])) < 1e-8) r[0] = T(0.0);
      else r[0] = T(c[1]) * diff_between_angles(sd_atan2(z[0], z[1]), c[0]);
      return true;
    }
    case OSFM_SIDE_TILT: {               // :67-90
      T R[3], z[3];
      shot_rotation<T>(x[0], x[1], R);
      const T ez[3] = {T(0.0), T(0.0), T(1.0)};
      aa_rotate_point(R, ez, z);
      const T l = sd_sqrt(z[0] * z[0] + z[1] * z[1]);
      r[0] = T(c[1]) * diff_between_angles(-sd_atan2(z[2], l), c[0]);
      return true;
    }
    case OSFM_SIDE_ROLL: {               // :92-136
      T R[3], ex_[3], ez_[3];
      shot_rotation<T>(x[0], x[1], R);
      const T ex[3] = {T(1.0), T(0.0), T(0.0)}, ez[3] = {T(0.0), T(0.0), T(1.0)};
      aa_rotate_point(R, ex, ex_);
      aa_rotate_point(R, ez, ez_);
      T a[3] = {ez_[1], -ez_[0], T(0.0)};
      const T la = sd_sqrt(a[0] * a[0] + a[1] * a[1]);
      const double eps = 1e-5;
      if (sd_val(la) < eps) { r[0] = T(0.0); return true; }
      a[0] = a[0] / la; a[1] = a[1] / la;
      const T b[3] = {ex_[1] * a[2] - ex_[2] * a[1], ex_[2] * a[0] - ex_[0] * a[2], ex_[0] * a[1] - ex_[1] * a[0]};
      const T sin_roll = ez_[0] * b[0] + ez_[1] * b[1] + ez_[2] * b[2];
      if (sd_val(sin_roll) <= -(1.0 - eps)) { r[0] = T(0.0); return true; }
      r[0] = T(c[1]) * diff_between_angles(sd_asin(sin_roll), c[0]);
      return true;
    }
    case OSFM_SIDE_RELATIVE_MOTION: {    // relative_motion_errors.h:14-72; c = Rts[7], scale_matrix[49], observed_scale
      const T* Ri = x[0]; const T* Rj = x[1];
      const T* si = x[2]; const T* sj = x[t.aux[0]];
      const T Rij[3] = {T(c[0]), T(c[1]), T(c[2])};
      const T nRi[3] = {-Ri[0], -Ri[1], -Ri[2]}, nRj[3] = {-Rj[0], -Rj[1], -Rj[2]};
      T e[7];
      mult_rotations3(Rij, nRi, Rj, e);
      const T dt[3] = {Ri[3] - Rj[3], Ri[4] - Rj[4], Ri[5] - Rj[5]};
      T rot[3];
      aa_rotate_point(nRj, dt, rot);
      for (int k = 0; k < 3; ++k) e[3 + k] = T(c[3 + k]) - sj[0] * rot[k];
      if (sd_val(si[0]) == 0.0 || sd_val(sj[0]) == 0.0) return false;
      e[6] = c[56] != 0.0 ? T(c[6]) - sj[0] / si[0] : T(0.0);
      for (int a = 0; a < 7; ++a) {
        T s(0.0);
        for (int b = 0; b < 7; ++b) s = s + T(c[7 + 7 * a + b]) * e[b];
        r[a] = s;
      }
      return true;
    }
    case OSFM_SIDE_RELATIVE_ROTATION: {  // :74-103; c = Rij[3], scale_matrix[9]; aux = rig camera block of i, of j (-1 unset)
      T Ri[3], Rj[3], e[3];
      shot_rotation<T>(x[0], t.aux[0] >= 0 ? x[t.aux[0]] : nullptr, Ri);
      shot_rotation<T>(x[1], t.aux[1] >= 0 ? x[t.aux[1]] : nullptr, Rj);
      const T Rij[3] = {T(c[0]), T(c[1]), T(c[2])};
      const T nRi[3] = {-Ri[0], -Ri[1], -Ri[2]};
      mult_rotations3(Rij, nRi, Rj, e);
      for (int a = 0; a < 3; ++a) r[a] = T(c[3 + 3 * a]) * e[0] + T(c[4 + 3 * a]) * e[1] + T(c[5 + 3 * a]) * e[2];
      return true;
    }
    case OSFM_SIDE_COMMON_POSITION: {    // :105-138; c = margin, scale
      T t1[3], t2[3];
      shot_position<T>(x[0], t.aux[0] >= 0 ? x[t.aux[0]] : nullptr, t1);
      shot_position<T>(x[1], t.aux[1] >= 0 ? x[t.aux[1]] : nullptr, t2);
      T e[3] = {t1[0] - t2[0], t1[1] - t2[1], t1[2] - t2[2]};
      for (int i = 0; i < 2; ++i) {
        const T m = sd_abs(e[i]) - T(c[0]);
        e[i] = sd_val(m) > 0.0 ? m : T(0.0);   // std::max(T(0), .) on Jets keeps the larger operand
      }
      for (int i = 0; i < 3; ++i) r[i] = T(c[1]) * e[i];
      return true;
    }
    case OSFM_SIDE_LINEAR_MOTION: {      // motion_prior_errors.h:13-76; c = alpha, position scale, orientation scale
      T R0[3], R1[3], R2[3], t0[3], t1[3], t2[3];
      const T* rc0 = t.aux[0] >= 0 ? x[t.aux[0]] : nullptr;
      const T* rc1 = t.aux[1] >= 0 ? x[t.aux[1]] : nullptr;
      const T* rc2 = t.aux[2] >= 0 ? x[t.aux[2]] : nullptr;
      shot_rotation<T>(x[0], rc0, R0); shot_position<T>(x[0], rc0, t0);
      shot_rotation<T>(x[1], rc1, R1); shot_position<T>(x[1], rc1, t1);
      shot_rotation<T>(x[2], rc2, R2); shot_position<T>(x[2], rc2, t2);
      const T a20[3] = {t2[0] - t0[0], t2[1] - t0[1], t2[2] - t0[2]};
      const T a10[3] = {t1[0] - t0[0], t1[1] - t0[1], t1[2] - t0[2]};
      const T n20 = sd_sqrt(a20[0] * a20[0] + a20[1] * a20[1] + a20[2] * a20[2]);
      const T n10 = sd_sqrt(a10[0] * a10[0] + a10[1] * a10[1] + a10[2] * a10[2]);
      for (int i = 0; i < 3; ++i) {
        if (sd_val(n20) > 1e-15) r[i] = T(c[1]) * (T(c[0]) - n10 / n20);
        else r[i] = T(c[1]) * (T(c[0]) * a20[i] - a10[i]);
      }
      const T nR0[3] = {-R0[0], -R0[1], -R0[2]}, nR1[3] = {-R1[0], -R1[1], -R1[2]};
      T A[3], B[3], e[3];
      mult_rotations(R2, nR0, A);
      for (int i = 0; i < 3; ++i) A[i] = T(c[0]) * A[i];
      mult_rotations(R0, nR1, B);
      mult_rotations(A, B, e);
      for (int i = 0; i < 3; ++i) r[3 + i] = T(c[2]) * e[i];
      return true;
    }
    case OSFM_SIDE_TRANSLATION_PRIOR: {  // absolute_motion_errors.h:180-202; c = prior norm (already max(norm, 1e-20))
      const T d[3] = {x[0][3] - x[1][3], x[0][4] - x[1][4], x[0][5] - x[1][5]};
      const T safe = sd_sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2] + T(1e-20));
      r[0] = sd_log(safe / T(c[0]));
      return true;
    }
    case OSFM_SIDE_PARAMETER_BARRIER: {  // parameters_errors.h:20-36; c = lower, upper; aux[0] = parameter index
      const T eps(1e-10);
      const T value = x[0][t.aux[0]];
      const T zero = T(2.0 * log((c[1] - c[0]) * 0.5));
      r[0] = sd_log(value - T(c[0]) + eps) + sd_log(T(c[1]) - value + eps) + zero;
      return true;
    }
    case OSFM_SIDE_STD_DEVIATION: {      // parameters_errors.h:7-18
      const T s2 = x[0][0] * x[0][0] + T(1e-20);
      r[0] = sd_log(T(1.0) / sd_sqrt(T(2.0 * M_PI) * s2));
      return true;
    }
    case OSFM_SIDE_POSITION_PRIOR: {     // prior_error.h:55-96 with SimilarityPriorTransform (data/bias.h:33-53)
      // blocks: rig instance, bias similarity [R | t | s], std-deviation scale; c = prior[3], 1/sigma[3], adjust flag
      const T* inst = x[0]; const T* bias = x[1]; const T* sd = x[2];
      const T prior[3] = {T(c[0]), T(c[1]), T(c[2])};
      T rp[3];
      aa_rotate_point(bias, prior, rp);
      for (int k = 0; k < 3; ++k) {
        const T pk = bias[6] * rp[k] + bias[3 + k];
        T sc(c[3 + k]);
        if (c[6] != 0.0) sc = sc / sd[0];
        r[k] = sc * (inst[3 + k] - pk);
      }
      return true;
    }
    // ---- ReconstructionAlignment (opensfm/src/bundle/reconstruction_alignment.h): shots [R | t] world-to-camera,
    //      reconstructions [R | t | scale] ----
    case OSFM_SIDE_RA_RELATIVE_MOTION: {          // :140-197; blocks [reconstruction a, shot i]; c = Rtai[6], scale_matrix[36]
      const T* rec = x[0]; const T* shot = x[1];
      const T Rit[3] = {-shot[0], -shot[1], -shot[2]};
      const T Rai[3] = {T(c[0]), T(c[1]), T(c[2])};
      const T tai[3] = {T(c[3]), T(c[4]), T(c[5])};
      const T Rait[3] = {-Rai[0], -Rai[1], -Rai[2]};
      T qRai[4], qRa[4], qRit[4], q1[4], q2[4], e[6];
      aa_to_quat(Rai, qRai); aa_to_quat(rec, qRa); aa_to_quat(Rit, qRit);
      quat_product(qRa, qRit, q1);
      quat_product(qRai, q1, q2);
      quat_to_aa(q2, e);
      T a[3], b[3], d[3];
      aa_rotate_point(Rait, tai, a);
      aa_rotate_point(Rit, shot + 3, b);
      aa_rotate_point(rec, b, d);
      for (int k = 0; k < 3; ++k) e[3 + k] = a[k] - rec[6] * d[k] + rec[3 + k];
      for (int i = 0; i < 6; ++i) {
        T s(0.0);
        for (int j = 0; j < 6; ++j) s = s + T(c[6 + 6 * i + j]) * e[j];
        r[i] = s;
      }
      return true;
    }
    case OSFM_SIDE_RA_ABSOLUTE_POSITION: {        // :199-222; block [shot]; c = prior[3], 1/std
      const T* shot = x[0];
      const T Rit[3] = {-shot[0], -shot[1], -shot[2]};
      T v[3];
      aa_rotate_point(Rit, shot + 3, v);
      for (int k = 0; k < 3; ++k) r[k] = T(c[3]) * (T(c[k]) + v[k]);
      return true;
    }
    case OSFM_SIDE_RA_RELATIVE_ABSOLUTE_POSITION: {   // :236-265; block [reconstruction]; c = prior[3], shot[6], 1/std
      double centre[3];
      ra_shot_centre(c + 3, centre);
      T tr[3];
      ra_transform_point(x[0], centre, tr);
      for (int k = 0; k < 3; ++k) r[k] = T(c[9]) * (T(c[k]) - tr[k]);
      return true;
    }
    case OSFM_SIDE_RA_COMMON_POINT: {             // :267-296; blocks [reconstruction a, b]; c = pa[3], pb[3], 1/std
      T ta[3], tb[3];
      ra_transform_point(x[0], c, ta);
      ra_transform_point(x[1], c + 3, tb);
      const T sf = x[0][6] + x[1][6];
      for (int k = 0; k < 3; ++k) r[k] = T(c[6]) * sf * (ta[k] - tb[k]);
      return true;
    }
    case OSFM_SIDE_RA_COMMON_CAMERA: {            // :298-365; blocks [reconstruction a, b]; c = shot_a[6], shot_b[6], 1/std_centre, 1/std_rotation
      double pa[3], pb[3];
      ra_shot_centre(c, pa);
      ra_shot_centre(c + 6, pb);
      T wa[3], wb[3];
      ra_transform_point(x[0], pa, wa);
      ra_transform_point(x[1], pb, wb);
      const T Rbt[3] = {-x[1][0], -x[1][1], -x[1][2]};
      const T Rbit[3] = {T(-c[6]), T(-c[7]), T(-c[8])};
      const T Rai[3] = {T(c[0]), T(c[1]), T(c[2])};
      T qRai[4], qRa[4], qRbt[4], qRbit[4], q1[4], q2[4], q3[4], e[3];
      aa_to_quat(Rai, qRai); aa_to_quat(x[0], qRa); aa_to_quat(Rbt, qRbt); aa_to_quat(Rbit, qRbit);
      quat_product(qRai, qRa, q1);
      quat_product(q1, qRbt, q2);
      quat_product(q2, qRbit, q3);
      quat_to_aa(q3, e);
      for (int k = 0; k < 3; ++k) { r[k] = e[k] * T(c[13]); r[3 + k] = T(c[12]) * (wa[k] - wb[k]); }
      return true;
    }
  }
  return false;
}

// parameter blocks of a term -> local column ranges
struct SideCols {
  SideBlock b[SIDE_MAX_BLOCKS];
  int start[SIDE_MAX_BLOCKS + 1];
};
__device__ __forceinline__ SideCols side_cols(const BAView& v, const BlkMaps& bm, const SideView& sv, const Params& p,
                                              const SideTerm& t) {
  SideCols sc;
  sc.start[0] = 0;
  for (int k = 0; k < t.nblocks; ++k) {
    sc.b[k] = side_block(v, bm, sv, p, t.kind[k], t.idx[k]);
    sc.start[k + 1] = sc.start[k] + sc.b[k].np;
  }
  return sc;
}
__device__ __forceinline__ int side_block_of(const SideCols& sc, int nblocks, int j) {
  int k = 0;
  while (k + 1 < nblocks && j >= sc.start[k + 1]) ++k;
  return k;
}

// A block a term lists twice (two shots of one rig instance) is one set of columns of J: the sum of its local copies.
// Only the first copy stands for it in the column norms, the gradient and S, so that a column whose copies cancel is 0.
__device__ __forceinline__ bool side_first_copy(const SideCols& sc, int kb) {
  for (int k = 0; k < kb; ++k)
    if (sc.b[k].col == sc.b[kb].col) return false;
  return true;
}
// entry j (in the first copy of block kb) of one row of J, summed over the copies of that block
__device__ __forceinline__ double side_column(const SideCols& sc, int nblocks, const double* row, int kb, int j) {
  double a = row[j];
  for (int k = kb + 1; k < nblocks; ++k)
    if (sc.b[k].col == sc.b[kb].col) a += row[sc.start[k] + (j - sc.start[kb])];
  return a;
}

// One CTA per term.  Thread j < nparams: column j of the Jacobian (dual seed on parameter j); thread 0 also
// writes the robustified residual and adds the cost.  with_cost = 0 on ranks that do not own the side terms.
__global__ void __launch_bounds__(SIDE_THREADS)
    side_linearize(SideView sv, BAView v, BlkMaps bm, Params p, Scalars* sc_out, int with_cost) {
  const SideTerm t = sv.terms[blockIdx.x];
  const SideCols sc = side_cols(v, bm, sv, p, t);
  const int NP = sc.start[t.nblocks];
  const int j = threadIdx.x;
  if (j >= NP) return;
  Dual1 xs[SIDE_MAX_PARAMS];
  Dual1* xp[SIDE_MAX_BLOCKS];
  for (int k = 0; k < t.nblocks; ++k) {
    xp[k] = xs + sc.start[k];
    for (int q = 0; q < sc.b[k].np; ++q) xs[sc.start[k] + q] = Dual1(sc.b[k].p[q]);
  }
  xs[j].d = 1.0;
  Dual1 r[SIDE_MAX_RES];
  const bool ok = side_eval<Dual1>(t, sv.consts + t.cofs, xp, r);
  double s = 0.0;
  for (int q = 0; q < t.nres; ++q) s += r[q].v * r[q].v;
  double w = 1.0;
  double rho = side_loss(t.loss, t.loss_a, s, &w);
  if (!ok) { w = 0.0; rho = __longlong_as_double(0x7ff8000000000000LL); }   // NaN cost: the step is rejected
  double* J = sv.J + sv.jofs[blockIdx.x];
  const int kb = side_block_of(sc, t.nblocks, j);
  const bool live = sc.b[kb].col >= 0;
  for (int q = 0; q < t.nres; ++q) J[q * NP + j] = live ? w * r[q].d : 0.0;
  if (j == 0) {
    double* ro = sv.r + sv.rofs[blockIdx.x];
    for (int q = 0; q < t.nres; ++q) ro[q] = w * r[q].v;
    bool any_free = false;   // all blocks constant: ceres drops the residual block from the minimised cost
    for (int k = 0; k < t.nblocks; ++k) any_free |= sc.b[k].col >= 0;
    if (with_cost && any_free) atomicAdd(&sc_out->cost, 0.5 * rho);
  }
}

// cost only (candidate evaluation): one thread per term
__global__ void side_cost(SideView sv, BAView v, BlkMaps bm, Params p, Scalars* sc_out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double cst = 0.0;
  if (i < sv.n) {
    const SideTerm t = sv.terms[i];
    const SideCols sc = side_cols(v, bm, sv, p, t);
    double xs[SIDE_MAX_PARAMS];
    double* xp[SIDE_MAX_BLOCKS];
    for (int k = 0; k < t.nblocks; ++k) {
      xp[k] = xs + sc.start[k];
      for (int q = 0; q < sc.b[k].np; ++q) xs[sc.start[k] + q] = sc.b[k].p[q];
    }
    double r[SIDE_MAX_RES];
    const bool ok = side_eval<double>(t, sv.consts + t.cofs, xp, r);
    double s = 0.0;
    for (int q = 0; q < t.nres; ++q) s += r[q] * r[q];
    double w;
    cst = 0.5 * side_loss(t.loss, t.loss_a, s, &w);
    if (!ok) cst = __longlong_as_double(0x7ff8000000000000LL);
    bool any_free = false;
    for (int k = 0; k < t.nblocks; ++k) any_free |= sc.b[k].col >= 0;
    if (!any_free) cst = 0.0;
  }
  const double tot = block_reduce_sum(cst);
  if (threadIdx.x == 0 && tot != 0.0) atomicAdd(&sc_out->cost, tot);
}

__global__ void __launch_bounds__(SIDE_THREADS)
    side_colnorm_grad(SideView sv, BAView v, BlkMaps bm, Params p, double* colnorm2, double* grad) {
  const SideTerm t = sv.terms[blockIdx.x];
  const SideCols sc = side_cols(v, bm, sv, p, t);
  const int NP = sc.start[t.nblocks];
  const int j = threadIdx.x;
  if (j >= NP) return;
  const int kb = side_block_of(sc, t.nblocks, j);
  if (sc.b[kb].col < 0 || !side_first_copy(sc, kb)) return;
  const int col = sc.b[kb].col + (j - sc.start[kb]);
  const double* J = sv.J + sv.jofs[blockIdx.x];
  const double* r = sv.r + sv.rofs[blockIdx.x];
  double n2 = 0.0, g = 0.0;
  for (int q = 0; q < t.nres; ++q) {
    const double a = side_column(sc, t.nblocks, J + q * NP, kb, j);
    n2 += a * a;
    g += a * r[q];
  }
  atomicAdd(&colnorm2[col], n2);
  atomicAdd(&grad[col], g);
}

// J^T J and J^T r of the terms into the block-sparse reduced system (upper blocks / upper triangles)
__global__ void __launch_bounds__(SIDE_THREADS)
    side_system(SideView sv, BAView v, BlkMaps bm, Params p, BsrView h, const double* __restrict__ scale,
                double* Sval, double* rhs) {
  const SideTerm t = sv.terms[blockIdx.x];
  const SideCols sc = side_cols(v, bm, sv, p, t);
  const int NP = sc.start[t.nblocks];
  const double* J = sv.J + sv.jofs[blockIdx.x];
  const double* r = sv.r + sv.rofs[blockIdx.x];
  for (int e = threadIdx.x; e < NP * NP; e += SIDE_THREADS) {
    const int j1 = e / NP, j2 = e - j1 * NP;
    const int k1 = side_block_of(sc, t.nblocks, j1), k2 = side_block_of(sc, t.nblocks, j2);
    const SideBlock& b1 = sc.b[k1];
    const SideBlock& b2 = sc.b[k2];
    if (b1.col < 0 || b2.col < 0 || !side_first_copy(sc, k1) || !side_first_copy(sc, k2)) continue;
    const int r1 = j1 - sc.start[k1], r2 = j2 - sc.start[k2];
    if (b1.blk > b2.blk || (b1.blk == b2.blk && r2 < r1)) continue;
    double val = 0.0;
    for (int q = 0; q < t.nres; ++q)
      val += side_column(sc, t.nblocks, J + q * NP, k1, j1) * side_column(sc, t.nblocks, J + q * NP, k2, j2);
    val *= scale[b1.col + r1] * scale[b2.col + r2];
    const int off = bsr_lookup(h, b1.blk, b2.blk);
    atomicAdd(&Sval[off + r1 * b2.np + r2], val);
    if (j1 == j2) {
      double g = 0.0;
      for (int q = 0; q < t.nres; ++q) g += side_column(sc, t.nblocks, J + q * NP, k1, j1) * r[q];
      atomicAdd(&rhs[b1.col + r1], g * scale[b1.col + r1]);
    }
  }
}

// structure: every pair of free blocks of a term owns a block of the reduced system
__global__ void side_enum_pairs(SideView sv, BAView v, BlkMaps bm, Params p, unsigned long long* tkeys, unsigned tmask,
                                int nblk) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= sv.n) return;
  const SideTerm t = sv.terms[i];
  const SideCols sc = side_cols(v, bm, sv, p, t);
  for (int a = 0; a < t.nblocks; ++a) {
    if (sc.b[a].blk < 0) continue;
    for (int b = a; b < t.nblocks; ++b) {
      if (sc.b[b].blk < 0) continue;
      const int lo = min(sc.b[a].blk, sc.b[b].blk), hi = max(sc.b[a].blk, sc.b[b].blk);
      bsr_insert(tkeys, tmask, (unsigned long long)lo * (unsigned)nblk + (unsigned)hi);
    }
  }
}

}  // namespace osfm
