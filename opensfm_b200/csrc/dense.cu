// DENSE: depthmaps of many shots at once, from views kept resident on the device.
//
// Replaces pydense (opensfm/src/dense/src/depthmap.cc) behind opensfm/dense.py: DepthmapEstimator's brute force
// (:184-204), PatchMatch and PatchMatch-sample (:206-490), DepthmapCleaner::Clean (:512-543) and
// DepthmapPruner::Prune (:565-625).  The restatement the results are checked against bit for bit is
// oracle/dense_oracle.cpp.  The one deliberate difference from the reference is the generator: every draw is
// Philox4x32-10 keyed by (seed, reference key) at counter (pixel, pass, draw, attempt), see dense_math.cuh.
//
// Layout: every view's gray, mask, RGB and label images in u8 slabs, and its raw depth, plane and clean depth in
// f32 slabs, all at one pixel offset per view.  An estimate submission's maps are laid out per reference in request
// order.  Kernels:
//   dn_brute_force   one thread per pixel, every plane against every view
//   dn_init          one thread per pixel: random plane, then the ignore mask
//   dn_propagate     one CTA per reference: forward and backward passes by anti-diagonals (i + j = k), which give
//                    the raster order's result because a pixel reads only itself and its two predecessors
//   dn_median, dn_post, dn_gate   PostProcess and compute_depthmap's gate into the raw slot cleaning reads
//   dn_clean         one thread per pixel over the raw slots
//   dn_prune_flag, dn_prune_write   one thread per pixel, then a scan and the compaction in raster order
// This file is compiled with -fmad=false: no product is contracted into an add anywhere.
#include <cub/cub.cuh>

#include <cmath>

#include "common.cuh"
#include "dense_math.cuh"

namespace osfm {
namespace {

using namespace dense;

constexpr int DN_MAX_PATCH = OSFM_DENSE_MAX_PATCH;
constexpr int DN_MAX_HPZ = (DN_MAX_PATCH - 1) / 2;
constexpr int DN_WD = 2 * DN_MAX_HPZ * DN_MAX_HPZ + 1;   // weight table columns: dx^2 + dy^2
constexpr int DN_MAX_VIEWS = OSFM_DENSE_MAX_VIEWS;
constexpr int DN_THREADS = 256;
constexpr double DN_Z_EPSILON = 1e-8;

struct DView {
  int w, h;
  long long off;
  double K[9], Kinv[9], R[9], t[3];
};

// one reference of an estimate submission
struct DRef {
  int n, first;          // list entries [first, first + n); entry first is the reference view
  int method, hpz, planes, iterations;
  uint32_t key;
  float min_var;
  double dmin, dmax;
  long long out;         // offset of its maps in the submission's outputs
};

// entry e of a list: its view, and Q = R_v R_ref^T, a = Q t_ref - t_v
struct DEntry {
  int view;
  double Q[9], a[3];
};

struct DArgs {
  const DView* views;
  const DRef* refs;
  const DEntry* entries;
  const uint8_t* gray;
  const uint8_t* mask;
  const float* weights;   // 256 x DN_WD
  uint32_t seed;
  float min_score;
  float* depth;
  float* plane;
  float* score;
  int* nghbr;
  float* median;
  float* raw_depth;
  float* raw_plane;
};

// ---- geometry, in the reference's expression types --------------------------------------------------------------

__device__ __forceinline__ void mat3(const double* A, const double* B, double* C) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      double s = 0.0;
      for (int k = 0; k < 3; ++k) s += A[3 * i + k] * B[3 * k + j];
      C[3 * i + j] = s;
    }
}

// PlaneInducedHomographyBaked: K2 (Q + a v^T) K1^-1 in fp64, rounded to f32
__device__ __forceinline__ void homography(const double* K2, const DEntry& e, const double* K1inv, const float* pl,
                                           float* H) {
  const double v[3] = {(double)pl[0], (double)pl[1], (double)pl[2]};
  double M[9], T[9], Hd[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) M[3 * i + j] = e.Q[3 * i + j] + e.a[i] * v[j];
  mat3(K2, M, T);
  mat3(T, K1inv, Hd);
  for (int k = 0; k < 9; ++k) H[k] = (float)Hd[k];
}

__device__ __forceinline__ float fmax_ref(float a, float b) { return a < b ? b : a; }   // std::max(a, b)

// PlaneFromDepthAndNormal
__device__ __forceinline__ void plane_from_depth(float x, float y, const double* Kinv, float depth, const float* n,
                                                 float* pl) {
  const double X[3] = {(double)x, (double)y, 1.0};
  float p[3];
  for (int i = 0; i < 3; ++i) {
    double s = 0.0;
    for (int k = 0; k < 3; ++k) s += (Kinv[3 * i + k] * (double)depth) * X[k];
    p[i] = (float)s;
  }
  float d = 0.f;
  for (int k = 0; k < 3; ++k) d += n[k] * p[k];
  const float r = 1.f / fmax_ref(1e-6f, -d);
  for (int k = 0; k < 3; ++k) pl[k] = n[k] * r;
}

// DepthOfPlaneBackprojection
__device__ __forceinline__ float depth_of_plane(double x, double y, const double* Kinv, const float* pl) {
  double r[3];
  for (int j = 0; j < 3; ++j) {
    double s = 0.0;
    for (int k = 0; k < 3; ++k) s += (double)pl[k] * Kinv[3 * k + j];
    r[j] = s;
  }
  double s = 0.0;
  s += r[0] * x;
  s += r[1] * y;
  s += r[2] * 1.0;
  const float denom = (float)(-s);
  return 1.0f / fmax_ref(1e-6f, denom);
}

// Backproject, fp64: R^T (depth K^-1 (x, y, 1) - t)
__device__ __forceinline__ void backproject(double x, double y, double depth, const DView& v, double* X) {
  const double P[3] = {x, y, 1.0};
  double q[3];
  for (int i = 0; i < 3; ++i) {
    double s = 0.0;
    for (int k = 0; k < 3; ++k) s += (v.Kinv[3 * i + k] * depth) * P[k];
    q[i] = s - v.t[i];
  }
  for (int i = 0; i < 3; ++i) {
    double s = 0.0;
    for (int k = 0; k < 3; ++k) s += v.R[3 * k + i] * q[k];
    X[i] = s;
  }
}

// Project, fp64: K (R x + t)
__device__ __forceinline__ void project(const float* x, const DView& v, double* out) {
  double y[3];
  for (int i = 0; i < 3; ++i) {
    double s = 0.0;
    for (int k = 0; k < 3; ++k) s += v.R[3 * i + k] * (double)x[k];
    y[i] = s + v.t[i];
  }
  for (int i = 0; i < 3; ++i) {
    double s = 0.0;
    for (int k = 0; k < 3; ++k) s += v.K[3 * i + k] * y[k];
    out[i] = s;
  }
}

// cv::normalize of a Vec3f: the norm's squares summed in f32, the scale 1 / norm in fp64
__device__ __forceinline__ void normalize3(const float* v, float* o) {
  float s = 0.f;
  for (int k = 0; k < 3; ++k) s += v[k] * v[k];
  const double nv = (double)sqrtf(s);
  const double sc = nv != 0.0 ? 1.0 / nv : 0.0;
  for (int k = 0; k < 3; ++k) o[k] = (float)((double)v[k] * sc);
}

// LinearInterpolation: 0 outside [0, cols - 1) x [0, rows - 1), and for NaN coordinates
template <class T>
__device__ __forceinline__ float interp(const T* im, int cols, int rows, float y, float x) {
  if (!(x >= 0.0f && x < (float)(cols - 1) && y >= 0.0f && y < (float)(rows - 1))) return 0.0f;
  const int ix = (int)x, iy = (int)y;
  const float dx = x - (float)ix, dy = y - (float)iy;
  const float im00 = (float)im[(long long)iy * cols + ix];
  const float im01 = (float)im[(long long)iy * cols + ix + 1];
  const float im10 = (float)im[(long long)(iy + 1) * cols + ix];
  const float im11 = (float)im[(long long)(iy + 1) * cols + ix + 1];
  const float im0 = (1.f - dx) * im00 + dx * im01;
  const float im1 = (1.f - dx) * im10 + dx * im11;
  return (1.f - dy) * im0 + dy * im1;
}

// ComputePlaneImageScore of plane at (i, j) against list entry e (local index > 0)
__device__ __forceinline__ float image_score(const DArgs& A, const DRef& r, const DView& v0, int i, int j, const float* pl, int e) {
  const DEntry& E = A.entries[r.first + e];
  const DView& vo = A.views[E.view];
  float H[9];
  homography(vo.K, E, v0.Kinv, pl, H);
  const float fj = (float)j, fi = (float)i;
  const float u = H[0] * fj + H[1] * fi + H[2];
  const float v = H[3] * fj + H[4] * fi + H[5];
  const float w = H[6] * fj + H[7] * fi + H[8];
  if (w == 0.0f) return -1.0f;
  const float ww = w * w;
  const float dfdx_x = (H[0] * w - H[6] * u) / ww;
  const float dfdx_y = (H[3] * w - H[6] * v) / ww;
  const float dfdy_x = (H[1] * w - H[7] * u) / ww;
  const float dfdy_y = (H[4] * w - H[7] * v) / ww;
  const float Hx0 = u / w, Hy0 = v / w;
  const uint8_t* im0 = A.gray + v0.off;
  const uint8_t* im2 = A.gray + vo.off;
  const float center = (float)im0[(long long)i * v0.w + j];
  float sx = 0.f, sy = 0.f, sxx = 0.f, syy = 0.f, sxy = 0.f, sw = 0.f;
  for (int dy = -r.hpz; dy <= r.hpz; ++dy) {
    for (int dx = -r.hpz; dx <= r.hpz; ++dx) {
      const float x1 = (float)im0[(long long)(i + dy) * v0.w + j + dx];
      const float x2 = Hx0 + dfdx_x * (float)dx + dfdy_x * (float)dy;
      const float y2 = Hy0 + dfdx_y * (float)dx + dfdy_y * (float)dy;
      const float y = interp(im2, vo.w, vo.h, y2, x2);
      const int dc = (int)fabsf(x1 - center);
      const float wt = __ldg(A.weights + dc * DN_WD + dx * dx + dy * dy);
      sx += wt * x1;
      sy += wt * y;
      sxx += wt * x1 * x1;
      syy += wt * y * y;
      sxy += wt * x1 * y;
      sw += wt;
    }
  }
  if (sw == 0.0f) return -1.0f;
  const float mx = sx / sw, my = sy / sw, mxx = sxx / sw, myy = syy / sw, mxy = sxy / sw;
  const float varx = mxx - mx * mx, vary = myy - my * my;
  if ((double)varx < 0.1 || (double)vary < 0.1) return -1.0f;
  return (mxy - mx * my) / sqrtf(varx * vary);
}

// ComputePlaneScore: the best view, strictly greater wins, starting from (-1, 0)
__device__ __forceinline__ void plane_score(const DArgs& A, const DRef& r, const DView& v0, int i, int j,
                                            const float* pl, float* score, int* nghbr) {
  *score = -1.0f;
  *nghbr = 0;
#pragma unroll 1
  for (int e = 1; e < r.n; ++e) {
    const float s = image_score(A, r, v0, i, j, pl, e);
    if (s > *score) {
      *score = s;
      *nghbr = e;
    }
  }
}

__device__ __forceinline__ void assign(const DArgs& A, long long p, float d, const float* pl, float s, int nb) {
  A.depth[p] = d;
  A.plane[3 * p] = pl[0];
  A.plane[3 * p + 1] = pl[1];
  A.plane[3 * p + 2] = pl[2];
  A.score[p] = s;
  A.nghbr[p] = nb;
}

// CheckPlaneCandidate (e < 0: every view) / CheckPlaneImageCandidate (view e)
__device__ __forceinline__ void check_candidate(const DArgs& A, const DRef& r, const DView& v0, int i, int j,
                                                const float* pl, int e) {
  float s;
  int nb = e;
  if (e < 0)
    plane_score(A, r, v0, i, j, pl, &s, &nb);
  else
    s = image_score(A, r, v0, i, j, pl, e);
  const long long p = r.out + (long long)i * v0.w + j;
  if (s > A.score[p]) assign(A, p, depth_of_plane((double)j, (double)i, v0.Kinv, pl), pl, s, nb);
}

__global__ void __launch_bounds__(DN_THREADS, 1) dn_brute_force(DArgs A, const int* which) {
  const DRef r = A.refs[which[blockIdx.y]];
  const DView& v0 = A.views[A.entries[r.first].view];
  const int W = v0.w - 2 * r.hpz, Hh = v0.h - 2 * r.hpz;
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= W * Hh) return;
  const int i = r.hpz + q / W, j = r.hpz + q % W;
  const float normal[3] = {0.f, 0.f, -1.f};
#pragma unroll 1
  for (int d = 0; d < r.planes; ++d) {
    float depth;
    if (r.planes <= 1)
      depth = (float)r.dmin;
    else
      depth = (float)(1.0 / (1.0 / r.dmin + (double)d * (1.0 / r.dmax - 1.0 / r.dmin) / (double)(r.planes - 1)));
    float pl[3];
    plane_from_depth((float)j, (float)i, v0.Kinv, depth, normal, pl);
    check_candidate(A, r, v0, i, j, pl, -1);
  }
}

__device__ __forceinline__ uint32_t pixel_counter(const DView& v0, int i, int j) {
  return (uint32_t)i * (uint32_t)v0.w + (uint32_t)j;
}

// RandomInitialization, then ComputeIgnoreMask (an ignored pixel's draws are not scored)
__global__ void __launch_bounds__(DN_THREADS) dn_init(DArgs A, const int* which) {
  const DRef r = A.refs[which[blockIdx.y]];
  const DView& v0 = A.views[A.entries[r.first].view];
  const int W = v0.w - 2 * r.hpz, Hh = v0.h - 2 * r.hpz;
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= W * Hh) return;
  const int i = r.hpz + q / W, j = r.hpz + q % W;
  const long long p = r.out + (long long)i * v0.w + j;
  const uint8_t* im0 = A.gray + v0.off;
  const int P = 2 * r.hpz + 1, n = P * P;
  float sum = 0.f;
  for (int u = -r.hpz; u <= r.hpz; ++u)
    for (int v = -r.hpz; v <= r.hpz; ++v) sum += (float)im0[(long long)(i + u) * v0.w + j + v];
  const float mean = sum / (float)n;
  float sum2 = 0.f;
  for (int u = -r.hpz; u <= r.hpz; ++u)
    for (int v = -r.hpz; v <= r.hpz; ++v) {
      const float x = (float)im0[(long long)(i + u) * v0.w + j + v];
      sum2 += (x - mean) * (x - mean);
    }
  const bool masked = A.mask[v0.off + (long long)i * v0.w + j] == 0;
  if (masked || sum2 / (float)n < r.min_var) {
    const float zero[3] = {0.f, 0.f, 0.f};
    assign(A, p, 0.f, zero, 0.f, 0);
    return;
  }
  const U4 x = philox(pixel_counter(v0, i, j), 0, DRAW_INIT, 0, A.seed, r.key);
  const float la = (float)dn_log(r.dmin), lb = (float)dn_log(r.dmax);
  const float depth = (float)dn_exp((double)(la + (lb - la) * dn_unit(x.x[0])));
  const float normal[3] = {-1.f + 2.f * dn_unit(x.x[1]), -1.f + 2.f * dn_unit(x.x[2]), -1.f};
  float pl[3];
  plane_from_depth((float)j, (float)i, v0.Kinv, depth, normal, pl);
  float s;
  int nb;
  if (r.method == OSFM_DENSE_PATCH_MATCH_SAMPLE) {
    nb = dn_index(x.x[3], 1, r.n - 1);
    s = image_score(A, r, v0, i, j, pl, nb);
  } else {
    plane_score(A, r, v0, i, j, pl, &s, &nb);
  }
  assign(A, p, depth, pl, s, nb);
}

// PatchMatchUpdatePixel; dir = -1 forward (reads (i-1, j), (i, j-1)), +1 backward (reads (i, j+1), (i+1, j))
__device__ void update_pixel(const DArgs& A, const DRef& r, const DView& v0, int i, int j, int dir, uint32_t pass) {
  const long long p = r.out + (long long)i * v0.w + j;
  if (A.depth[p] == 0.0f) return;
  const bool sample = r.method == OSFM_DENSE_PATCH_MATCH_SAMPLE;
  const long long adj[2] = {dir < 0 ? p - v0.w : p + 1, dir < 0 ? p - 1 : p + v0.w};
  for (int k = 0; k < 2; ++k) {
    const long long a = adj[k];
    if (A.depth[a] == 0.0f) continue;
    const float pl[3] = {A.plane[3 * a], A.plane[3 * a + 1], A.plane[3 * a + 2]};
    check_candidate(A, r, v0, i, j, pl, sample ? A.nghbr[a] : -1);
  }
  const uint32_t pix = pixel_counter(v0, i, j);
  float depth_range = 0.02f, normal_range = 0.5f;
  const int current = A.nghbr[p];
  for (int k = 0; k < 6; ++k) {
    const float nd = dn_normal(pix, pass, DRAW_PERTURB + 3 * k, A.seed, r.key);
    const float depth = A.depth[p] * (float)dn_exp((double)(depth_range * nd));
    const float cp[3] = {A.plane[3 * p], A.plane[3 * p + 1], A.plane[3 * p + 2]};
    if (cp[2] == 0.0f) continue;   // as the reference: the ranges do not decay for this k
    const float n0 = dn_normal(pix, pass, DRAW_PERTURB + 3 * k + 1, A.seed, r.key);
    const float n1 = dn_normal(pix, pass, DRAW_PERTURB + 3 * k + 2, A.seed, r.key);
    const float normal[3] = {-cp[0] / cp[2] + normal_range * n0, -cp[1] / cp[2] + normal_range * n1, -1.0f};
    float pl[3];
    plane_from_depth((float)j, (float)i, v0.Kinv, depth, normal, pl);
    check_candidate(A, r, v0, i, j, pl, sample ? current : -1);
    depth_range = (float)((double)depth_range * 0.3);
    normal_range = (float)((double)normal_range * 0.8);
  }
  if (!sample || r.n <= 2) return;
  int other = current;
  for (uint32_t a = 0; other == current; ++a) {
    const U4 x = philox(pix, pass, DRAW_OTHER_VIEW, a >> 2, A.seed, r.key);
    other = dn_index(x.x[a & 3], 1, r.n - 1);
  }
  const float pl[3] = {A.plane[3 * p], A.plane[3 * p + 1], A.plane[3 * p + 2]};
  check_candidate(A, r, v0, i, j, pl, other);
}

// Every iteration's forward and backward pass, one CTA per reference.  Pixels of one anti-diagonal depend only on the
// previous one, so the CTA walks the diagonals behind __syncthreads (which also orders its global stores).
__global__ void __launch_bounds__(DN_THREADS) dn_propagate(DArgs A, const int* which) {
  const DRef r = A.refs[which[blockIdx.x]];
  const DView& v0 = A.views[A.entries[r.first].view];
  const int i0 = r.hpz, i1 = v0.h - r.hpz - 1, j0 = r.hpz, j1 = v0.w - r.hpz - 1;
  if (i1 < i0 || j1 < j0) return;
  for (int it = 0; it < r.iterations; ++it) {
    for (int dir = -1; dir <= 1; dir += 2) {
      const uint32_t pass = 1 + 2 * it + (dir > 0);
      for (int s = 0; s <= (i1 - i0) + (j1 - j0); ++s) {
        const int k = dir < 0 ? i0 + j0 + s : i1 + j1 - s;   // i + j on this diagonal
        const int ilo = max(i0, k - j1), ihi = min(i1, k - j0);
        for (int i = ilo + (int)threadIdx.x; i <= ihi; i += blockDim.x) update_pixel(A, r, v0, i, k - i, dir, pass);
        __syncthreads();
      }
    }
  }
}

// cv::medianBlur(depth, 5) with replicated borders
__global__ void __launch_bounds__(DN_THREADS) dn_median(DArgs A, const int* which) {
  const DRef r = A.refs[which[blockIdx.y]];
  const DView& v0 = A.views[A.entries[r.first].view];
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= v0.w * v0.h) return;
  const int i = q / v0.w, j = q % v0.w;
  float v[25];
  int c = 0;
  for (int di = -2; di <= 2; ++di)
    for (int dj = -2; dj <= 2; ++dj) {
      const int ii = min(max(i + di, 0), v0.h - 1), jj = min(max(j + dj, 0), v0.w - 1);
      v[c++] = A.depth[r.out + (long long)ii * v0.w + jj];
    }
  for (int a = 0; a <= 12; ++a) {
    int m = a;
    for (int b = a + 1; b < 25; ++b)
      if (v[b] < v[m]) m = b;
    const float t = v[a];
    v[a] = v[m];
    v[m] = t;
  }
  A.median[r.out + q] = v[12];
}

__global__ void __launch_bounds__(DN_THREADS) dn_post(DArgs A, const int* which) {
  const DRef r = A.refs[which[blockIdx.y]];
  const DView& v0 = A.views[A.entries[r.first].view];
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= v0.w * v0.h) return;
  const float d = A.depth[r.out + q], m = A.median[r.out + q];
  if (d == 0.0f || (double)(fabsf(d - m) / d) > 0.05) A.depth[r.out + q] = 0.0f;
}

// compute_depthmap's gate (score > min_score in f32, depth < max_depth in fp64) into the reference view's raw slot
__global__ void __launch_bounds__(DN_THREADS) dn_gate(DArgs A) {
  const DRef r = A.refs[blockIdx.y];
  const DView& v0 = A.views[A.entries[r.first].view];
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= v0.w * v0.h) return;
  const float d = A.depth[r.out + q];
  const bool good = A.score[r.out + q] > A.min_score && (double)d < r.dmax;
  A.raw_depth[v0.off + q] = good ? d : 0.0f;
  for (int k = 0; k < 3; ++k) A.raw_plane[3 * (v0.off + q) + k] = A.plane[3 * (r.out + q) + k];
}

// ---- cleaning and pruning ---------------------------------------------------------------------------------------

struct DListArgs {
  const DView* views;
  const int* list_start;   // per reference, into list
  const int* list;         // view indices, reference first
  const long long* out;    // per reference: offset of its pixels in the submission
  float threshold;
  int min_consistent;
  const float* raw_depth;
  float* clean_depth;
  const float* plane;
  const uint8_t* rgb;
  const uint8_t* labels;
  uint8_t* keep;
  const long long* slot;   // exclusive scan of keep
  float* points;
  float* normals;
  uint8_t* colors;
  uint8_t* out_labels;
};

__global__ void __launch_bounds__(DN_THREADS) dn_clean(DListArgs L) {
  const int* lst = L.list + L.list_start[blockIdx.y];
  const int n = L.list_start[blockIdx.y + 1] - L.list_start[blockIdx.y];
  const DView& v0 = L.views[lst[0]];
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= v0.w * v0.h) return;
  const int i = q / v0.w, j = q % v0.w;
  const float depth = L.raw_depth[v0.off + q];
  double Xd[3];
  backproject((double)j, (double)i, (double)depth, v0, Xd);
  const float X[3] = {(float)Xd[0], (float)Xd[1], (float)Xd[2]};
  int consistent = 1;
  for (int o = 1; o < n; ++o) {
    const DView& vo = L.views[lst[o]];
    double rd[3];
    project(X, vo, rd);
    const float rp[3] = {(float)rd[0], (float)rd[1], (float)rd[2]};
    if ((double)rp[2] < DN_Z_EPSILON || isnan(rp[2])) continue;
    const float u = rp[0] / rp[2], v = rp[1] / rp[2], dpt = rp[2];
    const float dr = interp(L.raw_depth + vo.off, vo.w, vo.h, v, u);
    if (fabsf(dr - dpt) < dpt * L.threshold) ++consistent;
  }
  L.clean_depth[v0.off + q] = consistent >= L.min_consistent ? depth : 0.0f;
}

__device__ __forceinline__ float area_of(const float* nrm, float depth, const DView& v) {
  return (float)((double)(-nrm[2] / depth) * v.K[0]);
}

__global__ void __launch_bounds__(DN_THREADS) dn_prune_flag(DListArgs L) {
  const int* lst = L.list + L.list_start[blockIdx.y];
  const int n = L.list_start[blockIdx.y + 1] - L.list_start[blockIdx.y];
  const DView& v0 = L.views[lst[0]];
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= v0.w * v0.h) return;
  const int i = q / v0.w, j = q % v0.w;
  const float depth = L.clean_depth[v0.off + q];
  bool keep = depth > 0;
  if (keep) {
    float nrm[3];
    normalize3(L.plane + 3 * (v0.off + q), nrm);
    const float area = area_of(nrm, depth, v0);
    double Xd[3];
    backproject((double)j, (double)i, (double)depth, v0, Xd);
    const float X[3] = {(float)Xd[0], (float)Xd[1], (float)Xd[2]};
    for (int o = 1; o < n; ++o) {
      const DView& vo = L.views[lst[o]];
      double rp[3];
      project(X, vo, rp);
      if (rp[2] < DN_Z_EPSILON || isnan(rp[2])) continue;
      const long long iu = (long long)(rp[0] / rp[2] + 0.5), iv = (long long)(rp[1] / rp[2] + 0.5);
      if (iv < 0 || iv >= vo.h || iu < 0 || iu >= vo.w) continue;
      const long long at = vo.off + iv * vo.w + iu;
      const float da = L.clean_depth[at];
      if ((double)da > (double)(1.0f - L.threshold) * rp[2]) {
        float no[3];
        normalize3(L.plane + 3 * at, no);
        if (da == 0.0f || (double)(-no[2] / da) * vo.K[0] > (double)area) {
          keep = false;
          break;
        }
      }
    }
  }
  L.keep[L.out[blockIdx.y] + q] = keep;
}

__global__ void __launch_bounds__(DN_THREADS) dn_prune_write(DListArgs L) {
  const int* lst = L.list + L.list_start[blockIdx.y];
  const DView& v0 = L.views[lst[0]];
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= v0.w * v0.h) return;
  const long long g = L.out[blockIdx.y] + q;
  if (!L.keep[g]) return;
  const long long s = L.slot[g];
  const int i = q / v0.w, j = q % v0.w;
  const float depth = L.clean_depth[v0.off + q];
  float nrm[3];
  normalize3(L.plane + 3 * (v0.off + q), nrm);
  double Xd[3];
  backproject((double)j, (double)i, (double)depth, v0, Xd);
  for (int k = 0; k < 3; ++k) {
    float acc = 0.f;   // Matx33f(R^T) * normal
    for (int m = 0; m < 3; ++m) acc += (float)v0.R[3 * m + k] * nrm[m];
    L.points[3 * s + k] = (float)Xd[k];
    L.normals[3 * s + k] = acc;
    L.colors[3 * s + k] = L.rgb[3 * (v0.off + q) + k];
  }
  L.out_labels[s] = L.labels[v0.off + q];
}

// ---- the engine -------------------------------------------------------------------------------------------------

struct Dense : DeviceStream<6> {
  std::vector<DView> views;
  std::vector<uint8_t> has_raw, has_clean;
  bool has_gray = false, has_mask = false, has_color = false;
  long long pixels = 0;
  DevBuf<DView> d_views;
  DevBuf<uint8_t> d_gray, d_mask, d_rgb, d_labels;
  DevBuf<float> d_raw, d_plane, d_clean;
  // estimate
  DevBuf<DRef> d_refs;
  DevBuf<DEntry> d_entries;
  DevBuf<int> d_which;
  DevBuf<float> d_weights, d_depth, d_eplane, d_score, d_median;
  DevBuf<int> d_nghbr;
  // clean / prune
  DevBuf<int> d_list_start, d_list;
  DevBuf<long long> d_out, d_slot;
  DevBuf<uint8_t> d_keep, d_scan_tmp, d_colors, d_out_labels;
  DevBuf<float> d_points, d_normals;
  long long pruned = 0;
  bool timed[3] = {false, false, false};

  explicit Dense(int dev) : DeviceStream<6>(dev) {}

  // fails naming the bytes `what` needs when they exceed the device's free memory (before any allocation for it)
  static void fits(const char* what, long long bytes) {
    size_t free_b = 0, total_b = 0;
    OSFM_CUDA(cudaMemGetInfo(&free_b, &total_b));
    if (bytes > 0 && (size_t)bytes > free_b)
      throw std::runtime_error(std::string("dense: ") + what + " need " + std::to_string(bytes) +
                               " bytes of device memory, " + std::to_string(free_b) + " are free");
  }

  void set_views(int n, const int32_t* size, const double* K, const double* Kinv, const double* R, const double* t,
                 const uint8_t* gray, const uint8_t* mask, const uint8_t* rgb, const uint8_t* labels) {
    if (n < 0) throw ArgError("dense: negative number of views");
    if (n > 0 && (!size || !K || !Kinv || !R || !t)) throw ArgError("dense: null view geometry");
    std::vector<DView> v(n);
    long long off = 0;
    for (int k = 0; k < n; ++k) {
      if (size[2 * k] < 1 || size[2 * k + 1] < 1)
        throw ArgError("dense: view " + std::to_string(k) + " has an empty image");
      v[k].w = size[2 * k];
      v[k].h = size[2 * k + 1];
      v[k].off = off;
      off += (long long)v[k].w * v[k].h;
      std::copy(K + 9 * k, K + 9 * k + 9, v[k].K);
      std::copy(Kinv + 9 * k, Kinv + 9 * k + 9, v[k].Kinv);
      std::copy(R + 9 * k, R + 9 * k + 9, v[k].R);
      std::copy(t + 3 * k, t + 3 * k + 3, v[k].t);
    }
    fits("the views and their maps", off * (1 + 1 + 3 + 1 + 4 * 5));
    views = v;
    pixels = off;
    has_raw.assign(n, 0);
    has_clean.assign(n, 0);
    has_gray = gray != nullptr;
    has_mask = mask != nullptr;
    has_color = rgb != nullptr && labels != nullptr;
    upload(d_views, views.data(), views.size());
    upload(d_gray, gray, gray ? (size_t)off : 0);
    upload(d_mask, mask, mask ? (size_t)off : 0);
    upload(d_rgb, rgb, has_color ? (size_t)off * 3 : 0);
    upload(d_labels, labels, has_color ? (size_t)off : 0);
    d_raw.reserve((size_t)std::max(off, 1LL));
    d_clean.reserve((size_t)std::max(off, 1LL));
    d_plane.reserve((size_t)std::max(off * 3, 1LL));
    OSFM_CUDA(cudaStreamSynchronize(stream));
  }

  void check_view(int v) const {
    if (v < 0 || v >= (int)views.size())
      throw ArgError("dense: view index " + std::to_string(v) + " is out of range (" +
                     std::to_string(views.size()) + " views)");
  }

  void set_maps(int v, const float* raw, const float* plane, const float* clean) {
    check_view(v);
    const DView& V = views[v];
    const size_t np = (size_t)V.w * V.h;
    if (raw) OSFM_CUDA(cudaMemcpyAsync(d_raw.p + V.off, raw, np * 4, cudaMemcpyHostToDevice, stream));
    if (plane) OSFM_CUDA(cudaMemcpyAsync(d_plane.p + 3 * V.off, plane, np * 12, cudaMemcpyHostToDevice, stream));
    if (clean) OSFM_CUDA(cudaMemcpyAsync(d_clean.p + V.off, clean, np * 4, cudaMemcpyHostToDevice, stream));
    OSFM_CUDA(cudaStreamSynchronize(stream));
    if (raw && plane) has_raw[v] = 1;
    if (clean && plane) has_clean[v] = 1;
  }

  // views: every reference's list, checked; with `writes` (estimate and clean write the reference view's slot) no
  // two references may share a reference view.  Returns the pixel offset of every reference in the submission.
  std::vector<long long> check_lists(const char* what, int num_refs, const int32_t* list_start, const int32_t* list,
                                     int min_views, bool writes) {
    if (num_refs < 0) throw ArgError(std::string(what) + ": negative number of references");
    if (num_refs > 65535) throw ArgError(std::string(what) + ": more than 65535 references in one call");
    if (num_refs > 0 && (!list_start || !list)) throw ArgError(std::string(what) + ": null view lists");
    std::vector<long long> out(num_refs + 1, 0);
    if (num_refs > 0 && list_start[0] != 0) throw ArgError(std::string(what) + ": list_start[0] must be 0");
    for (int r = 0; r < num_refs; ++r) {
      const int n = list_start[r + 1] - list_start[r];
      if (n < min_views || n > DN_MAX_VIEWS)
        throw ArgError(std::string(what) + ": reference " + std::to_string(r) + " has " + std::to_string(n) +
                       " views; " + std::to_string(min_views) + " to " + std::to_string(DN_MAX_VIEWS) + " are needed");
      for (int e = list_start[r]; e < list_start[r + 1]; ++e) check_view(list[e]);
      for (int q = 0; writes && q < r; ++q)
        if (list[list_start[q]] == list[list_start[r]])
          throw ArgError(std::string(what) + ": references " + std::to_string(q) + " and " + std::to_string(r) +
                         " are both view " + std::to_string(list[list_start[r]]) + "; each view's maps have one slot");
      const DView& v0 = views[list[list_start[r]]];
      out[r + 1] = out[r] + (long long)v0.w * v0.h;
    }
    return out;
  }

  void estimate(int num_refs, const int32_t* list_start, const int32_t* list, const double* Q, const double* a,
                const int32_t* params, const double* depth_range, const float* min_patch_variance,
                const float* weights, uint32_t seed, double min_score, float* depth, float* plane, float* score,
                int32_t* nghbr) {
    timed[0] = false;
    const std::vector<long long> out = check_lists("estimate", num_refs, list_start, list, 2, true);
    if (num_refs == 0) return;
    if (!Q || !a || !params || !depth_range || !min_patch_variance || !weights)
      throw ArgError("estimate: null arrays");
    if (!has_gray || !has_mask) throw ArgError("estimate: the views have no gray images or masks");
    std::vector<DRef> refs(num_refs);
    std::vector<DEntry> entries(list_start[num_refs]);
    for (int e = 0; e < list_start[num_refs]; ++e) {
      entries[e].view = list[e];
      std::copy(Q + 9LL * e, Q + 9LL * e + 9, entries[e].Q);
      std::copy(a + 3LL * e, a + 3LL * e + 3, entries[e].a);
    }
    std::vector<int> bf, pm;
    for (int r = 0; r < num_refs; ++r) {
      DRef& R = refs[r];
      const std::string who = "estimate: reference " + std::to_string(r);
      R.n = list_start[r + 1] - list_start[r];
      R.first = list_start[r];
      R.method = params[5 * r];
      const int patch = params[5 * r + 1];
      R.planes = params[5 * r + 2];
      R.iterations = params[5 * r + 3];
      R.key = (uint32_t)params[5 * r + 4];
      R.dmin = depth_range[2 * r];
      R.dmax = depth_range[2 * r + 1];
      R.min_var = min_patch_variance[r];
      R.out = out[r];
      const DView& v0 = views[list[R.first]];
      if (R.method < OSFM_DENSE_BRUTE_FORCE || R.method > OSFM_DENSE_PATCH_MATCH_SAMPLE)
        throw ArgError(who + ": unknown method " + std::to_string(R.method));
      if (patch < 1 || patch % 2 == 0 || patch > DN_MAX_PATCH)
        throw ArgError(who + ": patch size " + std::to_string(patch) + " must be odd and at most " +
                       std::to_string(DN_MAX_PATCH));
      if (patch > v0.w || patch > v0.h)
        throw ArgError(who + ": patch size " + std::to_string(patch) + " exceeds the image size");
      R.hpz = (patch - 1) / 2;
      if (R.iterations < 0) throw ArgError(who + ": negative number of PatchMatch iterations");
      if (!(R.dmin > 0.0) || !(R.dmax > 0.0) || !std::isfinite(R.dmin) || !std::isfinite(R.dmax))
        throw ArgError(who + ": the depth range must be positive and finite");
      (R.method == OSFM_DENSE_BRUTE_FORCE ? bf : pm).push_back(r);
    }
    const long long total = out[num_refs];
    // depth, plane, score, nghbr and median of every reference pixel (buffers already large enough are not counted)
    fits("the estimate's maps", (total > (long long)d_depth.cap ? total * 28 : 0));
    upload(d_refs, refs.data(), refs.size());
    upload(d_entries, entries.data(), entries.size());
    upload(d_weights, weights, (size_t)256 * DN_WD);
    std::vector<int> which = bf;
    which.insert(which.end(), pm.begin(), pm.end());
    upload(d_which, which.data(), which.size());
    d_depth.reserve(total);
    d_eplane.reserve(total * 3);
    d_score.reserve(total);
    d_nghbr.reserve(total);
    d_median.reserve(total);
    OSFM_CUDA(cudaEventRecord(ev[0], stream));
    OSFM_CUDA(cudaMemsetAsync(d_depth.p, 0, total * 4, stream));
    OSFM_CUDA(cudaMemsetAsync(d_eplane.p, 0, total * 12, stream));
    OSFM_CUDA(cudaMemsetAsync(d_score.p, 0, total * 4, stream));
    OSFM_CUDA(cudaMemsetAsync(d_nghbr.p, 0, total * 4, stream));

    DArgs A;
    A.views = d_views.p;
    A.refs = d_refs.p;
    A.entries = d_entries.p;
    A.gray = d_gray.p;
    A.mask = d_mask.p;
    A.weights = d_weights.p;
    A.seed = seed;
    A.min_score = (float)min_score;
    A.depth = d_depth.p;
    A.plane = d_eplane.p;
    A.score = d_score.p;
    A.nghbr = d_nghbr.p;
    A.median = d_median.p;
    A.raw_depth = d_raw.p;
    A.raw_plane = d_plane.p;
    long long maxpix = 0;
    for (int r = 0; r < num_refs; ++r) maxpix = std::max(maxpix, out[r + 1] - out[r]);
    const unsigned gx = (unsigned)((maxpix + DN_THREADS - 1) / DN_THREADS);
    if (!bf.empty()) {
      dn_brute_force<<<dim3(gx, (unsigned)bf.size()), DN_THREADS, 0, stream>>>(A, d_which.p);
      OSFM_LAUNCH_CHECK();
    }
    if (!pm.empty()) {
      const int* w = d_which.p + bf.size();
      dn_init<<<dim3(gx, (unsigned)pm.size()), DN_THREADS, 0, stream>>>(A, w);
      OSFM_LAUNCH_CHECK();
      dn_propagate<<<(unsigned)pm.size(), DN_THREADS, 0, stream>>>(A, w);
      OSFM_LAUNCH_CHECK();
      dn_median<<<dim3(gx, (unsigned)pm.size()), DN_THREADS, 0, stream>>>(A, w);
      OSFM_LAUNCH_CHECK();
      dn_post<<<dim3(gx, (unsigned)pm.size()), DN_THREADS, 0, stream>>>(A, w);
      OSFM_LAUNCH_CHECK();
    }
    dn_gate<<<dim3(gx, (unsigned)num_refs), DN_THREADS, 0, stream>>>(A);
    OSFM_LAUNCH_CHECK();
    OSFM_CUDA(cudaEventRecord(ev[1], stream));
    if (depth) download(depth, d_depth.p, total);
    if (plane) download(plane, d_eplane.p, total * 3);
    if (score) download(score, d_score.p, total);
    if (nghbr) download(nghbr, d_nghbr.p, total);
    OSFM_CUDA(cudaStreamSynchronize(stream));
    for (int r = 0; r < num_refs; ++r) has_raw[list[list_start[r]]] = 1;
    timed[0] = true;
  }

  DListArgs list_args(int num_refs, const int32_t* list_start, const int32_t* list, const std::vector<long long>& out,
                      float threshold) {
    upload(d_list_start, list_start, num_refs + 1);
    upload(d_list, list, list_start[num_refs]);
    upload(d_out, out.data(), out.size());
    DListArgs L;
    L.views = d_views.p;
    L.list_start = d_list_start.p;
    L.list = d_list.p;
    L.out = d_out.p;
    L.threshold = threshold;
    L.raw_depth = d_raw.p;
    L.clean_depth = d_clean.p;
    L.plane = d_plane.p;
    L.rgb = d_rgb.p;
    L.labels = d_labels.p;
    return L;
  }

  void clean(int num_refs, const int32_t* list_start, const int32_t* list, float threshold, int min_consistent,
             float* clean_out) {
    timed[1] = false;
    const std::vector<long long> out = check_lists("clean", num_refs, list_start, list, 1, true);
    if (num_refs == 0) return;
    for (int e = 0; e < list_start[num_refs]; ++e)
      if (!has_raw[list[e]]) throw ArgError("clean: view " + std::to_string(list[e]) + " has no raw depthmap");
    DListArgs L = list_args(num_refs, list_start, list, out, threshold);
    L.min_consistent = min_consistent;
    long long maxpix = 0;
    for (int r = 0; r < num_refs; ++r) maxpix = std::max(maxpix, out[r + 1] - out[r]);
    OSFM_CUDA(cudaEventRecord(ev[2], stream));
    dn_clean<<<dim3((unsigned)((maxpix + DN_THREADS - 1) / DN_THREADS), (unsigned)num_refs), DN_THREADS, 0,
               stream>>>(L);
    OSFM_LAUNCH_CHECK();
    OSFM_CUDA(cudaEventRecord(ev[3], stream));
    if (clean_out)
      for (int r = 0; r < num_refs; ++r) {
        const DView& v0 = views[list[list_start[r]]];
        download(clean_out + out[r], d_clean.p + v0.off, out[r + 1] - out[r]);
      }
    OSFM_CUDA(cudaStreamSynchronize(stream));
    for (int r = 0; r < num_refs; ++r) has_clean[list[list_start[r]]] = 1;
    timed[1] = true;
  }

  void prune(int num_refs, const int32_t* list_start, const int32_t* list, float threshold, int64_t* counts) {
    timed[2] = false;
    pruned = 0;
    const std::vector<long long> out = check_lists("prune", num_refs, list_start, list, 1, false);
    if (num_refs == 0) return;
    if (!counts) throw ArgError("prune: null counts");
    if (!has_color) throw ArgError("prune: the views have no colour images and labels");
    for (int e = 0; e < list_start[num_refs]; ++e)
      if (!has_clean[list[e]]) throw ArgError("prune: view " + std::to_string(list[e]) + " has no clean depthmap");
    const long long total = out[num_refs];
    // flags, scan slots and, at worst, every pixel kept: 3 + 3 floats, 3 + 1 bytes
    fits("the pruner's buffers", (total + 1 > (long long)d_keep.cap ? (total + 1) * (1 + 8 + 28) : 0));
    DListArgs L = list_args(num_refs, list_start, list, out, threshold);
    d_keep.reserve(total + 1);
    d_slot.reserve(total + 1);
    L.keep = d_keep.p;
    L.slot = d_slot.p;
    long long maxpix = 0;
    for (int r = 0; r < num_refs; ++r) maxpix = std::max(maxpix, out[r + 1] - out[r]);
    const dim3 grid((unsigned)((maxpix + DN_THREADS - 1) / DN_THREADS), (unsigned)num_refs);
    OSFM_CUDA(cudaEventRecord(ev[4], stream));
    dn_prune_flag<<<grid, DN_THREADS, 0, stream>>>(L);
    OSFM_LAUNCH_CHECK();
    size_t tmp = 0;
    OSFM_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmp, d_keep.p, d_slot.p, total + 1, stream));
    d_scan_tmp.reserve(tmp);
    // keep[total], one past the flags, is cleared so that slot[total] is the kept count
    OSFM_CUDA(cudaMemsetAsync(d_keep.p + total, 0, 1, stream));
    OSFM_CUDA(cub::DeviceScan::ExclusiveSum(d_scan_tmp.p, tmp, d_keep.p, d_slot.p, total + 1, stream));
    std::vector<long long> slots(num_refs + 1);
    for (int r = 0; r <= num_refs; ++r) download(&slots[r], d_slot.p + out[r], 1);
    OSFM_CUDA(cudaStreamSynchronize(stream));
    const long long kept = slots[num_refs];
    d_points.reserve(std::max(kept * 3, 1LL));
    d_normals.reserve(std::max(kept * 3, 1LL));
    d_colors.reserve(std::max(kept * 3, 1LL));
    d_out_labels.reserve(std::max(kept, 1LL));
    L.points = d_points.p;
    L.normals = d_normals.p;
    L.colors = d_colors.p;
    L.out_labels = d_out_labels.p;
    dn_prune_write<<<grid, DN_THREADS, 0, stream>>>(L);
    OSFM_LAUNCH_CHECK();
    OSFM_CUDA(cudaEventRecord(ev[5], stream));
    OSFM_CUDA(cudaStreamSynchronize(stream));
    for (int r = 0; r < num_refs; ++r) counts[r] = slots[r + 1] - slots[r];
    pruned = kept;
    timed[2] = true;
  }
};

}  // namespace
}  // namespace osfm

struct osfm_dense : osfm::Handle<osfm::Dense> {
  using Handle::Handle;
  static constexpr const char* null_message = "null dense";
};

extern "C" {

int osfm_dense_create(int device, osfm_dense** out) { return osfm::create_handle(device, out); }
int osfm_dense_destroy(osfm_dense* h) { return osfm::destroy_handle(h); }

int osfm_dense_set_views(osfm_dense* h, int num_views, const int32_t* size, const double* K, const double* Kinv,
                         const double* R, const double* t, const uint8_t* gray, const uint8_t* mask,
                         const uint8_t* rgb, const uint8_t* labels) {
  return osfm::with_handle(h, [&](osfm::Dense& D) { D.set_views(num_views, size, K, Kinv, R, t, gray, mask, rgb, labels); });
}

int osfm_dense_set_maps(osfm_dense* h, int view, const float* raw_depth, const float* plane, const float* clean_depth) {
  return osfm::with_handle(h, [&](osfm::Dense& D) { D.set_maps(view, raw_depth, plane, clean_depth); });
}

int osfm_dense_estimate(osfm_dense* h, int num_refs, const int32_t* list_start, const int32_t* views, const double* Q,
                        const double* a, const int32_t* params, const double* depth_range,
                        const float* min_patch_variance, const float* weights, uint32_t seed, double min_score,
                        float* depth, float* plane, float* score, int32_t* nghbr) {
  return osfm::with_handle(h, [&](osfm::Dense& D) {
    D.estimate(num_refs, list_start, views, Q, a, params, depth_range, min_patch_variance, weights, seed, min_score,
               depth, plane, score, nghbr);
  });
}

int osfm_dense_clean(osfm_dense* h, int num_refs, const int32_t* list_start, const int32_t* views,
                     float same_depth_threshold, int min_consistent_views, float* clean_depth) {
  return osfm::with_handle(h, [&](osfm::Dense& D) {
    D.clean(num_refs, list_start, views, same_depth_threshold, min_consistent_views, clean_depth);
  });
}

int osfm_dense_prune(osfm_dense* h, int num_refs, const int32_t* list_start, const int32_t* views,
                     float same_depth_threshold, int64_t* counts) {
  return osfm::with_handle(h, [&](osfm::Dense& D) { D.prune(num_refs, list_start, views, same_depth_threshold, counts); });
}

int osfm_dense_get_pruned(osfm_dense* h, float* points, float* normals, uint8_t* colors, uint8_t* labels) {
  return osfm::with_handle(h, [&](osfm::Dense& D) {
    if (D.pruned > 0 && (!points || !normals || !colors || !labels)) throw osfm::ArgError("null outputs");
    D.download(points, D.d_points.p, (size_t)D.pruned * 3);
    D.download(normals, D.d_normals.p, (size_t)D.pruned * 3);
    D.download(colors, D.d_colors.p, (size_t)D.pruned * 3);
    D.download(labels, D.d_out_labels.p, (size_t)D.pruned);
    OSFM_CUDA(cudaStreamSynchronize(D.stream));
  });
}

int osfm_dense_last_device_ms(osfm_dense* h, float* estimate_ms, float* clean_ms, float* prune_ms) {
  return osfm::with_handle(h, [&](osfm::Dense& D) {
    if (!estimate_ms || !clean_ms || !prune_ms) throw osfm::ArgError("null ms");
    *estimate_ms = *clean_ms = *prune_ms = 0.f;
    if (D.timed[0]) OSFM_CUDA(cudaEventElapsedTime(estimate_ms, D.ev[0], D.ev[1]));
    if (D.timed[1]) OSFM_CUDA(cudaEventElapsedTime(clean_ms, D.ev[2], D.ev[3]));
    if (D.timed[2]) OSFM_CUDA(cudaEventElapsedTime(prune_ms, D.ev[4], D.ev[5]));
  });
}

}  // extern "C"
