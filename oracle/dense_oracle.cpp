// ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the shipped product.
//
// Raster-order restatement of pydense's DepthmapEstimator, DepthmapCleaner and DepthmapPruner
// (opensfm/src/dense/src/depthmap.cc), one reference shot at a time, in the reference's mixed f32 / f64 expression
// types, with plain arrays in place of cv::Mat / cv::Matx (a Matx product sums from 0 in k order; Vec3f / float
// multiplies by the f32 reciprocal; cv::normalize scales by 1 / norm in f64).  The generator is the deliberate
// difference: Philox4x32-10 keyed by (seed, key) at counter (pixel, pass, draw, attempt), with exp / log written
// from + - * / sqrt alone, so the engine draws the same variates.  Compiled with -ffp-contract=off.
//
// Differences from the reference where its behaviour is undefined: LinearInterpolation returns 0 for NaN
// coordinates, the pruner compares the int64 reprojection with the image bounds without narrowing it to int, and
// PatchMatch with patch size 1 is refused (its passes would read a pixel's neighbours outside the maps).
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

namespace {

// ---- generator ----------------------------------------------------------------------------------------------------

struct Words {
  uint32_t w[4];
};

Words philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1) {
  for (int round = 0; round < 10; ++round) {
    const uint64_t p0 = (uint64_t)0xD2511F53u * c0;
    const uint64_t p1 = (uint64_t)0xCD9E8D57u * c2;
    const uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0;
    const uint32_t n1 = (uint32_t)p1;
    const uint32_t n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1;
    const uint32_t n3 = (uint32_t)p0;
    c0 = n0, c1 = n1, c2 = n2, c3 = n3;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return Words{{c0, c1, c2, c3}};
}

double log_arith(double x) {
  uint64_t b;
  std::memcpy(&b, &x, 8);
  int e = (int)((b >> 52) & 0x7ff) - 1023;
  const uint64_t mb = (b & 0x000FFFFFFFFFFFFFull) | (1023ull << 52);
  double m;
  std::memcpy(&m, &mb, 8);
  if (m > 1.4142135623730951) {
    m = m * 0.5;
    e = e + 1;
  }
  const double s = (m - 1.0) / (m + 1.0);
  const double s2 = s * s;
  double term = s, sum = 0.0;
  for (int k = 0; k < 14; ++k) {
    sum = sum + term / (double)(2 * k + 1);
    term = term * s2;
  }
  return 2.0 * sum + (double)e * 0.6931471805599453;
}

double exp_arith(double x) {
  if (x > 700.0) return INFINITY;
  if (x < -700.0) return 0.0;
  const double q = x * 1.4426950408889634;
  const int k = (int)(q >= 0.0 ? q + 0.5 : q - 0.5);
  const double r = x - (double)k * 0.6931471805599453;
  double p = 1.0;
  for (int n = 20; n >= 1; --n) p = 1.0 + r * p / (double)n;
  const uint64_t sb = (uint64_t)(k + 1023) << 52;
  double scale;
  std::memcpy(&scale, &sb, 8);
  return p * scale;
}

float unit24(uint32_t x) { return (float)(x >> 8) * 5.9604644775390625e-8f; }
int index_in(uint32_t x, int lo, int n) { return lo + (int)(((uint64_t)x * (uint64_t)n) >> 32); }

float normal_variate(uint32_t pixel, uint32_t pass, uint32_t draw, uint32_t k0, uint32_t k1) {
  for (uint32_t attempt = 0;; ++attempt) {
    const Words r = philox4x32_10(pixel, pass, draw, attempt, k0, k1);
    const double u = (double)(int32_t)r.w[0] * 4.656612873077392578125e-10;
    const double v = (double)(int32_t)r.w[1] * 4.656612873077392578125e-10;
    const double s = u * u + v * v;
    if (s >= 1.0 || s == 0.0) continue;
    return (float)(u * std::sqrt(-2.0 * log_arith(s) / s));
  }
}

// ---- geometry -----------------------------------------------------------------------------------------------------

struct M3 {
  double v[9];
  double operator()(int i, int j) const { return v[3 * i + j]; }
};

M3 mul(const M3& A, const M3& B) {
  M3 C;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      double s = 0;
      for (int k = 0; k < 3; ++k) s += A(i, k) * B(k, j);
      C.v[3 * i + j] = s;
    }
  return C;
}

M3 load(const double* p) {
  M3 m;
  for (int k = 0; k < 9; ++k) m.v[k] = p[k];
  return m;
}

float max_ref(float a, float b) { return (a < b) ? b : a; }

// PlaneFromDepthAndNormal
void plane_from_depth_normal(float x, float y, const M3& Kinv, float depth, const float n[3], float out[3]) {
  M3 S;
  for (int k = 0; k < 9; ++k) S.v[k] = Kinv.v[k] * depth;
  const double X[3] = {x, y, 1.0};
  float p[3];
  for (int i = 0; i < 3; ++i) {
    double s = 0;
    for (int k = 0; k < 3; ++k) s += S(i, k) * X[k];
    p[i] = (float)s;
  }
  float dot = 0;
  for (int k = 0; k < 3; ++k) dot += n[k] * p[k];
  const float inv = 1.f / max_ref(1e-6f, -dot);
  for (int k = 0; k < 3; ++k) out[k] = n[k] * inv;
}

// DepthOfPlaneBackprojection
float depth_of_plane_backprojection(double x, double y, const M3& Kinv, const float pl[3]) {
  double row[3];
  for (int j = 0; j < 3; ++j) {
    double s = 0;
    for (int k = 0; k < 3; ++k) s += (double)pl[k] * Kinv(k, j);
    row[j] = s;
  }
  const double X[3] = {x, y, 1.0};
  double s = 0;
  for (int k = 0; k < 3; ++k) s += row[k] * X[k];
  const float denom = (float)(-s);
  return 1.0f / max_ref(1e-6f, denom);
}

void backproject(double x, double y, double depth, const M3& Kinv, const M3& R, const double* t, double out[3]) {
  M3 S;
  for (int k = 0; k < 9; ++k) S.v[k] = Kinv.v[k] * depth;
  const double X[3] = {x, y, 1.0};
  double q[3];
  for (int i = 0; i < 3; ++i) {
    double s = 0;
    for (int k = 0; k < 3; ++k) s += S(i, k) * X[k];
    q[i] = s - t[i];
  }
  for (int i = 0; i < 3; ++i) {
    double s = 0;
    for (int k = 0; k < 3; ++k) s += R(k, i) * q[k];
    out[i] = s;
  }
}

void project(const double X[3], const M3& K, const M3& R, const double* t, double out[3]) {
  double y[3];
  for (int i = 0; i < 3; ++i) {
    double s = 0;
    for (int k = 0; k < 3; ++k) s += R(i, k) * X[k];
    y[i] = s + t[i];
  }
  for (int i = 0; i < 3; ++i) {
    double s = 0;
    for (int k = 0; k < 3; ++k) s += K(i, k) * y[k];
    out[i] = s;
  }
}

void cv_normalize(const float v[3], float out[3]) {
  float s = 0;
  for (int k = 0; k < 3; ++k) s += v[k] * v[k];
  const double nv = std::sqrt(s);
  const double scale = nv ? 1. / nv : 0.;
  for (int k = 0; k < 3; ++k) out[k] = (float)(v[k] * scale);
}

template <class T>
float linear_interpolation(const T* im, int cols, int rows, float y, float x) {
  if (std::isnan(x) || std::isnan(y)) return 0.0f;
  if (x < 0.0f || x >= cols - 1 || y < 0.0f || y >= rows - 1) return 0.0f;
  int ix = static_cast<int>(x);
  int iy = static_cast<int>(y);
  float dx = x - ix;
  float dy = y - iy;
  float im00 = im[iy * cols + ix];
  float im01 = im[iy * cols + ix + 1];
  float im10 = im[(iy + 1) * cols + ix];
  float im11 = im[(iy + 1) * cols + ix + 1];
  float im0 = (1 - dx) * im00 + dx * im01;
  float im1 = (1 - dx) * im10 + dx * im11;
  return (1 - dy) * im0 + dy * im1;
}

struct NCC {
  float sx = 0, sy = 0, sxx = 0, syy = 0, sxy = 0, sw = 0;
  void push(float x, float y, float w) {
    sx += w * x;
    sy += w * y;
    sxx += w * x * x;
    syy += w * y * y;
    sxy += w * x * y;
    sw += w;
  }
  float get() const {
    if (sw == 0.0) return -1;
    float mx = sx / sw, my = sy / sw, mxx = sxx / sw, myy = syy / sw, mxy = sxy / sw;
    float varx = mxx - mx * mx, vary = myy - my * my;
    if (varx < 0.1 || vary < 0.1) return -1;
    return (mxy - mx * my) / std::sqrt(varx * vary);
  }
};

// PlaneInducedHomographyBaked: K2 (Q + a v^T) K1^-1 in fp64, rounded to f32
void baked_homography(const M3& K1inv, const M3& Q, const double* a, const M3& K2, const float pl[3], float H[9]) {
  M3 M;
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) M.v[3 * r + c] = Q(r, c) + a[r] * (double)pl[c];
  const M3 Hd = mul(mul(K2, M), K1inv);
  for (int k = 0; k < 9; ++k) H[k] = (float)Hd.v[k];
}

constexpr int MAX_HPZ = 7;
constexpr int WD = 2 * MAX_HPZ * MAX_HPZ + 1;

// ---- estimator ----------------------------------------------------------------------------------------------------

struct Estimator {
  int n;                           // views, reference first
  std::vector<int> W, H;
  std::vector<const uint8_t*> img;
  const uint8_t* mask;
  std::vector<M3> K, Q;
  M3 Kinv0;
  std::vector<const double*> a;
  int hpz, planes, iterations, method;
  float min_var;
  double dmin, dmax;
  const float* weights;
  uint32_t seed, key;
  // result
  float *depth, *plane, *score;
  int* nghbr;

  float image_score(int i, int j, const float pl[3], int other) const {
    float Hf[9];
    baked_homography(Kinv0, Q[other], a[other], K[other], pl, Hf);
    const float u = Hf[0] * j + Hf[1] * i + Hf[2];
    const float v = Hf[3] * j + Hf[4] * i + Hf[5];
    const float w = Hf[6] * j + Hf[7] * i + Hf[8];
    if (w == 0.0) return -1.0f;
    const float dfdx_x = (Hf[0] * w - Hf[6] * u) / (w * w);
    const float dfdx_y = (Hf[3] * w - Hf[6] * v) / (w * w);
    const float dfdy_x = (Hf[1] * w - Hf[7] * u) / (w * w);
    const float dfdy_y = (Hf[4] * w - Hf[7] * v) / (w * w);
    const float Hx0 = u / w, Hy0 = v / w;
    const int cols = W[0];
    const float center = img[0][i * cols + j];
    NCC ncc;
    for (int dy = -hpz; dy <= hpz; ++dy)
      for (int dx = -hpz; dx <= hpz; ++dx) {
        const float im1 = img[0][(i + dy) * cols + j + dx];
        const float x2 = Hx0 + dfdx_x * dx + dfdy_x * dy;
        const float y2 = Hy0 + dfdx_y * dx + dfdy_y * dy;
        const float im2 = linear_interpolation(img[other], W[other], H[other], y2, x2);
        const float dcolor = im1 - center;
        const float weight = weights[(int)std::fabs(dcolor) * WD + dx * dx + dy * dy];
        ncc.push(im1, im2, weight);
      }
    return ncc.get();
  }

  void plane_score(int i, int j, const float pl[3], float* s, int* nb) const {
    *s = -1.0f;
    *nb = 0;
    for (int other = 1; other < n; ++other) {
      const float t = image_score(i, j, pl, other);
      if (t > *s) {
        *s = t;
        *nb = other;
      }
    }
  }

  int at(int i, int j) const { return i * W[0] + j; }

  void assign(int i, int j, float d, const float pl[3], float s, int nb) {
    const int p = at(i, j);
    depth[p] = d;
    for (int k = 0; k < 3; ++k) plane[3 * p + k] = pl[k];
    score[p] = s;
    nghbr[p] = nb;
  }

  void check(int i, int j, const float pl[3], int view) {
    float s;
    int nb = view;
    if (view < 0)
      plane_score(i, j, pl, &s, &nb);
    else
      s = image_score(i, j, pl, view);
    if (s > score[at(i, j)]) assign(i, j, depth_of_plane_backprojection(j, i, Kinv0, pl), pl, s, nb);
  }

  void brute_force() {
    const float normal[3] = {0, 0, -1};
    for (int i = hpz; i < H[0] - hpz; ++i)
      for (int j = hpz; j < W[0] - hpz; ++j)
        for (int d = 0; d < planes; ++d) {
          float dep;
          if (planes <= 1)
            dep = dmin;
          else
            dep = 1 / (1 / dmin + d * (1 / dmax - 1 / dmin) / (planes - 1));
          float pl[3];
          plane_from_depth_normal(j, i, Kinv0, dep, normal, pl);
          check(i, j, pl, -1);
        }
  }

  float patch_variance(int i, int j) const {
    std::vector<float> patch;
    for (int u = -hpz; u <= hpz; ++u)
      for (int v = -hpz; v <= hpz; ++v) patch.push_back(img[0][(i + u) * W[0] + j + v]);
    const int cnt = (int)patch.size();
    float sum = 0;
    for (int k = 0; k < cnt; ++k) sum += patch[k];
    const float mean = sum / cnt;
    float sum2 = 0;
    for (int k = 0; k < cnt; ++k) sum2 += (patch[k] - mean) * (patch[k] - mean);
    return sum2 / cnt;
  }

  uint32_t pix(int i, int j) const { return (uint32_t)i * (uint32_t)W[0] + (uint32_t)j; }

  void random_initialization(bool sample) {
    const float la = (float)log_arith(dmin), lb = (float)log_arith(dmax);
    for (int i = hpz; i < H[0] - hpz; ++i)
      for (int j = hpz; j < W[0] - hpz; ++j) {
        const Words x = philox4x32_10(pix(i, j), 0, 0, 0, seed, key);
        const float dep = (float)exp_arith(la + (lb - la) * unit24(x.w[0]));
        const float normal[3] = {-1.f + 2.f * unit24(x.w[1]), -1.f + 2.f * unit24(x.w[2]), -1.f};
        float pl[3];
        plane_from_depth_normal(j, i, Kinv0, dep, normal, pl);
        int nb;
        float s;
        if (sample) {
          nb = index_in(x.w[3], 1, n - 1);
          s = image_score(i, j, pl, nb);
        } else {
          plane_score(i, j, pl, &s, &nb);
        }
        assign(i, j, dep, pl, s, nb);
      }
  }

  void ignore_mask() {
    const float zero[3] = {0, 0, 0};
    for (int i = hpz; i < H[0] - hpz; ++i)
      for (int j = hpz; j < W[0] - hpz; ++j)
        if (mask[at(i, j)] == 0 || patch_variance(i, j) < min_var) assign(i, j, 0.0f, zero, 0.0f, 0);
  }

  void update_pixel(int i, int j, const int adjacent[2][2], bool sample, uint32_t pass) {
    if (depth[at(i, j)] == 0.0f) return;
    for (int k = 0; k < 2; ++k) {
      const int ia = i + adjacent[k][0], ja = j + adjacent[k][1];
      if (depth[at(ia, ja)] == 0.0f) continue;
      const float* pa = plane + 3 * at(ia, ja);
      const float pl[3] = {pa[0], pa[1], pa[2]};
      check(i, j, pl, sample ? nghbr[at(ia, ja)] : -1);
    }
    float depth_range = 0.02;
    float normal_range = 0.5;
    const int current = nghbr[at(i, j)];
    for (int k = 0; k < 6; ++k) {
      const float cur_depth = depth[at(i, j)];
      const float dep = cur_depth * (float)exp_arith(depth_range * normal_variate(pix(i, j), pass, 1 + 3 * k, seed, key));
      const float* cp = plane + 3 * at(i, j);
      if (cp[2] == 0.0) continue;
      const float n0 = normal_variate(pix(i, j), pass, 1 + 3 * k + 1, seed, key);
      const float n1 = normal_variate(pix(i, j), pass, 1 + 3 * k + 2, seed, key);
      const float normal[3] = {-cp[0] / cp[2] + normal_range * n0, -cp[1] / cp[2] + normal_range * n1, -1.0f};
      float pl[3];
      plane_from_depth_normal(j, i, Kinv0, dep, normal, pl);
      check(i, j, pl, sample ? current : -1);
      depth_range *= 0.3;
      normal_range *= 0.8;
    }
    if (!sample || n <= 2) return;
    int other = current;
    for (uint32_t attempt = 0; other == current; ++attempt)
      other = index_in(philox4x32_10(pix(i, j), pass, 32, attempt / 4, seed, key).w[attempt % 4], 1, n - 1);
    const float* cp = plane + 3 * at(i, j);
    const float pl[3] = {cp[0], cp[1], cp[2]};
    check(i, j, pl, other);
  }

  void post_process();

  void patch_match(bool sample) {
    random_initialization(sample);
    ignore_mask();
    const int fwd[2][2] = {{-1, 0}, {0, -1}}, bwd[2][2] = {{0, 1}, {1, 0}};
    for (int it = 0; it < iterations; ++it) {
      for (int i = hpz; i < H[0] - hpz; ++i)
        for (int j = hpz; j < W[0] - hpz; ++j) update_pixel(i, j, fwd, sample, 1 + 2 * it);
      for (int i = H[0] - hpz - 1; i >= hpz; --i)
        for (int j = W[0] - hpz - 1; j >= hpz; --j) update_pixel(i, j, bwd, sample, 2 + 2 * it);
    }
    post_process();
  }
};

// cv::medianBlur(src, dst, 5) for f32, borders replicated
void median5(const float* src, int w, int h, float* dst) {
  for (int i = 0; i < h; ++i)
    for (int j = 0; j < w; ++j) {
      float v[25];
      int c = 0;
      for (int di = -2; di <= 2; ++di)
        for (int dj = -2; dj <= 2; ++dj) {
          int ii = i + di < 0 ? 0 : (i + di >= h ? h - 1 : i + di);
          int jj = j + dj < 0 ? 0 : (j + dj >= w ? w - 1 : j + dj);
          v[c++] = src[ii * w + jj];
        }
      // insertion sort, then the middle element
      for (int a = 1; a < 25; ++a) {
        const float t = v[a];
        int b = a - 1;
        while (b >= 0 && v[b] > t) {
          v[b + 1] = v[b];
          --b;
        }
        v[b + 1] = t;
      }
      dst[i * w + j] = v[12];
    }
}

void Estimator::post_process() {
  const int w = W[0], h = H[0];
  std::vector<float> filtered(w * h);
  median5(depth, w, h, filtered.data());
  for (int p = 0; p < w * h; ++p) {
    const float d = depth[p], m = filtered[p];
    if (d == 0.0 || std::fabs(d - m) / d > 0.05) depth[p] = 0;
  }
}

}  // namespace

extern "C" {

// One reference: views 0..n-1 (reference first), images and sizes per view, mask of the reference, K / Q / a per
// view, K^-1 of the reference.  method 0 brute force, 1 PatchMatch, 2 PatchMatch-sample.  Outputs of the reference's
// size, zero-initialised by the callee (AssignMatrices).  Returns 0, or -1 without touching the outputs for PatchMatch
// with patch size 1.
int dn_estimate(int n, const int* size, const uint8_t* const* images, const uint8_t* mask, const double* K,
                 const double* Kinv0, const double* Q, const double* a, int method, int patch, int planes,
                 int iterations, float min_var, double dmin, double dmax, const float* weights, uint32_t seed,
                 uint32_t key, float* depth, float* plane, float* score, int* nghbr) {
  if (patch == 1 && method != 0) return -1;
  Estimator E;
  E.n = n;
  for (int v = 0; v < n; ++v) {
    E.W.push_back(size[2 * v]);
    E.H.push_back(size[2 * v + 1]);
    E.img.push_back(images[v]);
    E.K.push_back(load(K + 9 * v));
    E.Q.push_back(load(Q + 9 * v));
    E.a.push_back(a + 3 * v);
  }
  E.mask = mask;
  E.Kinv0 = load(Kinv0);
  E.hpz = (patch - 1) / 2;
  E.planes = planes;
  E.iterations = iterations;
  E.method = method;
  E.min_var = min_var;
  E.dmin = dmin;
  E.dmax = dmax;
  E.weights = weights;
  E.seed = seed;
  E.key = key;
  const int np = size[0] * size[1];
  std::fill(depth, depth + np, 0.f);
  std::fill(plane, plane + 3 * np, 0.f);
  std::fill(score, score + np, 0.f);
  std::fill(nghbr, nghbr + np, 0);
  E.depth = depth;
  E.plane = plane;
  E.score = score;
  E.nghbr = nghbr;
  if (method == 0)
    E.brute_force();
  else
    E.patch_match(method == 2);
  return 0;
}

// DepthmapCleaner::Clean of view 0 against views 1..n-1
void dn_clean(int n, const int* size, const float* const* depths, const double* K, const double* Kinv,
              const double* R, const double* t, float threshold, int min_consistent, float* out) {
  const int w = size[0], h = size[1];
  const M3 Kinv0 = load(Kinv), R0 = load(R);
  for (int i = 0; i < h; ++i)
    for (int j = 0; j < w; ++j) {
      const float d = depths[0][i * w + j];
      double Xd[3];
      backproject(j, i, d, Kinv0, R0, t, Xd);
      const double X[3] = {(float)Xd[0], (float)Xd[1], (float)Xd[2]};
      int consistent = 1;
      for (int o = 1; o < n; ++o) {
        double rd[3];
        project(X, load(K + 9 * o), load(R + 9 * o), t + 3 * o, rd);
        const float r[3] = {(float)rd[0], (float)rd[1], (float)rd[2]};
        if (r[2] < 1e-8 || std::isnan(r[2])) continue;
        const float u = r[0] / r[2], v = r[1] / r[2], dp = r[2];
        const float da = linear_interpolation(depths[o], size[2 * o], size[2 * o + 1], v, u);
        if (std::fabs(da - dp) < dp * threshold) consistent++;
      }
      out[i * w + j] = consistent >= min_consistent ? d : 0;
    }
}

// DepthmapPruner::Prune of view 0 against views 1..n-1; outputs sized for every pixel of view 0; returns the count
long long dn_prune(int n, const int* size, const float* const* depths, const float* const* planes,
                   const uint8_t* rgb0, const uint8_t* labels0, const double* K, const double* Kinv,
                   const double* R, const double* t, float threshold, float* points, float* normals,
                   uint8_t* colors, uint8_t* labels) {
  const int w = size[0], h = size[1];
  const M3 Kinv0 = load(Kinv), R0 = load(R);
  float Rinv[9];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) Rinv[3 * r + c] = (float)R0(c, r);
  long long count = 0;
  for (int i = 0; i < h; ++i)
    for (int j = 0; j < w; ++j) {
      const float d = depths[0][i * w + j];
      if (d <= 0) continue;
      float nrm[3];
      cv_normalize(planes[0] + 3 * (i * w + j), nrm);
      const float area = -nrm[2] / d * K[0];
      double Xd[3];
      backproject(j, i, d, Kinv0, R0, t, Xd);
      const float Xf[3] = {(float)Xd[0], (float)Xd[1], (float)Xd[2]};
      const double X[3] = {Xf[0], Xf[1], Xf[2]};
      bool keep = true;
      for (int o = 1; o < n; ++o) {
        double r[3];
        project(X, load(K + 9 * o), load(R + 9 * o), t + 3 * o, r);
        if (r[2] < 1e-8 || std::isnan(r[2])) continue;
        const int64_t iu = static_cast<int64_t>(r[0] / r[2] + 0.5);
        const int64_t iv = static_cast<int64_t>(r[1] / r[2] + 0.5);
        const double dp = r[2];
        if (!(iv >= 0 && iv < size[2 * o + 1] && iu >= 0 && iu < size[2 * o])) continue;
        const int64_t q = iv * size[2 * o] + iu;
        const float da = depths[o][q];
        if (da > (1 - threshold) * dp) {
          float no[3];
          cv_normalize(planes[o] + 3 * q, no);
          if ((da == 0.0) || (-no[2] / da * K[9 * o] > area)) {
            keep = false;
            break;
          }
        }
      }
      if (!keep) continue;
      for (int k = 0; k < 3; ++k) {
        float s = 0;
        for (int m = 0; m < 3; ++m) s += Rinv[3 * k + m] * nrm[m];
        points[3 * count + k] = Xf[k];
        normals[3 * count + k] = s;
        colors[3 * count + k] = rgb0[3 * (i * w + j) + k];
      }
      labels[count] = labels0[i * w + j];
      ++count;
    }
  return count;
}

void dn_median5(const float* src, int w, int h, float* dst) { median5(src, w, h, dst); }

void dn_homography(const double* K1inv, const double* Q, const double* a, const double* K2, const float* plane,
                   float* H) {
  baked_homography(load(K1inv), load(Q), a, load(K2), plane, H);
}

// pieces the reference's depthmap_test.cc exercises
void dn_plane_from_depth_normal(float x, float y, const double* Kinv, float depth, const float* normal, float* out) {
  plane_from_depth_normal(x, y, load(Kinv), depth, normal, out);
}
float dn_depth_of_plane(double x, double y, const double* Kinv, const float* plane) {
  return depth_of_plane_backprojection(x, y, load(Kinv), plane);
}
void dn_backproject(double x, double y, double depth, const double* Kinv, const double* R, const double* t,
                    double* out) {
  backproject(x, y, depth, load(Kinv), load(R), t, out);
}
void dn_project(const double* X, const double* K, const double* R, const double* t, double* out) {
  project(X, load(K), load(R), t, out);
}
float dn_ncc(int n, const float* x, const float* y, const float* w) {
  NCC ncc;
  for (int k = 0; k < n; ++k) ncc.push(x[k], y[k], w[k]);
  return ncc.get();
}
double dn_log(double x) { return log_arith(x); }
double dn_exp(double x) { return exp_arith(x); }
float dn_normal(uint32_t pixel, uint32_t pass, uint32_t draw, uint32_t k0, uint32_t k1) {
  return normal_variate(pixel, pass, draw, k0, k1);
}
void dn_philox(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1, uint32_t* out) {
  const Words r = philox4x32_10(c0, c1, c2, c3, k0, k1);
  for (int k = 0; k < 4; ++k) out[k] = r.w[k];
}

}  // extern "C"
