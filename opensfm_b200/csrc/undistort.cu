// UNDISTORT: undistorted images, masks and segmentations of many shots per call, and the six perspective faces of
// a panorama.
//
// Replaces opensfm/undistort.py:166-232,360-403: pygeometry.compute_camera_mapping (ComputeCameraMapping,
// geometry/src/camera.cc:319-342), cv2.remap over its maps, render_perspective_view_of_a_panorama's face
// coordinates and the INTER_NEAREST resize of scale_image.  The restatement every rule is checked against is
// oracle/undistort_oracle.py.
//
// Layout: a job is one source image (u8 or u16, 1, 3 or 4 interleaved channels, row-major) and one output.  Its
// remap grid is the image the reference remaps into (the source's size for a camera, face_size^2 for a panorama
// face); its output is that grid after scale_image.  Kernels:
//   ud_sample   one thread per output pixel: the grid pixel cv2.resize(INTER_NEAREST) keeps there, its source
//               coordinate (ud_coord, fp64 rounded to f32 as the reference stores it), then cv2.remap's sampler
//   ud_maps     one thread per grid pixel: ud_coord into f32 maps, for tests and callers that remap themselves
// No map is materialised on the product path.  Jobs go through two page-locked staging slots on two streams, so one
// job's copies overlap the other's kernel; device memory is bounded by the two largest jobs in flight.
// This file is compiled with -fmad=false: the sampler's u16 sums and the mappings' products stay unfused.
#include <climits>
#include <cmath>

#include "ba_models.cuh"
#include "common.cuh"

namespace osfm {
namespace {

constexpr int UD_THREADS = 256;
constexpr int UD_SLOTS = 2;
constexpr int UD_CAMERA = OSFM_UNDISTORT_CAMERA, UD_FACE = OSFM_UNDISTORT_FACE, UD_MAPS = 2;
constexpr int UD_MAX_SIZE = 32766;   // cv2 saturates coordinates to int16 and refuses images this wide or wider

// Where the grid pixels of a job sample the source.
struct UMapping {
  int kind;                   // UD_CAMERA, UD_FACE or UD_MAPS
  int type;                   // camera: the source camera's projection type
  int gw, gh;                 // the remap grid
  int sw, sh;                 // the source image
  double p[OSFM_UNDISTORT_PARAMS];   // camera: values, p[12] the target focal; face: R_pano R_face^T row-major
  const float* mx;            // UD_MAPS: caller maps, gw x gh each
  const float* my;
};

struct UJob {
  UMapping m;
  int ch, bytes, interp, border;
  int ow, oh;                 // output; grid index of output pixel o = min(floor(o * ifx), g - 1)
  double ifx, ify;
  const void* src;
  void* dst;
};

// ---- mappings -----------------------------------------------------------------------------------------------------

// ComputeCameraMapping at grid pixel (u, v): to.Bearing(uv / max(w, h)) of the perspective target (UniformScale,
// Disto24 at k1 = k2 = 0, which is the identity, then (x, y, 1) / sqrt(x^2 + y^2 + 1)), from.Project of that
// bearing, times max(w, h), plus half the size.
__device__ float2 camera_coord(const UMapping& m, int u, int v) {
  const int n = max(m.gw, m.gh);
  const double inv = 1.0 / n;
  const double hw = m.gw * 0.5, hh = m.gh * 0.5;
  const double a = (inv * (u - hw)) / m.p[12], b = (inv * (v - hh)) / m.p[12];
  const double inv_norm = 1.0 / sqrt((a * a + b * b) + 1.0);
  const double bearing[3] = {a * inv_norm, b * inv_norm, inv_norm};
  double px[2];
  camera_project(m.type, m.p, bearing, px, nullptr, nullptr);
  return make_float2((float)(n * px[0] + hw), (float)(n * px[1] + hh));
}

// SphericalProjection::Forward (camera_projections_functions.h:216-223).
__device__ void spherical_project(const double* x, double* out) {
  const double inv = 1.0 / (2.0 * M_PI);
  const double lon = atan2(x[0], x[2]);
  const double lat = atan2(-x[1], sqrt(x[0] * x[0] + x[2] * x[2]));
  out[0] = lon * inv;
  out[1] = -lat * inv;
}

// render_perspective_view_of_a_panorama at face pixel (u, v): normalized_image_coordinates (in float32, as numpy
// evaluates it on the float32 pixel grid), the bearing of the focal-0.5 perspective face camera, rotated by
// R_pano R_face^T, the spherical projection and denormalized_image_coordinates in the panorama image.
__device__ float2 face_coord(const UMapping& m, int u, int v) {
  const int s = m.gw;
  const float fs = (float)s;
  const double a = (double)__fdiv_rn((float)(u + 0.5 - s / 2.0), fs) / 0.5;
  const double b = (double)__fdiv_rn((float)(v + 0.5 - s / 2.0), fs) / 0.5;
  const double inv_norm = 1.0 / sqrt((a * a + b * b) + 1.0);
  const double d[3] = {a * inv_norm, b * inv_norm, inv_norm};
  const double* R = m.p;
  double r[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) r[i] = (d[0] * R[3 * i] + d[1] * R[3 * i + 1]) + d[2] * R[3 * i + 2];
  double q[2];
  spherical_project(r, q);
  const int size = max(m.sw, m.sh);
  return make_float2((float)(q[0] * size - 0.5 + m.sw / 2.0), (float)(q[1] * size - 0.5 + m.sh / 2.0));
}

// The source coordinate of grid pixel (u, v): the one function behind both the sampler and the maps entry points.
__device__ __forceinline__ float2 ud_coord(const UMapping& m, int u, int v) {
  if (m.kind == UD_CAMERA) return camera_coord(m, u, v);
  if (m.kind == UD_FACE) return face_coord(m, u, v);
  const long long i = (long long)v * m.gw + u;
  return make_float2(m.mx[i], m.my[i]);
}

// ---- cv2.remap's sampler ------------------------------------------------------------------------------------------

// cvRound of a float on x86: half to even; NaN and results outside int32 give INT_MIN (cvtss2si's indefinite value).
__device__ __forceinline__ int cv_round(float v) {
  const float r = rintf(v);
  if (!(r >= -2147483648.f && r < 2147483648.f)) return INT_MIN;
  return (int)r;
}
__device__ __forceinline__ int sat16(int v) { return min(max(v, -32768), 32767); }

// The pixel at integer (x, y) under the border rule, or null for a constant-0 border tap.
template <class T, int C>
__device__ __forceinline__ const T* tap(const T* src, int w, int h, int border, int x, int y) {
  if (x < 0 || x >= w || y < 0 || y >= h) {
    if (border != OSFM_UNDISTORT_BORDER_WRAP) return nullptr;
    x %= w;
    if (x < 0) x += w;
    y %= h;
    if (y < 0) y += h;
  }
  return src + ((long long)y * w + x) * C;
}

template <class T, int C>
__device__ void sample(const UJob& J, float2 c, T* out) {
  const T* src = (const T*)J.src;
  const int w = J.m.sw, h = J.m.sh;
  if (J.interp == OSFM_UNDISTORT_NEAREST) {
    const T* p = tap<T, C>(src, w, h, J.border, sat16(cv_round(c.x)), sat16(cv_round(c.y)));
#pragma unroll
    for (int k = 0; k < C; ++k) out[k] = p ? p[k] : T(0);
    return;
  }
  // INTER_LINEAR: 5 fractional bits (INTER_TAB_SIZE 32), taps (X >> 5, Y >> 5) and their +1 neighbours
  const int X = cv_round(__fmul_rn(c.x, 32.f)), Y = cv_round(__fmul_rn(c.y, 32.f));
  const int fx = X & 31, fy = Y & 31;
  const int sx = sat16(X >> 5), sy = sat16(Y >> 5);
  const T* p[4] = {tap<T, C>(src, w, h, J.border, sx, sy), tap<T, C>(src, w, h, J.border, sx + 1, sy),
                   tap<T, C>(src, w, h, J.border, sx, sy + 1), tap<T, C>(src, w, h, J.border, sx + 1, sy + 1)};
  if (sizeof(T) == 1) {
    // 8 bit: weights 32768 wy wx (exact integers), (sum + 2^14) >> 15, saturated
    const int wt[4] = {(32 - fx) * (32 - fy) * 32, fx * (32 - fy) * 32, (32 - fx) * fy * 32, fx * fy * 32};
#pragma unroll
    for (int k = 0; k < C; ++k) {
      int acc = 0;
#pragma unroll
      for (int t = 0; t < 4; ++t) acc += (p[t] ? (int)p[t][k] : 0) * wt[t];
      out[k] = (T)min(max((acc + (1 << 14)) >> 15, 0), 255);
    }
  } else {
    // 16 bit: float weights wy wx, each product rounded, summed left to right, rounded half to even
    const float tx0 = 1.f - fx * (1.f / 32), tx1 = fx * (1.f / 32), ty0 = 1.f - fy * (1.f / 32), ty1 = fy * (1.f / 32);
    const float wt[4] = {__fmul_rn(ty0, tx0), __fmul_rn(ty0, tx1), __fmul_rn(ty1, tx0), __fmul_rn(ty1, tx1)};
#pragma unroll
    for (int k = 0; k < C; ++k) {
      float acc = __fmul_rn(p[0] ? (float)p[0][k] : 0.f, wt[0]);
#pragma unroll
      for (int t = 1; t < 4; ++t) acc = __fadd_rn(acc, __fmul_rn(p[t] ? (float)p[t][k] : 0.f, wt[t]));
      out[k] = (T)min(max((int)rintf(acc), 0), 65535);
    }
  }
}

template <class T, int C>
__global__ void __launch_bounds__(UD_THREADS) ud_sample(const UJob J) {
  const long long n = (long long)J.ow * J.oh;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int ox = (int)(i % J.ow), oy = (int)(i / J.ow);
    const int u = min((int)floor(ox * J.ifx), J.m.gw - 1);
    const int v = min((int)floor(oy * J.ify), J.m.gh - 1);
    T px[C];
    sample<T, C>(J, ud_coord(J.m, u, v), px);
    T* o = (T*)J.dst + i * C;
#pragma unroll
    for (int k = 0; k < C; ++k) o[k] = px[k];
  }
}

__global__ void __launch_bounds__(UD_THREADS) ud_maps(const UMapping m, float* mx, float* my) {
  const long long n = (long long)m.gw * m.gh;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float2 c = ud_coord(m, (int)(i % m.gw), (int)(i / m.gw));
    mx[i] = c.x;
    my[i] = c.y;
  }
}

unsigned grid_of(long long n) { return (unsigned)std::min<long long>((n + UD_THREADS - 1) / UD_THREADS, 1LL << 20); }

void launch_sample(const UJob& J, cudaStream_t st) {
  const unsigned g = grid_of((long long)J.ow * J.oh);
  const int key = J.bytes * 10 + J.ch;
  switch (key) {
    case 11: ud_sample<uint8_t, 1><<<g, UD_THREADS, 0, st>>>(J); break;
    case 13: ud_sample<uint8_t, 3><<<g, UD_THREADS, 0, st>>>(J); break;
    case 14: ud_sample<uint8_t, 4><<<g, UD_THREADS, 0, st>>>(J); break;
    case 21: ud_sample<uint16_t, 1><<<g, UD_THREADS, 0, st>>>(J); break;
    case 23: ud_sample<uint16_t, 3><<<g, UD_THREADS, 0, st>>>(J); break;
    case 24: ud_sample<uint16_t, 4><<<g, UD_THREADS, 0, st>>>(J); break;
    default: throw ArgError("undistort: no sampler for " + std::to_string(J.bytes) + "-byte samples with " +
                            std::to_string(J.ch) + " channels");
  }
  OSFM_LAUNCH_CHECK();
}

// ---- argument checks ----------------------------------------------------------------------------------------------

bool undistortable(int type) {
  return type == PT_PERSPECTIVE || type == PT_BROWN || type == PT_FISHEYE || type == PT_FISHEYE_OPENCV ||
         type == PT_FISHEYE62;
}

void check_image(const std::string& who, int w, int h, int ch, int bytes) {
  if (w < 1 || h < 1) throw ArgError(who + ": empty image " + std::to_string(w) + "x" + std::to_string(h));
  if (w > UD_MAX_SIZE || h > UD_MAX_SIZE)
    throw ArgError(who + ": image " + std::to_string(w) + "x" + std::to_string(h) + " exceeds " +
                   std::to_string(UD_MAX_SIZE) + " pixels a side");
  if (ch != 1 && ch != 3 && ch != 4) throw ArgError(who + ": " + std::to_string(ch) + " channels; 1, 3 or 4 are supported");
  if (bytes != 1 && bytes != 2)
    throw ArgError(who + ": " + std::to_string(bytes) + "-byte samples; uint8 and uint16 are supported");
}

void check_sampling(const std::string& who, int interp, int border) {
  if (interp != OSFM_UNDISTORT_NEAREST && interp != OSFM_UNDISTORT_LINEAR)
    throw ArgError(who + ": interpolation " + std::to_string(interp) + "; NEAREST and LINEAR are supported");
  if (border != OSFM_UNDISTORT_BORDER_CONSTANT && border != OSFM_UNDISTORT_BORDER_WRAP)
    throw ArgError(who + ": border " + std::to_string(border) + "; CONSTANT and WRAP are supported");
}

// The mapping of a camera or face job, checked.
UMapping mapping_of(const std::string& who, int kind, int type, const double* params, int gw, int gh, int sw, int sh) {
  if (!params) throw ArgError(who + ": null parameters");
  UMapping m{};
  m.kind = kind;
  m.type = type;
  m.gw = gw;
  m.gh = gh;
  m.sw = sw;
  m.sh = sh;
  std::copy(params, params + OSFM_UNDISTORT_PARAMS, m.p);
  if (gw < 1 || gh < 1) throw ArgError(who + ": empty remap grid");
  if (kind == UD_CAMERA) {
    if (!undistortable(type))
      throw ArgError(who + ": projection type " + std::to_string(type) +
                     " cannot be undistorted (perspective, brown, fisheye, fisheye_opencv and fisheye62 can)");
    if (gw != sw || gh != sh) throw ArgError(who + ": a camera's remap grid is its image");
    if (!(m.p[12] > 0.0) || !std::isfinite(m.p[12])) throw ArgError(who + ": the target focal must be positive");
  } else if (kind == UD_FACE) {
    if (gw != gh) throw ArgError(who + ": a panorama face is square");
  } else {
    throw ArgError(who + ": unknown mapping kind " + std::to_string(kind));
  }
  return m;
}

// ---- the engine ---------------------------------------------------------------------------------------------------

// One staging slot: a stream, page-locked and device buffers for one job's source and output, and its events
// (before the upload, after it, after the kernel, after the download).
struct Slot {
  cudaStream_t st = nullptr;
  cudaEvent_t ev[4] = {};
  PinnedBuf<uint8_t> h_src, h_dst;
  DevBuf<uint8_t> d_src, d_dst;
  int job = -1;
  void* user_dst = nullptr;
  size_t dst_bytes = 0;
};

struct Undistort : DeviceStream<2> {
  Slot slots[UD_SLOTS];
  DevBuf<float> d_mx, d_my;
  float ms[3] = {0.f, 0.f, 0.f};   // the last call's upload, kernel and download time

  explicit Undistort(int dev) : DeviceStream<2>(dev) {
    for (Slot& s : slots) {
      OSFM_CUDA(cudaStreamCreateWithFlags(&s.st, cudaStreamNonBlocking));
      for (auto& e : s.ev) OSFM_CUDA(cudaEventCreate(&e));
    }
  }
  ~Undistort() {
    for (Slot& s : slots) {
      for (auto& e : s.ev)
        if (e) cudaEventDestroy(e);
      if (s.st) cudaStreamDestroy(s.st);
    }
  }

  // fails naming the bytes when `bytes` more device memory than is free are needed
  static void fits(const std::string& what, long long bytes) {
    size_t free_b = 0, total_b = 0;
    OSFM_CUDA(cudaMemGetInfo(&free_b, &total_b));
    if (bytes > 0 && (size_t)bytes > free_b)
      throw std::runtime_error("undistort: " + what + " need " + std::to_string(bytes) + " bytes of device memory, " +
                               std::to_string(free_b) + " are free");
  }

  // waits for the slot's job, hands its output to the caller and adds its times
  void finish(Slot& s) {
    if (s.job < 0) return;
    OSFM_CUDA(cudaStreamSynchronize(s.st));
    std::memcpy(s.user_dst, s.h_dst.p, s.dst_bytes);
    float t;
    for (int k = 0; k < 3; ++k) {
      OSFM_CUDA(cudaEventElapsedTime(&t, s.ev[k], s.ev[k + 1]));
      ms[k] += t;
    }
    s.job = -1;
  }

  // stages job j's source into slot s, samples and downloads its output
  void submit(Slot& s, int j, const UJob& job, size_t src_bytes, size_t dst_bytes) {
    s.h_src.reserve(src_bytes);
    s.h_dst.reserve(dst_bytes);
    s.d_src.reserve(src_bytes);
    s.d_dst.reserve(dst_bytes);
    std::memcpy(s.h_src.p, job.src, src_bytes);
    UJob J = job;
    J.src = s.d_src.p;
    J.dst = s.d_dst.p;
    OSFM_CUDA(cudaEventRecord(s.ev[0], s.st));
    OSFM_CUDA(cudaMemcpyAsync(s.d_src.p, s.h_src.p, src_bytes, cudaMemcpyHostToDevice, s.st));
    OSFM_CUDA(cudaEventRecord(s.ev[1], s.st));
    launch_sample(J, s.st);
    OSFM_CUDA(cudaEventRecord(s.ev[2], s.st));
    OSFM_CUDA(cudaMemcpyAsync(s.h_dst.p, s.d_dst.p, dst_bytes, cudaMemcpyDeviceToHost, s.st));
    OSFM_CUDA(cudaEventRecord(s.ev[3], s.st));
    s.job = j;
    s.user_dst = job.dst;
    s.dst_bytes = dst_bytes;
  }

  // runs the jobs through the staging slots, in order; on failure every job in flight is drained first
  void run_jobs(const std::vector<UJob>& jobs) {
    ms[0] = ms[1] = ms[2] = 0.f;
    // device memory: every slot grows to the largest job it may hold
    size_t need = 0, have = 0;
    for (const Slot& s : slots) have += s.d_src.cap + s.d_dst.cap;
    for (const UJob& J : jobs) {
      const size_t b = (size_t)J.m.sw * J.m.sh * J.ch * J.bytes + (size_t)J.ow * J.oh * J.ch * J.bytes;
      need = std::max(need, b);
    }
    need *= std::min<size_t>(jobs.size(), UD_SLOTS);
    if (need > have) fits("the largest images in flight", (long long)(need - have));
    try {
      for (size_t j = 0; j < jobs.size(); ++j) {
        Slot& s = slots[j % UD_SLOTS];
        finish(s);
        const UJob& J = jobs[j];
        submit(s, (int)j, J, (size_t)J.m.sw * J.m.sh * J.ch * J.bytes, (size_t)J.ow * J.oh * J.ch * J.bytes);
      }
      for (size_t j = jobs.size() > UD_SLOTS ? jobs.size() - UD_SLOTS : 0; j < jobs.size(); ++j)
        finish(slots[j % UD_SLOTS]);
    } catch (...) {
      for (Slot& s : slots) {
        cudaStreamSynchronize(s.st);
        s.job = -1;
      }
      throw;
    }
  }

  void run(int num_jobs, const int32_t* desc, const double* params, const void* const* src, void* const* dst) {
    if (num_jobs < 0) throw ArgError("undistort: negative number of jobs");
    if (num_jobs > 0 && (!desc || !params || !src || !dst)) throw ArgError("undistort: null job arrays");
    std::vector<UJob> jobs(num_jobs);
    for (int j = 0; j < num_jobs; ++j) {
      const int32_t* d = desc + (size_t)OSFM_UNDISTORT_JOB_INTS * j;
      const std::string who = "undistort: job " + std::to_string(j);
      UJob& J = jobs[j];
      check_image(who, d[0], d[1], d[2], d[3]);
      check_sampling(who, d[4], d[5]);
      J.m = mapping_of(who, d[6], d[7], params + (size_t)OSFM_UNDISTORT_PARAMS * j, d[8], d[9], d[0], d[1]);
      J.ch = d[2];
      J.bytes = d[3];
      J.interp = d[4];
      J.border = d[5];
      J.ow = d[10];
      J.oh = d[11];
      if (J.ow < 1 || J.oh < 1) throw ArgError(who + ": empty output");
      J.ifx = 1.0 / ((double)J.ow / J.m.gw);
      J.ify = 1.0 / ((double)J.oh / J.m.gh);
      if (!src[j] || !dst[j]) throw ArgError(who + ": null image");
      J.src = src[j];
      J.dst = dst[j];
    }
    run_jobs(jobs);
  }

  void remap(const void* src, int sw, int sh, int ch, int bytes, const float* map_x, const float* map_y, int gw,
             int gh, int interp, int border, void* dst) {
    check_image("undistort remap", sw, sh, ch, bytes);
    check_sampling("undistort remap", interp, border);
    if (gw < 1 || gh < 1) throw ArgError("undistort remap: empty maps");
    if (!src || !map_x || !map_y || !dst) throw ArgError("undistort remap: null arrays");
    const size_t n = (size_t)gw * gh;
    const size_t src_bytes = (size_t)sw * sh * ch * bytes;
    if (n > d_mx.cap) fits("the maps", (long long)(8 * n + src_bytes + n * ch * bytes));
    upload(d_mx, map_x, n);
    upload(d_my, map_y, n);
    UJob J{};
    J.m.kind = UD_MAPS;
    J.m.gw = gw;
    J.m.gh = gh;
    J.m.sw = sw;
    J.m.sh = sh;
    J.m.mx = d_mx.p;
    J.m.my = d_my.p;
    J.ch = ch;
    J.bytes = bytes;
    J.interp = interp;
    J.border = border;
    J.ow = gw;
    J.oh = gh;
    J.ifx = J.ify = 1.0;
    J.src = src;
    J.dst = dst;
    OSFM_CUDA(cudaStreamSynchronize(stream));   // the maps are read from the slot's stream
    run_jobs({J});
  }

  void maps(const UMapping& m, float* map_x, float* map_y) {
    if (!map_x || !map_y) throw ArgError("undistort maps: null maps");
    const size_t n = (size_t)m.gw * m.gh;
    if (n > d_mx.cap) fits("the maps", (long long)(8 * n));
    d_mx.reserve(n);
    d_my.reserve(n);
    ms[0] = ms[1] = ms[2] = 0.f;
    OSFM_CUDA(cudaEventRecord(ev[0], stream));
    ud_maps<<<grid_of((long long)n), UD_THREADS, 0, stream>>>(m, d_mx.p, d_my.p);
    OSFM_LAUNCH_CHECK();
    OSFM_CUDA(cudaEventRecord(ev[1], stream));
    download(map_x, d_mx.p, n);
    download(map_y, d_my.p, n);
    OSFM_CUDA(cudaStreamSynchronize(stream));
    OSFM_CUDA(cudaEventElapsedTime(&ms[1], ev[0], ev[1]));
  }
};

}  // namespace
}  // namespace osfm

struct osfm_undistort : osfm::Handle<osfm::Undistort> {
  using Handle::Handle;
  static constexpr const char* null_message = "null undistort";
};

extern "C" {

int osfm_undistort_create(int device, osfm_undistort** out) { return osfm::create_handle(device, out); }
int osfm_undistort_destroy(osfm_undistort* h) { return osfm::destroy_handle(h); }

int osfm_undistort_camera_maps(osfm_undistort* h, int from_type, const double* params, int width, int height,
                               float* map_x, float* map_y) {
  return osfm::with_handle(h, [&](osfm::Undistort& U) {
    U.maps(osfm::mapping_of("undistort camera maps", OSFM_UNDISTORT_CAMERA, from_type, params, width, height, width,
                            height),
           map_x, map_y);
  });
}

int osfm_undistort_face_maps(osfm_undistort* h, int face_size, const double* rotation, int pano_width,
                             int pano_height, float* map_x, float* map_y) {
  return osfm::with_handle(h, [&](osfm::Undistort& U) {
    if (pano_width < 1 || pano_height < 1) throw osfm::ArgError("undistort face maps: empty panorama");
    U.maps(osfm::mapping_of("undistort face maps", OSFM_UNDISTORT_FACE, 0, rotation, face_size, face_size, pano_width,
                            pano_height),
           map_x, map_y);
  });
}

int osfm_undistort_remap(osfm_undistort* h, const void* src, int src_width, int src_height, int channels,
                         int bytes_per_sample, const float* map_x, const float* map_y, int width, int height,
                         int interpolation, int border, void* dst) {
  return osfm::with_handle(h, [&](osfm::Undistort& U) {
    U.remap(src, src_width, src_height, channels, bytes_per_sample, map_x, map_y, width, height, interpolation, border,
            dst);
  });
}

int osfm_undistort_run(osfm_undistort* h, int num_jobs, const int32_t* jobs, const double* params,
                       const void* const* src, void* const* dst) {
  return osfm::with_handle(h, [&](osfm::Undistort& U) { U.run(num_jobs, jobs, params, src, dst); });
}

int osfm_undistort_last_device_ms(osfm_undistort* h, float* upload_ms, float* kernel_ms, float* download_ms) {
  return osfm::with_handle(h, [&](osfm::Undistort& U) {
    if (!upload_ms || !kernel_ms || !download_ms) throw osfm::ArgError("null ms");
    *upload_ms = U.ms[0];
    *kernel_ms = U.ms[1];
    *download_ms = U.ms[2];
  });
}

}  // extern "C"
