// Bundle adjustment on H100 (sm_90a): Levenberg-Marquardt with Schur
// elimination of the points and PCG on the reduced camera system, all in fp64.
//
// Replaces bundle::BundleAdjuster::Run (opensfm/src/bundle/src/bundle_adjuster.cc:595-1121)
// = problem assembly + ceres::Solve(SPARSE_SCHUR) + ComputeReprojectionErrors, for the
// residual blocks the reference's default pipeline builds (sfm/src/ba_helpers.cc:581-763):
// point projections with a shared robust loss, camera-intrinsics priors (log-scale focal /
// aspect ratio), rig-instance position priors.  The LM rules are Ceres' (SURVEY.md §8c).
//
// HBM layout (SoA, observations sorted by point so that V_p, g_p, the Schur update
// and the back-substitution of a point touch one contiguous range):
//   obs_{shot,point,x,y,isig}[N]          observation records
//   r[nres][N], Jc[nres*wc][N], Jp[nres*3][N]   robustified residual / Jacobian planes
//   S[nc*nc], rhs[nc]                     reduced camera system (dense, symmetric)
//   Vinv[6][npf], vectors[nc + 3 npf]     per-point inverse blocks, LM vectors
//
// Kernels: ba_linearize (per observation); column norms and gradient over the segment chunk list when the camera
// side is 9 wide with 2 residual rows (ba_linearize_fused, ba_colnorm_grad_chunks: ba_schur_pipe.cuh), else a warp
// per segment (ba_colnorm_grad_seg), ba_colnorm_grad for the other observations; the segment Schur kernels
// (ba_reduced.cuh, ba_schur_pipe.cuh) and ba_schur (CTA per point: U, g_c, V^-1 and W V^-1 W^T scattered to S with
// fp64 atomics), ba_finish_system, PCG kernels (block-Jacobi), ba_backsub (warp per point), ba_model_change_alg,
// ba_update.
#include <algorithm>
#include <dlfcn.h>

#include <chrono>
#include <cstring>
#include <mutex>
#include <cmath>
#include <cstdlib>
#include <string>
#include <vector>

#include "ba_models.cuh"
#include "common.cuh"

// ncclUniqueId is 128 opaque bytes passed BY VALUE to ncclCommInitRank (nccl.h: NCCL_UNIQUE_ID_BYTES)
struct OsfmNcclId { char internal[128]; };

namespace osfm {

// ---------------------------------------------------------------------------
// Device-side problem view
// ---------------------------------------------------------------------------
struct BAView {
  int K, NI, NR, S, P;
  long long N;
  int nc, npf;      // reduced camera-side dimension, free local points
  int wc, nres;     // Jacobian plane counts
  int loss;
  double loss_a;
  const int *cam_type, *cam_off, *cam_np, *cam_poff, *inst_poff, *rc_poff, *pt_poff;
  const int *shot_inst, *shot_cam, *shot_rc, *shot_use_rc;
  const int *obs_shot, *obs_point;
  const double *obs_x, *obs_y, *obs_isig;
  const long long* obs_orig;
  const long long* pt_start;
  double *r, *Jc, *Jp;
};

struct Params {
  double *cam, *inst, *rc, *pts, *ext;
};

// scalar accumulators (device)
struct Scalars {
  double cost;
  double model_change;
  double step_norm2;
  double x_norm2;
  double grad_max_bits;  // max |g| via atomicMax on the bit pattern (non-negative doubles)
  double gdot;           // gradient . step (projected line search of bounded problems)
};

// Levenberg-Marquardt state of run(), owned by the device: the step control kernels (ba_lm_*) read and write it, the
// loop's other kernels and conditional nodes follow its branch word, the host reads it when the loop is done (and
// after every decision when the host drives the loop).
enum LmBranch { LM_EVAL = 1, LM_ACCEPT = 2, LM_PCG_CLASSIC = 4 };   // bits of LmState::branch
enum LmMessage { LM_MSG_MAX_ITERATIONS, LM_MSG_NO_FREE, LM_MSG_GTOL, LM_MSG_MIN_RADIUS, LM_MSG_INVALID, LM_MSG_PTOL,
                 LM_MSG_FTOL };
enum LmPhase { LM_PH_LIN, LM_PH_SCHUR, LM_PH_PCG, LM_PH_BACK, LM_PH_COUNT };   // the summary's phase timers
struct LmState {
  double radius, decrease_factor, cost, initial_cost, x_norm;
  int reuse_diagonal;
  int it, n_invalid, n_success, n_solves, n_eval, n_classic, pcg_total;   // n_eval: valid steps, n_classic: PCG fallbacks
  int termination, message;   // osfm_ba_summary::termination (1 while running), LmMessage
  int running;                // ba_lm_next: another iteration follows
  int branch;                 // LmBranch bits of the current iteration
  int pcg_path;               // OSFM_PCG_* that solved the last system (when the pipelined PCG ran first)
  unsigned long long phase_t0[LM_PH_COUNT], phase_ns[LM_PH_COUNT];   // %globaltimer stamps
  int phase_count[LM_PH_COUNT];
};
// Ceres' defaults (trust_region_minimizer / levenberg_marquardt_strategy)
constexpr double LM_RADIUS0 = 1e4, LM_MAX_RADIUS = 1e16, LM_MIN_RADIUS = 1e-32, LM_MIN_REL_DECREASE = 1e-3;
constexpr double LM_FTOL = 1e-6, LM_GTOL = 1e-10, LM_PTOL = 1e-8;

__device__ __forceinline__ double block_reduce_sum(double v) {
  __shared__ double sh[32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if (lane == 0) sh[w] = v;
  __syncthreads();
  const int nw = (blockDim.x + 31) >> 5;
  v = threadIdx.x < nw ? sh[threadIdx.x] : 0.0;
  if (w == 0) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  }
  return v;  // valid in thread 0
}

__device__ __forceinline__ void atomic_max_nonneg(double* addr, double v) {
  atomicMax(reinterpret_cast<unsigned long long*>(addr), (unsigned long long)__double_as_longlong(v));
}

// ---------------------------------------------------------------------------
// Per-observation kernels
// ---------------------------------------------------------------------------
// MODE 0: cost only (candidate evaluation).  MODE 1: residual + Jacobian planes (robustified).
// MODE 2: unscaled reprojection errors (bundle_adjuster.cc:531-566), written in original order.
// NB = minimum resident CTAs per SM the register allocation is held to (the kernel is latency-bound: at its
// natural 156 registers only 12 warps fit on an SM).
// TYPE >= 0: every camera of the problem has this projection type and no shot goes through a rig camera: the
// model dispatch, the parameter count and the Jacobian block sizes become compile-time constants, the blocks
// live in registers instead of a local-memory frame.
template <int MODE, int NB = 3, int TYPE = -1>
__global__ void __launch_bounds__(128, NB) ba_linearize(BAView v, Params p, Scalars* sc, double* reproj) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  double cost = 0.0;
  if (i < v.N) {
    const int shot = v.obs_shot[i];
    const int cam = v.shot_cam[shot];
    const int type = TYPE >= 0 ? TYPE : v.cam_type[cam];
    const int C = TYPE >= 0 ? model_num_params(TYPE >= 0 ? TYPE : 0) : v.cam_np[cam];
    const bool use_rc = TYPE >= 0 ? false : v.shot_use_rc[shot] != 0;
    const int pt = v.obs_point[i];
    double camp[MAX_CAM_PARAMS], ri[6], rc[6], X[3];
#pragma unroll
    for (int j = 0; j < MAX_CAM_PARAMS; ++j)
      if (j < C) camp[j] = p.cam[v.cam_off[cam] + j];
#pragma unroll
    for (int j = 0; j < 6; ++j) ri[j] = p.inst[6 * (size_t)v.shot_inst[shot] + j];
    if (use_rc) {
#pragma unroll
      for (int j = 0; j < 6; ++j) rc[j] = p.rc[6 * (size_t)v.shot_rc[shot] + j];
    }
#pragma unroll
    for (int j = 0; j < 3; ++j) X[j] = p.pts[3 * (size_t)pt + j];
    const double ox = v.obs_x[i], oy = v.obs_y[i];
    if (MODE == 2) {
      double r[3] = {0.0, 0.0, 0.0};
      observation_eval(type, camp, ri, rc, use_rc, X, ox, oy, 1.0, r, nullptr, nullptr, nullptr, nullptr);
      const long long o = v.obs_orig[i];
      reproj[3 * o] = r[0]; reproj[3 * o + 1] = r[1]; reproj[3 * o + 2] = r[2];
    } else if (MODE == 0) {
      double r[3];
      const int nres = observation_eval(type, camp, ri, rc, use_rc, X, ox, oy, v.obs_isig[i], r, nullptr, nullptr,
                                        nullptr, nullptr);
      double s = r[0] * r[0] + r[1] * r[1];
      if (nres == 3) s += r[2] * r[2];
      double w;
      cost = 0.5 * robust_loss(v.loss, v.loss_a, s, &w);
      // a residual block whose parameter blocks are all constant is not part of the minimised cost (ceres removes
      // it from the reduced program; its value only enters Summary::fixed_cost)
      if (v.cam_poff[cam] < 0 && v.inst_poff[v.shot_inst[shot]] < 0 && (!use_rc || v.rc_poff[v.shot_rc[shot]] < 0) &&
          v.pt_poff[pt] < 0)
        cost = 0.0;
    } else {
      double r[3], jc[3 * MAX_CAM_PARAMS], jri[18], jrc[18], jp[9];
      const int nres = observation_eval(type, camp, ri, rc, use_rc, X, ox, oy, v.obs_isig[i], r, jc, jri, jrc, jp);
      double s = r[0] * r[0] + r[1] * r[1];
      if (nres == 3) s += r[2] * r[2];
      double w;
      cost = 0.5 * robust_loss(v.loss, v.loss_a, s, &w);
      const bool pfree = v.pt_poff[pt] >= 0;
      if (!pfree && v.cam_poff[cam] < 0 && v.inst_poff[v.shot_inst[shot]] < 0 && (!use_rc || v.rc_poff[v.shot_rc[shot]] < 0))
        cost = 0.0;   // all blocks constant: not part of the minimised cost (see MODE 0)
      const size_t N = (size_t)v.N;
      if (TYPE >= 0) {
        // uniform projection type, no rig cameras: nres = 2 rows, wc = C + 6 columns, all indices compile-time
        constexpr int CC = TYPE == PT_PERSPECTIVE ? 3 : TYPE == PT_FISHEYE ? 3 : TYPE == PT_BROWN ? 9 : 1;
        const int wcl = v.wc;
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          v.r[k * N + i] = w * r[k];
          double* jcrow = v.Jc + (size_t)k * wcl * N + i;
#pragma unroll
          for (int j = 0; j < CC; ++j) jcrow[(size_t)j * N] = w * jc[k * CC + j];
#pragma unroll
          for (int j = 0; j < 6; ++j) jcrow[(size_t)(CC + j) * N] = w * jri[k * 6 + j];
          for (int j = CC + 6; j < wcl; ++j) jcrow[(size_t)j * N] = 0.0;
#pragma unroll
          for (int j = 0; j < 3; ++j) v.Jp[((size_t)k * 3 + j) * N + i] = pfree ? w * jp[k * 3 + j] : 0.0;
        }
        for (int k = 2; k < v.nres; ++k) {
          v.r[k * N + i] = 0.0;
          for (int j = 0; j < wcl; ++j) v.Jc[((size_t)k * wcl + j) * N + i] = 0.0;
          for (int j = 0; j < 3; ++j) v.Jp[((size_t)k * 3 + j) * N + i] = 0.0;
        }
      } else
      for (int k = 0; k < v.nres; ++k) {
        const bool live = k < nres;
        v.r[k * N + i] = live ? w * r[k] : 0.0;
        double* jcrow = v.Jc + (size_t)k * v.wc * N + i;
        for (int j = 0; j < v.wc; ++j) {
          double val = 0.0;
          if (live) {
            if (j < C) val = jc[k * C + j];
            else if (j < C + 6) val = jri[k * 6 + (j - C)];
            else if (use_rc && j < C + 12) val = jrc[k * 6 + (j - C - 6)];
          }
          jcrow[(size_t)j * N] = w * val;
        }
#pragma unroll
        for (int j = 0; j < 3; ++j) v.Jp[((size_t)k * 3 + j) * N + i] = (live && pfree) ? w * jp[k * 3 + j] : 0.0;
      }
    }
  }
  if (MODE != 2) {
    const double tot = block_reduce_sum(cost);
    if (threadIdx.x == 0 && tot != 0.0) atomicAdd(&sc->cost, tot);
  }
}

// Global column of local camera-side column j of an observation, or -1.
struct ObsCols {
  int g_cam, C, g_inst, g_rc;
  __device__ __forceinline__ int col(int j) const {
    if (j < C) return g_cam >= 0 ? g_cam + j : -1;
    if (j < C + 6) return g_inst >= 0 ? g_inst + (j - C) : -1;
    if (j < C + 12) return g_rc >= 0 ? g_rc + (j - C - 6) : -1;
    return -1;
  }
};
__device__ __forceinline__ ObsCols obs_cols(const BAView& v, long long i) {
  const int shot = v.obs_shot[i];
  const int cam = v.shot_cam[shot];
  ObsCols oc;
  oc.g_cam = v.cam_poff[cam];
  oc.C = v.cam_np[cam];
  oc.g_inst = v.inst_poff[v.shot_inst[shot]];
  oc.g_rc = v.shot_use_rc[shot] ? v.rc_poff[v.shot_rc[shot]] : -2;  // -2: no rig-camera columns at all
  return oc;
}

// Prior residual rows (camera prior bundle_adjuster.cc:568-593 / prior_error.h:78-95,
// position prior bundle_adjuster.cc:745-778): row value, column, derivative.
struct PriorView {
  int n_cam_rows, n_pos_rows;
  const int *cam_row_param, *cam_row_col, *cam_row_log;  // index into cam params / reduced column
  const double *cam_row_prior, *cam_row_scale;
  // linear rows on one component of a rig instance (kind 1: GPS position prior) or of a rig camera
  // (kind 2: DataPriorError<Pose>, bundle_adjuster.cc:779-790)
  const int *pos_row_kind, *pos_row_inst, *pos_row_axis, *pos_row_col;
  const double *pos_row_prior, *pos_row_scale;
};
__device__ __forceinline__ void prior_row(const PriorView& pv, const Params& p, int row, double* r, int* col,
                                          double* d) {
  if (row < pv.n_cam_rows) {
    const double val = p.cam[pv.cam_row_param[row]];
    const double sc = pv.cam_row_scale[row];
    *col = pv.cam_row_col[row];
    if (pv.cam_row_log[row]) {
      *r = sc * log(val / pv.cam_row_prior[row]);
      *d = sc / val;
    } else {
      *r = sc * (val - pv.cam_row_prior[row]);
      *d = sc;
    }
  } else {
    const int q = row - pv.n_cam_rows;
    const double sc = pv.pos_row_scale[q];
    *col = pv.pos_row_col[q];
    const double* base = pv.pos_row_kind[q] == 2 ? p.rc : p.inst;
    *r = sc * (base[6 * (size_t)pv.pos_row_inst[q] + pv.pos_row_axis[q]] - pv.pos_row_prior[q]);
    *d = sc;
  }
}

__global__ void ba_prior_cost(PriorView pv, Params p, Scalars* sc) {
  const int row = blockIdx.x * blockDim.x + threadIdx.x;
  double c = 0.0;
  if (row < pv.n_cam_rows + pv.n_pos_rows) {
    double r, d;
    int col;
    prior_row(pv, p, row, &r, &col, &d);
    c = 0.5 * r * r;
  }
  const double tot = block_reduce_sum(c);
  if (threadIdx.x == 0 && tot != 0.0) atomicAdd(&sc->cost, tot);
}

// Point priors (AddPointPrior, bundle_adjuster.cc:224-236; residual block :688-708, DataPriorError<Vec3d>):
// r_j = d_j (X_j - x0_j), d_j = 1 / max(sigma_j, eps), j over x, y (and z with an altitude prior).  Dense arrays in
// the caller's point order (d = 0: no row); local point np -> global_of[np].  Points with a prior are kept off the
// segment path (ba_order.cuh), so only ba_schur has to add them to V_p and g_p.
struct PointPriorView {
  const double* d;   // [3 * Pfull], nullptr when no point has a prior
  const double* x0;
  const int* global_of;
};
// MODE 0: cost.  1: cost + squared column norms + gradient.  3: adds J_p^T r to the right-hand side t[3][npf] of
// the back-substitution.  One thread per local point.
template <int MODE>
__global__ void ba_point_prior(PointPriorView pp, BAView v, Params p, double* colnorm2, double* grad, double* t, Scalars* sc) {
  const int np = blockIdx.x * blockDim.x + threadIdx.x;
  double acc = 0.0;
  if (np < v.P) {
    const int pf = v.pt_poff[np];
    const size_t g = (size_t)pp.global_of[np];
    if (pf >= 0) {
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        const double d = pp.d[3 * g + j];
        if (d == 0.0) continue;
        const double r = d * (p.pts[3 * (size_t)np + j] - pp.x0[3 * g + j]);
        const int col = v.nc + 3 * pf + j;
        if (MODE <= 1) acc += 0.5 * r * r;
        if (MODE == 1) { colnorm2[col] += d * d; grad[col] += d * r; }   // only this thread touches the point's columns here
        if (MODE == 3) t[(size_t)j * v.npf + pf] += d * r;
      }
    }
  }
  if (MODE <= 1) {
    const double tot = block_reduce_sum(acc);
    if (threadIdx.x == 0 && tot != 0.0) atomicAdd(&sc->cost, tot);
  }
}

// Squared column norms and gradient of the (unscaled, robustified) Jacobian.
// (camera-side columns of the observations i >= i0: the ones no segment covers)
__global__ void __launch_bounds__(256) ba_colnorm_grad(BAView v, long long i0, double* colnorm2, double* grad) {
  const long long i = i0 + (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= v.N) return;
  const size_t N = (size_t)v.N;
  const ObsCols oc = obs_cols(v, i);
  double r[3];
  for (int k = 0; k < v.nres; ++k) r[k] = v.r[k * N + i];
  for (int j = 0; j < v.wc; ++j) {
    const int g = oc.col(j);
    if (g < 0) continue;
    double n2 = 0.0, gr = 0.0;
    for (int k = 0; k < v.nres; ++k) {
      const double a = v.Jc[((size_t)k * v.wc + j) * N + i];
      n2 += a * a;
      gr += a * r[k];
    }
    atomicAdd(&colnorm2[g], n2);
    atomicAdd(&grad[g], gr);
  }
}

// Segmented sum over lanes holding consecutive observations of the same point (observations are
// sorted by point): after the call the LAST lane of every run holds the run's total.
template <int NV>
__device__ __forceinline__ void seg_scan_by_point(int pt, double (&val)[NV]) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int other = __shfl_up_sync(0xffffffffu, pt, o);
    const bool take = lane >= o && other == pt;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      const double up = __shfl_up_sync(0xffffffffu, val[k], o);
      if (take) val[k] += up;
    }
  }
}

// Point-side columns of the observations i >= i0: one thread per observation (coalesced plane reads), run totals
// by shuffles, one atomic per (run, column) -- a run is cut only at warp boundaries.
__global__ void __launch_bounds__(256) ba_colnorm_grad_points(BAView v, long long i0, double* colnorm2, double* grad) {
  const long long i = i0 + (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t N = (size_t)v.N;
  const bool in = i < v.N;
  const int pt = in ? v.obs_point[i] : -1;
  double val[6] = {0, 0, 0, 0, 0, 0};
  if (in) {
    for (int k = 0; k < v.nres; ++k) {
      const double rk = v.r[k * N + i];
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        const double a = v.Jp[((size_t)k * 3 + j) * N + i];
        val[j] += a * a;
        val[3 + j] += a * rk;
      }
    }
  }
  seg_scan_by_point<6>(pt, val);
  const int next = __shfl_down_sync(0xffffffffu, pt, 1);
  const bool tail = (threadIdx.x & 31) == 31 || next != pt;
  if (in && tail) {
    const int pf = v.pt_poff[pt];
    if (pf >= 0) {
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        atomicAdd(&colnorm2[v.nc + 3 * pf + j], val[j]);
        atomicAdd(&grad[v.nc + 3 * pf + j], val[3 + j]);
      }
    }
  }
}

// Camera-side columns of the segments (points seen by exactly the same k shots, ba_order.cuh): one
// warp per segment, lane = (point slot g, shot c) so that a lane always works on the same shot; the
// running sums stay in registers and a segment issues k * wc atomics instead of points * k * wc.
template <int WCT>
__global__ void __launch_bounds__(256, WCT ? 3 : 2) ba_colnorm_grad_seg(BAView v, const int* __restrict__ seg_start, int nseg,
                                                           double* colnorm2, double* grad) {
  const int s = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (s >= nseg) return;
  const int lane = threadIdx.x & 31;
  const int p0 = seg_start[s], np = seg_start[s + 1] - p0;
  const long long base = v.pt_start[p0];
  const int k = (int)(v.pt_start[p0 + 1] - base);
  const int G = 32 / k;
  const int g = lane / k, c = lane - g * k;
  const bool active = g < G;
  const size_t N = (size_t)v.N;
  const int wc = WCT ? WCT : v.wc;
  constexpr int WCU = WCT ? WCT : 16;
  double n2[WCU], gr[WCU];
#pragma unroll
  for (int j = 0; j < WCU; ++j) { n2[j] = 0.0; gr[j] = 0.0; }
  if (active) {
    for (int pi = g; pi < np; pi += G) {
      const size_t i = (size_t)(base + (long long)pi * k + c);
      for (int q = 0; q < v.nres; ++q) {
        const double rq = v.r[q * N + i];
#pragma unroll
        for (int j = 0; j < WCU; ++j) {
          if (j < wc) {
            const double a = v.Jc[((size_t)q * wc + j) * N + i];
            n2[j] += a * a;
            gr[j] += a * rq;
          }
        }
      }
    }
  }
  // lanes c, c + k, c + 2k, ... hold partial sums of the same shot
  for (int gg = 1; gg < G; ++gg) {
#pragma unroll
    for (int j = 0; j < WCU; ++j) {
      if (j < wc) {
        const double a = __shfl_down_sync(0xffffffffu, n2[j], gg * k);
        const double b = __shfl_down_sync(0xffffffffu, gr[j], gg * k);
        if (lane < k) { n2[j] += a; gr[j] += b; }
      }
    }
  }
  if (lane < k) {
    const ObsCols oc = obs_cols(v, base + c);
#pragma unroll
    for (int j = 0; j < WCU; ++j) {
      if (j < wc) {
        const int col = oc.col(j);
        if (col >= 0) {
          atomicAdd(&colnorm2[col], n2[j]);
          atomicAdd(&grad[col], gr[j]);
        }
      }
    }
  }
}

__global__ void ba_prior_colnorm_grad(PriorView pv, Params p, double* colnorm2, double* grad) {
  const int row = blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= pv.n_cam_rows + pv.n_pos_rows) return;
  double r, d;
  int col;
  prior_row(pv, p, row, &r, &col, &d);
  atomicAdd(&colnorm2[col], d * d);
  atomicAdd(&grad[col], d * r);
}

// scale = 1 / (1 + sqrt(colnorm2))   (Ceres jacobi_scaling)
__global__ void ba_make_scale(const double* colnorm2, double* scale, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) scale[i] = 1.0 / (1.0 + sqrt(colnorm2[i]));
}
// diag = clamp(colnorm2 * scale^2, 1e-6, 1e32), kept when the LM state reuses the diagonal; with diag_r, also the
// damping of this iteration diag_r = diag / radius
__global__ void ba_make_diag(const double* colnorm2, const double* scale, double* diag, int n, const LmState* st = nullptr,
                             double* diag_r = nullptr) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double d;
  if (st && st->reuse_diagonal) {
    d = diag[i];
  } else {
    d = fmin(fmax(colnorm2[i] * scale[i] * scale[i], 1e-6), 1e32);
    diag[i] = d;
  }
  if (diag_r) diag_r[i] = d * (1.0 / st->radius);
}
// Multi-GPU: everything rank-summed after a linearisation travels in ONE buffer
//   pack = [ colnorm2 (nc) | grad (nc) | cost | per-rank max |point gradient| (world) ]
__global__ void ba_pack_lin(const double* __restrict__ colnorm2, const double* __restrict__ grad, const Scalars* sc, int nc,
                            int rank, int world, double* __restrict__ pack) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < nc) { pack[i] = colnorm2[i]; pack[nc + i] = grad[i]; }
  if (i == 0) pack[2 * nc] = sc->cost;
  if (i < world) pack[2 * nc + 1 + i] = i == rank ? sc->grad_max_bits : 0.0;
}
__global__ void ba_unpack_lin(const double* __restrict__ pack, int nc, int world, double* __restrict__ colnorm2,
                              double* __restrict__ grad, Scalars* sc) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double v = 0.0;
  if (i < nc) { colnorm2[i] = pack[i]; grad[i] = pack[nc + i]; v = fabs(pack[nc + i]); }
  if (i < world) v = fmax(v, pack[2 * nc + 1 + i]);
  if (i == 0) sc->cost = pack[2 * nc];
#pragma unroll
  for (int o = 16; o; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  if ((threadIdx.x & 31) == 0 && v > 0.0) atomic_max_nonneg(&sc->grad_max_bits, v);
}
// one atomic per CTA: a C4 gradient has 600k entries, and per-warp atomics on one address serialise in L2
__global__ void __launch_bounds__(256) ba_grad_max(const double* grad, int n, Scalars* sc) {
  __shared__ double wmax[8];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double v = i < n ? fabs(grad[i]) : 0.0;
#pragma unroll
  for (int o = 16; o; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  if ((threadIdx.x & 31) == 0) wmax[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) v = fmax(v, wmax[w]);
    if (v > 0.0) atomic_max_nonneg(&sc->grad_max_bits, v);
  }
}

}  // namespace osfm
#include "ba_reduced.cuh"
#include "ba_schur_pipe.cuh"

#include <tuple>
#include <utility>

namespace osfm {
// The PCG kernels synchronise the whole grid through their own barrier (flags in global memory): every CTA must be
// resident at the same time.  A cooperative launch makes the runtime check that (it fails with
// cudaErrorCooperativeLaunchTooLarge instead of deadlocking when the grid cannot be co-resident).
template <typename... KArgs, size_t... I>
inline void launch_cooperative_impl(void (*kern)(KArgs...), int grid, int block, size_t smem, cudaStream_t st,
                                    std::tuple<KArgs...>& a, std::index_sequence<I...>) {
  void* ptrs[] = {static_cast<void*>(&std::get<I>(a))...};
  OSFM_CUDA(cudaLaunchCooperativeKernel(reinterpret_cast<const void*>(kern), dim3(grid), dim3(block), ptrs, smem, st));
}
template <typename... KArgs, typename... Args>
inline void launch_cooperative(void (*kern)(KArgs...), int grid, int block, size_t smem, cudaStream_t st, Args&&... args) {
  std::tuple<KArgs...> a(std::forward<Args>(args)...);
  launch_cooperative_impl(kern, grid, block, smem, st, a, std::index_sequence_for<KArgs...>{});
}
}  // namespace osfm
#include "ba_side.cuh"
#include "ba_order.cuh"
#include "ba_cov.cuh"
namespace osfm {

// ---------------------------------------------------------------------------
// Back-substitution: y_p = V^-1 (g_p - W^T y_c)  (scaled system).
// ba_backsub_rows: one thread per observation (coalesced plane reads) computes its share of
// g_p - W^T y_c, run totals by shuffles, one atomic per (run, coordinate) into t[3][npf];
// ba_backsub_points: one thread per point applies V^-1.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256) ba_backsub_rows(BAView v, const double* __restrict__ scale,
                                                       const double* __restrict__ y, double* __restrict__ t) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t N = (size_t)v.N;
  const bool in = i < v.N;
  const int pt = in ? v.obs_point[i] : -1;
  const int pf = in ? v.pt_poff[pt] : -1;
  double val[3] = {0.0, 0.0, 0.0};
  if (pf >= 0) {
    const int wc = v.wc;
    const ObsCols oc = obs_cols(v, i);
    for (int q = 0; q < v.nres; ++q) {
      double e = v.r[q * N + i];
      for (int j = 0; j < wc; ++j) {
        const int g = oc.col(j);
        if (g >= 0) e -= v.Jc[((size_t)q * wc + j) * N + i] * scale[g] * y[g];
      }
#pragma unroll
      for (int j = 0; j < 3; ++j) val[j] += v.Jp[((size_t)q * 3 + j) * N + i] * e;
    }
  }
  seg_scan_by_point<3>(pt, val);
  const int next = __shfl_down_sync(0xffffffffu, pt, 1);
  const bool tail = (threadIdx.x & 31) == 31 || next != pt;
  if (pf >= 0 && tail) {
    const size_t NP = (size_t)v.npf;
#pragma unroll
    for (int j = 0; j < 3; ++j) atomicAdd(&t[j * NP + pf], val[j]);
  }
}
__global__ void __launch_bounds__(256) ba_backsub_points(BAView v, const double* __restrict__ scale,
                                                         const double* __restrict__ Vinv, const double* __restrict__ t,
                                                         double* __restrict__ y) {
  const int pf = blockIdx.x * blockDim.x + threadIdx.x;
  if (pf >= v.npf) return;
  const size_t NP = (size_t)v.npf;
  const int nc = v.nc;
  const double t0 = t[pf] * scale[nc + 3 * pf], t1 = t[NP + pf] * scale[nc + 3 * pf + 1],
               t2 = t[2 * NP + pf] * scale[nc + 3 * pf + 2];
  const double a = Vinv[0 * NP + pf], b = Vinv[1 * NP + pf], c = Vinv[2 * NP + pf];
  const double d = Vinv[3 * NP + pf], e = Vinv[4 * NP + pf], f = Vinv[5 * NP + pf];
  y[nc + 3 * pf + 0] = a * t0 + b * t1 + c * t2;
  y[nc + 3 * pf + 1] = b * t0 + d * t1 + e * t2;
  y[nc + 3 * pf + 2] = c * t0 + e * t1 + f * t2;
}

// candidate = x - scale * y ; accumulates |delta|^2 and |candidate|^2 (free parameters only).
// which: 0 cameras, 1 instances, 2 rig cameras, 3 points.
__global__ void ba_update(int which, int count, const int* __restrict__ poff, const int* __restrict__ off,
                          const int* __restrict__ np, int stride, int base, const double* __restrict__ src,
                          double* __restrict__ dst, const double* __restrict__ scale, const double* __restrict__ y,
                          Scalars* sc, int accumulate_norms, const double* __restrict__ lower = nullptr,
                          double alpha = 1.0) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  double sn = 0.0, xn = 0.0;
  if (b < count) {
    const int o = which == 0 ? off[b] : b * stride;
    const int n = which == 0 ? np[b] : stride;
    const int g = poff[b];
    for (int j = 0; j < n; ++j) {
      double val = src[o + j];
      if (g >= 0) {
        const int gi = which == 3 ? base + 3 * g + j : g + j;
        double d = -alpha * scale[gi] * y[gi];
        if (lower && val + d < lower[o + j]) d = lower[o + j] - val;   // projection onto the bound (ceres bounded LM)
        sn += d * d;
        val += d;
        xn += val * val;
      }
      dst[o + j] = val;
    }
  }
  if (accumulate_norms) {
    const double t1 = block_reduce_sum(sn);
    const double t2 = block_reduce_sum(xn);
    if (threadIdx.x == 0) {
      if (t1 != 0.0) atomicAdd(&sc->step_norm2, t1);
      if (t2 != 0.0) atomicAdd(&sc->x_norm2, t2);
    }
  }
}

// gradient . delta with delta = -scale * y: camera side counted when cam_side != 0 (one rank), points always
__global__ void ba_grad_dot(int n, int nc, int cam_side, const double* __restrict__ grad, const double* __restrict__ scale,
                            const double* __restrict__ y, Scalars* sc) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double v = 0.0;
  if (i < n && (i >= nc || cam_side)) v = -grad[i] * scale[i] * y[i];
  const double t = block_reduce_sum(v);
  if (threadIdx.x == 0 && t != 0.0) atomicAdd(&sc->gdot, t);
}

// Model cost change of the step without another pass over the Jacobian.  Ceres evaluates
//   model_cost_change = -step^T (g + H step / 2),   H = J^T J, g = J^T r   (trust_region_minimizer.cc)
// from J step; the step solves (H + D) step = -g (D = LM diagonal / radius), so H step = -g - D step and
//   model_cost_change = (y^T g_s + y^T D y) / 2,   step = -y, g_s = scale * grad   (scaled variables)
// exactly when the linear system is solved exactly, and to the solver's 1e-8 relative residual here (every term of H
// and g -- observations, priors, side terms -- is in the system that was solved).
__global__ void ba_model_change_alg(int n, int nc, int cam_side, const double* __restrict__ grad, const double* __restrict__ scale,
                                    const double* __restrict__ diag, double inv_radius, const double* __restrict__ y, Scalars* sc) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double v = 0.0;
  if (i < n && (i >= nc || cam_side)) v = 0.5 * y[i] * (grad[i] * scale[i] + diag[i] * inv_radius * y[i]);
  const double t = block_reduce_sum(v);
  if (threadIdx.x == 0 && t != 0.0) atomicAdd(&sc->model_change, t);
}

// ---------------------------------------------------------------------------
// Levenberg-Marquardt step control (one thread each).  Ceres' trust_region_minimizer with the
// levenberg_marquardt_strategy: the same tests in the same order.  `cond`: when `set_cond`, the conditional node
// handle of the device-driven loop's graph that the kernel's decision drives.
// ---------------------------------------------------------------------------
// after the first linearisation and the |x| pass (Scalars: cost, max |g|, |x|^2); `has_free`: the problem (all ranks)
// has free parameters
__global__ void ba_lm_init(LmState* st, const Scalars* sc, int has_free) {
  st->radius = LM_RADIUS0;
  st->decrease_factor = 2.0;
  st->cost = st->initial_cost = sc->cost;
  st->x_norm = has_free ? sqrt(sc->x_norm2) : 0.0;
  st->termination = 1;
  st->message = LM_MSG_MAX_ITERATIONS;
  if (!has_free) { st->termination = 0; st->message = LM_MSG_NO_FREE; }
  else if (sc->grad_max_bits <= LM_GTOL) { st->termination = 0; st->message = LM_MSG_GTOL; }
}
// head of the loop: whether another iteration runs (the WHILE condition)
__global__ void ba_lm_next(LmState* st, int max_iterations, cudaGraphConditionalHandle cond, int set_cond) {
  int run = 0;
  if (st->termination == 1 && st->it < max_iterations) {
    if (st->radius < LM_MIN_RADIUS) { st->termination = 0; st->message = LM_MSG_MIN_RADIUS; }
    else { ++st->it; run = 1; }
  }
  st->running = run;
  st->branch = 0;
  if (set_cond) cudaGraphSetConditional(cond, run);
}
// after the pipelined PCG: the classic PCG from scratch when its recurrences stagnated or broke down
__global__ void ba_lm_pcg_check(LmState* st, const PcgState* pcg, int classic_path, cudaGraphConditionalHandle cond,
                                int set_cond) {
  const int fallback = pcg->converged ? 0 : 1;
  if (fallback) {
    st->pcg_total += pcg->iterations;
    st->pcg_path = classic_path;
    st->branch |= LM_PCG_CLASSIC;
    ++st->n_classic;
  } else {
    st->pcg_path = pcg->deflated ? OSFM_PCG_PIPELINED_DEFLATED : OSFM_PCG_PIPELINED;
  }
  if (set_cond) cudaGraphSetConditional(cond, fallback);
}
// after the candidate update: an invalid step (solver NaN, no model decrease, non-finite step) halves the radius
__global__ void ba_lm_check(LmState* st, const Scalars* sc, const PcgState* pcg, int nc, cudaGraphConditionalHandle cond,
                            int set_cond) {
  ++st->n_solves;
  bool ok = true;
  if (nc > 0) {
    st->pcg_total += pcg->iterations;
    if (!(pcg->rr_final == pcg->rr_final)) ok = false;
  }
  const double step_norm = sqrt(sc->step_norm2);
  int eval = 0;
  if (!ok || !(sc->model_change > 0.0) || !isfinite(step_norm)) {
    if (++st->n_invalid >= 5) {
      st->termination = 2;
      st->message = LM_MSG_INVALID;
    } else {
      st->radius *= 0.5;
      st->reuse_diagonal = 1;
    }
  } else {
    st->n_invalid = 0;
    ++st->n_eval;
    st->branch |= LM_EVAL;
    eval = 1;
  }
  if (set_cond) cudaGraphSetConditional(cond, eval);
}
// after the candidate cost (Scalars: candidate cost, |delta|^2, |candidate|^2): tolerances, then the ratio test
__global__ void ba_lm_step(LmState* st, const Scalars* sc, cudaGraphConditionalHandle cond, int set_cond) {
  int accept = 0;
  if (st->branch & LM_EVAL) {
    const double step_norm = sqrt(sc->step_norm2), cost_change = st->cost - sc->cost;
    if (step_norm <= LM_PTOL * (st->x_norm + LM_PTOL)) {
      st->termination = 0;
      st->message = LM_MSG_PTOL;
    } else if (fabs(cost_change) <= LM_FTOL * st->cost) {
      st->termination = 0;
      st->message = LM_MSG_FTOL;
    } else {
      const double rel = cost_change / sc->model_change;
      if (rel > LM_MIN_REL_DECREASE) {
        st->x_norm = sqrt(sc->x_norm2);
        st->radius = fmin(LM_MAX_RADIUS, st->radius / fmax(1.0 / 3.0, 1.0 - pow(2.0 * rel - 1.0, 3.0)));
        st->decrease_factor = 2.0;
        st->reuse_diagonal = 0;
        ++st->n_success;
        st->branch |= LM_ACCEPT;
        accept = 1;
      } else {
        st->radius /= st->decrease_factor;
        st->decrease_factor *= 2.0;
        st->reuse_diagonal = 1;
      }
    }
  }
  if (set_cond) cudaGraphSetConditional(cond, accept);
}
// after the relinearisation at an accepted step (Scalars: cost, max |g|)
__global__ void ba_lm_accepted(LmState* st, const Scalars* sc) {
  st->cost = sc->cost;
  if (sc->grad_max_bits <= LM_GTOL) { st->termination = 0; st->message = LM_MSG_GTOL; }
}
// phase timers: ends phase `stop` and starts phase `start` (-1: none) at the device's nanosecond clock
__global__ void ba_lm_phase(LmState* st, int stop, int start) {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  if (stop >= 0) { st->phase_ns[stop] += t - st->phase_t0[stop]; ++st->phase_count[stop]; }
  if (start >= 0) st->phase_t0[start] = t;
}

// single-observation device evaluation (test hook)
__global__ void ba_eval_one(int type, const double* in, int use_rc, double* out, int* nres_out) {
  // in: cam[16] ri[6] rc[6] X[3] obs[2] isig[1]
  double r[3] = {0, 0, 0}, jc[3 * MAX_CAM_PARAMS], jri[18], jrc[18], jp[9];
  for (int i = 0; i < 18; ++i) jrc[i] = 0.0;
  const int nres = observation_eval(type, in, in + 16, in + 22, use_rc != 0, in + 28, in[31], in[32], in[33], r, jc,
                                    jri, jrc, jp);
  *nres_out = nres;
  for (int i = 0; i < 3; ++i) out[i] = r[i];
  for (int i = 0; i < 48; ++i) out[3 + i] = jc[i];
  for (int i = 0; i < 18; ++i) out[51 + i] = jri[i];
  for (int i = 0; i < 18; ++i) out[69 + i] = jrc[i];
  for (int i = 0; i < 9; ++i) out[87 + i] = jp[i];
}

// ---------------------------------------------------------------------------
// NCCL, loaded at run time (libnccl.so.2: the copy torch already mapped if there is one, so that one
// process never mixes two NCCL versions).  Only the five entry points the all-reduce needs; the
// constants are nccl.h's (ncclFloat64 = 8, ncclSum = 0, ncclUniqueId = 128 bytes).
// ---------------------------------------------------------------------------
struct NcclApi {
  void* lib = nullptr;
  int (*GetUniqueId)(void*) = nullptr;
  int (*CommInitRank)(void**, int, OsfmNcclId, int) = nullptr;
  int (*AllReduce)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
  int (*CommDestroy)(void*) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
};
static NcclApi& nccl_api() {
  static NcclApi api;
  static std::once_flag once;
  std::call_once(once, []() {
    void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);
    if (!h) h = dlopen("libnccl.so.2", RTLD_NOW);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW);
    if (!h) return;
    api.lib = h;
    api.GetUniqueId = reinterpret_cast<int (*)(void*)>(dlsym(h, "ncclGetUniqueId"));
    api.CommInitRank = reinterpret_cast<int (*)(void**, int, OsfmNcclId, int)>(dlsym(h, "ncclCommInitRank"));
    api.AllReduce = reinterpret_cast<int (*)(const void*, void*, size_t, int, int, void*, cudaStream_t)>(dlsym(h, "ncclAllReduce"));
    api.CommDestroy = reinterpret_cast<int (*)(void*)>(dlsym(h, "ncclCommDestroy"));
    api.GetErrorString = reinterpret_cast<const char* (*)(int)>(dlsym(h, "ncclGetErrorString"));
  });
  if (!api.lib || !api.GetUniqueId || !api.CommInitRank || !api.AllReduce || !api.CommDestroy)
    throw std::runtime_error("NCCL (libnccl.so.2) is not available in this process");
  return api;
}
static void nccl_check(int rc, const char* what) {
  if (rc != 0) {
    NcclApi& a = nccl_api();
    throw std::runtime_error(std::string(what) + ": " + (a.GetErrorString ? a.GetErrorString(rc) : "NCCL error"));
  }
}

static int grid_for(long long n, int threads) { return (int)std::max<long long>(1, (n + threads - 1) / threads); }
static long long up16(long long x) { return (x + 15) / 16 * 16; }
// First item of each of G parts of items 0..n-1 whose prefix sums are w[0..n], cut where the sum reaches w[n] * c / G
static std::vector<int> balanced_cut(const std::vector<long long>& w, int G) {
  const int n = (int)w.size() - 1;
  std::vector<int> lo(G + 1, n);
  lo[0] = 0;
  for (int c = 1, i = 0; c < G; ++c) {
    const long long want = w[n] * c / G;
    while (i < n && w[i] < want) ++i;
    lo[c] = i;
  }
  return lo;
}
// OSFM_BA_TRACE=1, read once per process: host wall-clock per phase of run(), in-kernel clocks and all-reduce counts
// on stderr (diagnostics only)
static bool tracing() {
  static const bool on = [] {
    const char* e = getenv("OSFM_BA_TRACE");
    return e && e[0] == '1';
  }();
  return on;
}
// Every OSFM_BA_FALLBACK_* bit (osfm_ba_set_fallbacks; HOST_LOOP is the highest)
constexpr unsigned BA_FALLBACKS_ALL = 2 * OSFM_BA_FALLBACK_HOST_LOOP - 1;

// How linearize() forms the camera-side column norms and gradient of the segment observations (RunState::lin)
enum LinPath {
  LIN_NONE,       // no segments
  LIN_FUSED,      // ba_linearize_fused: with the planes, over the chunk list (also the sums of ba_point_blocks_sums)
  LIN_CHUNKS,     // ba_colnorm_grad_chunks over the chunk list
  LIN_SEGMENTS,   // ba_colnorm_grad_seg, a warp per segment (no chunk list: wc != 9 or nres != 2)
};

// What one run() derives from the problem, rebuilt by every run(): sizes, host tables, device views, kernel paths.
struct RunState {
  std::chrono::high_resolution_clock::time_point t_start, t_prev;   // run() start, last trace line
  int64_t launches0 = 0;
  // cameras, rig instances, rig cameras, ext blocks, side terms, shots, points of this rank / of the problem
  int K = 0, NI = 0, NR = 0, NE = 0, NT = 0, S = 0, P = 0, Pfull = 0;
  long long Nfull = 0, N = 0, n_fast_obs = 0, pair_bound = 0;   // observations: all, this rank's, in segments
  int nc = 0, nc_pad = 0, n = 0, nblk = 0, npf = 0, ngroups = 0, wc = 0, nres = 2, nseg = 0, P_fast = 0;
  size_t nz = 1;                  // max(n, 1)
  // free parameters of the whole problem (every rank's points): rank-independent, so the decisions that pair the
  // ranks' all-reduces depend on it, not on n (a rank's shard may hold no free point while other ranks' do)
  long long n_all = 0;
  int n_upper = 0, n_blocks_all = 0, pcg_grid = 1;
  long long s_upper_total = 0, s_total = 0, vb = 0;   // stored doubles: upper blocks, all blocks, ELL rows
  int uniform_type = -1;          // the projection type of every camera when no shot uses a rig camera, else -1
  bool constrained = false;       // a free ext parameter with a finite lower bound (ceres: Problem::IsConstrained)
  bool have_pp = false, add_priors = false;
  // host tables (-1 = constant)
  std::vector<int> cam_off, cam_np, cam_poff, inst_poff, rc_poff, ext_off, ext_poff, blk_off, blk_sz;
  std::vector<int> cam_blk, inst_blk, rc_blk, ext_blk, side_jofs, side_rofs, grp_b1, grp_b2;
  std::vector<int> pr_cam_param, pr_cam_col, pr_cam_log, pr_pos_kind, pr_pos_inst, pr_pos_axis, pr_pos_col;
  std::vector<int> pr_blk, pr_local;   // diagonal entry of every prior row inside its diagonal block
  std::vector<double> pr_cam_prior, pr_cam_scale, pr_pos_prior, pr_pos_scale;
  std::vector<int> row_M, cbase;       // ELL layout of the PCG mat-vec: block columns per block row, their base
  std::vector<long long> rowbase;      // and the first stored value of every block row
  std::vector<int> cov_inst, cov_bstart;   // free rig instances; starts of the Cholesky blocks (+ nc)
  int cov_m = 0, cov_nb1 = 0;              // instance columns (last in the dense S); blocks of the leading part
  // kernel paths
  int schur = OSFM_SCHUR_NONE;    // OSFM_SCHUR_*: the segment kernel of build_system
  LinPath lin = LIN_NONE;         // the segment column norms of linearize
  bool seg_tab = false;           // ba_seg_tables has run (gcol of every segment column)
  int sp_nchunks = 0;             // segment chunk list (0 = none)
  bool pcg_resident = false, pcg_pipe_ok = false;   // the classic PCG keeps S in shared memory; pipelined PCG fits
  int pcg_smem = 0, pcg_pipe_smem = 0;
  PcgResident pcg_res{};
  PcgPipe pcg_pipe{};
  // device views; d_rhs_p = [nc] right-hand side, d_S_p = block values (upper blocks first)
  BAView v{}; PriorView pv{}; SideView sv{}; PointPriorView ppv{}; BlkMaps bm{}; BsrView bsr{}; PcgLayout lay{};
  double *d_rhs_p = nullptr, *d_S_p = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;   // around the LM loop
  // Device-driven LM loop: the graph under capture (null: the host drives the loop and launches directly), the
  // nodes the next captured work depends on, the conditional handles of the iteration body, and the kernels captured
  // into each part of the body (unconditional part, PCG fallback, candidate cost, acceptance)
  cudaGraph_t cap_graph = nullptr;
  std::vector<cudaGraphNode_t> cap_deps;
  cudaGraphConditionalHandle h_pcg = 0, h_eval = 0, h_accept = 0;
  int64_t k_body = 0, k_pcg = 0, k_eval = 0, k_accept = 0;
  bool device_loop = false;
};

struct BA {
  int device = 0;
  cudaStream_t own_stream = nullptr, stream = nullptr;
  // osfm_ba_set_observations_async: the measurement arrays travel on their own stream while run() already sorts the indices
  cudaStream_t copy_stream = nullptr;
  cudaEvent_t ev_obs = nullptr;
  bool obs_pending = false;
  // host copies of the problem
  std::vector<int> cam_type, cam_const, cam_prior_log;
  std::vector<double> cam_params, cam_prior, cam_prior_sigma;
  std::vector<double> inst, inst_prior_pos, inst_prior_std;
  std::vector<int> inst_const, inst_has_prior;
  std::vector<double> rc, rc_prior, rc_prior_sigma;   // rig-camera pose priors: empty = none
  std::vector<int> rc_const;
  // ext blocks (biases, reconstruction scales, std-deviation scales), side terms, point priors
  std::vector<int> ext_size, ext_const;
  std::vector<double> ext_values, ext_lower;
  std::vector<osfm_side_term> side_terms;
  std::vector<double> side_consts;
  std::vector<int> pp_point, pp_alt;
  std::vector<double> pp_prior, pp_sigma;
  std::vector<int> shot_inst, shot_cam, shot_rc, shot_use_rc;
  std::vector<double> pts;
  std::vector<int> pt_const;
  long long n_obs_full = 0;  // observations live on the device only (d_raw_*)
  // options (defaults of bundle::BundleAdjuster(), bundle_adjuster.cc:24-44)
  int loss = OSFM_LOSS_CAUCHY;
  double loss_a = 1.0;
  int max_iterations = 500;
  bool compute_reproj = true;
  int rank = 0, world = 1;
  osfm_allreduce_fn allreduce = nullptr;
  void* allreduce_user = nullptr;
  void* nccl_comm = nullptr;   // own communicator (osfm_ba_set_nccl); used when no callback is set
  int nccl_rank = -1, nccl_world = 0;
  // results
  bool reproj_valid = false;
  osfm_ba_summary summary{};
  bool has_run = false;
  // osfm_ba_set_fallbacks: OSFM_BA_FALLBACK_* bits of the kernel paths every run() takes instead of the product path
  unsigned fallbacks = 0;
  // osfm_ba_capture_linear_system: raw copies of the reduced system at LM iteration cap_iter (0 = unarmed)
  int cap_iter = 0;
  bool cap_valid = false;
  osfm_ba_capture cap_info{};
  std::vector<double> cap_sbuf, cap_y, cap_scale, cap_diag, cap_grad;   // cap_sbuf = [rhs (nc_pad) | block values]
  std::vector<double> cap_cam, cap_inst, cap_rc, cap_pts, cap_ext;      // the linearisation point (points engine order)
  std::vector<double> cap_side_r, cap_side_J;                           // side_linearize's rows (rofs / jofs layout)
  std::vector<int4> cap_upper;
  std::vector<int> cap_blk_off, cap_blk_sz, cap_pt_poff, cap_global_of;
  int cap_nc_pad = 0;
  // osfm_ba_set_compute_covariances: rig-instance covariances after the LM loop (ba_cov.cuh)
  bool cov_on = false, cov_ran = false, cov_valid = false;
  int cov_status = OSFM_COV_OK;
  double cov_pass_ms = 0.0, cov_chol_ms = 0.0;
  std::vector<double> cov_out;             // NI x 36, row-major
  DevBuf<double> d_cov;                    // dense S | L22^-1 | diagonal-block inverses | original diagonal | NI x 36
  DevBuf<int> d_cov_perm, d_cov_inst, d_cov_flags;

  // device state
  DevBuf<int> d_cam_type, d_cam_off, d_cam_np, d_cam_poff, d_inst_poff, d_rc_poff, d_pt_poff;
  DevBuf<int> d_shot_inst, d_shot_cam, d_shot_rc, d_shot_use_rc, d_obs_shot, d_obs_point;
  DevBuf<double> d_obs_x, d_obs_y, d_obs_isig;
  DevBuf<long long> d_obs_orig, d_pt_start;
  DevBuf<double> d_cam[2], d_inst[2], d_rc[2], d_pts[2];
  DevBuf<double> d_r, d_Jc, d_Jp, d_Sbuf, d_Vinv, d_gp, d_slots;
  DevBuf<double> d_scale, d_colnorm2, d_grad, d_diag, d_y, d_bs_t;
  DevBuf<double> d_px, d_pr, d_pz, d_pp, d_pAp, d_Minv, d_reproj, d_full_pts;
  DevBuf<double> d_Wdef;                   // [PCG_ND][nc] deflation vectors of the pipelined PCG (pcg_gauge_vectors)
  DevBuf<unsigned long long> d_pm;         // [2][nc][2] m = M^-1 w of the pipelined PCG as flagged words, by parity
  DevBuf<int> d_blk_off, d_blk_sz, d_cam_blk, d_inst_blk, d_rc_blk;
  // block-sparse reduced system (ba_reduced.cuh)
  DevBuf<unsigned long long> d_tkeys, d_skeys, d_skeys2, d_rkeys, d_rkeys2;
  DevBuf<int> d_tvals, d_area, d_offs, d_row_ptr, d_row_col, d_row_off, d_diag_off, d_prior_diag_off;
  DevBuf<int> d_pr_blk, d_pr_local, d_g_obs_shot, d_g_obs_point;
  DevBuf<long long> d_g_pt_start;
  DevBuf<int4> d_upper;
  DevBuf<unsigned> d_count;
  DevBuf<char> d_cub;
  DevBuf<PcgState> d_pcg;
  DevBuf<int> d_seg_start;
  // raw observations as the caller gave them + scratch of the device-side ordering (ba_order.cuh)
  DevBuf<int> d_raw_shot, d_raw_point, d_ptc_full;
  DevBuf<double> d_raw_xy, d_raw_sigma, d_pts_in;
  DevBuf<unsigned long long> d_okeys, d_okeys2, d_pkey, d_pkey2;
  DevBuf<int> d_ovals, d_ovals2, d_pval, d_order, d_inv_order, d_global_of, d_free_flag, d_free_scan, d_head, d_run_head, d_nsel;
  DevBuf<long long> d_kk;
  DevBuf<char> d_seg_flags;
  DevBuf<OrderCounts> d_oc;
  PinnedBuf<OrderCounts> h_oc;
  DevBuf<double> d_rowsJ, d_rowsW, d_rowsY, d_Vig;
  DevBuf<int> d_row_M, d_qoff, d_blk_row, d_cbase, d_colidx, d_row_of, d_grp_b1, d_grp_b2;
  DevBuf<long long> d_rowbase;
  DevBuf<double> d_Spcg, d_Ap;
  PinnedBuf<PcgState> h_pcg;
  DevBuf<int> d_pcg_rowlo;
  DevBuf<int> d_pcg_grplo;
  DevBuf<char> d_grp_shared;               // per preconditioner group: its two block rows share one column list
  DevBuf<unsigned long long> d_prof;
  DevBuf<long long> d_tab_off, d_tab_sizes;
  DevBuf<int> d_sp_nch, d_sp_chunk0;       // chunks per segment / first chunk of every segment (ba_schur_pipe)
  DevBuf<SchurChunk> d_sp_chunks;
  DevBuf<int> d_sp_ftab;                   // flush destinations per segment (sp_flush_tables)
  DevBuf<int> d_tab;
  DevBuf<double> d_ptsum;                  // [9][npf] unscaled Jp^T Jp (upper) and Jp^T r per point (ba_linearize_fused)
  SmemOptIn opt_in_smem;                   // opt_in_smem(kernel, bytes): above 48 KB, once per handle
  int num_sms = 132;
  DevBuf<int> d_pr_cam_param, d_pr_cam_col, d_pr_cam_log, d_pr_pos_inst, d_pr_pos_axis, d_pr_pos_col;
  DevBuf<double> d_pr_cam_prior, d_pr_cam_scale, d_pr_pos_prior, d_pr_pos_scale;
  DevBuf<Scalars> d_sc;
  PinnedBuf<Scalars> h_sc;
  DevBuf<LmState> d_lm;
  PinnedBuf<LmState> h_lm;
  DevBuf<double> d_diag_r;                 // diag / radius of the current LM iteration
  DevBuf<int> d_pr_pos_kind, d_ext_off, d_ext_np, d_ext_poff, d_ext_blk, d_side_jofs, d_side_rofs;
  DevBuf<double> d_ext[2], d_ext_lower, d_side_consts, d_side_J, d_side_r, d_pp_d, d_pp_x0;
  DevBuf<SideTerm> d_side_terms;

  explicit BA(int dev) : device(dev) {
    OSFM_CUDA(cudaSetDevice(device));
    OSFM_CUDA(cudaStreamCreateWithFlags(&own_stream, cudaStreamNonBlocking));
    stream = own_stream;
    OSFM_CUDA(cudaStreamCreateWithFlags(&copy_stream, cudaStreamNonBlocking));
    OSFM_CUDA(cudaEventCreateWithFlags(&ev_obs, cudaEventDisableTiming));
    h_sc.reserve(1);
    h_pcg.reserve(1);
    d_lm.reserve(1);
    h_lm.reserve(1);
    OSFM_CUDA(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, device));
  }
  ~BA() {
    if (nccl_comm) { try { nccl_api().CommDestroy(nccl_comm); } catch (...) {} }
    if (copy_stream) { cudaStreamSynchronize(copy_stream); cudaStreamDestroy(copy_stream); }
    if (ev_obs) cudaEventDestroy(ev_obs);
    if (own_stream) cudaStreamDestroy(own_stream);
  }

  Scalars read_scalars() {
    OSFM_CUDA(cudaMemcpyAsync(h_sc.p, d_sc.p, sizeof(Scalars), cudaMemcpyDeviceToHost, stream));
    OSFM_CUDA(cudaStreamSynchronize(stream));
    return *h_sc.p;
  }
  const LmState& read_lm() {
    OSFM_CUDA(cudaMemcpyAsync(h_lm.p, d_lm.p, sizeof(LmState), cudaMemcpyDeviceToHost, stream));
    OSFM_CUDA(cudaStreamSynchronize(stream));
    return *h_lm.p;
  }
  // LM phase timer stamps (ba_lm_phase) around the work of the iteration
  void lm_phase(int stop, int start) {
    ba_lm_phase<<<1, 1, 0, stream>>>(d_lm.p, stop, start);
    OSFM_LAUNCH_CHECK();
  }
  // Device-driven loop: stream work from here on is captured into g, after the nodes rs.cap_deps
  void capture_begin(cudaGraph_t g) {
    rs.cap_graph = g;
    OSFM_CUDA(cudaStreamBeginCaptureToGraph(stream, g, rs.cap_deps.data(), nullptr, rs.cap_deps.size(),
                                            cudaStreamCaptureModeRelaxed));
  }
  // ... up to here; the nodes the capture ended with become rs.cap_deps
  void capture_end() {
    cudaStreamCaptureStatus status;
    const cudaGraphNode_t* deps = nullptr;
    size_t ndeps = 0;
    OSFM_CUDA(cudaStreamGetCaptureInfo(stream, &status, nullptr, nullptr, &deps, &ndeps));
    rs.cap_deps.assign(deps, deps + ndeps);
    cudaGraph_t g = nullptr;
    OSFM_CUDA(cudaStreamEndCapture(stream, &g));
  }
  // A conditional node of `type` on `handle` after the captured work; returns its body graph, the node becomes the
  // dependency of what follows
  cudaGraph_t add_conditional(cudaGraph_t g, cudaGraphConditionalHandle handle, cudaGraphConditionalNodeType type) {
    cudaGraphNodeParams p{};
    p.type = cudaGraphNodeTypeConditional;
    p.conditional.handle = handle;
    p.conditional.type = type;
    p.conditional.size = 1;
    cudaGraphNode_t node;
    OSFM_CUDA(cudaGraphAddNode(&node, g, rs.cap_deps.data(), rs.cap_deps.size(), &p));
    rs.cap_deps.assign(1, node);
    return p.conditional.phGraph_out[0];
  }
  // The work of `fn` when the LM state's branch word has `bit` set: read back by the host-driven loop; in the
  // device-driven loop, the body of an IF node on `handle` (set by the kernel before it).  Returns the kernels `fn`
  // launched.
  template <class F>
  int64_t lm_if(cudaGraphConditionalHandle handle, int bit, F fn) {
    const int64_t k0 = g_kernel_launches.load();
    if (!rs.cap_graph) {
      if (read_lm().branch & bit) fn();
      return 0;
    }
    cudaGraph_t outer = rs.cap_graph;
    capture_end();
    cudaGraph_t body = add_conditional(outer, handle, cudaGraphCondTypeIf);
    std::vector<cudaGraphNode_t> after = rs.cap_deps;
    rs.cap_deps.clear();
    capture_begin(body);
    fn();
    capture_end();
    rs.cap_deps = after;
    capture_begin(outer);
    return g_kernel_launches.load() - k0;
  }
  // OSFM_BA_TRACE: number of all-reduces and the host time spent issuing them (+ device time when traced)
  int ar_calls = 0;
  double ar_host_ms = 0.0, ar_dev_ms = 0.0;
  void allreduce_dev(double* buf, long long count) {
    if (world > 1) {
      const auto t0 = std::chrono::high_resolution_clock::now();
      cudaEvent_t e0 = nullptr, e1 = nullptr;
      if (tracing()) { cudaEventCreate(&e0); cudaEventCreate(&e1); cudaEventRecord(e0, stream); }
      struct Done {
        BA* self; std::chrono::high_resolution_clock::time_point t0; cudaEvent_t e0, e1;
        ~Done() {
          if (tracing()) {
            cudaEventRecord(e1, self->stream); cudaEventSynchronize(e1);
            float ms = 0.f; cudaEventElapsedTime(&ms, e0, e1); self->ar_dev_ms += ms;
            cudaEventDestroy(e0); cudaEventDestroy(e1);
          }
          ++self->ar_calls;
          self->ar_host_ms += std::chrono::duration<double, std::milli>(std::chrono::high_resolution_clock::now() - t0).count();
        }
      } done{this, t0, e0, e1};
      if (allreduce) {
        if (allreduce(buf, count, stream, allreduce_user) != 0) throw std::runtime_error("all-reduce callback failed");
      } else if (nccl_comm && nccl_world == world && nccl_rank == rank) {
        nccl_check(nccl_api().AllReduce(buf, buf, (size_t)count, /*ncclFloat64*/ 8, /*ncclSum*/ 0, nccl_comm, stream), "ncclAllReduce");
      } else {
        throw ArgError("world > 1 but neither an all-reduce callback nor an NCCL communicator is set");
      }
    }
  }
  void trace(const char* what) {   // OSFM_BA_TRACE=1: host wall-clock per phase of run() on stderr (diagnostics only)
    if (!tracing()) return;
    const auto now = std::chrono::high_resolution_clock::now();
    fprintf(stderr, "[osfm_ba] %-12s %8.3f ms\n", what, std::chrono::duration<double, std::milli>(now - rs.t_prev).count());
    rs.t_prev = now;
  }
  // ba_linearize at parameter set b, specialised when every camera has the same projection type.  Minimum blocks
  // per SM (NB): MODE 0 (cost) 3; MODE 1 (Jacobian) 5 perspective, 4 Brown, 5 fisheye, 3 generic.
  template <int MODE>
  void launch_linearize(int b) {
    const int grid = grid_for(rs.N, 128);
    switch (rs.uniform_type) {
      case PT_PERSPECTIVE: ba_linearize<MODE, MODE == 1 ? 5 : 3, PT_PERSPECTIVE><<<grid, 128, 0, stream>>>(rs.v, params_of(b), d_sc.p, nullptr); break;
      case PT_BROWN: ba_linearize<MODE, MODE == 1 ? 4 : 3, PT_BROWN><<<grid, 128, 0, stream>>>(rs.v, params_of(b), d_sc.p, nullptr); break;
      case PT_FISHEYE: ba_linearize<MODE, MODE == 1 ? 5 : 3, PT_FISHEYE><<<grid, 128, 0, stream>>>(rs.v, params_of(b), d_sc.p, nullptr); break;
      default: ba_linearize<MODE, 3><<<grid, 128, 0, stream>>>(rs.v, params_of(b), d_sc.p, nullptr); break;
    }
    OSFM_LAUNCH_CHECK();
  }
  // The five ba_update launches: parameter set dst = src - alpha * scale * y over cameras, rig instances, rig cameras,
  // points and ext blocks (ext blocks projected onto `lower` when given); accumulates |delta|^2 and |x|^2.
  void update_params(int src, int dst, double alpha, const double* lower) {
    const Params a = params_of(src), b = params_of(dst);
    const int K = rs.K, NI = rs.NI, NR = rs.NR, P = rs.P, NE = rs.NE;
    if (K) { ba_update<<<grid_for(K, 128), 128, 0, stream>>>(0, K, d_cam_poff.p, d_cam_off.p, d_cam_np.p, 0, 0, a.cam, b.cam, d_scale.p, d_y.p, d_sc.p, rank == 0, nullptr, alpha); OSFM_LAUNCH_CHECK(); }
    if (NI) { ba_update<<<grid_for(NI, 128), 128, 0, stream>>>(1, NI, d_inst_poff.p, nullptr, nullptr, 6, 0, a.inst, b.inst, d_scale.p, d_y.p, d_sc.p, rank == 0, nullptr, alpha); OSFM_LAUNCH_CHECK(); }
    if (NR) { ba_update<<<grid_for(NR, 128), 128, 0, stream>>>(2, NR, d_rc_poff.p, nullptr, nullptr, 6, 0, a.rc, b.rc, d_scale.p, d_y.p, d_sc.p, rank == 0, nullptr, alpha); OSFM_LAUNCH_CHECK(); }
    if (P) { ba_update<<<grid_for(P, 128), 128, 0, stream>>>(3, P, d_pt_poff.p, nullptr, nullptr, 3, rs.nc, a.pts, b.pts, d_scale.p, d_y.p, d_sc.p, 1, nullptr, alpha); OSFM_LAUNCH_CHECK(); }
    if (NE) { ba_update<<<grid_for(NE, 128), 128, 0, stream>>>(0, NE, d_ext_poff.p, d_ext_off.p, d_ext_np.p, 0, 0, a.ext, b.ext, d_scale.p, d_y.p, d_sc.p, rank == 0, lower, alpha); OSFM_LAUNCH_CHECK(); }
  }
  // |x|^2 of the free parameters of set b into Scalars::x_norm2
  void x_norm_pass(int b) {
    OSFM_CUDA(cudaMemsetAsync(&d_sc.p->x_norm2, 0, sizeof(double), stream));
    OSFM_CUDA(cudaMemsetAsync(d_y.p, 0, sizeof(double) * rs.nz, stream));
    update_params(b, b, 1.0, nullptr);
    allreduce_dev(&d_sc.p->x_norm2, 1);
  }
  // Parameter set 0 holds the accepted parameters, set 1 the candidate
  Params params_of(int b) { return Params{d_cam[b].p, d_inst[b].p, d_rc[b].p, d_pts[b].p, d_ext[b].p}; }
  RunState rs;

  void run();
  void plan_layout(), order_observations(), plan_prior_rows(), upload_problem(), discover_structure(), plan_pcg(),
      reserve_covariance(), build_segment_tables(), segment_table_scales();
  void eval_cost(int b), linearize(int b, bool timed);
  void build_system(const double* diag, double inv_radius, int* rank_flag, bool timed), back_substitute();
  void solve_reduced(), lm_iteration(), line_search(), accept_candidate(), run_lm_graph();
  void capture_linear_system(int it, double radius), covariance_pass(int termination);
  void write_results(osfm_ba_summary sum);
};

// Validation (errors mirror the reference's: missing ids -> runtime_error), layout of the reduced vector [free cameras |
// instances | rig cameras | ext blocks], side-term offsets, preconditioner groups, Jacobian plane widths.  Host only.
void BA::plan_layout() {
  const int K = (int)cam_type.size(), NI = (int)inst_const.size(), NR = (int)rc_const.size(), S = (int)shot_inst.size();
  const int NE = (int)ext_size.size(), NT = (int)side_terms.size();
  rs.K = K; rs.NI = NI; rs.NR = NR; rs.NE = NE; rs.NT = NT; rs.S = S; rs.Pfull = (int)pt_const.size(); rs.Nfull = n_obs_full;
  for (int s = 0; s < S; ++s) {
    if (shot_inst[s] < 0 || shot_inst[s] >= NI) throw ArgError("shot references a rig instance that doesn't exist");
    if (shot_cam[s] < 0 || shot_cam[s] >= K) throw ArgError("shot references a camera that doesn't exist");
    if (shot_use_rc[s] && (shot_rc[s] < 0 || shot_rc[s] >= NR))
      throw ArgError("shot references a rig camera that doesn't exist");
  }
  // (observation indices are checked on the device, ord_make_keys)
  trace("validate");

  // offset in the reduced vector and parameter-block id of every camera / rig instance / rig camera / ext block
  rs.cam_off.assign(K + 1, 0); rs.cam_np.assign(K, 0); rs.cam_poff.assign(K, -1); rs.inst_poff.assign(NI, -1);
  rs.rc_poff.assign(std::max(NR, 1), -1); rs.ext_off.assign(NE + 1, 0); rs.ext_poff.assign(std::max(NE, 1), -1);
  rs.cam_blk.assign(std::max(K, 1), -1); rs.inst_blk.assign(std::max(NI, 1), -1); rs.rc_blk.assign(std::max(NR, 1), -1);
  rs.ext_blk.assign(std::max(NE, 1), -1);
  int nc = 0;
  auto add_block = [&](int size, int& poff, int& blk) {
    poff = nc; blk = (int)rs.blk_off.size();
    rs.blk_off.push_back(nc); rs.blk_sz.push_back(size); nc += size;
  };
  for (int k = 0; k < K; ++k) {
    rs.cam_np[k] = model_num_params(cam_type[k]);
    rs.cam_off[k + 1] = rs.cam_off[k] + rs.cam_np[k];
  }
  for (int k = 0; k < K; ++k) if (!cam_const[k]) add_block(rs.cam_np[k], rs.cam_poff[k], rs.cam_blk[k]);
  for (int i = 0; i < NI; ++i) if (!inst_const[i]) add_block(6, rs.inst_poff[i], rs.inst_blk[i]);
  for (int i = 0; i < NR; ++i) if (!rc_const[i]) add_block(6, rs.rc_poff[i], rs.rc_blk[i]);
  for (int i = 0; i < NE; ++i) {
    if (ext_size[i] < 1 || ext_size[i] > MAXB) throw ArgError("ext block size must be in [1, 16]");
    rs.ext_off[i + 1] = rs.ext_off[i] + ext_size[i];
    if (ext_const[i]) continue;
    add_block(ext_size[i], rs.ext_poff[i], rs.ext_blk[i]);
    for (int j = 0; j < ext_size[i]; ++j) rs.constrained |= std::isfinite(ext_lower[rs.ext_off[i] + j]);
  }
  rs.nc = nc;
  rs.nblk = (int)rs.blk_off.size();
  rs.nc_pad = (nc + 15) / 16 * 16;  // rhs sits in front of the reduced system in one buffer
  // side terms: block references checked here (the reference's std::map::at / "doesn't exist" errors)
  rs.side_jofs.assign(NT + 1, 0); rs.side_rofs.assign(NT + 1, 0);
  for (int t = 0; t < NT; ++t) {
    const osfm_side_term& st = side_terms[t];
    if (st.type < 0 || st.type >= OSFM_SIDE_NUM_TYPES) throw ArgError("unknown side term type");
    if (st.nblocks < 1 || st.nblocks > SIDE_MAX_BLOCKS || st.nres < 1 || st.nres > SIDE_MAX_RES)
      throw ArgError("side term with a bad block / residual count");
    int np = 0;
    for (int b = 0; b < st.nblocks; ++b) {
      const int kd = st.kind[b], ix = st.idx[b];
      const int cnt = kd == SB_CAM ? K : kd == SB_INST ? NI : kd == SB_RIGCAM ? NR : kd == SB_EXT ? NE : -1;
      if (ix < 0 || ix >= cnt) throw ArgError("side term references a parameter block that doesn't exist");
      np += kd == SB_CAM ? model_num_params(cam_type[ix]) : kd == SB_EXT ? ext_size[ix] : 6;
    }
    if (np > SIDE_MAX_PARAMS) throw ArgError("side term with too many parameters");
    if (st.cofs < 0 || (size_t)st.cofs > side_consts.size()) throw ArgError("side term constants out of range");
    rs.side_jofs[t + 1] = rs.side_jofs[t] + st.nres * np;
    rs.side_rofs[t + 1] = rs.side_rofs[t] + st.nres;
  }

  // preconditioner groups: a camera and the rig instance that is its only user (and vice versa) are
  // merged into one diagonal block when they fit (C + 6 <= 16); everything else stays on its own
  {
    std::vector<int> cam_user(std::max(K, 1), -1), inst_cam(std::max(NI, 1), -1);  // -1 none, -2 several
    for (int s2 = 0; s2 < S; ++s2) {
      const int k = shot_cam[s2], i = shot_inst[s2];
      cam_user[k] = cam_user[k] == -1 || cam_user[k] == i ? i : -2;
      inst_cam[i] = inst_cam[i] == -1 || inst_cam[i] == k ? k : -2;
    }
    std::vector<char> inst_done(std::max(NI, 1), 0);
    for (int k = 0; k < K; ++k) {
      if (rs.cam_blk[k] < 0) continue;
      const int i = cam_user[k];
      if (i >= 0 && rs.inst_blk[i] >= 0 && inst_cam[i] == k && rs.cam_np[k] + 6 <= 16) {
        rs.grp_b1.push_back(rs.cam_blk[k]); rs.grp_b2.push_back(rs.inst_blk[i]); inst_done[i] = 1;
      } else {
        rs.grp_b1.push_back(rs.cam_blk[k]); rs.grp_b2.push_back(-1);
      }
    }
    for (int i = 0; i < NI; ++i)
      if (rs.inst_blk[i] >= 0 && !inst_done[i]) { rs.grp_b1.push_back(rs.inst_blk[i]); rs.grp_b2.push_back(-1); }
    for (int i = 0; i < NR; ++i)
      if (rs.rc_blk[i] >= 0) { rs.grp_b1.push_back(rs.rc_blk[i]); rs.grp_b2.push_back(-1); }
    for (int i = 0; i < NE; ++i)
      if (rs.ext_blk[i] >= 0) { rs.grp_b1.push_back(rs.ext_blk[i]); rs.grp_b2.push_back(-1); }
  }
  rs.ngroups = (int)rs.grp_b1.size();

  for (int s = 0; s < S; ++s) {
    rs.wc = std::max(rs.wc, rs.cam_np[shot_cam[s]] + 6 + (shot_use_rc[s] ? 6 : 0));
    if (cam_type[shot_cam[s]] == PT_SPHERICAL) rs.nres = 3;
  }
  rs.wc = std::max(rs.wc, 1);
  // one projection type for all cameras and no rig-camera shots -> specialised linearisation kernels
  if (!(fallbacks & OSFM_BA_FALLBACK_GENERIC_LINEARIZE) && K > 0) {
    int& t = rs.uniform_type;
    t = cam_type[0];
    for (int k = 1; k < K; ++k) if (cam_type[k] != t) t = -1;
    for (int s = 0; s < S && t >= 0; ++s) if (shot_use_rc[s]) t = -1;
    if (t != PT_PERSPECTIVE && t != PT_BROWN && t != PT_FISHEYE) t = -1;
  }
  if (rs.Nfull >= (1LL << 31)) throw ArgError("too many observations");
  for (int q : pp_point)
    if (q < 0 || q >= rs.Pfull) throw ArgError("point prior on a point that doesn't exist");
  rs.have_pp = !pp_point.empty();
  rs.add_priors = rank == 0;
}

// Orders the observations on the device (ba_order.cuh): shards points over ranks (p % world == rank), sorts by
// (point, shot) and puts points seen by exactly the same shots next to each other (segments of the fast Schur path).
// The segmented Schur path (ba_point_blocks + the segment kernels) is the default: points seen by the same shots
// share their camera-side rows, which the per-point kernel re-reads point by point.
void BA::order_observations() {
  const long long Nfull = rs.Nfull;
  const int S = rs.S, Pfull = rs.Pfull, wc = rs.wc;
  const int P = rs.P = Pfull > rank ? (Pfull - rank + world - 1) / world : 0;
  const size_t Nfz = (size_t)std::max<long long>(Nfull, 1), Pz = (size_t)std::max(P, 1);
  {
    std::vector<int> ptc = pt_const;
    for (int& c : ptc) c = c ? 1 : 0;
    for (int q : pp_point) ptc[q] |= 2;
    upload(d_ptc_full, ptc, stream);
    OSFM_CUDA(cudaStreamSynchronize(stream));  // ptc goes out of scope
  }
  upload(d_pts_in, pts, stream);
  d_okeys.reserve(Nfz); d_okeys2.reserve(Nfz); d_ovals.reserve(Nfz); d_ovals2.reserve(Nfz);
  d_g_pt_start.reserve((size_t)Pfull + 1);
  d_pkey.reserve(Pz); d_pkey2.reserve(Pz); d_pval.reserve(Pz); d_order.reserve(Pz); d_inv_order.reserve(Pz);
  d_global_of.reserve(Pz); d_free_flag.reserve(Pz + 1); d_free_scan.reserve(Pz + 1); d_kk.reserve(Pz + 1);
  d_pt_start.reserve(Pz + 1); d_pt_poff.reserve(Pz); d_head.reserve(Pz); d_run_head.reserve(Pz);
  d_seg_flags.reserve(Pz); d_seg_start.reserve(Pz + 1); d_nsel.reserve(1); d_oc.reserve(1); h_oc.reserve(1);
  d_pts[0].reserve(3 * Pz); d_pts[1].reserve(3 * Pz);
  int pbits = 1;
  while ((1LL << pbits) <= (long long)Pfull) ++pbits;
  {
    size_t t1 = 0, t2 = 0, t3 = 0, t4 = 0, t5 = 0, t6 = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, t1, d_okeys.p, d_okeys2.p, d_ovals.p, d_ovals2.p, (int)Nfull, 0, 32 + pbits, stream);
    cub::DeviceRadixSort::SortPairs(nullptr, t2, d_pkey.p, d_pkey2.p, d_pval.p, d_order.p, P, 0, 64, stream);
    cub::DeviceScan::ExclusiveSum(nullptr, t3, d_kk.p, d_pt_start.p, P + 1, stream);
    cub::DeviceScan::ExclusiveSum(nullptr, t4, d_free_flag.p, d_free_scan.p, P + 1, stream);
    cub::DeviceScan::InclusiveScan(nullptr, t5, d_head.p, d_run_head.p, OrdMax(), P, stream);
    cub::DeviceSelect::Flagged(nullptr, t6, thrust::counting_iterator<int>(0), d_seg_flags.p, d_seg_start.p, d_nsel.p, P, stream);
    d_cub.reserve(std::max({t1, t2, t3, t4, t5, t6}) + 256);
  }
  OSFM_CUDA(cudaMemsetAsync(d_oc.p, 0, sizeof(OrderCounts), stream));
  ord_make_keys<<<grid_for(Nfull, 256), 256, 0, stream>>>(Nfull, d_raw_shot.p, d_raw_point.p, S, Pfull, d_okeys.p, d_ovals.p, d_oc.p);
  OSFM_LAUNCH_CHECK();
  size_t tmpb = d_cub.cap;
  OSFM_CUDA(cub::DeviceRadixSort::SortPairs(d_cub.p, tmpb, d_okeys.p, d_okeys2.p, d_ovals.p, d_ovals2.p, (int)Nfull, 0, 32 + pbits, stream));
  const unsigned long long* okeys = d_okeys2.p;  // sorted keys / positions in the caller's list
  const int* ovals = d_ovals2.p;
  ord_point_starts<<<grid_for(Pfull + 1, 256), 256, 0, stream>>>(okeys, Nfull, Pfull, d_g_pt_start.p);
  OSFM_LAUNCH_CHECK();
  ord_pair_bound<<<grid_for(Pfull, 256), 256, 0, stream>>>(d_g_pt_start.p, Pfull, d_oc.p);
  OSFM_LAUNCH_CHECK();
  ord_signatures<<<grid_for(P, 256), 256, 0, stream>>>(okeys, d_g_pt_start.p, d_ptc_full.p, P, world, rank, wc,
                                                       (fallbacks & OSFM_BA_FALLBACK_PER_POINT_SCHUR) ? 0 : 1, SEG_KMAX,
                                                       SEG_NA, SEG_WCMAX, d_pkey.p, d_pval.p);
  OSFM_LAUNCH_CHECK();
  tmpb = d_cub.cap;
  OSFM_CUDA(cub::DeviceRadixSort::SortPairs(d_cub.p, tmpb, d_pkey.p, d_pkey2.p, d_pval.p, d_order.p, P, 0, 64, stream));
  ord_counts<<<grid_for(P + 1, 256), 256, 0, stream>>>(d_order.p, d_g_pt_start.p, d_ptc_full.p, P, world, rank, d_kk.p,
                                                       d_free_flag.p, d_inv_order.p, d_global_of.p);
  OSFM_LAUNCH_CHECK();
  tmpb = d_cub.cap;
  OSFM_CUDA(cub::DeviceScan::ExclusiveSum(d_cub.p, tmpb, d_kk.p, d_pt_start.p, P + 1, stream));
  tmpb = d_cub.cap;
  OSFM_CUDA(cub::DeviceScan::ExclusiveSum(d_cub.p, tmpb, d_free_flag.p, d_free_scan.p, P + 1, stream));
  ord_finish_points<<<grid_for(P + 1, 256), 256, 0, stream>>>(P, d_free_flag.p, d_free_scan.p, d_pt_start.p, d_global_of.p,
                                                              d_pts_in.p, d_pt_poff.p, d_pts[0].p, d_pts[1].p, d_oc.p);
  OSFM_LAUNCH_CHECK();
  OSFM_CUDA(cudaMemcpyAsync(h_oc.p, d_oc.p, sizeof(OrderCounts), cudaMemcpyDeviceToHost, stream));
  OSFM_CUDA(cudaStreamSynchronize(stream));
  if (h_oc.p->err & 1) throw ArgError("observation references a shot that doesn't exist");
  if (h_oc.p->err & 2) throw ArgError("observation references a point that doesn't exist");
  const long long N = rs.N = h_oc.p->n_local;
  rs.npf = h_oc.p->npf;
  rs.n = rs.nc + 3 * rs.npf;
  rs.n_all = rs.nc;
  for (int c : pt_const) rs.n_all += c ? 0 : 3;
  rs.nz = (size_t)std::max(rs.n, 1);
  {
    const size_t Nz0 = (size_t)std::max<long long>(N, 1);
    d_obs_orig.reserve(Nz0); d_obs_shot.reserve(Nz0); d_obs_point.reserve(Nz0);
    d_obs_x.reserve(Nz0); d_obs_y.reserve(Nz0); d_obs_isig.reserve(Nz0);
  }
  if (obs_pending) {   // image coordinates / standard deviations uploaded by osfm_ba_set_observations_async
    OSFM_CUDA(cudaStreamWaitEvent(stream, ev_obs, 0));
    obs_pending = false;
  }
  ord_gather_obs<<<grid_for(Nfull, 256), 256, 0, stream>>>(okeys, ovals, Nfull, d_g_pt_start.p, d_inv_order.p, d_pt_start.p, world,
                                                           rank, d_raw_xy.p, d_raw_sigma.p, d_obs_orig.p, d_obs_shot.p,
                                                           d_obs_point.p, d_obs_x.p, d_obs_y.p, d_obs_isig.p);
  OSFM_LAUNCH_CHECK();
  ord_seg_heads<<<grid_for(P, 256), 256, 0, stream>>>(P, d_pkey2.p, d_order.p, d_g_pt_start.p, okeys, d_ptc_full.p, world, rank,
                                                      d_head.p);
  OSFM_LAUNCH_CHECK();
  tmpb = d_cub.cap;
  OSFM_CUDA(cub::DeviceScan::InclusiveScan(d_cub.p, tmpb, d_head.p, d_run_head.p, OrdMax(), P, stream));
  ord_seg_flags<<<grid_for(P, 256), 256, 0, stream>>>(P, d_pkey2.p, d_run_head.p, d_seg_flags.p);
  OSFM_LAUNCH_CHECK();
  tmpb = d_cub.cap;
  OSFM_CUDA(cub::DeviceSelect::Flagged(d_cub.p, tmpb, thrust::counting_iterator<int>(0), d_seg_flags.p, d_seg_start.p, d_nsel.p, P,
                                       stream));
  ord_seg_finish<<<1, 32, 0, stream>>>(P, d_pkey2.p, d_pt_start.p, d_seg_start.p, d_nsel.p, d_oc.p);
  OSFM_LAUNCH_CHECK();
  if (world > 1) {  // the structure of the reduced system needs every point's shots on every rank
    d_g_obs_shot.reserve(Nfz); d_g_obs_point.reserve(Nfz);
    ord_split_keys<<<grid_for(Nfull, 256), 256, 0, stream>>>(okeys, Nfull, d_g_obs_shot.p, d_g_obs_point.p);
    OSFM_LAUNCH_CHECK();
  }
  OSFM_CUDA(cudaMemcpyAsync(h_oc.p, d_oc.p, sizeof(OrderCounts), cudaMemcpyDeviceToHost, stream));
  OSFM_CUDA(cudaStreamSynchronize(stream));
  rs.nseg = h_oc.p->nseg; rs.P_fast = h_oc.p->p_fast;
  rs.n_fast_obs = h_oc.p->n_fast; rs.pair_bound = (long long)h_oc.p->pair_bound;
  if (tracing())
    fprintf(stderr, "[osfm_ba] points %d (fast path %d in %d segments), observations %lld (fast path %lld), free points %d\n", P,
            rs.P_fast, rs.nseg, N, rs.n_fast_obs, rs.npf);
}

// Prior rows (rank 0 adds them; Ceres drops residuals of constant blocks), each with its diagonal entry
void BA::plan_prior_rows() {
  for (int k = 0; k < rs.K; ++k) {
    if (rs.cam_poff[k] < 0) continue;
    for (int j = 0; j < rs.cam_np[k]; ++j) {
      const int idx = rs.cam_off[k] + j;
      rs.pr_cam_param.push_back(idx);
      rs.pr_cam_col.push_back(rs.cam_poff[k] + j);
      rs.pr_cam_log.push_back(cam_prior_log[idx]);
      rs.pr_cam_prior.push_back(cam_prior[idx]);
      rs.pr_cam_scale.push_back(1.0 / std::max(cam_prior_sigma[idx], DBL_EPSILON));  // prior_error.h:31-35
      rs.pr_blk.push_back(rs.cam_blk[k]); rs.pr_local.push_back(j);
    }
  }
  // kind 1: rig-instance position (axes 3..5), kind 2: rig-camera pose
  auto pos_row = [&](int kind, int i, int axis, int poff, int blk, double prior, double sigma) {
    rs.pr_pos_kind.push_back(kind); rs.pr_pos_inst.push_back(i); rs.pr_pos_axis.push_back(axis); rs.pr_pos_col.push_back(poff + axis);
    rs.pr_pos_prior.push_back(prior);
    rs.pr_pos_scale.push_back(1.0 / std::max(sigma, DBL_EPSILON));
    rs.pr_blk.push_back(blk); rs.pr_local.push_back(axis);
  };
  for (int i = 0; i < rs.NI; ++i) {
    if (!inst_has_prior[i] || rs.inst_poff[i] < 0) continue;
    for (int j = 0; j < 3; ++j)
      pos_row(1, i, 3 + j, rs.inst_poff[i], rs.inst_blk[i], inst_prior_pos[3 * (size_t)i + j], inst_prior_std[3 * (size_t)i + j]);
  }
  for (int i = 0; i < rs.NR && !rc_prior.empty(); ++i) {   // DataPriorError<Pose> on every free rig camera (:779-790)
    if (rs.rc_poff[i] < 0) continue;
    for (int j = 0; j < 6; ++j)
      pos_row(2, i, j, rs.rc_poff[i], rs.rc_blk[i], rc_prior[6 * (size_t)i + j], rc_prior_sigma[6 * (size_t)i + j]);
  }
}

void BA::upload_problem() {
  const int NT = rs.NT, P = rs.P, Pfull = rs.Pfull, nc = rs.nc, npf = rs.npf, nres = rs.nres, wc = rs.wc;
  upload(d_cam_type, cam_type, stream); upload(d_cam_off, rs.cam_off, stream); upload(d_cam_np, rs.cam_np, stream);
  upload(d_cam_poff, rs.cam_poff, stream); upload(d_inst_poff, rs.inst_poff, stream); upload(d_rc_poff, rs.rc_poff, stream);
  upload(d_shot_inst, shot_inst, stream); upload(d_shot_cam, shot_cam, stream); upload(d_shot_rc, shot_rc, stream);
  upload(d_shot_use_rc, shot_use_rc, stream);
  std::vector<double> rc_h = rc;
  if (rc_h.empty()) rc_h.assign(6, 0.0);
  for (int b = 0; b < 2; ++b) {
    upload(d_cam[b], cam_params, stream); upload(d_inst[b], inst, stream); upload(d_rc[b], rc_h, stream);
  }
  upload(d_blk_off, rs.blk_off, stream); upload(d_blk_sz, rs.blk_sz, stream);
  upload(d_cam_blk, rs.cam_blk, stream); upload(d_inst_blk, rs.inst_blk, stream); upload(d_rc_blk, rs.rc_blk, stream);
  upload(d_pr_blk, rs.pr_blk, stream); upload(d_pr_local, rs.pr_local, stream);
  upload(d_grp_b1, rs.grp_b1, stream); upload(d_grp_b2, rs.grp_b2, stream);
  upload(d_pr_cam_param, rs.pr_cam_param, stream); upload(d_pr_cam_col, rs.pr_cam_col, stream);
  upload(d_pr_cam_log, rs.pr_cam_log, stream); upload(d_pr_cam_prior, rs.pr_cam_prior, stream);
  upload(d_pr_cam_scale, rs.pr_cam_scale, stream); upload(d_pr_pos_inst, rs.pr_pos_inst, stream);
  upload(d_pr_pos_axis, rs.pr_pos_axis, stream); upload(d_pr_pos_col, rs.pr_pos_col, stream);
  upload(d_pr_pos_kind, rs.pr_pos_kind, stream);
  // ext blocks, side terms, point priors
  std::vector<double> ev = ext_values, el = ext_lower;
  if (ev.empty()) { ev.assign(1, 0.0); el.assign(1, 0.0); }
  upload(d_ext[0], ev, stream); upload(d_ext[1], ev, stream); upload(d_ext_lower, el, stream);
  upload(d_ext_off, rs.ext_off, stream); upload(d_ext_np, ext_size, stream); upload(d_ext_poff, rs.ext_poff, stream);
  upload(d_ext_blk, rs.ext_blk, stream);
  upload(d_side_terms, side_terms, stream); upload(d_side_consts, side_consts, stream);
  upload(d_side_jofs, rs.side_jofs, stream); upload(d_side_rofs, rs.side_rofs, stream);
  d_side_J.reserve((size_t)rs.side_jofs[NT] + 1); d_side_r.reserve((size_t)rs.side_rofs[NT] + 1);
  std::vector<double> ppd, ppx;
  if (rs.have_pp) {
    ppd.assign(3 * (size_t)Pfull, 0.0); ppx.assign(3 * (size_t)Pfull, 0.0);
    for (size_t q = 0; q < pp_point.size(); ++q) {
      const size_t g = (size_t)pp_point[q];
      for (int j = 0; j < (pp_alt[q] ? 3 : 2); ++j) {
        ppd[3 * g + j] = 1.0 / std::max(pp_sigma[3 * q + j], DBL_EPSILON);   // prior_error.h:31-35
        ppx[3 * g + j] = pp_prior[3 * q + j];
      }
    }
    upload(d_pp_d, ppd, stream); upload(d_pp_x0, ppx, stream);
  }
  OSFM_CUDA(cudaStreamSynchronize(stream));  // local vectors go out of scope
  upload(d_pr_pos_prior, rs.pr_pos_prior, stream); upload(d_pr_pos_scale, rs.pr_pos_scale, stream);
  const size_t Nz = (size_t)std::max<long long>(rs.N, 1);
  d_r.reserve(nres * Nz); d_Jc.reserve((size_t)nres * wc * Nz); d_Jp.reserve((size_t)nres * 3 * Nz);
  d_Vinv.reserve(6 * (size_t)std::max(npf, 1)); d_gp.reserve(3 * (size_t)std::max(npf, 1));
  d_Vig.reserve(3 * (size_t)std::max(npf, 1)); d_bs_t.reserve(3 * (size_t)std::max(npf, 1));
  const size_t nz = rs.nz;
  d_scale.reserve(nz); d_colnorm2.reserve(nz); d_grad.reserve(nz); d_diag.reserve(nz); d_diag_r.reserve(nz); d_y.reserve(nz);
  d_px.reserve(std::max(nc, 1)); d_pr.reserve(std::max(nc, 1)); d_pz.reserve(std::max(nc, 1));
  d_pp.reserve(std::max(nc, 1)); d_pAp.reserve(std::max(nc, 1));
  d_pm.reserve(4 * (size_t)std::max(nc, 1));
  d_pcg.reserve(1);
  d_Minv.reserve((size_t)std::max(rs.ngroups, 1) * MAXB * MAXB);
  d_Ap.reserve(std::max(nc, 1));
  d_sc.reserve(1);

  BAView& v = rs.v;
  v.K = rs.K; v.NI = rs.NI; v.NR = rs.NR; v.S = rs.S; v.P = P; v.N = rs.N; v.nc = nc; v.npf = npf; v.wc = wc; v.nres = nres;
  v.loss = loss; v.loss_a = loss_a;
  v.cam_type = d_cam_type.p; v.cam_off = d_cam_off.p; v.cam_np = d_cam_np.p; v.cam_poff = d_cam_poff.p;
  v.inst_poff = d_inst_poff.p; v.rc_poff = d_rc_poff.p; v.pt_poff = d_pt_poff.p;
  v.shot_inst = d_shot_inst.p; v.shot_cam = d_shot_cam.p; v.shot_rc = d_shot_rc.p; v.shot_use_rc = d_shot_use_rc.p;
  v.obs_shot = d_obs_shot.p; v.obs_point = d_obs_point.p; v.obs_x = d_obs_x.p; v.obs_y = d_obs_y.p;
  v.obs_isig = d_obs_isig.p; v.obs_orig = d_obs_orig.p; v.pt_start = d_pt_start.p;
  v.r = d_r.p; v.Jc = d_Jc.p; v.Jp = d_Jp.p;
  PriorView& pv = rs.pv;
  pv.n_cam_rows = rs.add_priors ? (int)rs.pr_cam_param.size() : 0;
  pv.n_pos_rows = rs.add_priors ? (int)rs.pr_pos_inst.size() : 0;
  pv.cam_row_param = d_pr_cam_param.p; pv.cam_row_col = d_pr_cam_col.p; pv.cam_row_log = d_pr_cam_log.p;
  pv.cam_row_prior = d_pr_cam_prior.p; pv.cam_row_scale = d_pr_cam_scale.p;
  pv.pos_row_kind = d_pr_pos_kind.p;
  pv.pos_row_inst = d_pr_pos_inst.p; pv.pos_row_axis = d_pr_pos_axis.p; pv.pos_row_col = d_pr_pos_col.p;
  pv.pos_row_prior = d_pr_pos_prior.p; pv.pos_row_scale = d_pr_pos_scale.p;
  SideView& sv = rs.sv;
  sv.n = NT; sv.terms = d_side_terms.p; sv.consts = d_side_consts.p; sv.jofs = d_side_jofs.p; sv.rofs = d_side_rofs.p;
  sv.J = d_side_J.p; sv.r = d_side_r.p;
  sv.ext_off = d_ext_off.p; sv.ext_np = d_ext_np.p; sv.ext_poff = d_ext_poff.p; sv.ext_blk = d_ext_blk.p;
  rs.ppv = PointPriorView{rs.have_pp ? d_pp_d.p : nullptr, d_pp_x0.p, d_global_of.p};
  rs.bm = BlkMaps{d_cam_blk.p, d_inst_blk.p, d_rc_blk.p};
}

// Block-sparse structure of the reduced camera system (identical on every rank) and the block-row ELL layout of the
// PCG mat-vec
void BA::discover_structure() {
  const int nblk = rs.nblk, nc = rs.nc, NT = rs.NT;
  if (nblk > 0) {
    // global CSR by point (every rank needs the same structure, not only its shard)
    const int* g_shot = d_obs_shot.p;
    const int* g_point = d_obs_point.p;
    const long long* g_start = d_pt_start.p;
    if (world > 1) { g_shot = d_g_obs_shot.p; g_point = d_g_obs_point.p; g_start = d_g_pt_start.p; }
    const long long bound = std::min<long long>((long long)nblk * (nblk + 1) / 2, 9 * rs.pair_bound + nblk + 21LL * NT);
    unsigned tsize = 1024;
    while ((long long)tsize < 4 * bound) {
      if (tsize >= (1u << 28)) throw std::runtime_error("reduced camera system has too many block pairs");
      tsize <<= 1;
    }
    d_tkeys.reserve(tsize); d_tvals.reserve(tsize);
    OSFM_CUDA(cudaMemsetAsync(d_tkeys.p, 0xff, sizeof(unsigned long long) * tsize, stream));
    const long long n_enum = world > 1 ? rs.Nfull : rs.N;
    if (n_enum > 0) {   // only the shot tables of the view are used by the enumeration
      bsr_enum_pairs<<<grid_for(n_enum, 128), 128, 0, stream>>>(rs.v, rs.bm, g_shot, g_start, g_point, n_enum, d_tkeys.p,
                                                              tsize - 1, nblk);
      OSFM_LAUNCH_CHECK();
    }
    if (NT > 0) {
      side_enum_pairs<<<grid_for(NT, 128), 128, 0, stream>>>(rs.sv, rs.v, rs.bm, params_of(0), d_tkeys.p, tsize - 1, nblk);
      OSFM_LAUNCH_CHECK();
    }
    bsr_insert_diagonal<<<grid_for(nblk, 128), 128, 0, stream>>>(d_tkeys.p, tsize - 1, nblk);
    OSFM_LAUNCH_CHECK();
    const size_t cap = (size_t)(2 * bound + 16);
    d_skeys.reserve(cap); d_skeys2.reserve(cap); d_rkeys.reserve(cap); d_rkeys2.reserve(cap);
    d_area.reserve(cap); d_offs.reserve(cap); d_count.reserve(4);
    OSFM_CUDA(cudaMemsetAsync(d_count.p, 0, sizeof(unsigned), stream));
    bsr_compact<<<grid_for(tsize, 256), 256, 0, stream>>>(d_tkeys.p, tsize, nblk, d_skeys.p, d_count.p);
    OSFM_LAUNCH_CHECK();
    unsigned n_all_u = 0;
    OSFM_CUDA(cudaMemcpyAsync(&n_all_u, d_count.p, sizeof(unsigned), cudaMemcpyDeviceToHost, stream));
    OSFM_CUDA(cudaStreamSynchronize(stream));
    const int n_all = (int)n_all_u;
    rs.n_blocks_all = n_all;
    const int n_upper = rs.n_upper = nblk + (n_all - nblk) / 2;
    // sort: upper keys (bit 63 clear) first, each group ordered by (bi, bj)
    size_t tmp1 = 0, tmp2 = 0;
    cub::DeviceRadixSort::SortKeys(nullptr, tmp1, d_skeys.p, d_skeys2.p, n_all, 0, 64, stream);
    cub::DeviceScan::ExclusiveSum(nullptr, tmp2, d_area.p, d_offs.p, n_all, stream);
    d_cub.reserve(std::max(tmp1, tmp2) + 256);
    size_t tmp = d_cub.cap;
    OSFM_CUDA(cub::DeviceRadixSort::SortKeys(d_cub.p, tmp, d_skeys.p, d_skeys2.p, n_all, 0, 64, stream));
    g_kernel_launches.fetch_add(1);
    bsr_block_areas<<<grid_for(n_all, 256), 256, 0, stream>>>(d_skeys2.p, n_all, nblk, d_blk_sz.p, d_area.p);
    OSFM_LAUNCH_CHECK();
    tmp = d_cub.cap;
    OSFM_CUDA(cub::DeviceScan::ExclusiveSum(d_cub.p, tmp, d_area.p, d_offs.p, n_all, stream));
    g_kernel_launches.fetch_add(1);
    int last_off[2] = {0, 0}, last_area = 0, upper_end = 0;
    OSFM_CUDA(cudaMemcpyAsync(&last_off[0], d_offs.p + n_all - 1, sizeof(int), cudaMemcpyDeviceToHost, stream));
    OSFM_CUDA(cudaMemcpyAsync(&last_area, d_area.p + n_all - 1, sizeof(int), cudaMemcpyDeviceToHost, stream));
    if (n_upper < n_all)
      OSFM_CUDA(cudaMemcpyAsync(&upper_end, d_offs.p + n_upper, sizeof(int), cudaMemcpyDeviceToHost, stream));
    OSFM_CUDA(cudaStreamSynchronize(stream));
    rs.s_total = (long long)last_off[0] + last_area;
    rs.s_upper_total = n_upper < n_all ? upper_end : rs.s_total;
    // hash table values (inserting the mirrored keys) + plain key list, then block-row lists
    bsr_fill_table<<<grid_for(n_all, 256), 256, 0, stream>>>(d_skeys2.p, d_offs.p, n_all, d_tkeys.p, d_tvals.p, tsize - 1,
                                                            d_rkeys.p);
    OSFM_LAUNCH_CHECK();
    tmp = d_cub.cap;
    OSFM_CUDA(cub::DeviceRadixSort::SortKeys(d_cub.p, tmp, d_rkeys.p, d_rkeys2.p, n_all, 0, 64, stream));
    g_kernel_launches.fetch_add(1);
    BsrView& bsr = rs.bsr;
    bsr.tkeys = d_tkeys.p; bsr.tvals = d_tvals.p; bsr.tmask = tsize - 1; bsr.nblk = nblk;
    bsr.blk_off = d_blk_off.p; bsr.blk_sz = d_blk_sz.p;
    d_row_ptr.reserve(nblk + 2); d_row_col.reserve(n_all + 1); d_row_off.reserve(n_all + 1);
    bsr_rows<<<grid_for(n_all + 1, 256), 256, 0, stream>>>(d_rkeys2.p, n_all, bsr, d_row_ptr.p, d_row_col.p, d_row_off.p);
    OSFM_LAUNCH_CHECK();
    d_upper.reserve(n_upper + 1);
    bsr_upper_list<<<grid_for(n_upper, 256), 256, 0, stream>>>(d_skeys2.p, d_offs.p, n_upper, bsr, d_upper.p);
    OSFM_LAUNCH_CHECK();
    d_diag_off.reserve(nblk + 1);
    bsr_diag_offsets<<<grid_for(nblk, 128), 128, 0, stream>>>(bsr, d_diag_off.p);
    OSFM_LAUNCH_CHECK();
    const int npr = (int)rs.pr_blk.size();
    d_prior_diag_off.reserve(npr + 1);
    if (npr > 0) {
      bsr_prior_offsets<<<grid_for(npr, 128), 128, 0, stream>>>(d_pr_blk.p, d_pr_local.p, npr, d_diag_off.p, d_blk_sz.p,
                                                               d_prior_diag_off.p);
      OSFM_LAUNCH_CHECK();
    }
    d_Sbuf.reserve((size_t)std::max<long long>(rs.s_total, 1) + rs.nc_pad);
    // block-row ELL layout of the PCG mat-vec
    d_row_M.reserve(nblk + 1); d_qoff.reserve(n_all + 1); d_blk_row.reserve(n_all + 1);
    pcg_row_sizes<<<grid_for(nblk, 128), 128, 0, stream>>>(d_row_ptr.p, d_row_col.p, bsr, d_row_M.p, d_qoff.p, d_blk_row.p);
    OSFM_LAUNCH_CHECK();
    rs.row_M.resize(nblk);
    OSFM_CUDA(cudaMemcpyAsync(rs.row_M.data(), d_row_M.p, sizeof(int) * nblk, cudaMemcpyDeviceToHost, stream));
    OSFM_CUDA(cudaStreamSynchronize(stream));
    rs.rowbase.resize(nblk);
    rs.cbase.resize(nblk);
    long long cbt = 0;
    for (int b = 0; b < nblk; ++b) {
      rs.rowbase[b] = rs.vb; rs.cbase[b] = (int)cbt;
      rs.vb += (long long)rs.blk_sz[b] * rs.row_M[b];
      cbt += rs.row_M[b];
    }
    upload(d_rowbase, rs.rowbase, stream); upload(d_cbase, rs.cbase, stream);
    d_colidx.reserve((size_t)cbt + 1); d_row_of.reserve(nc + 1); d_Spcg.reserve((size_t)rs.vb + 1);
    pcg_fill_colidx<<<grid_for(n_all, 128), 128, 0, stream>>>(d_row_col.p, d_qoff.p, d_blk_row.p, n_all, bsr, d_cbase.p,
                                                             d_colidx.p, d_row_of.p);
    OSFM_LAUNCH_CHECK();
  }
  if (nblk == 0) d_Sbuf.reserve(rs.nc_pad + 16);
  rs.d_rhs_p = d_Sbuf.p;
  rs.d_S_p = d_Sbuf.p + rs.nc_pad;
}

// Shared-memory plans of the two persistent PCG kernels (one CTA per SM: the grid barrier needs every CTA resident)
void BA::plan_pcg() {
  const int nc = rs.nc, nblk = rs.nblk, ngroups = rs.ngroups;
  const int G = rs.pcg_grid =
      std::max(1, std::min(std::min(num_sms, PCG_MAX_CTAS), (nc + PCG_THREADS / 32 - 1) / (PCG_THREADS / 32)));
  if (nblk > 0) {
    const std::vector<int>& row_M = rs.row_M;
    int max_smem = 0;
    OSFM_CUDA(cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
    // resident PCG: contiguous scalar-row ranges per CTA, balanced by stored entries; usable when every CTA's
    // slice of S + its column indices (uint16) + p fit in shared memory
    {
      std::vector<long long> off(nc + 1, 0);
      std::vector<int> row_blk(nc, 0);
      bool monotone = true;
      for (int b = 0; b < nblk; ++b) {
        for (int r = 0; r < rs.blk_sz[b]; ++r) {
          off[rs.blk_off[b] + r] = rs.rowbase[b] + (long long)r * row_M[b];
          row_blk[rs.blk_off[b] + r] = b;
        }
        if (b > 0 && rs.blk_off[b] != rs.blk_off[b - 1] + rs.blk_sz[b - 1]) monotone = false;
      }
      off[nc] = rs.vb;
      const std::vector<int> row_lo = balanced_cut(off, G);
      long long ent_max = 0, col_max = 0;
      int rows_max = 0;
      for (int c = 0; c < G; ++c) {
        const int lo = row_lo[c], hi = row_lo[c + 1];
        if (hi <= lo) continue;
        ent_max = std::max(ent_max, off[hi] - off[lo]);
        const int b_lo = row_blk[lo], b_hi = row_blk[hi - 1];
        col_max = std::max<long long>(col_max, (long long)rs.cbase[b_hi] + row_M[b_hi] - rs.cbase[b_lo]);
        rows_max = std::max(rows_max, hi - lo);
      }
      const long long off_S = up16(8LL * nc), off_cols = off_S + up16(8 * ent_max), off_rows = off_cols + up16(2 * col_max);
      const long long total = off_rows + 12LL * rows_max;
      rs.pcg_resident = !(fallbacks & OSFM_BA_FALLBACK_STREAMED_PCG) && monotone && nc <= 65535 &&
                        total + 1024 <= max_smem;
      rs.pcg_smem = rs.pcg_resident ? (int)total : 0;
      if (tracing())
        fprintf(stderr, "[osfm_ba] pcg plan: classic resident %s, %lld B of shared memory per CTA, %d B available\n",
                rs.pcg_resident ? "on" : "off", total, max_smem - 1024);
      if (rs.pcg_resident) {
        upload(d_pcg_rowlo, row_lo, stream);
        PcgResident& pr = rs.pcg_res;
        pr.row_lo = d_pcg_rowlo.p; pr.off_S = (int)off_S; pr.off_cols = (int)off_cols;
        pr.off_rows = (int)off_rows; pr.max_rows = rows_max;
        OSFM_CUDA(cudaFuncSetAttribute(pcg_persistent<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, rs.pcg_smem));
      }
    }
    // pipelined PCG: whole preconditioner groups per CTA (ba_pcg_plan.h)
    {
      std::vector<int> row_ptr, row_col;
      download(row_ptr, d_row_ptr.p, nblk + 1, stream);
      download(row_col, d_row_col.p, rs.n_blocks_all, stream);
      OSFM_CUDA(cudaStreamSynchronize(stream));
      std::vector<char> shared(ngroups, 0);
      for (int g = 0; g < ngroups; ++g) shared[g] = pcg_rows_share_columns(row_ptr, row_col, rs.grp_b1[g], rs.grp_b2[g]);
      cudaFuncAttributes pipe_attr{};
      OSFM_CUDA(cudaFuncGetAttributes(&pipe_attr, pcg_pipelined));
      const PcgPipePlan plan = plan_pcg_pipelined(rs.grp_b1, rs.grp_b2, rs.blk_sz, row_M, shared, G,
                                                  (long long)max_smem - (long long)pipe_attr.sharedSizeBytes - 1024);
      rs.pcg_pipe_ok = !(fallbacks & OSFM_BA_FALLBACK_CLASSIC_PCG) && nc <= 65535 && plan.fits;
      rs.pcg_pipe_smem = rs.pcg_pipe_ok ? (int)plan.total : 0;
      if (tracing())
        fprintf(stderr, "[osfm_ba] pcg plan: pipelined %s, %lld B of shared memory per CTA, %lld B available (%d CTAs, "
                "worst CTA: %lld entries, %lld columns, %d rows, %d groups)\n", rs.pcg_pipe_ok ? "on" : "off", plan.total,
                plan.available, G, plan.max.ent, plan.max.cols, plan.max.rows, plan.max.groups);
      if (rs.pcg_pipe_ok) {
        upload(d_pcg_grplo, plan.grp_lo, stream);
        upload(d_grp_shared, shared, stream);
        PcgPipe& pp = rs.pcg_pipe;
        pp.grp_lo = d_pcg_grplo.p; pp.grp_shared = d_grp_shared.p; pp.off_S = (int)plan.off_S;
        pp.off_Minv = (int)plan.off_Minv; pp.off_vec = (int)plan.off_vec; pp.off_cols = (int)plan.off_cols;
        pp.off_rows = (int)plan.off_rows; pp.max_rows = plan.max.rows; pp.max_groups = plan.max.groups;
        pp.max_cols = (int)plan.max.cols; pp.off_defl = (int)plan.off_defl; pp.Wdef = nullptr;
        OSFM_CUDA(cudaFuncSetAttribute(pcg_pipelined, cudaFuncAttributeMaxDynamicSharedMemorySize, rs.pcg_pipe_smem));
      }
    }
    OSFM_CUDA(cudaStreamSynchronize(stream));  // the uploads above read host vectors of this function
  }
  PcgLayout& lay = rs.lay;
  lay.row_of = d_row_of.p; lay.row_M = d_row_M.p; lay.rowbase = d_rowbase.p; lay.cbase = d_cbase.p;
  lay.colidx = d_colidx.p; lay.ngroups = ngroups; lay.grp_b1 = d_grp_b1.p; lay.grp_b2 = d_grp_b2.p;
}

// Workspace of the covariance pass, claimed before the LM loop so that a problem too large for a dense S fails here
// (the pass itself runs after the loop)
void BA::reserve_covariance() {
  const int nc = rs.nc;
  for (int i = 0; i < rs.NI; ++i)
    if (rs.inst_poff[i] >= 0) rs.cov_inst.push_back(i);
  rs.cov_m = 6 * (int)rs.cov_inst.size();
  // leading and instance columns are blocked separately: L22's diagonal blocks are blocks of the Cholesky
  for (int k = 0; k < nc - rs.cov_m; k += COV_NB) rs.cov_bstart.push_back(k);
  rs.cov_nb1 = (int)rs.cov_bstart.size();
  for (int k = nc - rs.cov_m; k < nc; k += COV_NB) rs.cov_bstart.push_back(k);
  const size_t nblocks = rs.cov_bstart.size();
  rs.cov_bstart.push_back(nc);
  const size_t total = (size_t)nc * nc + (size_t)rs.cov_m * rs.cov_m + nblocks * COV_NB * COV_NB + (size_t)nc +
                       (size_t)rs.NI * 36 + 1;
  if (total > d_cov.cap) {
    size_t free_b = 0, total_b = 0;
    OSFM_CUDA(cudaMemGetInfo(&free_b, &total_b));
    if (total * sizeof(double) > free_b + d_cov.cap * sizeof(double)) {
      char msg[256];
      snprintf(msg, sizeof(msg),
               "covariance estimation needs %zu bytes of device memory for the dense reduced camera system "
               "(n_c = %d) and its workspace; %zu bytes are free", total * sizeof(double), nc, free_b);
      throw ArgError(msg);
    }
    d_cov.release();
    OSFM_CUDA(cudaMalloc(&d_cov.p, total * sizeof(double)));
    d_cov.cap = total;
  }
  d_cov_flags.reserve(COV_F_COUNT);
}

// Structure of the segments, before the first linearisation (the Jacobi scales of the tables follow in
// segment_table_scales()): the per-segment tables (columns, block offsets), the segment chunk list and the flush table
// of the persistent Schur kernel.  Decides the Schur path and the linearisation path of the run.
void BA::build_segment_tables() {
  const int nseg = rs.nseg, wc = rs.wc;
  // The tensor-core kernels add the same-shot blocks J^T J only in the tiles (t, t) and (t, t + 1): a shot's wc
  // columns must not span three 8-wide tiles, i.e. wc <= 9.  Wider camera sides (Brown: 9 + 6, rig cameras: + 6)
  // use the SIMT segment kernels.
  if (nseg > 0 && rs.nblk > 0 && wc <= 9) {
    d_tab_off.reserve((size_t)nseg + 1); d_tab_sizes.reserve((size_t)nseg + 1);
    ba_seg_table_sizes<<<grid_for(nseg + 1, 256), 256, 0, stream>>>(rs.v, d_seg_start.p, nseg, d_tab_sizes.p);
    OSFM_LAUNCH_CHECK();
    size_t tb = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, tb, d_tab_sizes.p, d_tab_off.p, nseg + 1, stream);
    d_cub.reserve(tb + 256);
    tb = d_cub.cap;
    OSFM_CUDA(cub::DeviceScan::ExclusiveSum(d_cub.p, tb, d_tab_sizes.p, d_tab_off.p, nseg + 1, stream));
    long long total_ints = 0;
    OSFM_CUDA(cudaMemcpyAsync(&total_ints, d_tab_off.p + nseg, sizeof(long long), cudaMemcpyDeviceToHost, stream));
    OSFM_CUDA(cudaStreamSynchronize(stream));
    d_tab.reserve((size_t)total_ints + 2);
    ba_seg_tables<<<nseg, 128, 0, stream>>>(rs.v, rs.bm, rs.bsr, d_seg_start.p, nullptr, d_tab_off.p, d_tab.p);
    OSFM_LAUNCH_CHECK();
    rs.seg_tab = true;
  }
  // The chunk list (ba_schur_pipe.cuh) of the camera side every chunk-list kernel is written for: a 3-parameter camera
  // and a pose per shot, 2-D residuals
  if (rs.seg_tab && wc == 9 && rs.nres == 2) {
    d_sp_nch.reserve((size_t)nseg + 1); d_sp_chunk0.reserve((size_t)nseg + 1);
    sp_chunk_counts<<<grid_for(nseg + 1, 256), 256, 0, stream>>>(rs.v, d_seg_start.p, nseg, d_sp_nch.p);
    OSFM_LAUNCH_CHECK();
    size_t tb = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, tb, d_sp_nch.p, d_sp_chunk0.p, nseg + 1, stream);
    d_cub.reserve(tb + 256);
    tb = d_cub.cap;
    OSFM_CUDA(cub::DeviceScan::ExclusiveSum(d_cub.p, tb, d_sp_nch.p, d_sp_chunk0.p, nseg + 1, stream));
    OSFM_CUDA(cudaMemcpyAsync(&rs.sp_nchunks, d_sp_chunk0.p + nseg, sizeof(int), cudaMemcpyDeviceToHost, stream));
    OSFM_CUDA(cudaStreamSynchronize(stream));
    d_sp_chunks.reserve((size_t)rs.sp_nchunks + 1);
    sp_fill_chunks<<<grid_for((long long)nseg * 32, 256), 256, 0, stream>>>(rs.v, d_seg_start.p, nseg, d_sp_chunk0.p,
                                                                          d_tab_off.p, d_sp_chunks.p);
    OSFM_LAUNCH_CHECK();
  }
  // the persistent Schur kernel runs over the chunk list; its flush table holds offset << 2 (the reduced system must
  // stay below 2^29 doubles) and takes 20 KB per segment
  const bool use_mma = !(fallbacks & OSFM_BA_FALLBACK_SIMT_SEGMENT_SCHUR) && wc <= 9;
  const bool use_pipe = use_mma && !(fallbacks & OSFM_BA_FALLBACK_CTA_PER_SEGMENT_SCHUR) && rs.sp_nchunks > 0 &&
                        rs.s_upper_total + (long long)rs.nc_pad < (1LL << 29) &&
                        (long long)nseg * SP_FT_SEG * (long long)sizeof(int) <= (8LL << 30);
  if (use_pipe) {
    d_sp_ftab.reserve((size_t)nseg * SP_FT_SEG);
    sp_flush_tables<<<nseg, SP_CONS_THREADS, 0, stream>>>(rs.v, d_seg_start.p, d_tab_off.p, d_tab.p, d_sp_ftab.p);
    OSFM_LAUNCH_CHECK();
  }
  rs.schur = nseg == 0 ? OSFM_SCHUR_NONE
             : !use_mma ? OSFM_SCHUR_SIMT_SEGMENT
             : use_pipe ? OSFM_SCHUR_PIPE : OSFM_SCHUR_MMA;
  if (rs.schur == OSFM_SCHUR_SIMT_SEGMENT) {
    const size_t rows = (size_t)rs.n_fast_obs * wc * 3 + 8;
    d_rowsJ.reserve(rows); d_rowsW.reserve(rows); d_rowsY.reserve(rows);
  }
  rs.lin = nseg == 0 ? LIN_NONE
           : rs.sp_nchunks == 0 ? LIN_SEGMENTS
           : rs.uniform_type == PT_PERSPECTIVE ? LIN_FUSED : LIN_CHUNKS;
}

// The Jacobi scale of every segment column into the tables, whenever d_scale has been (re)computed.
void BA::segment_table_scales() {
  if (!rs.seg_tab) return;
  ba_seg_scales<<<rs.nseg, 128, 0, stream>>>(rs.v, d_seg_start.p, d_scale.p, d_tab_off.p, d_tab.p);
  OSFM_LAUNCH_CHECK();
}

// cost at parameter set b (sum over ranks) into Scalars::cost
void BA::eval_cost(int b) {
  OSFM_CUDA(cudaMemsetAsync(&d_sc.p->cost, 0, sizeof(double), stream));
  if (rs.N > 0) launch_linearize<0>(b);
  const int npr_local = rs.pv.n_cam_rows + rs.pv.n_pos_rows;
  if (npr_local > 0) {
    ba_prior_cost<<<grid_for(npr_local, 128), 128, 0, stream>>>(rs.pv, params_of(b), d_sc.p);
    OSFM_LAUNCH_CHECK();
  }
  if (rs.NT > 0 && rs.add_priors) {
    side_cost<<<grid_for(rs.NT, 128), 128, 0, stream>>>(rs.sv, rs.v, rs.bm, params_of(b), d_sc.p);
    OSFM_LAUNCH_CHECK();
  }
  if (rs.have_pp && rs.P > 0) {
    ba_point_prior<0><<<grid_for(rs.P, 128), 128, 0, stream>>>(rs.ppv, rs.v, params_of(b), nullptr, nullptr, nullptr, d_sc.p);
    OSFM_LAUNCH_CHECK();
  }
  allreduce_dev(&d_sc.p->cost, 1);
}


// residual + Jacobian planes, column norms, gradient at parameter set b; the cost and max |g| into Scalars.  `timed`:
// into the linearisation phase timer.
void BA::linearize(int b, bool timed) {
  const long long N = rs.N, n_fast_obs = rs.n_fast_obs;
  const int nc = rs.nc, n = rs.n, nseg = rs.nseg, wc = rs.wc, NT = rs.NT;
  OSFM_CUDA(cudaMemsetAsync(d_sc.p, 0, sizeof(Scalars), stream));
  OSFM_CUDA(cudaMemsetAsync(d_colnorm2.p, 0, sizeof(double) * rs.nz, stream));
  OSFM_CUDA(cudaMemsetAsync(d_grad.p, 0, sizeof(double) * rs.nz, stream));
  if (N > 0 && rs.lin == LIN_FUSED) {
    // planes, cost and the segment observations' column norms / gradient / point sums in one pass; the observations
    // outside the segments get their sums from the plane-reading kernels
    d_ptsum.reserve(9 * (size_t)std::max(rs.npf, 1));
    const int grid = (int)((n_fast_obs + FL_WIN - 1) / FL_WIN + (N - n_fast_obs + FL_THREADS - 1) / FL_THREADS);
    if (timed) lm_phase(-1, LM_PH_LIN);
    ba_linearize_fused<PT_PERSPECTIVE><<<grid, FL_THREADS, 0, stream>>>(rs.v, params_of(b), d_sc.p, d_sp_chunks.p, rs.sp_nchunks,
                                                                        n_fast_obs, d_tab.p, d_colnorm2.p, d_grad.p, d_ptsum.p);
    OSFM_LAUNCH_CHECK();
    if (timed) lm_phase(LM_PH_LIN, -1);
    if (N > n_fast_obs) {
      ba_colnorm_grad_points<<<grid_for(N - n_fast_obs, 256), 256, 0, stream>>>(rs.v, n_fast_obs, d_colnorm2.p, d_grad.p);
      OSFM_LAUNCH_CHECK();
      ba_colnorm_grad<<<grid_for(N - n_fast_obs, 256), 256, 0, stream>>>(rs.v, n_fast_obs, d_colnorm2.p, d_grad.p);
      OSFM_LAUNCH_CHECK();
    }
  } else if (N > 0) {
    if (timed) lm_phase(-1, LM_PH_LIN);
    launch_linearize<1>(b);
    if (timed) lm_phase(LM_PH_LIN, -1);
    ba_colnorm_grad_points<<<grid_for(N, 256), 256, 0, stream>>>(rs.v, 0, d_colnorm2.p, d_grad.p);
    OSFM_LAUNCH_CHECK();
    if (rs.lin == LIN_CHUNKS) {   // no dependent index loads
      opt_in_smem(ba_colnorm_grad_chunks, CC_SMEM);
      const int grid = std::max(1, std::min(num_sms, (rs.sp_nchunks + CC_WARPS - 1) / CC_WARPS));
      ba_colnorm_grad_chunks<<<grid, 32 * CC_WARPS, CC_SMEM, stream>>>(rs.v, d_sp_chunks.p, rs.sp_nchunks, d_tab.p,
                                                                        d_colnorm2.p, d_grad.p);
      OSFM_LAUNCH_CHECK();
    } else if (rs.lin == LIN_SEGMENTS) {
      auto kern = wc == 9 ? ba_colnorm_grad_seg<9> : ba_colnorm_grad_seg<0>;
      kern<<<grid_for((long long)nseg * 32, 256), 256, 0, stream>>>(rs.v, d_seg_start.p, nseg, d_colnorm2.p, d_grad.p);
      OSFM_LAUNCH_CHECK();
    }
    if (N > n_fast_obs) {
      ba_colnorm_grad<<<grid_for(N - n_fast_obs, 256), 256, 0, stream>>>(rs.v, n_fast_obs, d_colnorm2.p, d_grad.p);
      OSFM_LAUNCH_CHECK();
    }
  }
  const int npr_local = rs.pv.n_cam_rows + rs.pv.n_pos_rows;
  if (npr_local > 0) {
    ba_prior_cost<<<grid_for(npr_local, 128), 128, 0, stream>>>(rs.pv, params_of(b), d_sc.p);
    OSFM_LAUNCH_CHECK();
    ba_prior_colnorm_grad<<<grid_for(npr_local, 128), 128, 0, stream>>>(rs.pv, params_of(b), d_colnorm2.p, d_grad.p);
    OSFM_LAUNCH_CHECK();
  }
  if (NT > 0) {   // every rank keeps the terms' Jacobians (rank 0 adds the system part, before the all-reduce)
    side_linearize<<<NT, SIDE_THREADS, 0, stream>>>(rs.sv, rs.v, rs.bm, params_of(b), d_sc.p, rs.add_priors ? 1 : 0);
    OSFM_LAUNCH_CHECK();
    if (rs.add_priors) {
      side_colnorm_grad<<<NT, SIDE_THREADS, 0, stream>>>(rs.sv, rs.v, rs.bm, params_of(b), d_colnorm2.p, d_grad.p);
      OSFM_LAUNCH_CHECK();
    }
  }
  if (rs.have_pp && rs.P > 0) {
    ba_point_prior<1><<<grid_for(rs.P, 128), 128, 0, stream>>>(rs.ppv, rs.v, params_of(b), d_colnorm2.p, d_grad.p, nullptr, d_sc.p);
    OSFM_LAUNCH_CHECK();
  }
  if (world > 1) {
    // local max over the point part, then one all-reduce for cost, camera-side sums and the per-rank maxima
    if (n > nc) {
      ba_grad_max<<<grid_for(n - nc, 256), 256, 0, stream>>>(d_grad.p + nc, n - nc, d_sc.p);
      OSFM_LAUNCH_CHECK();
    }
    const int npack = 2 * nc + 1 + world;
    d_slots.reserve(npack);
    const int gsz = std::max(nc, world);
    ba_pack_lin<<<grid_for(gsz, 256), 256, 0, stream>>>(d_colnorm2.p, d_grad.p, d_sc.p, nc, rank, world, d_slots.p);
    OSFM_LAUNCH_CHECK();
    allreduce_dev(d_slots.p, npack);
    ba_unpack_lin<<<grid_for(gsz, 256), 256, 0, stream>>>(d_slots.p, nc, world, d_colnorm2.p, d_grad.p, d_sc.p);
    OSFM_LAUNCH_CHECK();
  } else if (n > 0) {
    ba_grad_max<<<grid_for(n, 256), 256, 0, stream>>>(d_grad.p, n, d_sc.p);
    OSFM_LAUNCH_CHECK();
  }
}

// Reduced camera system at the accepted parameters (upper blocks accumulated with L2 atomics, all-reduced, priors
// and side terms added, mirrored), damped with diag * inv_radius.  The LM iteration (diag / radius of its state, 1)
// and the covariance pass (inv_radius = 0, rank_flag set: ba_cov.cuh) both build it here, through the same kernel
// path.  `timed`: into the Schur phase timer.
void BA::build_system(const double* diag, double inv_radius, int* rank_flag, bool timed) {
  const int nc = rs.nc, P = rs.P, P_fast = rs.P_fast, nseg = rs.nseg, wc = rs.wc;
  const bool trace_on = tracing();
  double *const d_rhs_p = rs.d_rhs_p, *const d_S_p = rs.d_S_p;
  if (nc > 0) OSFM_CUDA(cudaMemsetAsync(d_Sbuf.p, 0, sizeof(double) * ((size_t)rs.nc_pad + (size_t)rs.s_upper_total), stream));
  if (P > 0) {
    const size_t smem = (size_t)SCHUR_KC * wc * (2 * 3 * sizeof(double) + 2 * sizeof(int)) +
                        (size_t)SCHUR_KC * 8 * sizeof(int) + (size_t)SCHUR_KC * SCHUR_KC * 9 * sizeof(int);
    if (timed) lm_phase(-1, LM_PH_SCHUR);
    if (rs.schur != OSFM_SCHUR_NONE) {
      if (rs.lin == LIN_FUSED)   // the point sums of the linearisation
        ba_point_blocks_sums<<<grid_for(P_fast, PB_THREADS), PB_THREADS, 0, stream>>>(
            rs.v, P_fast, d_ptsum.p, d_scale.p, diag, inv_radius, d_Vinv.p, d_gp.p, d_Vig.p, rank_flag);
      else
        ba_point_blocks<<<grid_for(P_fast, PB_THREADS), PB_THREADS, 0, stream>>>(rs.v, P_fast, d_scale.p, diag, inv_radius,
                                                                               d_Vinv.p, d_gp.p, d_Vig.p, rank_flag);
      OSFM_LAUNCH_CHECK();
    }
    // the segment kernels add the segment points' camera-side blocks: with no free camera-side block (nc == 0) there
    // are none (and no segment tables or block structure to read); their point blocks are those above
    if (nc > 0 && (rs.schur == OSFM_SCHUR_PIPE || rs.schur == OSFM_SCHUR_MMA)) {
      unsigned long long* prof = nullptr;
      if (trace_on) {
        d_prof.reserve(16);
        OSFM_CUDA(cudaMemsetAsync(d_prof.p, 0, 16 * sizeof(unsigned long long), stream));
        prof = d_prof.p;
      }
      if (rs.schur == OSFM_SCHUR_PIPE) {
        auto kern = prof ? ba_schur_pipe<true> : ba_schur_pipe<false>;
        opt_in_smem(kern, (int)sizeof(SpSmem));
        const int grid = std::max(1, std::min(num_sms, rs.sp_nchunks));
        kern<<<grid, SP_THREADS, sizeof(SpSmem), stream>>>(rs.v, d_sp_chunks.p, rs.sp_nchunks, d_tab.p, d_scale.p, d_Vinv.p,
                                                          d_Vig.p, d_sp_ftab.p, d_S_p, d_rhs_p, prof);
        if (trace_on) {
          OSFM_LAUNCH_CHECK();
          unsigned long long hp[16];
          OSFM_CUDA(cudaMemcpyAsync(hp, d_prof.p, sizeof(hp), cudaMemcpyDeviceToHost, stream));
          OSFM_CUDA(cudaStreamSynchronize(stream));
          const unsigned long long nch = std::max<unsigned long long>(hp[3], 1);
          fprintf(stderr, "[osfm_ba] ba_schur_pipe (%d CTAs, %llu chunks) producer clocks / chunk: copy wait %llu buffer wait %llu build %llu\n",
                  grid, hp[3], hp[0] / nch, hp[1] / nch, hp[2] / nch);
          for (int gI = 0; gI < 2; ++gI) {
            const unsigned long long ns = std::max<unsigned long long>(hp[8 + 5 * gI], 1);
            fprintf(stderr, "[osfm_ba]   consumer group %d clocks / segment (%llu segments): tables %llu operand wait %llu mma %llu flush %llu\n",
                    gI, hp[8 + 5 * gI], hp[4 + 5 * gI] / ns, hp[5 + 5 * gI] / ns, hp[6 + 5 * gI] / ns, hp[7 + 5 * gI] / ns);
          }
        }
      } else {
        auto kern = wc == 9 ? ba_schur_mma<9> : ba_schur_mma<0>;
        opt_in_smem(kern, (int)sizeof(SegMmaSmem));
        kern<<<nseg, SM_THREADS, sizeof(SegMmaSmem), stream>>>(rs.v, d_seg_start.p, d_tab_off.p, d_tab.p, d_scale.p, d_Vinv.p,
                                                               d_Vig.p, d_S_p, d_rhs_p, prof);
      }
      OSFM_LAUNCH_CHECK();
      if (trace_on && rs.schur == OSFM_SCHUR_MMA) {
        unsigned long long hp[8];
        OSFM_CUDA(cudaMemcpyAsync(hp, d_prof.p, sizeof(hp), cudaMemcpyDeviceToHost, stream));
        OSFM_CUDA(cudaStreamSynchronize(stream));
        fprintf(stderr, "[osfm_ba] ba_schur_mma clocks / segment (thread 0): structure %llu offsets %llu loads %llu rows %llu mma %llu flush %llu\n",
                hp[0] / nseg, hp[1] / nseg, hp[2] / nseg, hp[3] / nseg, hp[4] / nseg, hp[5] / nseg);
      }
    } else if (nc > 0 && rs.schur == OSFM_SCHUR_SIMT_SEGMENT) {
      const long long n_fast = rs.n_fast_obs;
      ba_obs_rows<<<grid_for(n_fast * wc, 256), 256, 0, stream>>>(rs.v, rs.bm, rs.bsr, n_fast, d_scale.p, d_Vinv.p, d_Vig.p,
                                                                d_rowsJ.p, d_rowsW.p, d_rowsY.p, d_rhs_p);
      OSFM_LAUNCH_CHECK();
      auto kern = wc == 9 ? ba_schur_seg<9> : ba_schur_seg<0>;
      opt_in_smem(kern, (int)sizeof(SegSmem));
      kern<<<nseg, SEG_THREADS, sizeof(SegSmem), stream>>>(rs.v, rs.bm, rs.bsr, d_seg_start.p, n_fast, d_rowsJ.p, d_rowsW.p,
                                                           d_rowsY.p, d_S_p);
      OSFM_LAUNCH_CHECK();
    }
    if (P > P_fast) {
      ba_schur<<<P - P_fast, SCHUR_THREADS, smem, stream>>>(rs.v, rs.bm, rs.bsr, d_scale.p, diag, inv_radius, d_S_p,
                                                           d_rhs_p, d_Vinv.p, d_gp.p, P_fast, rs.ppv, d_pts[0].p, rank_flag);
      OSFM_LAUNCH_CHECK();
    }
    if (timed) lm_phase(LM_PH_SCHUR, -1);
  }
  if (nc > 0) {
    // the side terms' blocks: rank 0 adds them to its partial system before the exchange.  Several terms add to one
    // entry with atomics, in an order that changes from run to run; added on every rank after the exchange, they left
    // each rank with a slightly different system and the ranks' camera sides apart by a few 1e-12.
    if (rs.NT > 0 && rs.add_priors) {
      side_system<<<rs.NT, SIDE_THREADS, 0, stream>>>(rs.sv, rs.v, rs.bm, params_of(0), rs.bsr, d_scale.p, d_S_p, d_rhs_p);
      OSFM_LAUNCH_CHECK();
    }
    // the one exchange step of the LM iteration: sum of the partial reduced systems over ranks
    if (world > 1) allreduce_dev(d_Sbuf.p, (long long)rs.nc_pad + rs.s_upper_total);  // rhs + upper blocks, one call
    // every rank then adds the (replicated) prior rows, one addition per entry, and the damping to its copy of the
    // reduced system: the copies stay identical.
    PriorView pall = rs.pv;
    pall.n_cam_rows = (int)rs.pr_cam_param.size();
    pall.n_pos_rows = (int)rs.pr_pos_inst.size();
    const int nall = pall.n_cam_rows + pall.n_pos_rows;
    if (nall > 0) {
      ba_prior_system<<<grid_for(nall, 128), 128, 0, stream>>>(pall, params_of(0), d_scale.p, d_prior_diag_off.p,
                                                              d_S_p, d_rhs_p);
      OSFM_LAUNCH_CHECK();
    }
    ba_finish_system<<<grid_for((long long)rs.n_upper * 32, 256), 256, 0, stream>>>(d_upper.p, rs.n_upper, rs.bsr, d_S_p,
                                                                                  diag, inv_radius);
    OSFM_LAUNCH_CHECK();
  }
}

// PCG on the damped reduced system, |r| <= 1e-8 |b|, into y: the pipelined kernel, and the classic one from scratch
// when its recurrences stagnate or break down (ba_lm_pcg_check decides on the device).
void BA::solve_reduced() {
  const int nc = rs.nc;
  lm_phase(-1, LM_PH_PCG);
  pcg_convert<<<grid_for((long long)rs.n_blocks_all * 32, 256), 256, 0, stream>>>(
      rs.d_S_p, d_row_col.p, d_row_off.p, d_qoff.p, d_blk_row.p, rs.n_blocks_all, rs.bsr, d_row_M.p, d_rowbase.p, d_Spcg.p);
  OSFM_LAUNCH_CHECK();
  pcg_factor_groups<<<grid_for((long long)rs.ngroups * 32, 32 * PFG_WARPS), 32 * PFG_WARPS, 0, stream>>>(rs.d_S_p, rs.bsr, d_diag_off.p, d_grp_b1.p, d_grp_b2.p,
                                                                rs.ngroups, d_Minv.p);
  OSFM_LAUNCH_CHECK();
  OSFM_CUDA(cudaMemsetAsync(d_pcg.p, 0, sizeof(PcgState), stream));
  // the flagged words of pcg_pipelined start every solve at generation 0, which no exchange waits for
  if (rs.pcg_pipe_ok) OSFM_CUDA(cudaMemsetAsync(d_pm.p, 0, sizeof(unsigned long long) * 4 * (size_t)nc, stream));
  const int max_pcg = std::min(2 * nc + 100, 5000);
  const int classic_path = rs.pcg_resident ? OSFM_PCG_CLASSIC_RESIDENT : OSFM_PCG_CLASSIC_STREAMED;
  auto classic = [&]() {
    launch_cooperative(rs.pcg_resident ? pcg_persistent<true> : pcg_persistent<false>, rs.pcg_grid, PCG_THREADS, rs.pcg_smem,
                       stream, d_Spcg.p, rs.lay, rs.bsr, d_Minv.p, rs.d_rhs_p, d_px.p, d_pr.p, d_pz.p, d_pp.p, d_pAp.p, d_Ap.p,
                       d_pcg.p, nc, max_pcg, 1e-16, rs.pcg_res);
    OSFM_LAUNCH_CHECK();
    if (tracing()) {
      OSFM_CUDA(cudaMemcpyAsync(h_pcg.p, d_pcg.p, PCG_STATE_HEADER, cudaMemcpyDeviceToHost, stream));
      OSFM_CUDA(cudaStreamSynchronize(stream));
      const PcgState& h = *h_pcg.p;
      const int its = std::max(h.iterations, 1);
      fprintf(stderr, "[osfm_ba] pcg %d its, CTA0 clocks/it: stage %lld matvec %lld reduce1 %lld phaseB %lld reduce2 %lld (resident %d)\n",
              h.iterations, h.prof[0] / its, h.prof[1] / its, h.prof[2] / its, h.prof[3] / its, h.prof[4] / its, (int)rs.pcg_resident);
    }
  };
  if (rs.pcg_pipe_ok) {
    launch_cooperative(pcg_pipelined, rs.pcg_grid, PCG_THREADS, rs.pcg_pipe_smem, stream, d_Spcg.p, rs.lay, rs.bsr, d_Minv.p,
                       rs.d_rhs_p, d_px.p, d_pm.p, d_pcg.p, nc, max_pcg, 1e-16, rs.pcg_pipe);
    OSFM_LAUNCH_CHECK();
    if (tracing()) {
      OSFM_CUDA(cudaMemcpyAsync(h_pcg.p, d_pcg.p, PCG_STATE_HEADER, cudaMemcpyDeviceToHost, stream));
      OSFM_CUDA(cudaStreamSynchronize(stream));
      const PcgState& h = *h_pcg.p;
      const int its = std::max(h.iterations, 1);
      fprintf(stderr, "[osfm_ba] pipelined pcg %d its converged %d, CTA0 clocks/it: post %lld stage %lld matvec %lld collect %lld"
              " update %lld\n", h.iterations, h.converged, h.prof[0] / its, h.prof[1] / its, h.prof[2] / its, h.prof[3] / its,
              h.prof[4] / its);
    }
    ba_lm_pcg_check<<<1, 1, 0, stream>>>(d_lm.p, d_pcg.p, classic_path, rs.h_pcg, rs.cap_graph != nullptr);
    OSFM_LAUNCH_CHECK();
    rs.k_pcg = lm_if(rs.h_pcg, LM_PCG_CLASSIC, [&]() {
      OSFM_CUDA(cudaMemsetAsync(d_pcg.p, 0, sizeof(PcgState), stream));
      classic();
    });
  } else {
    classic();
  }
  OSFM_CUDA(cudaMemcpyAsync(d_y.p, d_px.p, sizeof(double) * nc, cudaMemcpyDeviceToDevice, stream));
  lm_phase(LM_PH_PCG, -1);
}

// back-substitution: the point part of y from its camera part
void BA::back_substitute() {
  const int P = rs.P, npf = rs.npf;
  if (P == 0 || npf == 0) return;
  lm_phase(-1, LM_PH_BACK);
  OSFM_CUDA(cudaMemsetAsync(d_bs_t.p, 0, sizeof(double) * 3 * (size_t)npf, stream));
  if (rs.N > 0) {
    ba_backsub_rows<<<grid_for(rs.N, 256), 256, 0, stream>>>(rs.v, d_scale.p, d_y.p, d_bs_t.p);
    OSFM_LAUNCH_CHECK();
  }
  if (rs.have_pp) {
    ba_point_prior<3><<<grid_for(P, 128), 128, 0, stream>>>(rs.ppv, rs.v, params_of(0), nullptr, nullptr, d_bs_t.p, d_sc.p);
    OSFM_LAUNCH_CHECK();
  }
  ba_backsub_points<<<grid_for(npf, 256), 256, 0, stream>>>(rs.v, d_scale.p, d_Vinv.p, d_bs_t.p, d_y.p);
  OSFM_LAUNCH_CHECK();
  lm_phase(LM_PH_BACK, -1);
}

// osfm_ba_capture_linear_system: raw copies of the system the PCG solved, the dense expansion is host code in
// osfm_ba_get_captured_system
void BA::capture_linear_system(int it, double radius) {
  const int nc = rs.nc, n = rs.n, P = rs.P;
  const int pcg_path = rs.pcg_pipe_ok ? read_lm().pcg_path : rs.pcg_resident ? OSFM_PCG_CLASSIC_RESIDENT : OSFM_PCG_CLASSIC_STREAMED;
  OSFM_CUDA(cudaMemcpyAsync(h_pcg.p, d_pcg.p, PCG_STATE_HEADER, cudaMemcpyDeviceToHost, stream));
  download(cap_sbuf, d_Sbuf.p, (size_t)rs.nc_pad + (size_t)rs.s_total, stream);
  download(cap_upper, d_upper.p, rs.n_upper, stream);
  download(cap_y, d_px.p, nc, stream);
  download(cap_scale, d_scale.p, n, stream); download(cap_diag, d_diag.p, n, stream); download(cap_grad, d_grad.p, n, stream);
  download(cap_pt_poff, d_pt_poff.p, P, stream); download(cap_global_of, d_global_of.p, P, stream);
  const Params xp = params_of(0);
  download(cap_cam, xp.cam, cam_params.size(), stream); download(cap_inst, xp.inst, inst.size(), stream);
  download(cap_rc, xp.rc, rc.size(), stream); download(cap_pts, xp.pts, 3 * (size_t)P, stream);
  download(cap_ext, xp.ext, ext_values.size(), stream);
  download(cap_side_r, d_side_r.p, rs.side_rofs[rs.NT], stream);
  download(cap_side_J, d_side_J.p, rs.side_jofs[rs.NT], stream);
  OSFM_CUDA(cudaStreamSynchronize(stream));
  cap_blk_off = rs.blk_off; cap_blk_sz = rs.blk_sz; cap_nc_pad = rs.nc_pad;
  cap_info = osfm_ba_capture{};
  cap_info.iteration = it; cap_info.nc = nc; cap_info.n = n; cap_info.wc = rs.wc; cap_info.nres = rs.nres;
  cap_info.radius = radius;
  cap_info.nseg = rs.nseg; cap_info.p_fast = rs.P_fast; cap_info.p_slow = P - rs.P_fast;
  cap_info.schur_kernel = rs.schur;
  cap_info.sp_nchunks = rs.sp_nchunks;
  cap_info.pcg_kernel = pcg_path;
  cap_info.pcg_rescued = rs.pcg_pipe_ok && pcg_path != OSFM_PCG_PIPELINED_DEFLATED && pcg_path != OSFM_PCG_PIPELINED;
  cap_info.pcg_iterations = h_pcg.p->iterations;
  cap_info.pcg_rr = h_pcg.p->rr_final;
  cap_valid = true;
}

// Rig-instance covariances (ba_cov.cuh) at the accepted parameters: not after a FAILURE termination, as in the reference
void BA::covariance_pass(int termination) {
  const int nc = rs.nc, n = rs.n, NI = rs.NI;
  cov_out.assign((size_t)NI * 36, 0.0);
  cov_status = OSFM_COV_SOLVER_FAILURE;
  cov_pass_ms = cov_chol_ms = 0.0;
  if (termination != 2) {
    const std::vector<int>& cov_inst = rs.cov_inst;
    const std::vector<int>& cov_bstart = rs.cov_bstart;
    double* const A = d_cov.p;                                   // dense S -> L, column-major, ld nc
    double* const X = A + (size_t)nc * nc;                       // L22^-1, ld m
    double* const W = X + (size_t)rs.cov_m * rs.cov_m;           // inverse of every diagonal block of L
    double* const d0 = W + (cov_bstart.size() - 1) * COV_NB * COV_NB;   // diagonal of S before the factorisation
    double* const out = d0 + nc;
    int* const flags = d_cov_flags.p;
    const int m = rs.cov_m, n1 = nc - rs.cov_m;
    std::vector<int> perm(std::max(nc, 1));
    {
      std::vector<char> is_inst(std::max(nc, 1), 0);
      for (size_t q = 0; q < cov_inst.size(); ++q)
        for (int j = 0; j < 6; ++j) {
          perm[rs.inst_poff[cov_inst[q]] + j] = n1 + 6 * (int)q + j;
          is_inst[rs.inst_poff[cov_inst[q]] + j] = 1;
        }
      for (int g = 0, lead = 0; g < nc; ++g)
        if (!is_inst[g]) perm[g] = lead++;
    }
    upload(d_cov_perm, perm, stream);
    std::vector<int> inst_list = cov_inst;
    if (inst_list.empty()) inst_list.push_back(0);
    upload(d_cov_inst, inst_list, stream);
    OSFM_CUDA(cudaMemsetAsync(flags, 0, sizeof(int) * COV_F_COUNT, stream));
    const int potrf_smem = 2 * COV_NB * (COV_NB + 1) * (int)sizeof(double);
    const int gemm_smem = 2 * COV_NB * COV_LDS * (int)sizeof(double);
    opt_in_smem(cov_potrf_diag, potrf_smem);
    for (auto k : {cov_gemm<COV_TRSM>, cov_gemm<COV_SYRK>, cov_gemm<COV_TRI_DIAG>, cov_gemm<COV_TRI_UPD>}) opt_in_smem(k, gemm_smem);
    cudaEvent_t ce[4];
    for (auto& e : ce) OSFM_CUDA(cudaEventCreate(&e));
    OSFM_CUDA(cudaEventRecord(ce[0], stream));
    // re-linearise at the accepted parameters with the Jacobi scale of this point (the LM keeps the first one)
    linearize(0, false);
    if (n > 0) {
      ba_make_scale<<<grid_for(n, 256), 256, 0, stream>>>(d_colnorm2.p, d_scale.p, n);
      OSFM_LAUNCH_CHECK();
      // the diagonal only has to be finite: the system is built with inv_radius = 0
      ba_make_diag<<<grid_for(n, 256), 256, 0, stream>>>(d_colnorm2.p, d_scale.p, d_diag.p, n);
      OSFM_LAUNCH_CHECK();
    }
    segment_table_scales();   // the tensor-core Schur kernels read the scale from their segment tables
    build_system(d_diag.p, 0.0, flags + COV_F_POINT_RANK, false);
    OSFM_CUDA(cudaEventRecord(ce[1], stream));
    auto tiles = [](int k) { return (k + COV_NB - 1) / COV_NB; };
    CovGemm g{A, nc, X, m, n1, nullptr, 0, 0, flags};
    if (nc > 0) {
      OSFM_CUDA(cudaMemsetAsync(A, 0, sizeof(double) * (size_t)nc * nc, stream));
      OSFM_CUDA(cudaMemsetAsync(d0, 0, sizeof(double) * (size_t)nc, stream));
      cov_densify<<<grid_for((long long)rs.n_upper * 32, 256), 256, 0, stream>>>(d_upper.p, rs.n_upper, rs.bsr, rs.d_S_p,
                                                                                d_cov_perm.p, nc, A, d0);
      OSFM_LAUNCH_CHECK();
      // blocked right-looking Cholesky: diagonal block, panel below it, trailing update
      for (size_t b = 0; b + 1 < cov_bstart.size(); ++b) {
        const int k0 = cov_bstart[b], kb = cov_bstart[b + 1] - k0, rem = nc - k0 - kb;
        cov_potrf_diag<<<1, COV_THREADS, 2 * COV_NB * (COV_NB + 1) * sizeof(double), stream>>>(
            A, nc, k0, kb, d0, W + b * COV_NB * COV_NB, flags);
        OSFM_LAUNCH_CHECK();
        if (rem == 0) continue;
        g.W = W + b * COV_NB * COV_NB; g.k0 = k0; g.kb = kb;
        cov_gemm<COV_TRSM><<<dim3(tiles(rem), 1), COV_THREADS, gemm_smem, stream>>>(g);
        OSFM_LAUNCH_CHECK();
        cov_gemm<COV_SYRK><<<dim3(tiles(rem), tiles(rem)), COV_THREADS, gemm_smem, stream>>>(g);
        OSFM_LAUNCH_CHECK();
      }
    }
    OSFM_CUDA(cudaEventRecord(ce[2], stream));
    if (m > 0) {
      // X = L22^-1: X_k = W_kk X_k, then X_i -= L22_ik X_k below, block row by block row
      cov_identity<<<grid_for((long long)m * m, 256), 256, 0, stream>>>(X, m);
      OSFM_LAUNCH_CHECK();
      for (size_t b = rs.cov_nb1; b + 1 < cov_bstart.size(); ++b) {
        const int k0 = cov_bstart[b] - n1, kb = cov_bstart[b + 1] - cov_bstart[b], rem = m - k0 - kb;
        g.W = W + b * COV_NB * COV_NB; g.k0 = k0; g.kb = kb;
        cov_gemm<COV_TRI_DIAG><<<dim3(1, tiles(k0 + kb)), COV_THREADS, gemm_smem, stream>>>(g);
        OSFM_LAUNCH_CHECK();
        if (rem == 0) continue;
        cov_gemm<COV_TRI_UPD><<<dim3(tiles(rem), tiles(k0 + kb)), COV_THREADS, gemm_smem, stream>>>(g);
        OSFM_LAUNCH_CHECK();
      }
      OSFM_CUDA(cudaMemsetAsync(out, 0, sizeof(double) * (size_t)NI * 36, stream));
      cov_blocks<<<(int)cov_inst.size(), COV_THREADS, 0, stream>>>(X, m, d_cov_inst.p, d_inst_poff.p, d_scale.p, flags,
                                                                   out, flags);
      OSFM_LAUNCH_CHECK();
    }
    OSFM_CUDA(cudaEventRecord(ce[3], stream));
    int hf[COV_F_COUNT];
    OSFM_CUDA(cudaMemcpyAsync(hf, flags, sizeof(hf), cudaMemcpyDeviceToHost, stream));
    if (m > 0) OSFM_CUDA(cudaMemcpyAsync(cov_out.data(), out, sizeof(double) * cov_out.size(), cudaMemcpyDeviceToHost, stream));
    OSFM_CUDA(cudaStreamSynchronize(stream));
    float ms_pass = 0.f, ms_chol = 0.f;
    OSFM_CUDA(cudaEventElapsedTime(&ms_pass, ce[0], ce[3]));
    OSFM_CUDA(cudaEventElapsedTime(&ms_chol, ce[1], ce[2]));
    for (auto& e : ce) cudaEventDestroy(e);
    cov_pass_ms = ms_pass; cov_chol_ms = ms_chol;
    cov_status = hf[COV_F_POINT_RANK] ? OSFM_COV_POINT_RANK_DEFICIENT
                 : hf[COV_F_CHOL]     ? OSFM_COV_CAMERA_RANK_DEFICIENT
                 : hf[COV_F_NONFINITE] ? OSFM_COV_NON_FINITE : OSFM_COV_OK;
    if (tracing() && hf[COV_F_CHOL])
      fprintf(stderr, "[osfm_ba] covariances: reduced system rank deficient at dense column %d\n", hf[COV_F_CHOL_COL]);
  }
  cov_valid = cov_status == OSFM_COV_OK;
  if (!cov_valid) {   // bundle_adjuster.cc:1177-1192: the default for every instance, replacing whatever was computed
    std::fill(cov_out.begin(), cov_out.end(), 0.0);
    for (int i = 0; i < NI; ++i)
      for (int j = 0; j < 6; ++j) cov_out[(size_t)i * 36 + j * 7] = j < 3 ? 1e-5 : 1e-2;
  }
  cov_ran = true;
  trace("covariances");
}

// Accepted parameters, points and reprojection errors back to the caller; the summary of the run (`sum` holds the
// LM loop's counts and costs)
void BA::write_results(osfm_ba_summary sum) {
  const int cur = 0, P = rs.P, Pfull = rs.Pfull;
  const long long Nfull = rs.Nfull;
  download(cam_params, d_cam[cur].p, cam_params.size(), stream); download(inst, d_inst[cur].p, inst.size(), stream);
  download(rc, d_rc[cur].p, rc.size(), stream); download(ext_values, d_ext[cur].p, ext_values.size(), stream);
  d_full_pts.reserve(3 * (size_t)std::max(Pfull, 1));
  if (world > 1) OSFM_CUDA(cudaMemsetAsync(d_full_pts.p, 0, sizeof(double) * 3 * (size_t)Pfull, stream));
  if (P > 0) {
    ord_scatter_points<<<grid_for(P, 256), 256, 0, stream>>>(P, d_pts[cur].p, d_global_of.p, d_full_pts.p);
    OSFM_LAUNCH_CHECK();
  }
  allreduce_dev(d_full_pts.p, 3 * (long long)Pfull);
  download(pts, d_full_pts.p, 3 * (size_t)Pfull, stream);
  // the reprojection errors stay on the device until osfm_ba_get_reprojection_errors fetches them
  reproj_valid = false;
  if (compute_reproj && Nfull > 0) {
    d_reproj.reserve(3 * (size_t)Nfull);
    OSFM_CUDA(cudaMemsetAsync(d_reproj.p, 0, sizeof(double) * 3 * (size_t)Nfull, stream));
    if (rs.N > 0) {
      ba_linearize<2><<<grid_for(rs.N, 128), 128, 0, stream>>>(rs.v, params_of(cur), d_sc.p, d_reproj.p);
      OSFM_LAUNCH_CHECK();
    }
    allreduce_dev(d_reproj.p, 3 * Nfull);
    reproj_valid = true;
  }
  OSFM_CUDA(cudaStreamSynchronize(stream));
  trace("results");
  if (tracing() && world > 1)
    fprintf(stderr, "[osfm_ba] rank %d: %d all-reduces, host %.3f ms, device (traced, serialised) %.3f ms\n", rank, ar_calls,
            ar_host_ms, ar_dev_ms);
  float dev_ms = 0.f;
  OSFM_CUDA(cudaEventElapsedTime(&dev_ms, rs.ev0, rs.ev1));
  cudaEventDestroy(rs.ev0); cudaEventDestroy(rs.ev1);
  const LmState& lm = read_lm();
  sum.time_device_ms = dev_ms;
  sum.time_linearize_ms = lm.phase_ns[LM_PH_LIN] * 1e-6;
  sum.linearize_launches = lm.phase_count[LM_PH_LIN];
  sum.time_schur_ms = lm.phase_ns[LM_PH_SCHUR] * 1e-6;
  sum.schur_launches = lm.phase_count[LM_PH_SCHUR];
  sum.time_pcg_ms = lm.phase_ns[LM_PH_PCG] * 1e-6;
  sum.time_backsub_ms = lm.phase_ns[LM_PH_BACK] * 1e-6;
  sum.num_observations_local = rs.N;
  sum.reduced_dim = rs.nc;
  sum.reduced_blocks = rs.n_blocks_all;
  sum.reduced_nnz = rs.s_total;
  sum.jac_planes = rs.nres * (rs.wc + 3 + 1);
  // kernels executed: the device-driven loop's graph ran the kernels captured into its body once per iteration and
  // those of its conditional bodies once per time taken
  sum.kernel_launches = g_kernel_launches.load() - rs.launches0;
  if (rs.device_loop)
    sum.kernel_launches += (int64_t)(lm.it - 1) * rs.k_body + (int64_t)(lm.n_classic - 1) * rs.k_pcg +
                           (int64_t)(lm.n_eval - 1) * rs.k_eval + (int64_t)(lm.n_success - 1) * rs.k_accept;
  sum.device_loop = rs.device_loop ? 1 : 0;
  sum.time_run_s = std::chrono::duration<double>(std::chrono::high_resolution_clock::now() - rs.t_start).count();
  summary = sum;
  has_run = true;
}

// One LM iteration after ba_lm_next started it: the damped reduced system, its solve, the candidate and its model
// cost change, the candidate cost, and at an accepted step the relinearisation.  Only enqueues work: the host-driven
// loop reads the LM state at each decision, the device-driven loop captures this once into its graph.
void BA::lm_iteration() {
  const int n = rs.n, nc = rs.nc;
  const int graph = rs.cap_graph != nullptr;
  ba_make_diag<<<grid_for(n, 256), 256, 0, stream>>>(d_colnorm2.p, d_scale.p, d_diag.p, n, d_lm.p, d_diag_r.p);
  OSFM_LAUNCH_CHECK();
  build_system(d_diag_r.p, 1.0, nullptr, true);
  OSFM_CUDA(cudaMemsetAsync(d_y.p, 0, sizeof(double) * rs.nz, stream));
  if (nc > 0) {
    solve_reduced();
    if (cap_iter > 0 && read_lm().it == cap_iter) capture_linear_system(cap_iter, h_lm.p->radius);
  }
  back_substitute();
  OSFM_CUDA(cudaMemsetAsync(&d_sc.p->model_change, 0, sizeof(double) * 3, stream));  // model_change, step_norm2, x_norm2
  if (n > 0) {
    ba_model_change_alg<<<grid_for(n, 256), 256, 0, stream>>>(n, nc, rank == 0, d_grad.p, d_scale.p, d_diag_r.p, 1.0, d_y.p, d_sc.p);
    OSFM_LAUNCH_CHECK();
  }
  update_params(0, 1, 1.0, d_ext_lower.p);
  if (world > 1) allreduce_dev(&d_sc.p->model_change, 3);
  ba_lm_check<<<1, 1, 0, stream>>>(d_lm.p, d_sc.p, d_pcg.p, nc, rs.h_eval, graph);
  OSFM_LAUNCH_CHECK();
  rs.k_eval = lm_if(rs.h_eval, LM_EVAL, [&]() {
    eval_cost(1);
    if (rs.constrained) line_search();
  });
  ba_lm_step<<<1, 1, 0, stream>>>(d_lm.p, d_sc.p, rs.h_accept, graph);
  OSFM_LAUNCH_CHECK();
  rs.k_accept = lm_if(rs.h_accept, LM_ACCEPT, [&]() { accept_candidate(); });
}

// Ceres: a problem with parameter bounds is "constrained": TrustRegionMinimizer::DoLineSearch runs a projected Armijo
// search along the step (sufficient decrease 1e-4, at most 20 contractions; bisection here, Ceres' default
// interpolates a cubic) and the candidate is the point it accepts.  The model cost change stays that of the full
// step, as in Ceres.  Host code (host-driven loop): leaves the accepted candidate, its cost and norms in Scalars.
void BA::line_search() {
  const int n = rs.n, nc = rs.nc;
  const double cost = read_lm().cost;
  double cand_cost = read_scalars().cost;
  auto step_to = [&](double alpha) {   // candidate = Project(x - alpha * scale * y) and its cost
    OSFM_CUDA(cudaMemsetAsync(&d_sc.p->step_norm2, 0, sizeof(double) * 2, stream));
    update_params(0, 1, alpha, d_ext_lower.p);
    if (world > 1) allreduce_dev(&d_sc.p->step_norm2, 2);
    eval_cost(1);
  };
  OSFM_CUDA(cudaMemsetAsync(&d_sc.p->gdot, 0, sizeof(double), stream));
  ba_grad_dot<<<grid_for(n, 256), 256, 0, stream>>>(n, nc, rank == 0, d_grad.p, d_scale.p, d_y.p, d_sc.p);
  OSFM_LAUNCH_CHECK();
  if (world > 1) allreduce_dev(&d_sc.p->gdot, 1);
  const double g0 = read_scalars().gdot;
  double alpha = 1.0;
  for (int ls = 0; ls < 20; ++ls) {
    if (ls > 0) { step_to(alpha); cand_cost = read_scalars().cost; }
    if (std::isfinite(cand_cost) && cand_cost <= cost + 1e-4 * g0 * alpha) return;
    alpha *= 0.5;
  }
  step_to(1.0);
}

// The candidate (parameter set 1) becomes the accepted set 0, relinearised there
void BA::accept_candidate() {
  const Params a = params_of(0), c = params_of(1);
  auto copy = [&](double* dst, const double* src, size_t count) {
    if (count) OSFM_CUDA(cudaMemcpyAsync(dst, src, sizeof(double) * count, cudaMemcpyDeviceToDevice, stream));
  };
  copy(a.cam, c.cam, cam_params.size());
  copy(a.inst, c.inst, inst.size());
  copy(a.rc, c.rc, rc.size());
  copy(a.pts, c.pts, 3 * (size_t)rs.P);
  copy(a.ext, c.ext, ext_values.size());
  linearize(0, true);
  ba_lm_accepted<<<1, 1, 0, stream>>>(d_lm.p, d_sc.p);
  OSFM_LAUNCH_CHECK();
}

// The device-driven loop: ba_lm_next, then WHILE (running) { lm_iteration(); ba_lm_next }, captured into one graph
// and launched once.  The counts of kernels captured into each part turn the graph's run into kernels executed.
void BA::run_lm_graph() {
  cudaGraph_t g = nullptr;
  OSFM_CUDA(cudaGraphCreate(&g, 0));
  cudaGraphConditionalHandle h_while;
  OSFM_CUDA(cudaGraphConditionalHandleCreate(&h_while, g, 0, 0));
  rs.cap_deps.clear();
  capture_begin(g);
  ba_lm_next<<<1, 1, 0, stream>>>(d_lm.p, max_iterations, h_while, 1);
  OSFM_LAUNCH_CHECK();
  capture_end();
  cudaGraph_t body = add_conditional(g, h_while, cudaGraphCondTypeWhile);
  OSFM_CUDA(cudaGraphConditionalHandleCreate(&rs.h_pcg, body, 0, 0));
  OSFM_CUDA(cudaGraphConditionalHandleCreate(&rs.h_eval, body, 0, 0));
  OSFM_CUDA(cudaGraphConditionalHandleCreate(&rs.h_accept, body, 0, 0));
  rs.cap_deps.clear();
  const int64_t k0 = g_kernel_launches.load();
  capture_begin(body);
  lm_iteration();
  ba_lm_next<<<1, 1, 0, stream>>>(d_lm.p, max_iterations, h_while, 1);
  OSFM_LAUNCH_CHECK();
  capture_end();
  rs.cap_graph = nullptr;
  rs.k_body = g_kernel_launches.load() - k0 - rs.k_pcg - rs.k_eval - rs.k_accept;
  cudaGraphExec_t exec = nullptr;
  OSFM_CUDA(cudaGraphInstantiate(&exec, g, 0));
  OSFM_CUDA(cudaGraphLaunch(exec, stream));
  OSFM_CUDA(cudaGraphExecDestroy(exec));   // released when the launch completes
  OSFM_CUDA(cudaGraphDestroy(g));
}

void BA::run() {
  OSFM_CUDA(cudaSetDevice(device));
  rs = RunState{};
  rs.t_start = rs.t_prev = std::chrono::high_resolution_clock::now();
  ar_calls = 0; ar_host_ms = 0.0; ar_dev_ms = 0.0;
  if (cam_type.empty() && n_obs_full > 0) throw ArgError("observations but no cameras");
  if (cap_iter > 0 && world > 1) throw ArgError("the linear-system capture supports world == 1 only");
  if (cov_on && world > 1) throw ArgError("covariance estimation supports world == 1 only");
  cap_valid = cov_ran = false;
  if (!cov_on) d_cov.release();   // the dense workspace of an earlier armed run (n_c^2 + m^2 doubles and more)
  rs.launches0 = g_kernel_launches.load();

  plan_layout();
  trace("layout");
  order_observations();
  trace("sort");
  plan_prior_rows();
  trace("priors");
  upload_problem();
  OSFM_CUDA(cudaEventCreate(&rs.ev0)); OSFM_CUDA(cudaEventCreate(&rs.ev1));
  trace("upload");
  trace("pre-struct");
  discover_structure();
  plan_pcg();
  trace("structure");
  if (cov_on) reserve_covariance();

  // ---- Levenberg-Marquardt (Ceres trust_region_minimizer / levenberg_marquardt_strategy) ----
  // The step control is device code (ba_lm_*).  One process, no bounds, no capture and no trace: the loop is one CUDA
  // graph launch (a WHILE node around the iteration body).  Otherwise the host drives the same body and reads the
  // LM state after each decision: the all-reduce callback and the projected line search are host code.
  const int n = rs.n, nc = rs.nc;
  // The graph is built for the pipelined PCG with the classic one as its conditional fallback; a problem whose
  // pipelined plan does not fit runs the host-driven loop.
  rs.device_loop = world == 1 && !rs.constrained && cap_iter == 0 && !tracing() &&
                   !(fallbacks & OSFM_BA_FALLBACK_HOST_LOOP) && rs.pcg_pipe_ok && stream != cudaStreamLegacy;
  if (world > 1) {  // all ranks enter the timed region together (their set-up times differ)
    OSFM_CUDA(cudaMemsetAsync(d_sc.p, 0, sizeof(Scalars), stream));
    allreduce_dev(&d_sc.p->cost, 1);
    OSFM_CUDA(cudaStreamSynchronize(stream));
  }
  OSFM_CUDA(cudaMemsetAsync(d_lm.p, 0, sizeof(LmState), stream));
  OSFM_CUDA(cudaEventRecord(rs.ev0, stream));
  build_segment_tables();
  linearize(0, true);
  if (n > 0) {
    ba_make_scale<<<grid_for(n, 256), 256, 0, stream>>>(d_colnorm2.p, d_scale.p, n);
    OSFM_LAUNCH_CHECK();
  }
  segment_table_scales();   // the scale is constant from here on
  // deflation vectors of the reduced solve: the similarity gauge at the initial poses, in the scaled variables
  if (!(fallbacks & OSFM_BA_FALLBACK_UNDEFLATED_PCG) && rs.pcg_pipe_ok && rs.NI > 0 && nc > 0) {
    d_Wdef.reserve((size_t)PCG_ND * nc);
    OSFM_CUDA(cudaMemsetAsync(d_Wdef.p, 0, sizeof(double) * PCG_ND * (size_t)nc, stream));
    pcg_gauge_vectors<<<grid_for(rs.NI, 128), 128, 0, stream>>>(rs.NI, d_inst_poff.p, params_of(0).inst, d_colnorm2.p,
                                                                    d_scale.p, nc, d_Wdef.p);
    OSFM_LAUNCH_CHECK();
    rs.pcg_pipe.Wdef = d_Wdef.p;
  }
  // every rank takes part in the |x| all-reduce and leaves the loop together: decided on the whole problem's size
  if (rs.n_all > 0) x_norm_pass(0);
  ba_lm_init<<<1, 1, 0, stream>>>(d_lm.p, d_sc.p, rs.n_all > 0 ? 1 : 0);
  OSFM_LAUNCH_CHECK();
  if (rs.device_loop) {
    run_lm_graph();
  } else {
    for (;;) {
      ba_lm_next<<<1, 1, 0, stream>>>(d_lm.p, max_iterations, 0, 0);
      OSFM_LAUNCH_CHECK();
      if (!read_lm().running) break;
      lm_iteration();
    }
  }
  OSFM_CUDA(cudaEventRecord(rs.ev1, stream));
  static const char* const messages[] = {"Maximum number of iterations reached.", "No free parameters.",
                                         "Gradient tolerance reached.", "Minimum trust region radius reached.",
                                         "Too many consecutive invalid steps.", "Parameter tolerance reached.",
                                         "Function tolerance reached."};
  const LmState lm = read_lm();
  const int termination = lm.termination;
  osfm_ba_summary sum{};
  sum.iterations = lm.it;
  sum.successful_steps = lm.n_success;
  sum.linear_solves = lm.n_solves;
  sum.pcg_iterations = lm.pcg_total;
  sum.termination = termination;
  sum.initial_cost = lm.initial_cost;
  eval_cost(0);
  sum.final_cost = read_scalars().cost;
  snprintf(sum.message, sizeof(sum.message), "%s", messages[lm.message]);
  trace("lm");

  if (cov_on) covariance_pass(termination);
  write_results(sum);
}

}  // namespace osfm

// ---------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------
struct osfm_ba : osfm::Handle<osfm::BA> {
  using Handle::Handle;
  static constexpr const char* null_message = "null ba handle";
};
using osfm::ArgError;

extern "C" {

int osfm_camera_num_params(int projection_type) {
  if (projection_type < 0 || projection_type > 9) return -1;
  return osfm::model_num_params(projection_type);
}

int osfm_ba_create(int device, osfm_ba** out) { return osfm::create_handle(device, out); }
int osfm_ba_destroy(osfm_ba* ba) { return osfm::destroy_handle(ba); }

int osfm_ba_set_cameras(osfm_ba* ba, int n, const int32_t* type, const double* params, const int32_t* constant,
                        const double* prior, const double* prior_sigma, const int32_t* prior_log) {
  return osfm::with_handle(ba, [&](osfm::BA& b) {
    if (n < 0 || (n > 0 && (!type || !params || !constant || !prior || !prior_sigma || !prior_log)))
      throw ArgError("bad camera arrays");
    int total = 0;
    for (int k = 0; k < n; ++k) {
      if (type[k] < 0 || type[k] > 9) throw ArgError("Invalid ProjectionType");  // camera_instances.h:232
      total += osfm::model_num_params(type[k]);
    }
    b.cam_type.assign(type, type + n);
    b.cam_const.assign(constant, constant + n);
    b.cam_params.assign(params, params + total);
    b.cam_prior.assign(prior, prior + total);
    b.cam_prior_sigma.assign(prior_sigma, prior_sigma + total);
    b.cam_prior_log.assign(prior_log, prior_log + total);
  });
}
int osfm_ba_set_rig_instances(osfm_ba* ba, int n, const double* pose6, const int32_t* constant,
                              const int32_t* has_position_prior, const double* prior_position3,
                              const double* prior_std3) {
  return osfm::with_handle(ba, [&](osfm::BA& b) {
    if (n < 0 || (n > 0 && (!pose6 || !constant))) throw ArgError("bad rig instance arrays");
    b.inst.assign(pose6, pose6 + 6 * (size_t)n);
    b.inst_const.assign(constant, constant + n);
    b.inst_has_prior.assign(n, 0);
    b.inst_prior_pos.assign(3 * (size_t)n, 0.0);
    b.inst_prior_std.assign(3 * (size_t)n, 1.0);
    if (has_position_prior) {
      if (!prior_position3 || !prior_std3) throw ArgError("position prior arrays missing");
      b.inst_has_prior.assign(has_position_prior, has_position_prior + n);
      b.inst_prior_pos.assign(prior_position3, prior_position3 + 3 * (size_t)n);
      b.inst_prior_std.assign(prior_std3, prior_std3 + 3 * (size_t)n);
    }
  });
}
int osfm_ba_set_rig_cameras(osfm_ba* ba, int n, const double* pose6, const int32_t* constant) {
  return osfm::with_handle(ba, [&](osfm::BA& b) {
    if (n < 0 || (n > 0 && (!pose6 || !constant))) throw ArgError("bad rig camera arrays");
    b.rc.assign(pose6, pose6 + 6 * (size_t)n);
    b.rc_const.assign(constant, constant + n);
    b.rc_prior.clear();
    b.rc_prior_sigma.clear();
  });
}
int osfm_ba_set_rig_camera_priors(osfm_ba* ba, const double* prior6, const double* sigma6) {
  return osfm::with_handle(ba, [&](osfm::BA& b) {
    const size_t n = b.rc_const.size();
    if (!prior6 || !sigma6) { b.rc_prior.clear(); b.rc_prior_sigma.clear(); }
    else { b.rc_prior.assign(prior6, prior6 + 6 * n); b.rc_prior_sigma.assign(sigma6, sigma6 + 6 * n); }
  });
}
int osfm_ba_set_point_priors(osfm_ba* ba, int n, const int32_t* point, const double* prior3, const double* sigma3,
                             const int32_t* has_altitude) {
  return osfm::with_handle(ba, [&](osfm::BA& b) {
    if (n < 0 || (n > 0 && (!point || !prior3 || !sigma3 || !has_altitude))) throw ArgError("bad point prior arrays");
    b.pp_point.assign(point, point + n);
    b.pp_prior.assign(prior3, prior3 + 3 * (size_t)n);
    b.pp_sigma.assign(sigma3, sigma3 + 3 * (size_t)n);
    b.pp_alt.assign(has_altitude, has_altitude + n);
  });
}
int osfm_ba_set_ext_blocks(osfm_ba* ba, int n, const int32_t* size, const double* values, const int32_t* constant,
                           const double* lower_bound) {
  return osfm::with_handle(ba, [&](osfm::BA& b) {
    if (n < 0 || (n > 0 && (!size || !values || !constant || !lower_bound))) throw ArgError("bad ext block arrays");
    size_t total = 0;
    for (int i = 0; i < n; ++i) {
      if (size[i] < 1 || size[i] > 16) throw ArgError("ext block size must be in [1, 16]");
      total += (size_t)size[i];
    }
    b.ext_size.assign(size, size + n);
    b.ext_const.assign(constant, constant + n);
    b.ext_values.assign(values, values + total);
    b.ext_lower.assign(lower_bound, lower_bound + total);
  });
}
int osfm_ba_get_ext_blocks(osfm_ba* ba, double* values) {
  return osfm::with_handle(ba, [&](osfm::BA& b) { std::copy(b.ext_values.begin(), b.ext_values.end(), values); });
}
int osfm_ba_set_side_terms(osfm_ba* ba, int n, const osfm_side_term* terms, int64_t nconsts, const double* consts) {
  return osfm::with_handle(ba, [&](osfm::BA& b) {
    if (n < 0 || nconsts < 0 || (n > 0 && !terms) || (nconsts > 0 && !consts)) throw ArgError("bad side term arrays");
    b.side_terms.assign(terms, terms + n);
    b.side_consts.assign(consts, consts + nconsts);
    for (const auto& t : b.side_terms)
      if (t.loss < -1 || t.loss > OSFM_LOSS_TUKEY) throw ArgError("ceres::LossFunction with that name not found.");
  });
}
int osfm_ba_set_shots(osfm_ba* ba, int n, const int32_t* rig_instance, const int32_t* camera,
                      const int32_t* rig_camera, const int32_t* use_rig_camera) {
  return osfm::with_handle(ba, [&](osfm::BA& b) {
    if (n < 0 || (n > 0 && (!rig_instance || !camera || !rig_camera || !use_rig_camera))) throw ArgError("bad shot arrays");
    b.shot_inst.assign(rig_instance, rig_instance + n);
    b.shot_cam.assign(camera, camera + n);
    b.shot_rc.assign(rig_camera, rig_camera + n);
    b.shot_use_rc.assign(use_rig_camera, use_rig_camera + n);
  });
}
int osfm_ba_set_points(osfm_ba* ba, int n, const double* xyz, const int32_t* constant) {
  return osfm::with_handle(ba, [&](osfm::BA& b) {
    if (n < 0 || (n > 0 && (!xyz || !constant))) throw ArgError("bad point arrays");
    b.pts.assign(xyz, xyz + 3 * (size_t)n);
    b.pt_const.assign(constant, constant + n);
  });
}
int osfm_ba_set_observations(osfm_ba* ba, int64_t n, const int32_t* shot, const int32_t* point, const double* xy,
                             const double* std_deviation) {
  return osfm::with_handle(ba, [&](osfm::BA& b) {
    if (n < 0 || (n > 0 && (!shot || !point || !xy || !std_deviation))) throw ArgError("bad observation arrays");
    // straight to the device: the ordering, the index checks and the 1/sigma happen there (ba_order.cuh)
    if (b.obs_pending) { OSFM_CUDA(cudaStreamSynchronize(b.copy_stream)); b.obs_pending = false; }
    const size_t nz = (size_t)std::max<int64_t>(n, 1);
    b.d_raw_shot.reserve(nz); b.d_raw_point.reserve(nz); b.d_raw_xy.reserve(2 * nz); b.d_raw_sigma.reserve(nz);
    if (n > 0) {
      OSFM_CUDA(cudaMemcpyAsync(b.d_raw_shot.p, shot, sizeof(int32_t) * n, cudaMemcpyHostToDevice, b.own_stream));
      OSFM_CUDA(cudaMemcpyAsync(b.d_raw_point.p, point, sizeof(int32_t) * n, cudaMemcpyHostToDevice, b.own_stream));
      OSFM_CUDA(cudaMemcpyAsync(b.d_raw_xy.p, xy, sizeof(double) * 2 * n, cudaMemcpyHostToDevice, b.own_stream));
      OSFM_CUDA(cudaMemcpyAsync(b.d_raw_sigma.p, std_deviation, sizeof(double) * n, cudaMemcpyHostToDevice, b.own_stream));
      OSFM_CUDA(cudaStreamSynchronize(b.own_stream));
    }
    b.n_obs_full = n;
    b.has_run = false;
  });
}
int osfm_ba_set_observations_async(osfm_ba* ba, int64_t n, const int32_t* shot, const int32_t* point, const double* xy,
                                   const double* std_deviation) {
  return osfm::with_handle(ba, [&](osfm::BA& b) {
    if (n < 0 || (n > 0 && (!shot || !point || !xy || !std_deviation))) throw ArgError("bad observation arrays");
    if (b.obs_pending) { OSFM_CUDA(cudaStreamSynchronize(b.copy_stream)); b.obs_pending = false; }
    const size_t nz = (size_t)std::max<int64_t>(n, 1);
    b.d_raw_shot.reserve(nz); b.d_raw_point.reserve(nz); b.d_raw_xy.reserve(2 * nz); b.d_raw_sigma.reserve(nz);
    if (n > 0) {
      // the indices are what the ordering needs first: they are on the device when the call returns; the measurements
      // follow on the copy stream and run() waits for them (an event) right before the kernel that gathers them
      OSFM_CUDA(cudaMemcpyAsync(b.d_raw_shot.p, shot, sizeof(int32_t) * n, cudaMemcpyHostToDevice, b.own_stream));
      OSFM_CUDA(cudaMemcpyAsync(b.d_raw_point.p, point, sizeof(int32_t) * n, cudaMemcpyHostToDevice, b.own_stream));
      OSFM_CUDA(cudaMemcpyAsync(b.d_raw_xy.p, xy, sizeof(double) * 2 * n, cudaMemcpyHostToDevice, b.copy_stream));
      OSFM_CUDA(cudaMemcpyAsync(b.d_raw_sigma.p, std_deviation, sizeof(double) * n, cudaMemcpyHostToDevice, b.copy_stream));
      OSFM_CUDA(cudaEventRecord(b.ev_obs, b.copy_stream));
      b.obs_pending = true;
      OSFM_CUDA(cudaStreamSynchronize(b.own_stream));
    }
    b.n_obs_full = n;
    b.has_run = false;
  });
}
int osfm_ba_set_options(osfm_ba* ba, int loss, double loss_threshold, int max_iterations, const char* linear_solver,
                        int compute_reprojection_errors) {
  return osfm::with_handle(ba, [&](osfm::BA& b) {
    if (loss < 0 || loss > 4) throw ArgError("ceres::LossFunction with that name not found.");  // bundle_adjuster.cc:427
    if (linear_solver) {
      const std::string s(linear_solver);
      // ceres::StringToLinearSolverType names (bundle_adjuster.cc:1105-1109)
      static const char* known[] = {"DENSE_NORMAL_CHOLESKY", "DENSE_QR", "SPARSE_NORMAL_CHOLESKY", "DENSE_SCHUR",
                                    "SPARSE_SCHUR", "ITERATIVE_SCHUR", "CGNR"};
      bool found = false;
      for (const char* k : known) found |= (s == k);
      if (!found) throw std::runtime_error("Linear solver type " + s + " doesn't exist.");
    }
    b.loss = loss;
    b.loss_a = loss_threshold;
    b.max_iterations = max_iterations;
    b.compute_reproj = compute_reprojection_errors != 0;
  });
}
int osfm_ba_set_distributed(osfm_ba* ba, int rank, int world, osfm_allreduce_fn fn, void* user) {
  return osfm::with_handle(ba, [&](osfm::BA& b) {
    if (world < 1 || rank < 0 || rank >= world) throw ArgError("bad rank/world");
    if (world > 1 && !fn && !(b.nccl_comm && b.nccl_world == world && b.nccl_rank == rank))
      throw ArgError("world > 1 needs an all-reduce callback or osfm_ba_set_nccl");
    b.rank = rank; b.world = world; b.allreduce = fn; b.allreduce_user = user;
  });
}
int osfm_nccl_unique_id(char* out128) {
  OSFM_API_BEGIN
  if (!out128) throw ArgError("null id buffer");
  OsfmNcclId id;
  osfm::nccl_check(osfm::nccl_api().GetUniqueId(&id), "ncclGetUniqueId");
  std::memcpy(out128, id.internal, 128);
  OSFM_API_END
}
int osfm_ba_set_nccl(osfm_ba* ba, int rank, int world, const char* id128) {
  return osfm::with_handle(ba, [&](osfm::BA& b) {
    if (world < 2 || rank < 0 || rank >= world || !id128) throw ArgError("bad rank/world/id");
    if (b.nccl_comm) { osfm::nccl_api().CommDestroy(b.nccl_comm); b.nccl_comm = nullptr; }
    OsfmNcclId id;
    std::memcpy(id.internal, id128, 128);
    osfm::nccl_check(osfm::nccl_api().CommInitRank(&b.nccl_comm, world, id, rank), "ncclCommInitRank");
    b.nccl_rank = rank; b.nccl_world = world;
  });
}
int osfm_ba_set_stream(osfm_ba* ba, void* cuda_stream) {
  return osfm::with_handle(ba, [&](osfm::BA& b) {
    b.stream = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : b.own_stream;
  });
}
int osfm_ba_run(osfm_ba* ba) {
  return osfm::with_handle(ba, [&](osfm::BA& b) {
    try {
      b.run();
    } catch (...) {
      // an asynchronous observation upload must not outlive the call: the caller may free its arrays now
      if (b.obs_pending) { cudaStreamSynchronize(b.copy_stream); b.obs_pending = false; }
      throw;
    }
  });
}
int osfm_ba_get_summary(osfm_ba* ba, osfm_ba_summary* out) {
  return osfm::with_handle(ba, [&](osfm::BA& b) {
    if (!out) throw ArgError("null out");
    *out = b.summary;
  });
}
int osfm_ba_get_cameras(osfm_ba* ba, double* params_flat) {
  return osfm::with_handle(ba, [&](osfm::BA& b) { std::copy(b.cam_params.begin(), b.cam_params.end(), params_flat); });
}
int osfm_ba_get_rig_instances(osfm_ba* ba, double* pose6) {
  return osfm::with_handle(ba, [&](osfm::BA& b) { std::copy(b.inst.begin(), b.inst.end(), pose6); });
}
int osfm_ba_get_rig_cameras(osfm_ba* ba, double* pose6) {
  return osfm::with_handle(ba, [&](osfm::BA& b) { std::copy(b.rc.begin(), b.rc.end(), pose6); });
}
int osfm_ba_get_points(osfm_ba* ba, double* xyz) {
  return osfm::with_handle(ba, [&](osfm::BA& b) { std::copy(b.pts.begin(), b.pts.end(), xyz); });
}
int osfm_ba_get_reprojection_errors(osfm_ba* ba, double* out_n_by_3) {
  return osfm::with_handle(ba, [&](osfm::BA& b) {
    if (!b.has_run) throw std::runtime_error("run() has not been called");
    if (b.n_obs_full > 0) {
      if (b.reproj_valid)
        OSFM_CUDA(cudaMemcpy(out_n_by_3, b.d_reproj.p, sizeof(double) * 3 * (size_t)b.n_obs_full, cudaMemcpyDeviceToHost));
      else
        std::fill(out_n_by_3, out_n_by_3 + 3 * (size_t)b.n_obs_full, 0.0);
    }
  });
}

int osfm_ba_eval_observation(int device, int projection_type, const double* camera, const double* rig_instance,
                             const double* rig_camera, int use_rig_camera, const double* point,
                             const double* observed, double std_deviation, double* r, double* jac_camera,
                             double* jac_instance, double* jac_rig_camera, double* jac_point, int* num_residuals) {
  OSFM_API_BEGIN
  if (projection_type < 0 || projection_type > 9) throw ArgError("Invalid ProjectionType");
  OSFM_CUDA(cudaSetDevice(device));
  const int C = osfm::model_num_params(projection_type);
  double in[34] = {0};
  for (int i = 0; i < C; ++i) in[i] = camera[i];
  for (int i = 0; i < 6; ++i) in[16 + i] = rig_instance[i];
  for (int i = 0; i < 6; ++i) in[22 + i] = rig_camera ? rig_camera[i] : 0.0;
  for (int i = 0; i < 3; ++i) in[28 + i] = point[i];
  in[31] = observed[0]; in[32] = observed[1]; in[33] = 1.0 / std_deviation;
  double *d_in = nullptr, *d_out = nullptr;
  int* d_n = nullptr;
  OSFM_CUDA(cudaMalloc(&d_in, sizeof(in)));
  OSFM_CUDA(cudaMalloc(&d_out, sizeof(double) * 96));
  OSFM_CUDA(cudaMalloc(&d_n, sizeof(int)));
  OSFM_CUDA(cudaMemcpy(d_in, in, sizeof(in), cudaMemcpyHostToDevice));
  osfm::ba_eval_one<<<1, 1>>>(projection_type, d_in, use_rig_camera, d_out, d_n);
  OSFM_LAUNCH_CHECK();
  double out[96];
  int nres = 0;
  OSFM_CUDA(cudaMemcpy(out, d_out, sizeof(out), cudaMemcpyDeviceToHost));
  OSFM_CUDA(cudaMemcpy(&nres, d_n, sizeof(int), cudaMemcpyDeviceToHost));
  cudaFree(d_in); cudaFree(d_out); cudaFree(d_n);
  for (int i = 0; i < nres; ++i) r[i] = out[i];
  for (int i = 0; i < nres * C; ++i) jac_camera[i] = out[3 + i];
  for (int i = 0; i < nres * 6; ++i) jac_instance[i] = out[51 + i];
  for (int i = 0; i < nres * 6; ++i) jac_rig_camera[i] = out[69 + i];
  for (int i = 0; i < nres * 3; ++i) jac_point[i] = out[87 + i];
  if (num_residuals) *num_residuals = nres;
  OSFM_API_END
}

int osfm_ba_capture_linear_system(osfm_ba* ba, int iteration) {
  return osfm::with_handle(ba, [&](osfm::BA& b) {
    if (iteration < 0) throw ArgError("capture iteration must be >= 0");
    if (iteration > 0 && b.world != 1) throw ArgError("the linear-system capture supports world == 1 only");
    b.cap_iter = iteration;
  });
}

int osfm_ba_set_fallbacks(osfm_ba* ba, unsigned mask) {
  return osfm::with_handle(ba, [&](osfm::BA& b) {
    if (mask & ~osfm::BA_FALLBACKS_ALL) throw ArgError("unknown OSFM_BA_FALLBACK_* bits");
    b.fallbacks = mask;
  });
}

int osfm_ba_get_captured_system(osfm_ba* ba, osfm_ba_capture* info, double* S, double* rhs, double* y, double* scale,
                                double* diag, double* grad) {
  return osfm::with_handle(ba, [&](osfm::BA& b) {
    if (!b.cap_valid) throw std::runtime_error("no linear system was captured (not armed, or the run ended earlier)");
    const int nc = b.cap_info.nc, n = b.cap_info.n;
    if (nc > 8192) throw ArgError("reduced system too large for a dense copy (nc > 8192)");
    if (info) *info = b.cap_info;
    if (S) {
      std::fill(S, S + (size_t)nc * nc, 0.0);
      const double* val = b.cap_sbuf.data() + b.cap_nc_pad;
      for (const int4& u : b.cap_upper) {
        const int oi = b.cap_blk_off[u.x], oj = b.cap_blk_off[u.y], si = b.cap_blk_sz[u.x], sj = b.cap_blk_sz[u.y];
        for (int r = 0; r < si; ++r)   // block (bi, bj), row-major si x sj
          for (int c = 0; c < sj; ++c) S[(size_t)(oi + r) * nc + oj + c] = val[u.z + r * sj + c];
        if (u.w >= 0)
          for (int r = 0; r < sj; ++r)   // its own lower block (bj, bi), row-major sj x si
            for (int c = 0; c < si; ++c) S[(size_t)(oj + r) * nc + oi + c] = val[u.w + r * si + c];
      }
    }
    if (rhs) std::copy(b.cap_sbuf.begin(), b.cap_sbuf.begin() + nc, rhs);
    if (y) std::copy(b.cap_y.begin(), b.cap_y.end(), y);
    // point side: engine order -> free points by ascending caller index
    std::vector<int> dst(std::max(n, 1));
    for (int i = 0; i < nc; ++i) dst[i] = i;
    {
      std::vector<std::pair<int, int>> fp;   // (caller index, engine free index)
      for (size_t q = 0; q < b.cap_pt_poff.size(); ++q)
        if (b.cap_pt_poff[q] >= 0) fp.emplace_back(b.cap_global_of[q], b.cap_pt_poff[q]);
      if (nc + 3 * (int)fp.size() != n) throw std::runtime_error("captured point layout is inconsistent");
      std::sort(fp.begin(), fp.end());
      for (size_t k = 0; k < fp.size(); ++k)
        for (int j = 0; j < 3; ++j) dst[nc + 3 * fp[k].second + j] = nc + 3 * (int)k + j;
    }
    auto scatter = [&](const std::vector<double>& src, double* out) {
      if (out)
        for (int i = 0; i < n; ++i) out[dst[i]] = src[i];
    };
    scatter(b.cap_scale, scale);
    scatter(b.cap_diag, diag);
    scatter(b.cap_grad, grad);
  });
}

int osfm_ba_get_captured_side_rows(osfm_ba* ba, double* r, double* J) {
  return osfm::with_handle(ba, [&](osfm::BA& b) {
    if (!b.cap_valid) throw std::runtime_error("no linear system was captured (not armed, or the run ended earlier)");
    if (r) std::copy(b.cap_side_r.begin(), b.cap_side_r.end(), r);
    if (J) std::copy(b.cap_side_J.begin(), b.cap_side_J.end(), J);
  });
}

int osfm_ba_get_captured_parameters(osfm_ba* ba, double* cam_params, double* inst_pose6, double* rig_camera_pose6,
                                    double* points, double* ext_values) {
  return osfm::with_handle(ba, [&](osfm::BA& b) {
    if (!b.cap_valid) throw std::runtime_error("no linear system was captured (not armed, or the run ended earlier)");
    if (cam_params) std::copy(b.cap_cam.begin(), b.cap_cam.end(), cam_params);
    if (inst_pose6) std::copy(b.cap_inst.begin(), b.cap_inst.end(), inst_pose6);
    if (rig_camera_pose6) std::copy(b.cap_rc.begin(), b.cap_rc.end(), rig_camera_pose6);
    if (ext_values) std::copy(b.cap_ext.begin(), b.cap_ext.end(), ext_values);
    if (points)   // engine order -> the caller's
      for (size_t q = 0; q < b.cap_global_of.size(); ++q)
        for (int j = 0; j < 3; ++j) points[3 * (size_t)b.cap_global_of[q] + j] = b.cap_pts[3 * q + j];
  });
}

int osfm_ba_set_compute_covariances(osfm_ba* ba, int enable) {
  return osfm::with_handle(ba, [&](osfm::BA& b) { b.cov_on = enable != 0; });
}

int osfm_ba_get_covariances(osfm_ba* ba, int* valid, int* status, double* out) {
  return osfm::with_handle(ba, [&](osfm::BA& b) {
    if (!b.cov_ran) throw std::runtime_error("the last run() did not compute covariances (not armed, or it failed)");
    if (valid) *valid = b.cov_valid ? 1 : 0;
    if (status) *status = b.cov_status;
    if (out) std::copy(b.cov_out.begin(), b.cov_out.end(), out);
  });
}

int osfm_ba_get_covariance_timing(osfm_ba* ba, double* pass_ms, double* cholesky_ms) {
  return osfm::with_handle(ba, [&](osfm::BA& b) {
    if (!b.cov_ran) throw std::runtime_error("the last run() did not compute covariances (not armed, or it failed)");
    if (pass_ms) *pass_ms = b.cov_pass_ms;
    if (cholesky_ms) *cholesky_ms = b.cov_chol_ms;
  });
}

}  // extern "C"
