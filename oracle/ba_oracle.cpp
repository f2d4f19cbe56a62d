// ORACLE — TEST INFRASTRUCTURE ONLY (see ba_functors.hpp header).
//
// C entry points (ctypes) around the restated functors, plus the bulk
// (OpenMP) pieces of one Levenberg-Marquardt iteration that oracle/ba_lm.py
// drives: robustified linearisation, normal-equation blocks, Schur complement
// on the points, back-substitution, model cost change.  This is the
// "CPU restatement of the Ceres path (not Ceres)" of BASELINE.md §3: Ceres is
// a third-party dependency absent from the OpenSfM tree (conda ceres-solver 2.1,
// conda.yml:10); its published algorithm is restated (SURVEY.md §8c box) and
// anchored on the reference's call sites:
//   opensfm/src/bundle/src/bundle_adjuster.cc:595-1121 (problem assembly),
//   :414-429 (loss functions), :568-593 (camera prior, log-scale focal),
//   :745-778 (rig-instance position prior), :1196-1208 (reprojection errors).
#include <omp.h>

#include <algorithm>
#include <cstdint>
#include <vector>

#include "ba_functors.hpp"
#include "ba_side_terms.hpp"

using namespace oracle;

namespace {

enum Loss { TRIVIAL = 0, HUBER = 1, SOFTLONE = 2, CAUCHY = 3, ARCTAN = 4 };

// ceres::LossFunction::Evaluate for the five losses CreateLossFunction
// (bundle_adjuster.cc:414-429) can return; rho[0]=rho(s), rho[1]=rho'(s).
// (rho'' <= 0 for all of them, so Ceres' corrector reduces to sqrt(rho').)
inline void loss_eval(int loss, double a, double s, double* rho) {
  const double kMin = DBL_MIN;
  switch (loss) {
    case TRIVIAL: rho[0] = s; rho[1] = 1.0; return;
    case HUBER: {
      const double b = a * a;
      if (s > b) {
        const double r = std::sqrt(s);
        rho[0] = 2.0 * a * r - b;
        rho[1] = std::max(kMin, a / r);
      } else {
        rho[0] = s; rho[1] = 1.0;
      }
      return;
    }
    case SOFTLONE: {
      const double b = a * a, c = 1.0 / b;
      const double sum = 1.0 + s * c, tmp = std::sqrt(sum);
      rho[0] = 2.0 * b * (tmp - 1.0);
      rho[1] = std::max(kMin, 1.0 / tmp);
      return;
    }
    case CAUCHY: {
      const double b = a * a, c = 1.0 / b;
      const double sum = 1.0 + s * c, inv = 1.0 / sum;
      rho[0] = b * std::log(sum);
      rho[1] = std::max(kMin, inv);
      return;
    }
    case ARCTAN: {
      const double b = 1.0 / (a * a);
      const double sum = 1.0 + s * s * b, inv = 1.0 / sum;
      rho[0] = a * std::atan2(s, a);
      rho[1] = std::max(kMin, inv);
      return;
    }
  }
  throw std::runtime_error("bad loss");
}

struct Problem {
  // structure
  int K = 0, NI = 0, NR = 0, S = 0, P = 0;
  int64_t N = 0;
  std::vector<int> cam_type, cam_off, cam_np;
  std::vector<int> shot_inst, shot_cam, shot_rc, shot_use_rc;
  std::vector<int> obs_shot, obs_point;
  std::vector<double> obs_xy, obs_sigma;
  // free/constant -> offsets in the reduced (camera-side) vector, -1 = constant
  std::vector<int> cam_poff, inst_poff, rc_poff, pt_poff;  // pt_poff: index of free point or -1
  int nc = 0, npts_free = 0;
  // priors
  std::vector<double> cam_prior, cam_prior_sigma;  // same layout as cam params
  std::vector<int> cam_prior_log;                  // 1 = logarithmic (focal, aspect ratio)
  std::vector<int> inst_has_prior;
  std::vector<double> inst_prior_pos, inst_prior_std;
  // current values
  std::vector<double> cam, inst, rc, pts;
  // loss
  int loss = SOFTLONE;
  double loss_a = 1.0;
  // linearisation storage
  int wc = 0;  // camera-side Jacobian width per observation (max over obs)
  std::vector<int> obs_nres;
  std::vector<double> r;   // N x 3   (robustified)
  std::vector<double> Jc;  // N x 3 x wc
  std::vector<double> Jp;  // N x 3 x 3
  std::vector<int64_t> pt_start;  // CSR over points (obs sorted by point)
  std::vector<int64_t> pt_obs;
  // prior residual rows: stored as (row value, global column, derivative)
  struct PriorRow { double r; int col; double d; };
  std::vector<PriorRow> prior_rows;
  std::vector<double> scale;  // Jacobi column scaling, size nc + 3*npts_free (1 if unset)
  // ---- secondary residuals (bundle_adjuster.cc:610-625, 672-790, 817-1101) ----
  // ext blocks: camera biases (7), reconstruction scales (1), std-deviation scales (1)
  int NE = 0;
  std::vector<int> ext_off, ext_np, ext_poff;
  std::vector<double> ext, ext_lower;
  struct SideTerm { int type, nres, nblocks, kind[6], idx[6], loss; double loss_a; int cofs, aux[4]; };
  std::vector<SideTerm> side_terms;
  std::vector<double> side_consts;
  struct DenseRows { int nres, ncols; int cols[MAXD]; double J[7 * MAXD]; double r[7]; };  // robustified rows
  std::vector<DenseRows> side_rows;
  std::vector<int> pp_of_point;            // per point: index of its prior or -1
  std::vector<double> pp_prior, pp_sigma;  // per prior: xyz
  std::vector<int> pp_alt;
  std::vector<double> rc_prior, rc_prior_sigma;  // empty = no rig-camera priors
};

// parameter block (kind 0 camera, 1 rig instance, 2 rig camera, 3 ext) -> values, size, reduced column
struct BlockRef { const double* p; int np; int col; };
inline BlockRef block_ref(const Problem& pb, int kind, int idx) {
  switch (kind) {
    case 0: return {&pb.cam[pb.cam_off[idx]], pb.cam_np[idx], pb.cam_poff[idx]};
    case 1: return {&pb.inst[6 * (size_t)idx], 6, pb.inst_poff[idx]};
    case 2: return {&pb.rc[6 * (size_t)idx], 6, pb.rc_poff[idx]};
    default: return {&pb.ext[pb.ext_off[idx]], pb.ext_np[idx], pb.ext_poff[idx]};
  }
}

// Cost of the side terms at the current parameters; with_rows: also their robustified residuals and Jacobians
// (ceres::Jet-style forward differentiation of the templated functors, Corrector with rho'' <= 0).
inline double eval_side_terms(Problem* pb, bool with_rows) {
  double cost = 0.0;
  if (with_rows) pb->side_rows.assign(pb->side_terms.size(), Problem::DenseRows());
  for (size_t t = 0; t < pb->side_terms.size(); ++t) {
    const Problem::SideTerm& st = pb->side_terms[t];
    BlockRef br[6];
    int start[7] = {0};
    for (int b = 0; b < st.nblocks; ++b) {
      br[b] = block_ref(*pb, st.kind[b], st.idx[b]);
      start[b + 1] = start[b] + br[b].np;
    }
    const int NP = start[st.nblocks];
    const double* c = pb->side_consts.data() + st.cofs;
    double rho[2] = {0.0, 1.0};
    double rv[7];
    bool ok;
    Problem::DenseRows rows;
    rows.nres = st.nres; rows.ncols = NP;
    if (with_rows) {
      std::vector<Dual> x(NP);
      const Dual* xp[6];
      for (int b = 0; b < st.nblocks; ++b) {
        xp[b] = x.data() + start[b];
        for (int q = 0; q < br[b].np; ++q) x[start[b] + q] = Dual::variable(br[b].p[q], start[b] + q);
      }
      Dual r[7];
      ok = side_residual<Dual>(st.type, c, st.aux, xp, r);
      for (int k = 0; k < st.nres; ++k) {
        rv[k] = r[k].v;
        for (int j = 0; j < NP; ++j) rows.J[k * MAXD + j] = r[k].d[j];
      }
      for (int b = 0; b < st.nblocks; ++b)
        for (int q = 0; q < br[b].np; ++q) rows.cols[start[b] + q] = br[b].col >= 0 ? br[b].col + q : -1;
    } else {
      std::vector<double> x(NP);
      const double* xp[6];
      for (int b = 0; b < st.nblocks; ++b) {
        xp[b] = x.data() + start[b];
        for (int q = 0; q < br[b].np; ++q) x[start[b] + q] = br[b].p[q];
      }
      ok = side_residual<double>(st.type, c, st.aux, xp, rv);
    }
    double s = 0.0;
    for (int k = 0; k < st.nres; ++k) s += rv[k] * rv[k];
    if (st.loss < 0) { rho[0] = s; rho[1] = 1.0; }
    else if (st.loss == 5) tukey_loss(st.loss_a, s, rho);
    else loss_eval(st.loss, st.loss_a, s, rho);
    if (!ok) { cost = std::nan(""); rho[1] = 0.0; }
    bool any_free = false;  // Ceres removes residual blocks whose parameter blocks are all constant (fixed_cost)
    for (int b = 0; b < st.nblocks; ++b) any_free |= br[b].col >= 0;
    if (any_free) cost += 0.5 * rho[0];
    if (with_rows) {
      const double w = std::sqrt(rho[1]);
      for (int k = 0; k < st.nres; ++k) {
        rows.r[k] = w * rv[k];
        for (int j = 0; j < NP; ++j) rows.J[k * MAXD + j] *= w;
      }
      pb->side_rows[t] = rows;
    }
  }
  return cost;
}

// Columns of the camera-side Jacobian of one observation:
// local layout [camera C | instance 6 | rig camera 6].
struct ObsCols {
  int goff[3];  // global offsets (or -1)
  int lsz[3];
  int lstart[3];
};
inline ObsCols obs_cols(const Problem& pb, int shot) {
  ObsCols oc;
  const int cam = pb.shot_cam[shot];
  oc.goff[0] = pb.cam_poff[cam]; oc.lsz[0] = pb.cam_np[cam]; oc.lstart[0] = 0;
  oc.goff[1] = pb.inst_poff[pb.shot_inst[shot]]; oc.lsz[1] = 6; oc.lstart[1] = oc.lsz[0];
  oc.goff[2] = pb.shot_use_rc[shot] ? pb.rc_poff[pb.shot_rc[shot]] : -1; oc.lsz[2] = 6;
  oc.lstart[2] = oc.lsz[0] + 6;
  return oc;
}

// every parameter block of the observation's residual block is constant: Ceres drops the block from the reduced
// program (its cost only enters Summary::fixed_cost, not the minimised cost the tolerances look at)
inline bool obs_all_constant(const Problem& pb, int64_t i) {
  const int shot = pb.obs_shot[i];
  return pb.cam_poff[pb.shot_cam[shot]] < 0 && pb.inst_poff[pb.shot_inst[shot]] < 0 &&
         (!pb.shot_use_rc[shot] || pb.rc_poff[pb.shot_rc[shot]] < 0) && pb.pt_poff[pb.obs_point[i]] < 0;
}

}  // namespace

extern "C" {

int oracle_camera_num_params(int type) { return camera_num_params(type); }

void oracle_project(int type, const double* params, const double* point, double* out2) {
  camera_project<double>(type, point, params, out2);
}

int oracle_reproj_analytic(int type, const double* camera, const double* rig_instance, const double* rig_camera,
                           int use_rig_camera, const double* point, const double* observed, double sigma,
                           double* r, double* jc, double* ji, double* jrc, double* jp) {
  return reprojection_analytic(type, camera, rig_instance, rig_camera, use_rig_camera != 0, point, observed, sigma,
                               r, jc, ji, jrc, jp);
}

int oracle_reproj_autodiff(int type, const double* camera, const double* rig_instance, const double* rig_camera,
                           int use_rig_camera, const double* point, const double* observed, double sigma,
                           double* r, double* jc, double* ji, double* jrc, double* jp) {
  return reprojection_autodiff(type, camera, rig_instance, rig_camera, use_rig_camera != 0, point, observed, sigma,
                               r, jc, ji, jrc, jp);
}

void oracle_loss(int loss, double a, double s, double* rho2) { loss_eval(loss, a, s, rho2); }

// ---------------------------------------------------------------------------
// Bulk problem handle.
// ---------------------------------------------------------------------------
void* oba_create(int K, const int* cam_type, const double* cam_params, const int* cam_const,
                 const double* cam_prior, const double* cam_prior_sigma, const int* cam_prior_log,
                 int NI, const double* inst, const int* inst_const, const int* inst_has_prior,
                 const double* inst_prior_pos, const double* inst_prior_std,
                 int NR, const double* rc, const int* rc_const,
                 int S, const int* shot_inst, const int* shot_cam, const int* shot_rc, const int* shot_use_rc,
                 int P, const double* pts, const int* pt_const,
                 int64_t N, const int* obs_shot, const int* obs_point, const double* obs_xy,
                 const double* obs_sigma, int loss, double loss_a) {
  Problem* pb = new Problem();
  pb->K = K; pb->NI = NI; pb->NR = NR; pb->S = S; pb->P = P; pb->N = N;
  pb->cam_type.assign(cam_type, cam_type + K);
  pb->cam_off.resize(K + 1);
  pb->cam_np.resize(K);
  pb->cam_off[0] = 0;
  for (int k = 0; k < K; ++k) {
    pb->cam_np[k] = camera_num_params(cam_type[k]);
    pb->cam_off[k + 1] = pb->cam_off[k] + pb->cam_np[k];
  }
  const int ncp = pb->cam_off[K];
  pb->cam.assign(cam_params, cam_params + ncp);
  pb->cam_prior.assign(cam_prior, cam_prior + ncp);
  pb->cam_prior_sigma.assign(cam_prior_sigma, cam_prior_sigma + ncp);
  pb->cam_prior_log.assign(cam_prior_log, cam_prior_log + ncp);
  pb->inst.assign(inst, inst + 6 * (size_t)NI);
  pb->rc.assign(rc, rc + 6 * (size_t)NR);
  pb->pts.assign(pts, pts + 3 * (size_t)P);
  pb->inst_has_prior.assign(inst_has_prior, inst_has_prior + NI);
  pb->inst_prior_pos.assign(inst_prior_pos, inst_prior_pos + 3 * (size_t)NI);
  pb->inst_prior_std.assign(inst_prior_std, inst_prior_std + 3 * (size_t)NI);
  pb->shot_inst.assign(shot_inst, shot_inst + S);
  pb->shot_cam.assign(shot_cam, shot_cam + S);
  pb->shot_rc.assign(shot_rc, shot_rc + S);
  pb->shot_use_rc.assign(shot_use_rc, shot_use_rc + S);
  pb->obs_shot.assign(obs_shot, obs_shot + N);
  pb->obs_point.assign(obs_point, obs_point + N);
  pb->obs_xy.assign(obs_xy, obs_xy + 2 * N);
  pb->obs_sigma.assign(obs_sigma, obs_sigma + N);
  pb->loss = loss; pb->loss_a = loss_a;
  // reduced-vector layout: [free cameras | free instances | free rig cameras]
  int off = 0;
  pb->cam_poff.resize(K); pb->inst_poff.resize(NI); pb->rc_poff.resize(NR); pb->pt_poff.resize(P);
  for (int k = 0; k < K; ++k) { pb->cam_poff[k] = cam_const[k] ? -1 : off; if (!cam_const[k]) off += pb->cam_np[k]; }
  for (int i = 0; i < NI; ++i) { pb->inst_poff[i] = inst_const[i] ? -1 : off; if (!inst_const[i]) off += 6; }
  for (int i = 0; i < NR; ++i) { pb->rc_poff[i] = rc_const[i] ? -1 : off; if (!rc_const[i]) off += 6; }
  pb->nc = off;
  int nf = 0;
  for (int p = 0; p < P; ++p) pb->pt_poff[p] = pt_const[p] ? -1 : nf++;
  pb->npts_free = nf;
  int wc = 0;
  for (int s = 0; s < S; ++s) wc = std::max(wc, pb->cam_np[pb->shot_cam[s]] + 6 + (pb->shot_use_rc[s] ? 6 : 0));
  pb->wc = wc;
  // CSR of observations per point
  pb->pt_start.assign(P + 1, 0);
  for (int64_t i = 0; i < N; ++i) pb->pt_start[obs_point[i] + 1]++;
  for (int p = 0; p < P; ++p) pb->pt_start[p + 1] += pb->pt_start[p];
  pb->pt_obs.resize(N);
  std::vector<int64_t> fill(pb->pt_start.begin(), pb->pt_start.end() - 1);
  for (int64_t i = 0; i < N; ++i) pb->pt_obs[fill[obs_point[i]]++] = i;
  pb->scale.assign(pb->nc + 3 * (size_t)nf, 1.0);
  return pb;
}

// Secondary residuals of the problem (call right after oba_create): ext blocks extend the reduced vector
// [.. | free ext blocks]; term records = 21 ints each (type, nres, nblocks, kind[6], idx[6], loss, cofs, aux[4]).
void oba_set_secondary(void* h, int NE, const int* ext_size, const double* ext_values, const int* ext_const,
                       const double* ext_lower, int NT, const int* term_ints, const double* term_loss_a, int nconsts,
                       const double* consts, int NPP, const int* pp_point, const double* pp_prior,
                       const double* pp_sigma, const int* pp_alt, int has_rc_prior, const double* rc_prior,
                       const double* rc_sigma) {
  Problem* pb = static_cast<Problem*>(h);
  pb->NE = NE;
  pb->ext_off.assign(NE + 1, 0); pb->ext_np.assign(ext_size, ext_size + NE); pb->ext_poff.assign(NE, -1);
  int off = pb->nc;
  for (int i = 0; i < NE; ++i) {
    pb->ext_off[i + 1] = pb->ext_off[i] + ext_size[i];
    if (!ext_const[i]) { pb->ext_poff[i] = off; off += ext_size[i]; }
  }
  pb->nc = off;
  pb->ext.assign(ext_values, ext_values + pb->ext_off[NE]);
  pb->ext_lower.assign(ext_lower, ext_lower + pb->ext_off[NE]);
  pb->side_terms.resize(NT);
  for (int t = 0; t < NT; ++t) {
    const int* q = term_ints + 21 * t;
    Problem::SideTerm& st = pb->side_terms[t];
    st.type = q[0]; st.nres = q[1]; st.nblocks = q[2];
    for (int b = 0; b < 6; ++b) { st.kind[b] = q[3 + b]; st.idx[b] = q[9 + b]; }
    st.loss = q[15]; st.cofs = q[16];
    for (int b = 0; b < 4; ++b) st.aux[b] = q[17 + b];
    st.loss_a = term_loss_a[t];
  }
  pb->side_consts.assign(consts, consts + nconsts);
  pb->pp_of_point.assign(pb->P, -1);
  for (int q = 0; q < NPP; ++q) pb->pp_of_point[pp_point[q]] = q;
  pb->pp_prior.assign(pp_prior, pp_prior + 3 * (size_t)NPP);
  pb->pp_sigma.assign(pp_sigma, pp_sigma + 3 * (size_t)NPP);
  pb->pp_alt.assign(pp_alt, pp_alt + NPP);
  if (has_rc_prior) {
    pb->rc_prior.assign(rc_prior, rc_prior + 6 * (size_t)pb->NR);
    pb->rc_prior_sigma.assign(rc_sigma, rc_sigma + 6 * (size_t)pb->NR);
  }
  pb->scale.assign(pb->nc + 3 * (size_t)pb->npts_free, 1.0);
}
void oba_get_ext(void* h, double* ext) {
  Problem* pb = static_cast<Problem*>(h);
  std::copy(pb->ext.begin(), pb->ext.end(), ext);
}
void oba_set_ext(void* h, const double* ext) {
  Problem* pb = static_cast<Problem*>(h);
  std::copy(ext, ext + pb->ext.size(), pb->ext.begin());
}

void oba_destroy(void* h) { delete static_cast<Problem*>(h); }
int oba_nc(void* h) { return static_cast<Problem*>(h)->nc; }
int oba_npts_free(void* h) { return static_cast<Problem*>(h)->npts_free; }

void oba_get_params(void* h, double* cam, double* inst, double* rc, double* pts) {
  Problem* pb = static_cast<Problem*>(h);
  std::copy(pb->cam.begin(), pb->cam.end(), cam);
  std::copy(pb->inst.begin(), pb->inst.end(), inst);
  std::copy(pb->rc.begin(), pb->rc.end(), rc);
  std::copy(pb->pts.begin(), pb->pts.end(), pts);
}
void oba_set_params(void* h, const double* cam, const double* inst, const double* rc, const double* pts) {
  Problem* pb = static_cast<Problem*>(h);
  std::copy(cam, cam + pb->cam.size(), pb->cam.begin());
  std::copy(inst, inst + pb->inst.size(), pb->inst.begin());
  std::copy(rc, rc + pb->rc.size(), pb->rc.begin());
  std::copy(pts, pts + pb->pts.size(), pb->pts.begin());
}

// x <- x + delta, delta laid out [reduced camera side (nc) | free points (3 each)].
void oba_plus(void* h, const double* delta) {
  Problem* pb = static_cast<Problem*>(h);
  for (int k = 0; k < pb->K; ++k)
    if (pb->cam_poff[k] >= 0)
      for (int j = 0; j < pb->cam_np[k]; ++j) pb->cam[pb->cam_off[k] + j] += delta[pb->cam_poff[k] + j];
  for (int i = 0; i < pb->NI; ++i)
    if (pb->inst_poff[i] >= 0)
      for (int j = 0; j < 6; ++j) pb->inst[6 * i + j] += delta[pb->inst_poff[i] + j];
  for (int i = 0; i < pb->NR; ++i)
    if (pb->rc_poff[i] >= 0)
      for (int j = 0; j < 6; ++j) pb->rc[6 * i + j] += delta[pb->rc_poff[i] + j];
  for (int p = 0; p < pb->P; ++p)
    if (pb->pt_poff[p] >= 0)
      for (int j = 0; j < 3; ++j) pb->pts[3 * p + j] += delta[pb->nc + 3 * pb->pt_poff[p] + j];
  // ext blocks: projected onto their lower bounds (scales >= 0, std-deviation scales >= 1e-10; ceres bounded LM)
  for (int i = 0; i < pb->NE; ++i)
    if (pb->ext_poff[i] >= 0)
      for (int j = 0; j < pb->ext_np[i]; ++j) {
        double& v = pb->ext[pb->ext_off[i] + j];
        v = std::max(v + delta[pb->ext_poff[i] + j], pb->ext_lower[pb->ext_off[i] + j]);
      }
}

// Norm of the free parameters (Ceres' x_norm).
double oba_x_norm(void* h) {
  Problem* pb = static_cast<Problem*>(h);
  double s = 0.0;
  for (int k = 0; k < pb->K; ++k)
    if (pb->cam_poff[k] >= 0)
      for (int j = 0; j < pb->cam_np[k]; ++j) { const double v = pb->cam[pb->cam_off[k] + j]; s += v * v; }
  for (int i = 0; i < pb->NI; ++i)
    if (pb->inst_poff[i] >= 0)
      for (int j = 0; j < 6; ++j) { const double v = pb->inst[6 * i + j]; s += v * v; }
  for (int i = 0; i < pb->NR; ++i)
    if (pb->rc_poff[i] >= 0)
      for (int j = 0; j < 6; ++j) { const double v = pb->rc[6 * i + j]; s += v * v; }
  for (int p = 0; p < pb->P; ++p)
    if (pb->pt_poff[p] >= 0)
      for (int j = 0; j < 3; ++j) { const double v = pb->pts[3 * p + j]; s += v * v; }
  for (int i = 0; i < pb->NE; ++i)
    if (pb->ext_poff[i] >= 0)
      for (int j = 0; j < pb->ext_np[i]; ++j) { const double v = pb->ext[pb->ext_off[i] + j]; s += v * v; }
  return std::sqrt(s);
}

// Prior residual rows at the current parameters.
// Camera prior: DataPriorError<Camera> with LOGARITHMIC scale on focal and
// aspect ratio (bundle_adjuster.cc:568-593, prior_error.h:78-95), added for
// every camera (:783-787); scale = 1/max(sigma, eps) (prior_error.h:31-35).
// Position prior: DataPriorError<Pose, SimilarityPriorTransform> on TX,TY,TZ
// with the (constant, identity) bias (bundle_adjuster.cc:745-778, bias.h:33-53).
static void build_prior_rows(Problem* pb) {
  pb->prior_rows.clear();
  for (int k = 0; k < pb->K; ++k) {
    if (pb->cam_poff[k] < 0) continue;  // constant block: residual is a constant, dropped by Ceres
    if (pb->cam_type[k] == SPHERICAL) {
      // single dummy parameter: prior keeps it at its value
    }
    for (int j = 0; j < pb->cam_np[k]; ++j) {
      const int idx = pb->cam_off[k] + j;
      const double sc = 1.0 / std::max(pb->cam_prior_sigma[idx], DBL_EPSILON);
      Problem::PriorRow row;
      row.col = pb->cam_poff[k] + j;
      if (pb->cam_prior_log[idx]) {
        row.r = sc * std::log(pb->cam[idx] / pb->cam_prior[idx]);
        row.d = sc / pb->cam[idx];
      } else {
        row.r = sc * (pb->cam[idx] - pb->cam_prior[idx]);
        row.d = sc;
      }
      pb->prior_rows.push_back(row);
    }
  }
  for (int i = 0; i < pb->NI; ++i) {
    if (!pb->inst_has_prior[i] || pb->inst_poff[i] < 0) continue;
    for (int j = 0; j < 3; ++j) {
      const double sc = 1.0 / std::max(pb->inst_prior_std[3 * i + j], DBL_EPSILON);
      Problem::PriorRow row;
      row.col = pb->inst_poff[i] + 3 + j;
      row.r = sc * (pb->inst[6 * i + 3 + j] - pb->inst_prior_pos[3 * i + j]);
      row.d = sc;
      pb->prior_rows.push_back(row);
    }
  }
  // DataPriorError<Pose> on every rig camera with sigma GetDefaultRigPoseSigma (bundle_adjuster.cc:779-790)
  if (!pb->rc_prior.empty())
    for (int i = 0; i < pb->NR; ++i) {
      if (pb->rc_poff[i] < 0) continue;
      for (int j = 0; j < 6; ++j) {
        const double sc = 1.0 / std::max(pb->rc_prior_sigma[6 * i + j], DBL_EPSILON);
        pb->prior_rows.push_back({sc * (pb->rc[6 * i + j] - pb->rc_prior[6 * i + j]), pb->rc_poff[i] + j, sc});
      }
    }
  // point priors DataPriorError<Vec3d> on x, y (, z) (bundle_adjuster.cc:688-708): columns on the point side
  for (int p = 0; p < pb->P && !pb->pp_of_point.empty(); ++p) {
    const int q = pb->pp_of_point[p], pf = pb->pt_poff[p];
    if (q < 0 || pf < 0) continue;
    for (int j = 0; j < (pb->pp_alt[q] ? 3 : 2); ++j) {
      const double sc = 1.0 / std::max(pb->pp_sigma[3 * q + j], DBL_EPSILON);
      pb->prior_rows.push_back({sc * (pb->pts[3 * p + j] - pb->pp_prior[3 * q + j]), pb->nc + 3 * pf + j, sc});
    }
  }
}

// Cost = 1/2 sum_blocks rho(|r|^2) (Ceres), projections through the shared loss
// (bundle_adjuster.cc:799-814), priors without loss.  Optionally returns the
// unscaled residuals of ComputeReprojectionErrors (sigma = 1,
// bundle_adjuster.cc:531-566,1196-1208) in reproj[N x 3].
double oba_cost(void* h, double* reproj) {
  Problem* pb = static_cast<Problem*>(h);
  double cost = 0.0;
#pragma omp parallel for reduction(+ : cost) schedule(static)
  for (int64_t i = 0; i < pb->N; ++i) {
    const int shot = pb->obs_shot[i];
    const int cam = pb->shot_cam[shot];
    double r[3];
    const int nres = reprojection_residual<double>(
        pb->cam_type[cam], &pb->cam[pb->cam_off[cam]], &pb->inst[6 * pb->shot_inst[shot]],
        &pb->rc[6 * pb->shot_rc[shot]], pb->shot_use_rc[shot] != 0, &pb->pts[3 * pb->obs_point[i]],
        &pb->obs_xy[2 * i], pb->obs_sigma[i], r);
    double s = 0.0;
    for (int k = 0; k < nres; ++k) s += r[k] * r[k];
    double rho[2];
    loss_eval(pb->loss, pb->loss_a, s, rho);
    if (!obs_all_constant(*pb, i)) cost += 0.5 * rho[0];
    if (reproj) {
      for (int k = 0; k < 3; ++k) reproj[3 * i + k] = k < nres ? r[k] * pb->obs_sigma[i] : 0.0;
    }
  }
  build_prior_rows(pb);
  for (const auto& row : pb->prior_rows) cost += 0.5 * row.r * row.r;
  cost += eval_side_terms(pb, false);
  return cost;
}

// Robustified residuals and Jacobians at the current parameters (Ceres
// Corrector with rho'' <= 0: r <- sqrt(rho') r, J <- sqrt(rho') J).  Returns cost.
double oba_linearize(void* h) {
  Problem* pb = static_cast<Problem*>(h);
  const int wc = pb->wc;
  pb->obs_nres.resize(pb->N);
  pb->r.assign(3 * (size_t)pb->N, 0.0);
  pb->Jc.assign(3 * (size_t)wc * pb->N, 0.0);
  pb->Jp.assign(9 * (size_t)pb->N, 0.0);
  double cost = 0.0;
#pragma omp parallel for reduction(+ : cost) schedule(static)
  for (int64_t i = 0; i < pb->N; ++i) {
    const int shot = pb->obs_shot[i];
    const int cam = pb->shot_cam[shot];
    const int C = pb->cam_np[cam];
    double r[3], jc[3 * 16], ji[18], jrc[18], jp[9];
    const int nres = reprojection_analytic(
        pb->cam_type[cam], &pb->cam[pb->cam_off[cam]], &pb->inst[6 * pb->shot_inst[shot]],
        &pb->rc[6 * pb->shot_rc[shot]], pb->shot_use_rc[shot] != 0, &pb->pts[3 * pb->obs_point[i]],
        &pb->obs_xy[2 * i], pb->obs_sigma[i], r, jc, ji, jrc, jp);
    double s = 0.0;
    for (int k = 0; k < nres; ++k) s += r[k] * r[k];
    double rho[2];
    loss_eval(pb->loss, pb->loss_a, s, rho);
    if (!obs_all_constant(*pb, i)) cost += 0.5 * rho[0];
    const double w = std::sqrt(rho[1]);
    pb->obs_nres[i] = nres;
    double* R = &pb->r[3 * i];
    double* JC = &pb->Jc[3 * (size_t)wc * i];
    double* JP = &pb->Jp[9 * i];
    const bool pfree = pb->pt_poff[pb->obs_point[i]] >= 0;
    for (int k = 0; k < nres; ++k) {
      R[k] = w * r[k];
      for (int j = 0; j < C; ++j) JC[k * wc + j] = w * jc[k * C + j];
      for (int j = 0; j < 6; ++j) JC[k * wc + C + j] = w * ji[k * 6 + j];
      if (pb->shot_use_rc[shot])
        for (int j = 0; j < 6; ++j) JC[k * wc + C + 6 + j] = w * jrc[k * 6 + j];
      for (int j = 0; j < 3; ++j) JP[k * 3 + j] = pfree ? w * jp[k * 3 + j] : 0.0;
    }
  }
  build_prior_rows(pb);
  for (const auto& row : pb->prior_rows) cost += 0.5 * row.r * row.r;
  cost += eval_side_terms(pb, true);
  return cost;
}

void oba_set_scale(void* h, const double* scale) {
  Problem* pb = static_cast<Problem*>(h);
  std::copy(scale, scale + pb->scale.size(), pb->scale.begin());
}

// Squared column norms of the (unscaled) Jacobian and the gradient J^T r
// (unscaled), both laid out [nc | 3 * npts_free].
void oba_colnorm_gradient(void* h, double* colnorm2, double* grad) {
  Problem* pb = static_cast<Problem*>(h);
  const int wc = pb->wc;
  const size_t n = pb->nc + 3 * (size_t)pb->npts_free;
  std::fill(colnorm2, colnorm2 + n, 0.0);
  std::fill(grad, grad + n, 0.0);
  for (int64_t i = 0; i < pb->N; ++i) {
    const int shot = pb->obs_shot[i];
    const ObsCols oc = obs_cols(*pb, shot);
    const double* R = &pb->r[3 * i];
    const double* JC = &pb->Jc[3 * (size_t)wc * i];
    const double* JP = &pb->Jp[9 * i];
    const int nres = pb->obs_nres[i];
    for (int b = 0; b < 3; ++b) {
      if (oc.goff[b] < 0) continue;
      for (int j = 0; j < oc.lsz[b]; ++j)
        for (int k = 0; k < nres; ++k) {
          const double v = JC[k * wc + oc.lstart[b] + j];
          colnorm2[oc.goff[b] + j] += v * v;
          grad[oc.goff[b] + j] += v * R[k];
        }
    }
    const int pf = pb->pt_poff[pb->obs_point[i]];
    if (pf >= 0)
      for (int j = 0; j < 3; ++j)
        for (int k = 0; k < nres; ++k) {
          const double v = JP[k * 3 + j];
          colnorm2[pb->nc + 3 * pf + j] += v * v;
          grad[pb->nc + 3 * pf + j] += v * R[k];
        }
  }
  for (const auto& row : pb->prior_rows) {
    colnorm2[row.col] += row.d * row.d;
    grad[row.col] += row.d * row.r;
  }
  for (const auto& rows : pb->side_rows)
    for (int j = 0; j < rows.ncols; ++j) {
      if (rows.cols[j] < 0) continue;
      for (int k = 0; k < rows.nres; ++k) {
        const double v = rows.J[k * MAXD + j];
        colnorm2[rows.cols[j]] += v * v;
        grad[rows.cols[j]] += v * rows.r[k];
      }
    }
}

// Reduced camera system for the *scaled* Jacobian Js = J diag(scale) and LM
// diagonal D (given as D^2 = diag2, length nc + 3 npf):
//   S = (U + D_c^2) - sum_p W_p (V_p + D_p^2)^-1 W_p^T,
//   rhs = g_c - sum_p W_p (V_p + D_p^2)^-1 g_p,   g = Js^T r
// (Ceres SchurEliminator on the normal equations of min |Js y - r|^2 + |D y|^2;
// the step is -y).  S is dense nc x nc row-major (symmetric, full storage).
void oba_schur(void* h, const double* diag2, double* Sout, double* rhs) {
  Problem* pb = static_cast<Problem*>(h);
  const int wc = pb->wc, nc = pb->nc;
  std::fill(Sout, Sout + (size_t)nc * nc, 0.0);
  std::fill(rhs, rhs + nc, 0.0);
  const double* sc = pb->scale.data();
  const int nth = omp_get_max_threads();
  // U and g_c (observations of constant points included)
  std::vector<std::vector<double>> Sloc(nth), rloc(nth);
#pragma omp parallel
  {
    const int t = omp_get_thread_num();
    std::vector<double>& Sl = Sloc[t];
    std::vector<double>& rl = rloc[t];
    Sl.assign((size_t)nc * nc, 0.0);
    rl.assign(nc, 0.0);
    std::vector<double> Wbuf, jbuf;
    std::vector<int> gcol;
#pragma omp for schedule(dynamic, 64)
    for (int p = 0; p < pb->P; ++p) {
      const int64_t b = pb->pt_start[p], e = pb->pt_start[p + 1];
      const int pf = pb->pt_poff[p];
      const int no = (int)(e - b);
      if (no == 0) continue;
      // scaled per-observation camera-side Jacobians with their global columns
      jbuf.assign((size_t)no * 3 * wc, 0.0);
      gcol.assign((size_t)no * wc, -1);
      double V[9] = {0}, gp[3] = {0};
      Wbuf.assign((size_t)no * wc * 3, 0.0);
      for (int a = 0; a < no; ++a) {
        const int64_t i = pb->pt_obs[b + a];
        const ObsCols oc = obs_cols(*pb, pb->obs_shot[i]);
        const double* R = &pb->r[3 * i];
        const double* JC = &pb->Jc[3 * (size_t)wc * i];
        const double* JP = &pb->Jp[9 * i];
        const int nres = pb->obs_nres[i];
        double* jb = &jbuf[(size_t)a * 3 * wc];
        int* gc = &gcol[(size_t)a * wc];
        for (int bk = 0; bk < 3; ++bk) {
          if (oc.goff[bk] < 0) continue;
          for (int j = 0; j < oc.lsz[bk]; ++j) {
            const int lc = oc.lstart[bk] + j;
            gc[lc] = oc.goff[bk] + j;
            for (int k = 0; k < nres; ++k) jb[k * wc + lc] = JC[k * wc + lc] * sc[gc[lc]];
          }
        }
        double jp[9] = {0};
        if (pf >= 0)
          for (int k = 0; k < nres; ++k)
            for (int j = 0; j < 3; ++j) jp[k * 3 + j] = JP[k * 3 + j] * sc[nc + 3 * pf + j];
        // U += Jc^T Jc, g_c += Jc^T r
        for (int c1 = 0; c1 < wc; ++c1) {
          if (gc[c1] < 0) continue;
          double g = 0.0;
          for (int k = 0; k < nres; ++k) g += jb[k * wc + c1] * R[k];
          rl[gc[c1]] += g;
          for (int c2 = 0; c2 < wc; ++c2) {
            if (gc[c2] < 0) continue;
            double v = 0.0;
            for (int k = 0; k < nres; ++k) v += jb[k * wc + c1] * jb[k * wc + c2];
            Sl[(size_t)gc[c1] * nc + gc[c2]] += v;
          }
        }
        if (pf >= 0) {
          for (int j1 = 0; j1 < 3; ++j1) {
            for (int k = 0; k < nres; ++k) gp[j1] += jp[k * 3 + j1] * R[k];
            for (int j2 = 0; j2 < 3; ++j2)
              for (int k = 0; k < nres; ++k) V[j1 * 3 + j2] += jp[k * 3 + j1] * jp[k * 3 + j2];
          }
          double* W = &Wbuf[(size_t)a * wc * 3];
          for (int c1 = 0; c1 < wc; ++c1)
            for (int j = 0; j < 3; ++j) {
              double v = 0.0;
              for (int k = 0; k < nres; ++k) v += jb[k * wc + c1] * jp[k * 3 + j];
              W[c1 * 3 + j] = v;
            }
        }
      }
      if (pf < 0) continue;
      if (!pb->pp_of_point.empty() && pb->pp_of_point[p] >= 0) {  // point prior rows: diagonal
        const int q = pb->pp_of_point[p];
        for (int j = 0; j < (pb->pp_alt[q] ? 3 : 2); ++j) {
          const double d = sc[nc + 3 * pf + j] / std::max(pb->pp_sigma[3 * q + j], DBL_EPSILON);
          const double rr = (pb->pts[3 * p + j] - pb->pp_prior[3 * q + j]) / std::max(pb->pp_sigma[3 * q + j], DBL_EPSILON);
          V[j * 3 + j] += d * d;
          gp[j] += d * rr;
        }
      }
      for (int j = 0; j < 3; ++j) V[j * 3 + j] += diag2[nc + 3 * pf + j];
      // inverse of symmetric 3x3
      double Vi[9];
      {
        const double a = V[0], b_ = V[1], c = V[2], d = V[4], e_ = V[5], f = V[8];
        const double A = d * f - e_ * e_, B = c * e_ - b_ * f, Cc = b_ * e_ - c * d;
        const double det = a * A + b_ * B + c * Cc;
        const double id = 1.0 / det;
        Vi[0] = A * id; Vi[1] = B * id; Vi[2] = Cc * id;
        Vi[3] = Vi[1]; Vi[4] = (a * f - c * c) * id; Vi[5] = (b_ * c - a * e_) * id;
        Vi[6] = Vi[2]; Vi[7] = Vi[5]; Vi[8] = (a * d - b_ * b_) * id;
      }
      double Vig[3];
      for (int j = 0; j < 3; ++j) Vig[j] = Vi[j * 3] * gp[0] + Vi[j * 3 + 1] * gp[1] + Vi[j * 3 + 2] * gp[2];
      for (int a = 0; a < no; ++a) {
        const int* gca = &gcol[(size_t)a * wc];
        const double* Wa = &Wbuf[(size_t)a * wc * 3];
        for (int c1 = 0; c1 < wc; ++c1) {
          if (gca[c1] < 0) continue;
          double WVi[3];
          for (int j = 0; j < 3; ++j)
            WVi[j] = Wa[c1 * 3] * Vi[j] + Wa[c1 * 3 + 1] * Vi[3 + j] + Wa[c1 * 3 + 2] * Vi[6 + j];
          rl[gca[c1]] -= Wa[c1 * 3] * Vig[0] + Wa[c1 * 3 + 1] * Vig[1] + Wa[c1 * 3 + 2] * Vig[2];
          for (int a2 = 0; a2 < no; ++a2) {
            const int* gcb = &gcol[(size_t)a2 * wc];
            const double* Wb = &Wbuf[(size_t)a2 * wc * 3];
            for (int c2 = 0; c2 < wc; ++c2) {
              if (gcb[c2] < 0) continue;
              Sl[(size_t)gca[c1] * nc + gcb[c2]] -=
                  WVi[0] * Wb[c2 * 3] + WVi[1] * Wb[c2 * 3 + 1] + WVi[2] * Wb[c2 * 3 + 2];
            }
          }
        }
      }
    }
  }
  for (int t = 0; t < nth; ++t) {
    if (Sloc[t].empty()) continue;
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < (int64_t)nc * nc; ++i) Sout[i] += Sloc[t][i];
    for (int i = 0; i < nc; ++i) rhs[i] += rloc[t][i];
  }
  for (const auto& row : pb->prior_rows) {
    if (row.col >= nc) continue;  // point-side rows went into V_p / g_p above
    const double d = row.d * sc[row.col];
    Sout[(size_t)row.col * nc + row.col] += d * d;
    rhs[row.col] += d * row.r;
  }
  for (const auto& rows : pb->side_rows)
    for (int j1 = 0; j1 < rows.ncols; ++j1) {
      const int c1 = rows.cols[j1];
      if (c1 < 0) continue;
      for (int k = 0; k < rows.nres; ++k) rhs[c1] += rows.J[k * MAXD + j1] * sc[c1] * rows.r[k];
      for (int j2 = 0; j2 < rows.ncols; ++j2) {
        const int c2 = rows.cols[j2];
        if (c2 < 0) continue;
        double v = 0.0;
        for (int k = 0; k < rows.nres; ++k) v += rows.J[k * MAXD + j1] * rows.J[k * MAXD + j2];
        Sout[(size_t)c1 * nc + c2] += v * sc[c1] * sc[c2];
      }
    }
  for (int i = 0; i < nc; ++i) Sout[(size_t)i * nc + i] += diag2[i];
}

// Back-substitution y_p = (V_p + D_p^2)^-1 (g_p - W_p^T y_c) for the scaled
// system; y laid out [nc | 3 npf] with y[0:nc] = y_c given.
void oba_backsub(void* h, const double* diag2, double* y) {
  Problem* pb = static_cast<Problem*>(h);
  const int wc = pb->wc, nc = pb->nc;
  const double* sc = pb->scale.data();
#pragma omp parallel for schedule(dynamic, 256)
  for (int p = 0; p < pb->P; ++p) {
    const int pf = pb->pt_poff[p];
    if (pf < 0) continue;
    double V[9] = {0}, t[3] = {0};
    for (int64_t q = pb->pt_start[p]; q < pb->pt_start[p + 1]; ++q) {
      const int64_t i = pb->pt_obs[q];
      const ObsCols oc = obs_cols(*pb, pb->obs_shot[i]);
      const double* R = &pb->r[3 * i];
      const double* JC = &pb->Jc[3 * (size_t)wc * i];
      const double* JP = &pb->Jp[9 * i];
      const int nres = pb->obs_nres[i];
      // e = r - Jc_s y_c   (per residual row)
      double e[3];
      for (int k = 0; k < nres; ++k) {
        double acc = R[k];
        for (int bk = 0; bk < 3; ++bk) {
          if (oc.goff[bk] < 0) continue;
          for (int j = 0; j < oc.lsz[bk]; ++j) {
            const int g = oc.goff[bk] + j;
            acc -= JC[k * wc + oc.lstart[bk] + j] * sc[g] * y[g];
          }
        }
        e[k] = acc;
      }
      for (int j1 = 0; j1 < 3; ++j1) {
        const double s1 = sc[nc + 3 * pf + j1];
        for (int k = 0; k < nres; ++k) t[j1] += JP[k * 3 + j1] * s1 * e[k];
        for (int j2 = 0; j2 < 3; ++j2) {
          const double s2 = sc[nc + 3 * pf + j2];
          for (int k = 0; k < nres; ++k) V[j1 * 3 + j2] += JP[k * 3 + j1] * s1 * JP[k * 3 + j2] * s2;
        }
      }
    }
    if (!pb->pp_of_point.empty() && pb->pp_of_point[p] >= 0) {
      const int q = pb->pp_of_point[p];
      for (int j = 0; j < (pb->pp_alt[q] ? 3 : 2); ++j) {
        const double dd = sc[nc + 3 * pf + j] / std::max(pb->pp_sigma[3 * q + j], DBL_EPSILON);
        const double rr = (pb->pts[3 * p + j] - pb->pp_prior[3 * q + j]) / std::max(pb->pp_sigma[3 * q + j], DBL_EPSILON);
        V[j * 3 + j] += dd * dd;
        t[j] += dd * rr;
      }
    }
    for (int j = 0; j < 3; ++j) V[j * 3 + j] += diag2[nc + 3 * pf + j];
    const double a = V[0], b_ = V[1], c = V[2], d = V[4], e_ = V[5], f = V[8];
    const double A = d * f - e_ * e_, B = c * e_ - b_ * f, Cc = b_ * e_ - c * d;
    const double id = 1.0 / (a * A + b_ * B + c * Cc);
    const double Vi[9] = {A * id, B * id, Cc * id, B * id, (a * f - c * c) * id, (b_ * c - a * e_) * id,
                          Cc * id, (b_ * c - a * e_) * id, (a * d - b_ * b_) * id};
    for (int j = 0; j < 3; ++j) y[nc + 3 * pf + j] = Vi[j * 3] * t[0] + Vi[j * 3 + 1] * t[1] + Vi[j * 3 + 2] * t[2];
  }
}

// Ceres: model_residuals = Js * step; model_cost_change =
// -model_residuals . (r + model_residuals / 2)   (trust_region_minimizer).
double oba_model_cost_change(void* h, const double* step) {
  Problem* pb = static_cast<Problem*>(h);
  const int wc = pb->wc, nc = pb->nc;
  const double* sc = pb->scale.data();
  double total = 0.0;
#pragma omp parallel for reduction(+ : total) schedule(static)
  for (int64_t i = 0; i < pb->N; ++i) {
    const ObsCols oc = obs_cols(*pb, pb->obs_shot[i]);
    const double* R = &pb->r[3 * i];
    const double* JC = &pb->Jc[3 * (size_t)wc * i];
    const double* JP = &pb->Jp[9 * i];
    const int nres = pb->obs_nres[i];
    const int pf = pb->pt_poff[pb->obs_point[i]];
    for (int k = 0; k < nres; ++k) {
      double m = 0.0;
      for (int bk = 0; bk < 3; ++bk) {
        if (oc.goff[bk] < 0) continue;
        for (int j = 0; j < oc.lsz[bk]; ++j) {
          const int g = oc.goff[bk] + j;
          m += JC[k * wc + oc.lstart[bk] + j] * sc[g] * step[g];
        }
      }
      if (pf >= 0)
        for (int j = 0; j < 3; ++j) m += JP[k * 3 + j] * sc[nc + 3 * pf + j] * step[nc + 3 * pf + j];
      total += -m * (R[k] + 0.5 * m);
    }
  }
  for (const auto& row : pb->prior_rows) {
    const double m = row.d * sc[row.col] * step[row.col];
    total += -m * (row.r + 0.5 * m);
  }
  for (const auto& rows : pb->side_rows)
    for (int k = 0; k < rows.nres; ++k) {
      double m = 0.0;
      for (int j = 0; j < rows.ncols; ++j)
        if (rows.cols[j] >= 0) m += rows.J[k * MAXD + j] * sc[rows.cols[j]] * step[rows.cols[j]];
      total += -m * (rows.r[k] + 0.5 * m);
    }
  return total;
}

}  // extern "C"
