/* opensfm_b200 — C ABI of the H100-native hot paths of OpenSfM.
 *
 * Plain C, plain pointers and sizes; no torch / pybind types.  Every entry
 * point returns 0 on success and a non-zero code on failure; the message of
 * the last failure on the calling thread is osfm_last_error().
 *
 * Two paths (SURVEY.md §8):
 *   MATCH  brute-force descriptor matching + Lowe ratio test, replacing
 *          opensfm/matching.py:723-777 (cv2.BFMatcher.knnMatch k=2).
 *   BA     bundle adjustment, replacing bundle::BundleAdjuster
 *          (opensfm/src/bundle/bundle_adjuster.h:178-299,
 *           opensfm/src/bundle/src/bundle_adjuster.cc) behind pybundle /
 *          sfm::BAHelpers (opensfm/src/sfm/src/ba_helpers.cc:117,408,581).
 * and, between them, TRACKS: linking matches into tracks, replacing
 *          tracking.create_tracks_manager (opensfm/tracking.py:72-150), and
 *          triangulating them, replacing TrackTriangulator.triangulate
 *          (opensfm/reconstruction.py:1032-1073).
 *
 * There is no CPU fallback: every call needs a CUDA device (H100, sm_90a).
 *
 * Handles (osfm_matcher, osfm_ba, osfm_tracks, osfm_rotransac, osfm_resect, osfm_relpose, osfm_dense) own a CUDA stream and
 * workspaces on the device they were created on, and every call on a handle makes that device current on the calling thread.  Calls on one handle
 * are serialised and may come from any thread; calls on different handles do not wait for each other.  A callback
 * (today only the all-reduce of osfm_ba_set_distributed) must not call into the handle that called it.
 */
#ifndef OPENSFM_B200_H_
#define OPENSFM_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define OSFM_OK 0
#define OSFM_ERR_CUDA 1
#define OSFM_ERR_ARG 2
#define OSFM_ERR_RUNTIME 3

const char* osfm_last_error(void);
int osfm_version(void);
/* number of this library's kernels launched by the calling process so far */
int64_t osfm_kernel_launch_count(void);

/* ------------------------------------------------------------------------
 * MATCH
 * ---------------------------------------------------------------------- */
typedef struct osfm_matcher osfm_matcher;

/* A matcher owns one CUDA stream and its workspaces on `device`.  Threads that
 * match at the same time use a matcher each: matching.match_brute_force is
 * called concurrently from joblib threads (opensfm/context.py:59-64). */
int osfm_matcher_create(int device, osfm_matcher** out);
int osfm_matcher_destroy(osfm_matcher* m);

/* One-shot, host buffers: the drop-in for
 *   matching.match_brute_force(f1, f2, config, maskij)            (matching.py:723-756)
 *   matching.match_brute_force_symmetric(fi, fj, config, maskij)  (matching.py:759-777)
 * f1: n1 x dim, f2: n2 x dim, row-major, float32 (L2, "BruteForce") or
 * uint8 (Hamming, "BruteForce-Hamming", dim = bytes per descriptor).
 * mask: NULL or n1 x n2 bytes, non-zero = allowed (matching.py:745).
 * out_match[i] = matched index in f2 for row i of f1, or -1.  For the one-way
 * call the reference's list is [(i, out_match[i]) for i ascending if >= 0]. */
int osfm_bf_match_f32(osfm_matcher* m, const float* f1, int n1, const float* f2, int n2, int dim,
                      double lowes_ratio, const uint8_t* mask, int symmetric, int32_t* out_match);
int osfm_bf_match_u8(osfm_matcher* m, const uint8_t* f1, int n1, const uint8_t* f2, int n2, int nbytes,
                     double lowes_ratio, const uint8_t* mask, int symmetric, int32_t* out_match);

/* Resident descriptor sets + batched pair list: the drop-in for the pair loop of
 * matching.match_images_with_pairs (matching.py:63-98).  Descriptors are
 * uploaded once; a pair list is matched in one submission. */
int osfm_matcher_add_f32(osfm_matcher* m, const float* desc, int n, int dim, int* out_id);
int osfm_matcher_add_u8(osfm_matcher* m, const uint8_t* desc, int n, int nbytes, int* out_id);
/* Upload `count` descriptor matrices (desc[i] is n[i] x dim) with one host synchronisation at the end:
 * the per-image loop of matching.match_images_with_pairs loading features (matching.py:70-82). */
int osfm_matcher_add_batch_f32(osfm_matcher* m, int count, const float* const* desc, const int* n, int dim, int* out_ids);
int osfm_matcher_add_batch_u8(osfm_matcher* m, int count, const uint8_t* const* desc, const int* n, int nbytes,
                              int* out_ids);
/* uint8-STORED descriptors compared with L2 ("BruteForce"): HAHOG / SIFT are integers 0..255 and live as uint8 on
 * disk (opensfm/features.py:169-170, 526-534); the reference widens them to float32 on load.  Uploading the bytes
 * and widening on the device moves a quarter of the data; results are identical to adding the float32 matrix. */
int osfm_matcher_add_u8_l2(osfm_matcher* m, const uint8_t* desc, int n, int dim, int* out_id);
int osfm_matcher_add_batch_u8_l2(osfm_matcher* m, int count, const uint8_t* const* desc, const int* n, int dim,
                                 int* out_ids);
int osfm_matcher_remove(osfm_matcher* m, int id);
int osfm_matcher_clear(osfm_matcher* m);
/* Enqueue matching of npairs pairs (ids_a[p], ids_b[p]).  Results stay on the
 * device until fetched.  Total result length = sum_p n(ids_a[p]). */
int osfm_matcher_match_pairs_async(osfm_matcher* m, int npairs, const int* ids_a, const int* ids_b,
                                   double lowes_ratio, int symmetric);
/* Guided matching (matching._match_descriptors_guided_impl, matching.py:260-338): unit bearing vectors of a
 * resident set (n x 3 float32, feature_loader.load_bearings), then a pair list with the relative pose of image b
 * w.r.t. image a -- pose12[p] = [R (cam b -> cam a) row-major, 9 | origin of b in a, 3] as doubles
 * (pose.get_R_cam_to_world(), pose.get_origin()).  The epipolar mask
 * compute_inliers_bearing_epipolar(b1, b2, pose, threshold) (matching.py:847-868,
 * geometry/src/triangulation.cc:195-219) is evaluated on the device into a bitmask that never leaves HBM, and
 * the pairs are matched like osfm_matcher_match_pairs_async with that mask (transposed for the b -> a pass). */
int osfm_matcher_set_bearings(osfm_matcher* m, int id, const float* bearings_n_by_3);
int osfm_matcher_match_pairs_guided_async(osfm_matcher* m, int npairs, const int* ids_a, const int* ids_b,
                                          const double* pose12, double threshold, double lowes_ratio, int symmetric);
/* Test hook: the epipolar bitmask the last guided submission built for its pair `pair`, in both layouts the
 * matcher uses -- F: n1 rows of ceil(n2 / 32) words (bit j % 32 of word j / 32 = feature j of image b passes for
 * feature i of image a), T: n2 rows of ceil(n1 / 32) words, the transpose.  Fails if the last submission was not
 * guided or `pair` is out of range. */
int osfm_matcher_get_epipolar_masks(osfm_matcher* m, int pair, uint32_t* F, uint32_t* T);
int osfm_matcher_sync(osfm_matcher* m);
/* Copy the last batch's results to the host: concatenated per pair, n(ids_a[p]) entries each. */
int osfm_matcher_fetch(osfm_matcher* m, int32_t* out_match, int64_t capacity);
/* The last batch as the reference's lists: (query, train) int32 rows packed pair after pair in query order
 * (matching.py:749-756, 775-777), compacted on the device.  offsets_out[npairs + 1] = first row of every pair,
 * *total_rows = offsets_out[npairs] rows written to pairs_out (capacity_rows >= sum of n(ids_a[p]) always fits). */
int osfm_matcher_fetch_pairs(osfm_matcher* m, int64_t* offsets_out, int32_t* pairs_out, int64_t capacity_rows,
                             int64_t* total_rows);
/* Milliseconds spent on the device by the last batch (CUDA events on the matcher's stream). */
int osfm_matcher_last_device_ms(osfm_matcher* m, float* ms_total, float* ms_distance_kernel);
/* 0 = pick automatically, 1 = force the exact SIMT kernel, 2 = force the tensor-core (wgmma) kernel
 * (fails at match time if the descriptors are not exactly representable). */
int osfm_matcher_set_kernel(osfm_matcher* m, int which);
/* Which distance kernel the last batch used: 1 = SIMT, 2 = tensor cores bf16 (L2), 3 = tensor cores fp8 (Hamming). */
int osfm_matcher_last_kernel(osfm_matcher* m);
/* Device memory held by the matcher's descriptor slabs (bytes reserved / bytes in use by live sets). */
int osfm_matcher_device_bytes(osfm_matcher* m, int64_t* reserved, int64_t* in_use);

/* WORDS matcher: features::match_using_words (opensfm/src/features/src/matching.cc:24-88; pyfeatures, called by
 * matching.match_words, matching.py:636-656).  words1: n1 x words_per_feature nearest visual words of every feature
 * of image 1; words2: the nearest word of every feature of image 2 (words2[:, 0] in the reference's call).
 * out_match[i] = matched feature of image 2 or -1; the reference returns the rows (i, out_match[i]) with a match. */
int osfm_match_words(osfm_matcher* m, const float* f1, int n1, const int32_t* words1, int words_per_feature,
                     const float* f2, int n2, const int32_t* words2, int dim, float lowes_ratio, int max_checks,
                     int32_t* out_match);
/* features::compute_vlad_distances (matching.cc:122-145): Euclidean distance of VLAD descriptor `query` to each of
 * the n descriptors (n x dim float32, row-major), sqrt(sum (double(a) - double(b))^2); out_n[query] = 0. */
int osfm_vlad_distances(osfm_matcher* m, const float* vlad, int n, int dim, int query, double* out_n);

/* VLAD pair selection (pairs_selection.match_candidates_with_vlad, opensfm/pairs_selection.py:351-431, 471-490,
 * 764-795; vlad.py).  osfm_matcher_vlad_compute: the VLAD descriptor of each listed resident set against
 * `centers` (ncenters x dim float32, row-major) -- features::compute_vlad_descriptor (matching.cc:90-119), bit for
 * bit, then vlad.signed_square_root_normalize -- kept on the device with the set.  out_valid[i] = 0 for Hamming
 * sets and sets of another dimension (they get no descriptor, as unnormalized_vlad returns None).  float32 and
 * uint8-stored L2 sets are read as float32.  Fails (OSFM_ERR_ARG) on non-finite centres or descriptors. */
int osfm_matcher_vlad_compute(osfm_matcher* m, int count, const int* set_ids, const float* centers, int ncenters, int dim,
                              int* out_valid);
/* Copy one set's VLAD descriptor (ncenters * dim floats): unnormalised if `unnormalized`, else normalised. */
int osfm_matcher_vlad_get(osfm_matcher* m, int set_id, int unnormalized, float* out);
/* For every reference set r, the k nearest candidate sets by (distance, candidate index) -- a stable argsort of the
 * distances over the candidates in the given order, NaN last -- among the candidates j with bit j % 32 of
 * cand_mask_bits[r * ceil(ncand / 32) + j / 32] set (NULL: all) other than r's own set.  camera_labels: NULL, or
 * nref + ncand ints (the references' labels, then the candidates'): then the k nearest of r's camera and the k
 * nearest of other cameras (pairs_from_neighbors).  Distances as osfm_vlad_distances, computed block by block on
 * the device.  Output: the selected (column, distance) of reference r in rows out_offsets[r] .. out_offsets[r + 1]
 * of out_cols / out_dist, columns ascending; out_offsets has nref + 1 entries, the outputs room for
 * nref * min(k, ncand) rows (twice that with camera labels). */
int osfm_matcher_vlad_select(osfm_matcher* m, int nref, const int* ref_ids, int ncand, const int* cand_ids,
                             const uint32_t* cand_mask_bits, const int* camera_labels, int k, int64_t* out_offsets,
                             int32_t* out_cols, double* out_dist);

/* BoW pair selection (pairs_selection.match_candidates_with_bow, opensfm/pairs_selection.py:281-348, 690-727;
 * bow.py).  osfm_matcher_bow_words: the k nearest of the nwords vocabulary words (nwords x dim float32, row-major)
 * of every row of each listed resident set, as cv2 BruteForce knnMatch(desc, vocab, k) returns them (bow.py
 * map_to_words): ranked by the float32 square root of the squared distance summed in cv2's order, ties to the lower
 * word.  1 <= k <= 64; min(k, nwords) words per row.  The rows of set i are rows out_offsets[i] .. out_offsets[i + 1]
 * of out_words (out_offsets: count + 1 entries; out_words: NULL, or room for all rows of the valid sets); the first
 * word of every row stays on the device with the set.  out_valid[i] = 0 for Hamming sets and sets of another
 * dimension (no rows).  float32 and uint8-stored L2 sets are read as float32.  Fails (OSFM_ERR_ARG) on non-finite
 * vocabulary or descriptor elements. */
int osfm_matcher_bow_words(osfm_matcher* m, int count, const int* set_ids, const float* vocab, int nwords, int dim,
                           int k, int64_t* out_offsets, int32_t* out_words, int* out_valid);
/* One-shot osfm_matcher_bow_words of n x dim float32 descriptors from host memory: out = n x min(k, nwords). */
int osfm_bow_map_to_words(osfm_matcher* m, const float* desc, int n, int dim, const float* vocab, int nwords, int k,
                          int32_t* out);
/* BagOfWords.histogram of each listed set's resident first words: h = bincount(words, nwords) * weights, h / h.sum(),
 * float64 in numpy's order (bit for bit), kept on the device with the set.  out_valid[i] = 0 for sets without
 * words of an nwords-word vocabulary (osfm_matcher_bow_words) and sets of 8 or fewer rows (load_histograms). */
int osfm_matcher_bow_histograms(osfm_matcher* m, int count, const int* set_ids, const double* weights, int nwords,
                                int* out_valid);
/* Copy one set's BoW histogram (nwords doubles). */
int osfm_matcher_bow_get(osfm_matcher* m, int set_id, double* out);
/* One-shot BagOfWords.histogram of n word indices from host memory (no minimum count): out = nwords doubles. */
int osfm_bow_histogram(osfm_matcher* m, const int32_t* words, int n, const double* weights, int nwords, double* out);
/* osfm_matcher_vlad_select over the BoW histograms, with the distance np.fabs(h - h2).sum() (numpy's pairwise
 * order, bit for bit).  cand_order: NULL (every candidate, ties to the lower column), or nref x ncand ints, the
 * position of candidate j in reference r's own candidate list or -1 if it is not in it: then only listed candidates
 * are eligible and ties go to the earlier position (bow_distances walks each list in the given order). */
int osfm_matcher_bow_select(osfm_matcher* m, int nref, const int* ref_ids, int ncand, const int* cand_ids,
                            const int32_t* cand_order, const int* camera_labels, int k, int64_t* out_offsets,
                            int32_t* out_cols, double* out_dist);
/* np.fabs(h - h2).sum() of histogram `query` and each of the n histograms (n x len float64, row-major), in numpy's
 * pairwise order; out_n[query] = 0. */
int osfm_bow_distances(osfm_matcher* m, const double* hist, int n, int len, int query, double* out_n);

/* ------------------------------------------------------------------------
 * BA
 * ---------------------------------------------------------------------- */
typedef struct osfm_ba osfm_ba;

/* geometry::ProjectionType (opensfm/src/geometry/camera_instances.h:8-20) */
enum {
  OSFM_PERSPECTIVE = 0, OSFM_BROWN = 1, OSFM_FISHEYE = 2, OSFM_FISHEYE_OPENCV = 3, OSFM_FISHEYE62 = 4,
  OSFM_FISHEYE624 = 5, OSFM_SPHERICAL = 6, OSFM_DUAL = 7, OSFM_RADIAL = 8, OSFM_SIMPLE_RADIAL = 9
};
/* ceres loss names accepted by CreateLossFunction (bundle_adjuster.cc:414-429) */
enum { OSFM_LOSS_TRIVIAL = 0, OSFM_LOSS_HUBER = 1, OSFM_LOSS_SOFTLONE = 2, OSFM_LOSS_CAUCHY = 3, OSFM_LOSS_ARCTAN = 4,
       OSFM_LOSS_TUKEY = 5 /* side terms only (common position, bundle_adjuster.cc:905) */ };

int osfm_ba_create(int device, osfm_ba** out);
int osfm_ba_destroy(osfm_ba* ba);
int osfm_camera_num_params(int projection_type);

/* Bulk SoA setters — replace the string-keyed AddCamera / AddRigInstance /
 * AddRigCamera / AddPoint / AddPointProjectionObservation calls
 * (bundle_adjuster.cc:94-260).  All arrays are host memory and are copied. */
int osfm_ba_set_cameras(osfm_ba* ba, int n, const int32_t* type, const double* params /*flat*/,
                        const int32_t* constant, const double* prior /*flat*/, const double* prior_sigma /*flat*/,
                        const int32_t* prior_log /*flat*/);
int osfm_ba_set_rig_instances(osfm_ba* ba, int n, const double* pose6, const int32_t* constant,
                              const int32_t* has_position_prior, const double* prior_position3,
                              const double* prior_std3);
int osfm_ba_set_rig_cameras(osfm_ba* ba, int n, const double* pose6, const int32_t* constant);
int osfm_ba_set_shots(osfm_ba* ba, int n, const int32_t* rig_instance, const int32_t* camera,
                      const int32_t* rig_camera, const int32_t* use_rig_camera);
int osfm_ba_set_points(osfm_ba* ba, int n, const double* xyz, const int32_t* constant);
int osfm_ba_set_observations(osfm_ba* ba, int64_t n, const int32_t* shot, const int32_t* point,
                             const double* xy, const double* std_deviation);
/* The same for PAGE-LOCKED arrays: the indices are on the device when the call returns, xy and std_deviation may
 * still be in flight on a copy stream (osfm_ba_run waits for them right before the kernel that needs them, i.e. the
 * upload overlaps the device-side ordering): both arrays must stay valid and unchanged until osfm_ba_run returns.
 * With pageable memory the copies are staged by the driver and the call behaves like osfm_ba_set_observations. */
int osfm_ba_set_observations_async(osfm_ba* ba, int64_t n, const int32_t* shot, const int32_t* point,
                                   const double* xy, const double* std_deviation);

/* Rig-camera pose priors: DataPriorError<Pose> with sigma GetDefaultRigPoseSigma, one per rig camera
 * (bundle_adjuster.cc:779-790; residual dropped when the rig camera is constant).  prior6 / sigma6: n x 6
 * in the order [rx, ry, rz, tx, ty, tz]; NULL removes the priors.  Call after osfm_ba_set_rig_cameras. */
int osfm_ba_set_rig_camera_priors(osfm_ba* ba, const double* prior6, const double* sigma6);
/* Point priors (GCP): AddPointPrior (bundle_adjuster.cc:224-236, residual :688-708): residuals on x, y
 * (and z when has_altitude) with scale 1 / max(sigma, eps).  n priors on points point[i]. */
int osfm_ba_set_point_priors(osfm_ba* ba, int n, const int32_t* point, const double* prior3, const double* sigma3,
                             const int32_t* has_altitude);
/* Extra parameter blocks of the camera side: camera biases (7: [R | t | scale], data/bias.h:10-31), per-instance
 * reconstruction scales (1, lower bound 0, bundle_adjuster.cc:672-685), std-deviation scales of the position-prior
 * groups (1, lower bound 1e-10, :727-736).  values / lower_bound are flat over the blocks (-inf = unbounded). */
int osfm_ba_set_ext_blocks(osfm_ba* ba, int n, const int32_t* size, const double* values, const int32_t* constant,
                           const double* lower_bound);
int osfm_ba_get_ext_blocks(osfm_ba* ba, double* values);

/* Side terms: the O(#shots) residual blocks next to the point projections.  Each names up to 6 parameter blocks
 * (kind: 0 camera, 1 rig instance, 2 rig camera, 3 ext block; idx within the kind), a ceres loss (-1 = none) and
 * `nconst` constants starting at consts[cofs].  Types, blocks and constants (reference functor):
 *   UP_VECTOR           [inst, rigcam]  c = unit acceleration[3], 1/std          absolute_motion_errors.h:12-39
 *   PAN / TILT / ROLL   [inst, rigcam]  c = angle, 1/std                         :41-136
 *   RELATIVE_MOTION     [inst_i, inst_j, scale_i(, scale_j)]  c = Rts[7], scale_matrix[49] row-major,
 *                       observed_scale; aux[0] = block of scale_j (2 or 3)       relative_motion_errors.h:14-72
 *   RELATIVE_ROTATION   [inst_i, inst_j(, rigcam_i)(, rigcam_j)]  c = Rij[3], scale_matrix[9];
 *                       aux[0], aux[1] = rig-camera block of i, j or -1          :74-103
 *   COMMON_POSITION     same blocks / aux; c = margin, 1/std                     :105-138
 *   LINEAR_MOTION       [inst0, inst1, inst2(, rigcams)]  c = alpha, 1/pos_std, 1/ori_std; aux[0..2] = rig-camera
 *                       blocks or -1                                             motion_prior_errors.h:13-76
 *   TRANSLATION_PRIOR   [inst1, inst2]  c = max(prior norm, 1e-20)               absolute_motion_errors.h:180-202
 *   PARAMETER_BARRIER   [camera]  c = lower, upper; aux[0] = parameter index     parameters_errors.h:20-36
 *   STD_DEVIATION       [ext]                                                    parameters_errors.h:7-18
 *   POSITION_PRIOR      [inst, bias ext(7), std-scale ext(1)]  c = prior[3], 1/sigma[3], adjust flag
 *                       (the general form of the position prior: bias transform + scale group,
 *                        bundle_adjuster.cc:745-778, data/bias.h:33-53) */
enum {
  OSFM_SIDE_UP_VECTOR = 0, OSFM_SIDE_PAN = 1, OSFM_SIDE_TILT = 2, OSFM_SIDE_ROLL = 3, OSFM_SIDE_RELATIVE_MOTION = 4,
  OSFM_SIDE_RELATIVE_ROTATION = 5, OSFM_SIDE_COMMON_POSITION = 6, OSFM_SIDE_LINEAR_MOTION = 7,
  OSFM_SIDE_TRANSLATION_PRIOR = 8, OSFM_SIDE_PARAMETER_BARRIER = 9, OSFM_SIDE_STD_DEVIATION = 10,
  OSFM_SIDE_POSITION_PRIOR = 11,
  /* ReconstructionAlignment (opensfm/src/bundle/reconstruction_alignment.h:140-365): "shots" are rig-instance blocks
   * holding [R | t] world-to-camera, "reconstructions" are 7-parameter ext blocks [R | t | scale] (scale >= 0.1):
   *   RA_RELATIVE_MOTION             [reconstruction, shot]  c = Rtai[6], scale_matrix[36]
   *   RA_ABSOLUTE_POSITION           [shot]                  c = position[3], 1/std
   *   RA_RELATIVE_ABSOLUTE_POSITION  [reconstruction]        c = position[3], shot[6], 1/std
   *   RA_COMMON_POINT                [reconstruction a, b]   c = point_a[3], point_b[3], 1/std
   *   RA_COMMON_CAMERA               [reconstruction a, b]   c = shot_a[6], shot_b[6], 1/std_centre, 1/std_rotation */
  OSFM_SIDE_RA_RELATIVE_MOTION = 12, OSFM_SIDE_RA_ABSOLUTE_POSITION = 13, OSFM_SIDE_RA_RELATIVE_ABSOLUTE_POSITION = 14,
  OSFM_SIDE_RA_COMMON_POINT = 15, OSFM_SIDE_RA_COMMON_CAMERA = 16, OSFM_SIDE_NUM_TYPES = 17
};
typedef struct {
  int32_t type, nres, nblocks;
  int32_t kind[6], idx[6];
  int32_t loss;          /* OSFM_LOSS_*, or -1 for no loss function */
  double loss_a;
  int32_t cofs;          /* index of the term's first constant in `consts` */
  int32_t aux[4];
} osfm_side_term;
int osfm_ba_set_side_terms(osfm_ba* ba, int n, const osfm_side_term* terms, int64_t nconsts, const double* consts);
/* SetPointProjectionLossFunction / SetMaxNumIterations / SetLinearSolverType
 * (bundle_adjuster.cc:262-372).  linear_solver: "SPARSE_SCHUR", "DENSE_SCHUR",
 * "ITERATIVE_SCHUR" are all served by Schur elimination + PCG; unknown names fail
 * like ceres::StringToLinearSolverType (bundle_adjuster.cc:1105-1109). */
int osfm_ba_set_options(osfm_ba* ba, int loss, double loss_threshold, int max_iterations,
                        const char* linear_solver, int compute_reprojection_errors);
/* Multi-GPU: this process holds shard `rank` of `world` (observations are
 * sharded by point).  allreduce_sum(buf, count, user) must sum `count` doubles
 * at device pointer `buf` across ranks on `stream` (NCCL); NULL when world == 1. */
typedef int (*osfm_allreduce_fn)(void* device_buf, int64_t count, void* stream, void* user);
int osfm_ba_set_distributed(osfm_ba* ba, int rank, int world, osfm_allreduce_fn fn, void* user);
/* Alternative to the callback: the library opens libnccl.so.2 itself and owns a communicator.
 * Rank 0 calls osfm_nccl_unique_id, the caller broadcasts the 128 bytes by its own means, every rank calls
 * osfm_ba_set_nccl (collective), then osfm_ba_set_distributed(ba, rank, world, NULL, NULL).  The all-reduces
 * of a run are then plain ncclAllReduce calls on the library's stream (no host code in between). */
int osfm_nccl_unique_id(char* out128);
int osfm_ba_set_nccl(osfm_ba* ba, int rank, int world, const char* id128);
/* Use an externally owned stream (e.g. torch's current stream); NULL = own stream. */
int osfm_ba_set_stream(osfm_ba* ba, void* cuda_stream);

/* BundleAdjuster::Run (bundle_adjuster.cc:595-1121). */
int osfm_ba_run(osfm_ba* ba);

typedef struct {
  int iterations;             /* LM iterations executed (successful + unsuccessful) */
  int successful_steps;
  int linear_solves;
  int pcg_iterations;         /* total CG iterations */
  int termination;            /* 0 CONVERGENCE, 1 NO_CONVERGENCE, 2 FAILURE */
  double initial_cost, final_cost;
  double time_run_s;          /* wall time of run() (ba_helpers.cc:749-753) */
  double time_device_ms;      /* CUDA-event time of the LM loop */
  /* phase times: summed device-clock (%globaltimer) spans of the linearise+accumulate kernel, the Schur-complement
     kernels, the PCG solves and the back-substitution inside the LM loop */
  double time_linearize_ms;
  int64_t linearize_launches;
  double time_schur_ms;
  int64_t schur_launches;
  double time_pcg_ms;
  double time_backsub_ms;
  int64_t num_observations_local; /* observations held by this rank */
  int reduced_dim;            /* dimension of the reduced camera system */
  int reduced_blocks;         /* stored blocks of the block-sparse reduced system (both triangles) */
  int64_t reduced_nnz;        /* stored doubles of the reduced system */
  int jac_planes;             /* doubles stored per observation: nres * (wc + 3 + 1) */
  int64_t kernel_launches;     /* kernels executed by run() (the device-driven loop's graph counted per execution) */
  char message[128];
  int device_loop;             /* 1: the LM loop ran as one CUDA graph with device-side step control */
} osfm_ba_summary;
int osfm_ba_get_summary(osfm_ba* ba, osfm_ba_summary* out);

int osfm_ba_get_cameras(osfm_ba* ba, double* params_flat);
int osfm_ba_get_rig_instances(osfm_ba* ba, double* pose6);
int osfm_ba_get_rig_cameras(osfm_ba* ba, double* pose6);
int osfm_ba_get_points(osfm_ba* ba, double* xyz);
/* ComputeReprojectionErrors (bundle_adjuster.cc:1196-1208): unscaled residuals,
 * n x 3 (third column 0 for 2-D errors), observation order. */
int osfm_ba_get_reprojection_errors(osfm_ba* ba, double* out_n_by_3);

/* Single-observation evaluation on the device (test hook for the per-observation
 * kernel; ReprojectionError2DAnalytic::Evaluate, projection_errors.h:67-207).
 * Outputs: r[3], jac_camera[3*C], jac_instance[18], jac_rig_camera[18], jac_point[9]. */
int osfm_ba_eval_observation(int device, int projection_type, const double* camera, const double* rig_instance,
                             const double* rig_camera, int use_rig_camera, const double* point,
                             const double* observed, double std_deviation, double* r, double* jac_camera,
                             double* jac_instance, double* jac_rig_camera, double* jac_point, int* num_residuals);

/* Linear-system capture (test hook for the Schur-complement and PCG kernels).  Arms a capture of the damped
 * reduced camera system at LM iteration `iteration` (1-based) of the next osfm_ba_run; 0 disarms.  Single-GPU
 * only (world == 1, else OSFM_ERR_ARG).  Unarmed, run() computes exactly what it computes without the hook. */
int osfm_ba_capture_linear_system(osfm_ba* ba, int iteration);
/* Fallback paths (test and A/B hook).  Every run() of the handle takes the kernel paths `mask` names instead of the
 * product path; each is a path some inputs take anyway, so a test can compare it with the default on any scene.
 * 0 = the product path; sticky until the next call.  Bits outside the enum fail with OSFM_ERR_ARG. */
enum { OSFM_BA_FALLBACK_PER_POINT_SCHUR = 1,        /* every point through the per-point ba_schur */
       OSFM_BA_FALLBACK_SIMT_SEGMENT_SCHUR = 2,     /* SIMT segment kernels instead of the tensor-core ones */
       OSFM_BA_FALLBACK_CTA_PER_SEGMENT_SCHUR = 4,  /* ba_schur_mma (one CTA per segment), not ba_schur_pipe */
       OSFM_BA_FALLBACK_GENERIC_LINEARIZE = 8,      /* generic ba_linearize even for uniform scenes */
       OSFM_BA_FALLBACK_CLASSIC_PCG = 16,           /* the classic PCG only, not the pipelined one */
       OSFM_BA_FALLBACK_STREAMED_PCG = 32,          /* the classic PCG streams S from memory */
       OSFM_BA_FALLBACK_UNDEFLATED_PCG = 64,        /* the pipelined PCG without gauge deflation */
       OSFM_BA_FALLBACK_HOST_LOOP = 128 };          /* the host drives the LM loop, no CUDA graph */
int osfm_ba_set_fallbacks(osfm_ba* ba, unsigned mask);
enum { OSFM_SCHUR_NONE = 0, OSFM_SCHUR_PIPE = 1, OSFM_SCHUR_MMA = 2, OSFM_SCHUR_SIMT_SEGMENT = 3 };
enum { OSFM_PCG_PIPELINED_DEFLATED = 1, OSFM_PCG_PIPELINED = 2, OSFM_PCG_CLASSIC_RESIDENT = 3,
       OSFM_PCG_CLASSIC_STREAMED = 4 };
typedef struct {
  int iteration;              /* LM iteration captured */
  int nc, n, wc, nres;        /* reduced dimension, nc + 3 * free points, camera-side width, residuals / observation */
  double radius;              /* trust-region radius of the iteration: S holds D_c / radius on its diagonal */
  int nseg, p_fast, p_slow;   /* segments; points in segments; points through the per-point ba_schur */
  int schur_kernel;           /* OSFM_SCHUR_*: the segment kernel that ran (NONE when no point is in a segment) */
  int sp_nchunks;             /* chunks of the segment chunk list (0 = none: no segments, or wc != 9 or nres != 2) */
  int pcg_kernel;             /* OSFM_PCG_*: the solver that produced y */
  int pcg_rescued;            /* 1 = the pipelined PCG's result was rejected and the classic PCG re-solved */
  int pcg_iterations;         /* iterations of the solver that produced y */
  double pcg_rr;              /* |r|^2 that solver reported at exit */
} osfm_ba_capture;
/* What the last armed run captured.  S: dense nc x nc row-major, every stored block expanded from its own storage
 * (upper and lower blocks separately, blocks that are not stored stay 0) after priors, side terms, damping and
 * mirroring, i.e. the matrix the PCG receives; rhs[nc]; y[nc] the PCG solution; scale[n], diag[n] (the undamped
 * LM diagonal) and grad[n] with the point side in the caller's order (free points by ascending index).  Any
 * output may be NULL.  Fails when nothing was captured or nc > 8192. */
int osfm_ba_get_captured_system(osfm_ba* ba, osfm_ba_capture* info, double* S, double* rhs, double* y, double* scale,
                                double* diag, double* grad);
/* The side terms' rows of the captured linearisation, robustified (sqrt(rho') r and sqrt(rho') J), terms in the order
 * osfm_ba_set_side_terms got them: r holds each term's nres residuals, J each term's nres x np block row-major (np =
 * the sizes of its blocks in the order it lists them; the columns of constant blocks are 0).  Either may be NULL. */
int osfm_ba_get_captured_side_rows(osfm_ba* ba, double* r, double* J);
/* The parameters at which the captured system was linearised, laid out like osfm_ba_get_cameras /
 * _rig_instances / _rig_cameras / _points / _ext_blocks.  Any output may be NULL. */
int osfm_ba_get_captured_parameters(osfm_ba* ba, double* cam_params, double* inst_pose6, double* rig_camera_pose6,
                                    double* points, double* ext_values);

/* Rig-instance pose covariances (bundle_adjuster.cc:1123-1194).  When enabled, run() ends with a covariance pass
 * at the accepted parameters: (J^T J)^-1 of the robustified Jacobian over every non-constant block, bounds ignored,
 * each rig instance's 6 x 6 diagonal block in its [rx, ry, rz, tx, ty, tz] order.  Single GPU only (run() fails
 * with world > 1), and run() fails when the dense n_c x n_c reduced system does not fit in device memory. */
int osfm_ba_set_compute_covariances(osfm_ba* ba, int enable);
enum {
  OSFM_COV_OK = 0,                     /* computed, every block finite: valid */
  OSFM_COV_SOLVER_FAILURE = 1,         /* the solve terminated with FAILURE: not computed */
  OSFM_COV_POINT_RANK_DEFICIENT = 2,   /* a point's 3x3 block failed the pivot test */
  OSFM_COV_CAMERA_RANK_DEFICIENT = 3,  /* the reduced camera system failed the pivot test */
  OSFM_COV_NON_FINITE = 4              /* a covariance entry is not finite */
};
/* Result of the last run(), which must have been armed.  out: NI x 36, row-major 6 x 6 per instance in the
 * caller's order; constant instances get zeros.  Invalid (status != OSFM_COV_OK): every instance gets
 * diag(1e-5, 1e-5, 1e-5, 1e-2, 1e-2, 1e-2).  Any output may be NULL. */
int osfm_ba_get_covariances(osfm_ba* ba, int* valid, int* status, double* out);
/* Device time of the last covariance pass (CUDA events): the whole pass and the Cholesky of the reduced system. */
int osfm_ba_get_covariance_timing(osfm_ba* ba, double* pass_ms, double* cholesky_ms);

/* ------------------------------------------------------------------------
 * TRACKS
 * ---------------------------------------------------------------------- */
typedef struct osfm_tracks osfm_tracks;

/* Links pair matches into tracks: tracking.create_tracks_manager (opensfm/tracking.py:72-150) and, for all image
 * pairs at once, TracksManager::GetAllPairsConnectivity / GetAllCommonObservations (tracks_manager.cc:285-350).
 * A handle owns one CUDA stream and its workspaces on `device`; they are reused from call to call. */
int osfm_tracks_create(int device, osfm_tracks** out);
int osfm_tracks_destroy(osfm_tracks* t);
/* Connected components of the graph whose nodes are features and whose edges are match rows, filtered like
 * _good_track (tracking.py:238-244): at least min_length features and no two of one image.
 * num_features[i] = features of image i; has_features[i] = 0 for an image that occurs in matches but has no
 * feature file: its features count in the filter and are left out of the output (tracking.py:98 vs :106).  Pair p
 * owns rows [match_start[p], match_start[p + 1]) of matches (int32 x 2: feature in pair_a[p], feature in
 * pair_b[p]); a pair may be listed several times and in either order.  Tracks with at least one observation to
 * output are numbered 0 .. T - 1 by their smallest (image, feature), so the result does not depend on the order of
 * pairs or rows.  Returns T and the number of observations N.  Fails with OSFM_ERR_RUNTIME, naming the first
 * offending row, if an image or feature index is out of range, and with OSFM_ERR_ARG for more than 2^31 - 1
 * features or match rows in all. */
int osfm_tracks_build(osfm_tracks* t, int num_images, const int32_t* num_features, const uint8_t* has_features,
                      int64_t num_pairs, const int32_t* pair_a, const int32_t* pair_b, const int64_t* match_start,
                      const int32_t* matches, int min_length, int64_t* num_tracks, int64_t* num_observations);
/* The last build's observations sorted by (track, image): obs_track / obs_image / obs_feature have N entries,
 * track t owns rows [track_start[t], track_start[t + 1]) (T + 1 entries). */
int osfm_tracks_get(osfm_tracks* t, int32_t* obs_track, int32_t* obs_image, int32_t* obs_feature,
                    int64_t* track_start);
/* For the last build, every image pair a < b with a track in common and the observations they share.  Returns the
 * number of such pairs Q and the total number of shared tracks R over all pairs (a track of L observations counts
 * L (L - 1) / 2 times).  R is known before the pair lists are built; if the device cannot hold them (about 33 R
 * bytes) the call fails with OSFM_ERR_CUDA and a message giving R, and the handle stays usable. */
int osfm_tracks_common(osfm_tracks* t, int64_t* num_pairs, int64_t* num_common);
/* Pairs ascending by (pair_a, pair_b), Q entries; pair q owns rows [pair_start[q], pair_start[q + 1]) (Q + 1
 * entries; the run length is the pair's connectivity) of common_obs_a / common_obs_b (R entries): rows of
 * osfm_tracks_get's arrays, the observation in pair_a[q] and the one of the same track in pair_b[q], tracks
 * ascending inside a pair. */
int osfm_tracks_get_common(osfm_tracks* t, int32_t* pair_a, int32_t* pair_b, int64_t* pair_start,
                           int64_t* common_obs_a, int64_t* common_obs_b);
/* Device time of the last osfm_tracks_build (kernels, sorts and scans, after the uploads) and the last
 * osfm_tracks_common (CUDA events on the handle's stream). */
int osfm_tracks_last_device_ms(osfm_tracks* t, float* ms_build, float* ms_common);

/* Triangulates the handle's tracks from its device-resident observations: TrackTriangulator.triangulate
 * (opensfm/reconstruction.py:1032-1073) of every selected track, i.e. TriangulateBearingsMidpoint with its angle,
 * reprojection and depth tests (geometry/src/triangulation.cc:137-177) and PointRefinement (:221-233), in fp64.
 * num_images / num_observations / num_tracks must be the handle's (osfm_tracks_build).  Per image: image_rt
 * (row-major R^T of the world-to-camera rotation, 9), image_origin (3), image_in (1 if the image is in the
 * reconstruction); only observations in such images are used.  Per observation, in osfm_tracks_get's order:
 * bearings (camera frame, 3; read only in images of the reconstruction).  Per track: selected (0 / 1).
 * threshold is the reprojection angle and min_ray_angle the least ray angle, both in radians; iterations bounds the
 * refinement.  Out per track: status (OSFM_TRI_*) and points (3; NaN unless the status is OSFM_TRI_OK). */
#define OSFM_TRI_NOT_SELECTED 0
#define OSFM_TRI_TOO_FEW 1          /* fewer than 2 observations in images of the reconstruction */
#define OSFM_TRI_BAD_ANGLE 2        /* no pair of rays at an angle in [min_ray_angle, pi - min_ray_angle] */
#define OSFM_TRI_BAD_REPROJECTION 3 /* the midpoint fails the reprojection or the depth test */
#define OSFM_TRI_OK 4
int osfm_tracks_triangulate(osfm_tracks* t, int num_images, const double* image_rt, const double* image_origin,
                            const uint8_t* image_in, int64_t num_observations, const double* bearings,
                            int64_t num_tracks, const uint8_t* selected, double threshold, double min_ray_angle,
                            double min_depth, int iterations, int8_t* status, double* points);
/* Device time of the last osfm_tracks_triangulate (CUDA events around its kernel, after the uploads). */
int osfm_tracks_last_triangulate_ms(osfm_tracks* t, float* ms);

/* ------------------------------------------------------------------------
 * ROTATION-ONLY RANSAC OF IMAGE PAIRS
 * ---------------------------------------------------------------------- */
typedef struct osfm_rotransac osfm_rotransac;

/* Ranks image pairs for the reconstruction bootstrap: pyrobust's ransac_relative_rotation with RANSAC scoring, as
 * compute_image_pairs runs it (opensfm/reconstruction.py:208-244), and the chord inliers of its rotation, for many
 * pairs at once.  The rules, including the one deliberate difference (a 3-row sample takes the proper Kabsch
 * rotation), are stated in oracle/rotation_ransac_oracle.py.  A handle owns one CUDA stream, its workspaces on
 * `device` and the shared sample stream of mt19937(42). */
int osfm_rotransac_create(int device, osfm_rotransac** out);
int osfm_rotransac_destroy(osfm_rotransac* h);
/* bearings: num_bearings x 3 fp64 unit vectors.  Pair p owns rows [pair_start[p], pair_start[p + 1]) (pair_start[0]
 * = 0); row r pairs bearing row_a[r] of the first image with bearing row_b[r] of the second.  threshold is the
 * angle of compute_image_pairs (4 * five_point_algo_threshold): RANSAC inliers have |1 - (M b1) . b2| below
 * 1 - cos(threshold), chord inliers ||R b2 - b1|| below threshold with R = lo_model^T.  iterations >= 1 (the
 * reference passes 1000).  Outputs: lo_model (9 per pair, row-major), the RANSAC inlier count and the chord inlier
 * count of every pair, and the chord inlier mask of every row.  A pair of fewer than 3 rows, or a row naming a
 * bearing outside [0, num_bearings), fails with OSFM_ERR_ARG naming it. */
int osfm_rotransac_run(osfm_rotransac* h, int64_t num_bearings, const double* bearings, int64_t num_pairs,
                       const int64_t* pair_start, const int64_t* row_a, const int64_t* row_b, double threshold,
                       int iterations, double* lo_model, int32_t* ransac_inliers, int32_t* chord_inliers,
                       uint8_t* chord_mask);
/* Device time of the last osfm_rotransac_run (CUDA events around its kernels, after the uploads). */
int osfm_rotransac_last_device_ms(osfm_rotransac* h, float* ms);
/* Test hooks.  The generator outputs kept on the device (65536 unless set; a pair that uses them all continues from
 * the generator state saved after them).  Tracing: with capacity > 0 the next runs record, per pair, every sample
 * index drawn (minimal samples: rows; local optimisation: positions in the best inlier list), in order, up to
 * capacity of them; get_trace returns, per pair, how many were drawn, how many generator outputs were consumed,
 * and the indices (num_pairs x capacity). */
int osfm_rotransac_set_stream_prefix(osfm_rotransac* h, int64_t length);
int osfm_rotransac_set_trace(osfm_rotransac* h, int capacity);
int osfm_rotransac_get_trace(osfm_rotransac* h, int32_t* count, int64_t* stream_used, int32_t* indices);

/* ------------------------------------------------------------------------
 * ABSOLUTE-POSE RANSAC OF SHOTS (RESECTION)
 * ---------------------------------------------------------------------- */
typedef struct osfm_resect osfm_resect;

/* Resects shots against the reconstructed points: pyrobust's ransac_absolute_pose with RANSAC scoring (P3P samples,
 * Lu's orthogonal iteration in local optimisation), as resect runs it through multiview.absolute_pose_ransac
 * (opensfm/reconstruction.py:695-762), and the chord inliers of the resulting pose, for many shots at once.  The
 * rules, including the deliberate differences, are stated in oracle/absolute_pose_oracle.py.  A handle owns one CUDA
 * stream, its workspaces on `device` and the shared sample stream of mt19937(42). */
int osfm_resect_create(int device, osfm_resect** out);
int osfm_resect_destroy(osfm_resect* h);
/* bearings: num_bearings x 3 fp64 (normalised on the device); points: num_points x 3 fp64 world points.  Shot s
 * owns rows [shot_start[s], shot_start[s + 1]) (shot_start[0] = 0); row r pairs bearing row_bearing[r] with point
 * row_point[r].  threshold is resect's angle (resection_threshold): RANSAC inliers have |1 - b . normalize(R X + t)|
 * below 1 - cos(threshold), chord inliers ||normalize(R (X - o)) - b|| below threshold, o = -R^T t.  iterations >= 1
 * (resect passes 1000).  Outputs: lo_model (12 per shot: [R | t] row-major, world to camera), the RANSAC inlier count
 * and the chord inlier count of every shot, and the chord inlier mask of every row.  A shot of fewer than 3 rows, or
 * a row naming a bearing or point outside its table, fails with OSFM_ERR_ARG naming it. */
int osfm_resect_run(osfm_resect* h, int64_t num_bearings, const double* bearings, int64_t num_points,
                    const double* points, int64_t num_shots, const int64_t* shot_start, const int64_t* row_bearing,
                    const int64_t* row_point, double threshold, int iterations, double* lo_model,
                    int32_t* ransac_inliers, int32_t* chord_inliers, uint8_t* chord_mask);
/* Device time of the last osfm_resect_run (CUDA events around its kernels, after the uploads). */
int osfm_resect_last_device_ms(osfm_resect* h, float* ms);
/* Test hooks, as osfm_rotransac_set_stream_prefix / set_trace / get_trace, per shot. */
int osfm_resect_set_stream_prefix(osfm_resect* h, int64_t length);
int osfm_resect_set_trace(osfm_resect* h, int capacity);
int osfm_resect_get_trace(osfm_resect* h, int32_t* count, int64_t* stream_used, int32_t* indices);

/* ------------------------------------------------------------------------
 * FIVE-POINT RELATIVE-POSE RANSAC OF IMAGE PAIRS
 * ---------------------------------------------------------------------- */
typedef struct osfm_relpose osfm_relpose;

/* Estimates the relative pose of image pairs: pyrobust's ransac_relative_pose with RANSAC scoring (five-point
 * samples, EssentialNPoints in local optimisation), as two_view_reconstruction_general runs it through
 * multiview.relative_pose_ransac, for many pairs at once.  The rules, including the deliberate differences, are
 * stated in oracle/relative_pose_oracle.py.  A handle owns one CUDA stream, its workspaces on `device` and the shared
 * sample stream of mt19937(42). */
int osfm_relpose_create(int device, osfm_relpose** out);
int osfm_relpose_destroy(osfm_relpose* h);
/* bearings: num_bearings x 3 fp64 (normalised on the device).  Pair p owns rows [pair_start[p], pair_start[p + 1])
 * (pair_start[0] = 0); row r pairs bearing row_a[r] of the first image with bearing row_b[r] of the second.
 * threshold is an angle: inliers have |1 - (px . x + py . y) / 2| below 1 - cos(threshold), px and py the midpoint
 * of the row seen from both cameras.  iterations >= 1 (two_view_reconstruction_general passes 1000).  Outputs:
 * lo_model (12 per pair: [R | t] row-major, x2 = R x1 + t, |t| = 1), the RANSAC inlier count of every pair and the
 * inlier mask of lo_model over every row.  A pair of fewer than 5 rows, or a row naming a bearing outside the table,
 * fails with OSFM_ERR_ARG naming it. */
int osfm_relpose_run(osfm_relpose* h, int64_t num_bearings, const double* bearings, int64_t num_pairs,
                     const int64_t* pair_start, const int64_t* row_a, const int64_t* row_b, double threshold,
                     int iterations, double* lo_model, int32_t* ransac_inliers, uint8_t* inlier_mask);
/* two_view_reconstruction_general's steps after the plane homography, for many pairs in one call: the RANSAC of
 * osfm_relpose_run (same inputs, same checks, same threshold angle), then on the device, per pair, from its lo_model:
 * the bearing inliers of the pose [R^T | -R^T t] (and, when check_reversal = 1, of its transpose), the TinySolver
 * refinement of RelativePoseRefinement on more than 5 inliers (refine_iterations = max_num_iterations), the inliers
 * of the refined pose, the Necker rule of two_view_reconstruction_5pt with reversal_ratio, and the inliers of the
 * plane motion.  The rules are stated in oracle/two_view_oracle.py.
 *   threshold         the angle of RANSAC and the chord bound of the bearing inliers (five_point_algo_threshold)
 *   plane_pose        12 per pair: the plane motion [R_p | t_p] row-major (motion_from_plane_homography's first),
 *                     whose inliers are those of (R_p^T, -R_p^T t_p); NaN when the pair has none
 * Outputs: lo_model and ransac_inliers as osfm_relpose_run; pose (24 per pair: each configuration's final [R | t],
 * row-major, in compute_inliers_bearings' convention, NaN for a configuration not run); counts (3 per pair: final
 * inliers of each configuration, then of the plane motion); chosen (per pair: 0 or 1, the configuration the 5-point
 * result keeps, -1 for none); mask_5pt and mask_plane (per row: the inliers of the 5-point and plane results).
 * refine_iterations >= 1, check_reversal 0 or 1, reversal_ratio not NaN; otherwise, or on the conditions of
 * osfm_relpose_run, OSFM_ERR_ARG. */
int osfm_relpose_two_view(osfm_relpose* h, int64_t num_bearings, const double* bearings, int64_t num_pairs,
                          const int64_t* pair_start, const int64_t* row_a, const int64_t* row_b, double threshold,
                          int ransac_iterations, int refine_iterations, int check_reversal, double reversal_ratio,
                          const double* plane_pose, double* lo_model, int32_t* ransac_inliers, double* pose,
                          int32_t* counts, int32_t* chosen, uint8_t* mask_5pt, uint8_t* mask_plane);
/* Device time of the last osfm_relpose_run or osfm_relpose_two_view (CUDA events around its kernels, after the
 * uploads). */
int osfm_relpose_last_device_ms(osfm_relpose* h, float* ms);
/* The same split into the RANSAC kernels and the two-view kernel (0 when the last call was osfm_relpose_run). */
int osfm_relpose_last_stage_ms(osfm_relpose* h, float* ransac_ms, float* two_view_ms);
/* Test hooks, as osfm_rotransac_set_stream_prefix / set_trace / get_trace, per pair. */
int osfm_relpose_set_stream_prefix(osfm_relpose* h, int64_t length);
int osfm_relpose_set_trace(osfm_relpose* h, int capacity);
int osfm_relpose_get_trace(osfm_relpose* h, int32_t* count, int64_t* stream_used, int32_t* indices);

/* ------------------------------------------------------------------------
 * DENSE DEPTHMAPS
 * ---------------------------------------------------------------------- */
typedef struct osfm_dense osfm_dense;

#define OSFM_DENSE_BRUTE_FORCE 0
#define OSFM_DENSE_PATCH_MATCH 1
#define OSFM_DENSE_PATCH_MATCH_SAMPLE 2
#define OSFM_DENSE_MAX_PATCH 15
#define OSFM_DENSE_MAX_VIEWS 32

/* pydense's DepthmapEstimator, DepthmapCleaner and DepthmapPruner (opensfm/src/dense/src/depthmap.cc) for many
 * reference shots per call, over views kept resident on the handle.  The rules are restated in
 * oracle/dense_oracle.cpp; the one deliberate difference is the generator: every variate is Philox4x32-10 keyed by
 * (seed, the reference's key) at counter (pixel, pass, draw, attempt).  A handle owns one CUDA stream and its
 * workspaces on `device`. */
int osfm_dense_create(int device, osfm_dense** out);
int osfm_dense_destroy(osfm_dense* h);
/* Replaces the handle's views (and forgets every map).  size: 2 per view (width, height); K, Kinv, R: 9 per view
 * row-major fp64; t: 3 per view.  gray, mask, labels: every view's pixels in view order, row-major; rgb: 3 per
 * pixel.  gray and mask are needed to estimate, rgb and labels to prune; each may be null otherwise.  Fails with
 * OSFM_ERR_RUNTIME naming the bytes needed when the views and their maps do not fit in device memory. */
int osfm_dense_set_views(osfm_dense* h, int num_views, const int32_t* size, const double* K, const double* Kinv,
                         const double* R, const double* t, const uint8_t* gray, const uint8_t* mask,
                         const uint8_t* rgb, const uint8_t* labels);
/* Uploads maps of one view computed earlier: raw depth (as compute_depthmap saves it), plane (3 per pixel) and clean
 * depth; each may be null.  A view has a raw map once raw depth and plane are set, a clean map once clean depth and
 * plane are. */
int osfm_dense_set_maps(osfm_dense* h, int view, const float* raw_depth, const float* plane, const float* clean_depth);
/* Estimates the depthmap of num_refs references.  Reference r's views are views[list_start[r] .. list_start[r+1]),
 * itself first, 2 to OSFM_DENSE_MAX_VIEWS of them.  Per list entry e: Q (9) = R_v R_ref^T and a (3) = Q t_ref - t_v.
 * params: 5 per reference (method, patch_size, num_depth_planes, patchmatch_iterations, generator key);
 * depth_range: 2 per reference (min, max); min_patch_variance: per reference; weights: the bilateral weight table,
 * 256 x (2 ((OSFM_DENSE_MAX_PATCH - 1) / 2)^2 + 1) f32 indexed by (|dcolor|, dx^2 + dy^2).  The ungated maps (depth,
 * plane 3 per pixel, score, nghbr as the list-local view index) are written per reference in request order, each of
 * its view's size; any may be null.  The reference view's raw slot gets the depth gated by score > (float)min_score
 * and depth < max, and the plane.  An even or too-large patch, patch size 1 with a PatchMatch method (its passes
 * would read a pixel's neighbours outside the maps), an unknown method, a bad depth range, a view out of range or two
 * references of the same view fails with OSFM_ERR_ARG, before anything is launched; maps that do not fit in device
 * memory fail with OSFM_ERR_RUNTIME naming the bytes needed. */
int osfm_dense_estimate(osfm_dense* h, int num_refs, const int32_t* list_start, const int32_t* views, const double* Q,
                        const double* a, const int32_t* params, const double* depth_range,
                        const float* min_patch_variance, const float* weights, uint32_t seed, double min_score,
                        float* depth, float* plane, float* score, int32_t* nghbr);
/* DepthmapCleaner::Clean of every reference over the raw slots of its views (reference first, each with a raw map),
 * into the reference's clean slot (two references of the same view fail with OSFM_ERR_ARG); clean_depth (nullable) receives the maps per reference in request order. */
int osfm_dense_clean(osfm_dense* h, int num_refs, const int32_t* list_start, const int32_t* views,
                     float same_depth_threshold, int min_consistent_views, float* clean_depth);
/* DepthmapPruner::Prune of every reference over the clean depth and plane of its views (reference first, each with a
 * clean map) and the reference's colour and labels.  counts: per reference, the points kept; the points themselves,
 * in raster order per reference and references in request order, come from osfm_dense_get_pruned. */
int osfm_dense_prune(osfm_dense* h, int num_refs, const int32_t* list_start, const int32_t* views,
                     float same_depth_threshold, int64_t* counts);
/* The last prune's points (3 f32 each), normals (3 f32), colours (3 u8) and labels (u8). */
int osfm_dense_get_pruned(osfm_dense* h, float* points, float* normals, uint8_t* colors, uint8_t* labels);
/* Device time of the last estimate, clean and prune (CUDA events around their kernels, after the uploads). */
int osfm_dense_last_device_ms(osfm_dense* h, float* estimate_ms, float* clean_ms, float* prune_ms);

#ifdef __cplusplus
}
#endif
#endif /* OPENSFM_B200_H_ */
