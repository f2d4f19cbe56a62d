// TRIANGULATE: the tracks of a tracks handle triangulated on the device (triangulate.cu).  The handle's engine
// (tracks.cu) owns the workspace and passes its device-resident observation arrays; nothing of the topology is
// uploaded again.
#pragma once
#include "common.cuh"

namespace osfm {

// per-track result codes (include/opensfm_b200.h)
enum TriStatus : int8_t {
  TRI_NOT_SELECTED = 0,
  TRI_TOO_FEW = 1,        // fewer than 2 observations in images of the reconstruction
  TRI_BAD_ANGLE = 2,      // no pair of rays at an angle in [min_angle, pi - min_angle]
  TRI_BAD_REPROJECTION = 3,   // the midpoint fails the reprojection or the depth test of some observation
  TRI_OK = 4,
};

struct TriWorkspace {
  DevBuf<double> image_rt, image_origin, bearings, X;
  DevBuf<unsigned char> image_in, selected;
  DevBuf<int8_t> status;
  bool timed = false;
};

// The tracks' device arrays: T tracks, nobs observations sorted by (track, image), obs_image in [0, I).  The
// tracks handle keeps nobs below 2^31, so the kernel indexes observations with int.
struct TriTopology {
  int I, T;
  long long nobs;
  const int* obs_image;
  const long long* track_start;
};

void triangulate_tracks(TriWorkspace& w, cudaStream_t stream, cudaEvent_t ev_start, cudaEvent_t ev_end,
                        const TriTopology& topo, const double* image_rt, const double* image_origin,
                        const uint8_t* image_in, const double* bearings, const uint8_t* selected, double threshold,
                        double min_ray_angle, double min_depth, int iterations, int8_t* status, double* X);

}  // namespace osfm
