// host_intr_cols.cc -- the product's obs_intr_cols (theiasfm_b200/csrc/tba_camera_models.cuh) compiled for the host: the J_i that
// linearize_obs returns against the one the passes over a compact linearisation rebuild from the normalised image point (u, v)
// with the identity corrector (tests/test_compact_intrinsics_host.py).  Nothing here is used by the product.
#define __device__
#define __host__
#define __forceinline__ inline
#define __restrict__
#ifndef _GNU_SOURCE
#define _GNU_SOURCE
#endif
#include <cmath>
using std::atan;
using std::atan2;
using std::fabs;
using std::fmax;
using std::sqrt;
using std::tan;

#include "../theiasfm_b200/csrc/tba_camera_models.cuh"

extern "C" {

// One observation through cam_prep + linearize_obs<all 10 intrinsics columns>: Ji[20] and uv[2] as linearize_obs returns them,
// Jr[20] rebuilt by obs_intr_cols from uv with P = I.  Returns 0 when the projection fails.
int host_intr_cols(int model, const double* ext, const double* intr, const double* pt, const double* xy, int loss_type, double loss_width,
                   double* Ji, double* uv, double* Jr) {
  double rec[tba::kCamRec];
  tba::cam_prep(ext + 3, rec);
  double r[2], rho0, Ja[6], Jw[6], Jh[2];
  if (!tba::linearize_obs<0x3FFu>(model, ext, rec, intr, pt[0], pt[1], pt[2], pt[3], xy[0], xy[1], loss_type, loss_width, r, rho0, Ja, Jw,
                                  Jh, Ji, uv))
    return 0;
  tba::obs_intr_cols<0x3FFu>(model, uv[0], uv[1], intr, 1.0, 0.0, 0.0, 1.0, Jr);
  return 1;
}

}  // extern "C"
