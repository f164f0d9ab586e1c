// tba_camera_models.cuh -- device-side reprojection residual + ANALYTIC Jacobian.
//
// What it must equal (reference): ReprojectionError<CameraModel>::operator()
// (src/theia/sfm/camera/reprojection_error.h:51-95) instantiated for
// PinholeCameraModel (pinhole_camera_model.h:181-210,241-257) and
// PinholeRadialTangentialCameraModel (pinhole_radial_tangential_camera_model.h:190-219,
// 250-291), differentiated the way ceres::AutoDiffCostFunction<.., 2, 6, K, 4>
// (create_reprojection_error_cost_function.h:60-90) does.  The derivation is NOT a
// transcription of any reference code (the reference has no analytic Jacobian):
//
//   a = X - h C,  q = R(w) a,  (u,v) = q_xy / q_z,  (ud,vd) = distort(u,v),  pix = K2 (ud,vd) + c
//   J_q  = K2 * D' * (1/q_z) [[1,0,-u],[0,1,-v]]                       (2x3)
//   J_a  = J_q R           = dpix/dX_{0..2}
//   J_h  = -J_a C          = dpix/dh           (homogeneous coordinate, track.h:87)
//   J_C  = -h J_a          = dpix/dC
//   J_w  = -(J_q x q) J_l(w)   exact derivative of Rodrigues' formula (left Jacobian of SO(3));
//          -(J_q x a)          in the first-order branch theta^2 <= DBL_EPSILON of
//                              ceres::AngleAxisRotatePoint (q = a + w x a).
//
// Only J_a, J_w, J_h and the free intrinsics columns are stored per observation
// ("compact linearisation", DESIGN.md section 4); J_C is rebuilt from J_a and h.
#pragma once
#include <cstdint>
#include <cfloat>

#include "tba_camera_models_ext.cuh"  // FISHEYE / FOV / DIVISION_UNDISTORTION (only in EXT = true instantiations)

// '#pragma unroll' only where the device compiler sees it (the host pass of __host__ __device__ code warns otherwise)
#ifdef __CUDA_ARCH__
#define TBA_UNROLL _Pragma("unroll")
#else
#define TBA_UNROLL
#endif

namespace tba {

constexpr int kModelPinhole = 0;
constexpr int kModelRadTan = 1;

// Per-camera record written by k_cam_prep: R (row-major 9), L = J_l(w) (9), small-angle flag, pad.
constexpr int kCamRec = 20;

__host__ __device__ constexpr int popcount10(uint32_t m) {
  int n = 0;
  for (int i = 0; i < 10; ++i) n += (m >> i) & 1u;
  return n;
}
// index of the j-th set bit of m (compile-time use)
__host__ __device__ constexpr int nth_bit(uint32_t m, int j) {
  int n = 0;
  for (int i = 0; i < 10; ++i) {
    if ((m >> i) & 1u) {
      if (n == j) return i;
      ++n;
    }
  }
  return 0;
}

// Rotation matrix and left Jacobian of SO(3) for one camera, in two steps so that kernels can gather a COMPACT record
// (the angle-axis w from ext + four scalars = 56 bytes instead of the 160-byte matrix record) and rebuild R and J_l in
// registers with exactly the arithmetic cam_prep itself uses (bit-identical values everywhere):
//   s4 = {c, S, B, Cc}:  c = cos(th), S = sin(th)/th, B = (1 - cos th)/th^2 = 2 sin^2(th/2)/th^2, Cc = (th - sin th)/th^3;
//   R   = c I + S [w]x + B w w^T,     J_l = (1 - Cc th^2) I + B [w]x + Cc w w^T;
//   first-order branch of ceres::AngleAxisRotatePoint (th^2 <= DBL_EPSILON): s4 = {1, 1, 0, 0}, R = I + [w]x, J_l = I
//   (B == 0 identifies it: B ~ 1/2 whenever the Rodrigues branch runs).
__host__ __device__ inline void cam_scalars(const double* __restrict__ w, double s4[4]) {
  const double th2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2];
  if (th2 > DBL_EPSILON) {
    const double th = sqrt(th2);
    double s, c;
    sincos(th, &s, &c);
    const double sh = sin(0.5 * th);
    s4[0] = c;
    s4[1] = s / th;
    s4[2] = 2.0 * sh * sh / th2;
    if (th < 0.05) s4[3] = 1.0 / 6.0 - th2 * (1.0 / 120.0 - th2 * (1.0 / 5040.0 - th2 * (1.0 / 362880.0 - th2 / 39916800.0)));
    else s4[3] = (th - s) / (th2 * th);
  } else {
    s4[0] = 1.0; s4[1] = 1.0; s4[2] = 0.0; s4[3] = 0.0;
  }
}
__host__ __device__ inline void cam_rec_expand(const double w0, const double w1, const double w2, const double c, const double S,
                                               const double B, const double Cc, double* __restrict__ rec) {
  double* R = rec;
  double* L = rec + 9;
  const double Sw0 = S * w0, Sw1 = S * w1, Sw2 = S * w2;
  const double B01 = B * w0 * w1, B02 = B * w0 * w2, B12 = B * w1 * w2;
  R[0] = c + B * w0 * w0; R[1] = B01 - Sw2;       R[2] = B02 + Sw1;
  R[3] = B01 + Sw2;       R[4] = c + B * w1 * w1; R[5] = B12 - Sw0;
  R[6] = B02 - Sw1;       R[7] = B12 + Sw0;       R[8] = c + B * w2 * w2;
  const double th2 = w0 * w0 + w1 * w1 + w2 * w2;
  const double d = 1.0 - Cc * th2;
  const double Bw0 = B * w0, Bw1 = B * w1, Bw2 = B * w2;
  const double C01 = Cc * w0 * w1, C02 = Cc * w0 * w2, C12 = Cc * w1 * w2;
  L[0] = d + Cc * w0 * w0; L[1] = C01 - Bw2;        L[2] = C02 + Bw1;
  L[3] = C01 + Bw2;        L[4] = d + Cc * w1 * w1; L[5] = C12 - Bw0;
  L[6] = C02 - Bw1;        L[7] = C12 + Bw0;        L[8] = d + Cc * w2 * w2;
  rec[18] = B == 0.0 ? 1.0 : 0.0;  // first-order branch
  rec[19] = 0.0;
}
__host__ __device__ inline void cam_prep(const double* __restrict__ w, double* __restrict__ rec, double* __restrict__ s4_out = nullptr) {
  double s4[4];
  cam_scalars(w, s4);
  cam_rec_expand(w[0], w[1], w[2], s4[0], s4[1], s4[2], s4[3], rec);
  if (s4_out) { s4_out[0] = s4[0]; s4_out[1] = s4[1]; s4_out[2] = s4[2]; s4_out[3] = s4[3]; }
}

// ceres::LossFunction::Evaluate for the six types create_loss_function.cc:42-71 maps to.
__host__ __device__ inline void loss_evaluate(int type, double a, double s, double rho[3]) {
  switch (type) {
    case 1: {  // HUBER
      const double b = a * a;
      if (s > b) { const double r = sqrt(s); rho[0] = 2.0 * a * r - b; rho[1] = fmax(DBL_MIN, a / r); rho[2] = -rho[1] / (2.0 * s); }
      else { rho[0] = s; rho[1] = 1.0; rho[2] = 0.0; }
      break; }
    case 2: {  // SOFTLONE
      const double b = a * a, c = 1.0 / b, sum = 1.0 + s * c, tmp = sqrt(sum);
      rho[0] = 2.0 * b * (tmp - 1.0); rho[1] = fmax(DBL_MIN, 1.0 / tmp); rho[2] = -(c * rho[1]) / (2.0 * sum);
      break; }
    case 3: {  // CAUCHY
      const double b = a * a, c = 1.0 / b, sum = 1.0 + s * c, inv = 1.0 / sum;
      rho[0] = b * log(sum); rho[1] = fmax(DBL_MIN, inv); rho[2] = -c * (inv * inv);
      break; }
    case 4: {  // ARCTAN
      const double b = 1.0 / (a * a), sum = 1.0 + s * s * b, inv = 1.0 / sum;
      rho[0] = a * atan2(s, a); rho[1] = fmax(DBL_MIN, inv); rho[2] = -2.0 * s * b * (inv * inv);
      break; }
    case 5: {  // TUKEY
      const double a2 = a * a;
      if (s <= a2) { const double v = 1.0 - s / a2, v2 = v * v; rho[0] = a2 / 6.0 * (1.0 - v2 * v); rho[1] = 0.5 * v2; rho[2] = -1.0 / a2 * v; }
      else { rho[0] = a2 / 6.0; rho[1] = 0.0; rho[2] = 0.0; }
      break; }
    default: rho[0] = s; rho[1] = 1.0; rho[2] = 0.0;
  }
}

// Camera::ProjectPoint (camera.cc:204-213) without any guard: pixel and camera-frame depth coordinate q_z
// (the caller divides by h for the depth ProjectPoint returns).  a = X - h C is also returned for the callers' guards.
__host__ __device__ inline void project_pixel(int model, const double* __restrict__ C, const double* __restrict__ R,
                                     const double* __restrict__ k, const double X0, const double X1, const double X2, const double h,
                                     double& px, double& py, double& qz, double& a_sq) {
  const double a0 = X0 - h * C[0], a1 = X1 - h * C[1], a2 = X2 - h * C[2];
  a_sq = a0 * a0 + a1 * a1 + a2 * a2;
  const double q0 = R[0] * a0 + R[1] * a1 + R[2] * a2;
  const double q1 = R[3] * a0 + R[4] * a1 + R[5] * a2;
  const double q2 = R[6] * a0 + R[7] * a1 + R[8] * a2;
  qz = q2;
  const double u = q0 / q2, v = q1 / q2;
  const double r2 = u * u + v * v;
  double ud, vd;
  if (model == kModelPinhole) {
    const double d = 1.0 + r2 * (k[5] + k[6] * r2);
    ud = u * d; vd = v * d;
  } else {
    const double rd = 1.0 + k[5] * r2 + k[6] * r2 * r2 + k[7] * r2 * r2 * r2;
    const double tx = k[9] * (r2 + 2.0 * u * u) + 2.0 * k[8] * u * v;
    const double ty = k[8] * (r2 + 2.0 * v * v) + 2.0 * k[9] * u * v;
    ud = u * rd + tx; vd = v * rd + ty;
  }
  px = k[0] * ud + k[2] * vd + k[3];
  py = k[0] * k[1] * vd + k[4];
}

// Projection only (the double instantiation of the functor). Returns false if ||a||^2 < 1e-8.
__host__ __device__ inline bool reproject(int model, const double* __restrict__ C, const double* __restrict__ R,
                                 const double* __restrict__ k, const double X0, const double X1, const double X2,
                                 const double h, const double x, const double y, double& r0, double& r1) {
  double px, py, qz, a_sq;
  project_pixel(model, C, R, k, X0, X1, X2, h, px, py, qz, a_sq);
  if (a_sq < 1e-8) return false;
  r0 = px - x;
  r1 = py - y;
  return true;
}

// Explicitly rounded product, sum and fused multiply-add: what obs_intr_cols computes with them does not depend on how the compiler
// contracts the code around each call site.
__host__ __device__ inline double mul_rn(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;  // only ever an operand of add_rn / fma_rn below, so no sum is left to contract it into
#endif
}
__host__ __device__ inline double add_rn(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;  // host builds of these helpers are compiled without contraction (tests) or see only rounded operands
#endif
}
__host__ __device__ inline double fma_rn(double a, double b, double c) {
#ifdef __CUDA_ARCH__
  return __fma_rn(a, b, c);
#else
  return fma(a, b, c);
#endif
}

// The free intrinsics columns of one PINHOLE / PINHOLE_RADIAL_TANGENTIAL observation from its normalised image point
// (u, v) = q_xy / q_z and the group's intrinsics k, with the loss corrector P applied: Ji[j] = P00 c0 + P01 c1 and
// Ji[NI + j] = P10 c0 + P11 c1 for the j-th column (c0, c1) of IMASK.  linearize_obs takes its J_i from here, and the passes over
// a compact linearisation (kernels: kCompactIntr) rebuild J_i from the stored (u, v) with P = I, which is what the TRIVIAL loss
// gives: every operation is rounded explicitly, so both produce the same bits.  The roundings are the ones nvcc chose for these
// columns when linearize_obs computed them inline (r2 = u u + v v from two rounded products, 2 u u + r2 rounded on its own in
// dk_9, the other sums fused), so J_i, and every solve, keeps the values it had before this helper existed.
template <uint32_t IMASK>
__host__ __device__ inline void obs_intr_cols(int model, double u, double v, const double* __restrict__ k, double P00, double P01,
                                              double P10, double P11, double* Ji) {
  constexpr int NI = popcount10(IMASK);
  if (NI == 0) return;
  const double f = k[0], ar = k[1], sk = k[2];
  const double r2 = add_rn(mul_rn(u, u), mul_rn(v, v));
  double ud, vd, dk[10][2];  // dk[j] = d(ud,vd)/dk_j, j >= 5
  if (model == kModelPinhole) {
    const double d = fma_rn(r2, fma_rn(k[6], r2, k[5]), 1.0);
    ud = mul_rn(u, d); vd = mul_rn(v, d);
    const double r4 = mul_rn(r2, r2);
    dk[5][0] = mul_rn(r2, u); dk[5][1] = mul_rn(r2, v);
    dk[6][0] = mul_rn(r4, u); dk[6][1] = mul_rn(r4, v);
    dk[7][0] = dk[7][1] = dk[8][0] = dk[8][1] = dk[9][0] = dk[9][1] = 0.0;
  } else {
    const double r4 = mul_rn(r2, r2), r6 = mul_rn(r4, r2);
    const double rd = fma_rn(mul_rn(k[7], r4), r2, fma_rn(k[6], r4, fma_rn(k[5], r2, 1.0)));
    const double t1 = k[8], t2 = k[9];
    const double uv2 = mul_rn(2.0 * u, v), eu = fma_rn(2.0 * u, u, r2), ev = fma_rn(2.0 * v, v, r2);
    ud = fma_rn(mul_rn(2.0 * t1, u), v, fma_rn(u, rd, mul_rn(t2, eu)));
    vd = fma_rn(mul_rn(2.0 * t2, u), v, fma_rn(v, rd, mul_rn(t1, ev)));
    dk[5][0] = mul_rn(r2, u); dk[5][1] = mul_rn(r2, v);
    dk[6][0] = mul_rn(r4, u); dk[6][1] = mul_rn(r4, v);
    dk[7][0] = mul_rn(r6, u); dk[7][1] = mul_rn(r6, v);
    dk[8][0] = uv2; dk[8][1] = ev;
    dk[9][0] = add_rn(r2, mul_rn(2.0 * u, u)); dk[9][1] = uv2;
  }
  const double far = mul_rn(f, ar);
  double col[10][2];
  col[0][0] = ud;  col[0][1] = mul_rn(ar, vd);  // d/df
  col[1][0] = 0.0; col[1][1] = mul_rn(f, vd);   // d/da
  col[2][0] = vd;  col[2][1] = 0.0;             // d/ds
  col[3][0] = 1.0; col[3][1] = 0.0;             // d/dcx
  col[4][0] = 0.0; col[4][1] = 1.0;             // d/dcy
  TBA_UNROLL
  for (int j = 5; j < 10; ++j) {                // distortion params: K2 * d(ud,vd)/dk_j
    col[j][0] = fma_rn(f, dk[j][0], mul_rn(sk, dk[j][1]));
    col[j][1] = mul_rn(far, dk[j][1]);
  }
  TBA_UNROLL
  for (int j = 0; j < NI; ++j) {
    constexpr uint32_t M = IMASK;
    const int idx = nth_bit(M, j);
    Ji[j] = fma_rn(P00, col[idx][0], mul_rn(P01, col[idx][1]));
    Ji[NI + j] = fma_rn(P10, col[idx][0], mul_rn(P11, col[idx][1]));
  }
}

// Residual + analytic Jacobian + robust-loss correction (ceres Corrector).
//   Ja[6] = rows of dpix/dX_{0..2}; Jw[6] = rows of dpix/dw; Jh[2]; Ji[2*NI] = row0 cols | row1 cols
// of the stored intrinsics columns (bits of IMASK).  r[2] is the robustified residual,
// rho0 the loss value (cost contribution 0.5 * rho0); uv (optional) receives the normalised image point (u, v).
template <uint32_t IMASK>
__host__ __device__ inline bool linearize_obs(int model, const double* __restrict__ C, const double* __restrict__ rec,
                                     const double* __restrict__ k, const double X0, const double X1, const double X2,
                                     const double h, const double x, const double y, int loss_type, double loss_width,
                                     double r[2], double& rho0, double Ja[6], double Jw[6], double Jh[2], double* Ji,
                                     double* uv = nullptr) {
  constexpr int NI = popcount10(IMASK);
  const double* R = rec;
  const double* L = rec + 9;
  const bool small = rec[18] != 0.0;
  const double a0 = X0 - h * C[0], a1 = X1 - h * C[1], a2 = X2 - h * C[2];
  if (a0 * a0 + a1 * a1 + a2 * a2 < 1e-8) return false;
  const double q0 = R[0] * a0 + R[1] * a1 + R[2] * a2;
  const double q1 = R[3] * a0 + R[4] * a1 + R[5] * a2;
  const double q2 = R[6] * a0 + R[7] * a1 + R[8] * a2;
  const double iz = 1.0 / q2;
  const double u = q0 * iz, v = q1 * iz;
  const double r2 = u * u + v * v;
  // distortion and its 2x2 derivative D' = d(ud,vd)/d(u,v)
  double ud, vd, D00, D01, D10, D11;
  if (model == kModelPinhole) {
    const double d = 1.0 + r2 * (k[5] + k[6] * r2);
    const double dd = 2.0 * k[5] + 4.0 * k[6] * r2;
    ud = u * d; vd = v * d;
    D00 = d + u * u * dd; D01 = u * v * dd; D10 = D01; D11 = d + v * v * dd;
  } else {
    const double r4 = r2 * r2;
    const double rd = 1.0 + k[5] * r2 + k[6] * r4 + k[7] * r4 * r2;
    const double rdp = k[5] + 2.0 * k[6] * r2 + 3.0 * k[7] * r4;  // d rd / d r2
    const double t1 = k[8], t2 = k[9];
    ud = u * rd + t2 * (r2 + 2.0 * u * u) + 2.0 * t1 * u * v;
    vd = v * rd + t1 * (r2 + 2.0 * v * v) + 2.0 * t2 * u * v;
    D00 = rd + 2.0 * u * u * rdp + 6.0 * t2 * u + 2.0 * t1 * v;
    D01 = 2.0 * u * v * rdp + 2.0 * t2 * v + 2.0 * t1 * u;
    D10 = 2.0 * u * v * rdp + 2.0 * t1 * u + 2.0 * t2 * v;
    D11 = rd + 2.0 * v * v * rdp + 6.0 * t1 * v + 2.0 * t2 * u;
  }
  const double f = k[0], ar = k[1], sk = k[2];
  const double rr0 = f * ud + sk * vd + k[3] - x;
  const double rr1 = f * ar * vd + k[4] - y;
  // robust loss (ResidualBlock::Evaluate + Corrector): P = sqrt(rho') (I - alpha r r^T / |r|^2)
  const double s = rr0 * rr0 + rr1 * rr1;
  double rho[3];
  loss_evaluate(loss_type, loss_width, s, rho);
  rho0 = rho[0];
  const double sq = sqrt(rho[1]);
  double P00 = sq, P01 = 0.0, P10 = 0.0, P11 = sq, rscale = sq;
  if (!(s == 0.0 || rho[2] <= 0.0)) {
    const double Dd = 1.0 + 2.0 * s * rho[2] / rho[1];
    const double alpha = 1.0 - sqrt(Dd);
    rscale = sq / (1.0 - alpha);
    const double an = alpha / s;
    P00 = sq * (1.0 - an * rr0 * rr0); P01 = -sq * an * rr0 * rr1; P10 = P01; P11 = sq * (1.0 - an * rr1 * rr1);
  }
  r[0] = rr0 * rscale; r[1] = rr1 * rscale;
  // A = P * K2 * D',  K2 = [[f, sk],[0, f*ar]]
  const double K00 = f * D00 + sk * D10, K01 = f * D01 + sk * D11;
  const double K10 = f * ar * D10, K11 = f * ar * D11;
  const double A00 = P00 * K00 + P01 * K10, A01 = P00 * K01 + P01 * K11;
  const double A10 = P10 * K00 + P11 * K10, A11 = P10 * K01 + P11 * K11;
  // J_q = A * (1/q_z) [[1,0,-u],[0,1,-v]]
  const double Jq00 = A00 * iz, Jq01 = A01 * iz, Jq02 = -(A00 * u + A01 * v) * iz;
  const double Jq10 = A10 * iz, Jq11 = A11 * iz, Jq12 = -(A10 * u + A11 * v) * iz;
  // J_a = J_q R
  Ja[0] = Jq00 * R[0] + Jq01 * R[3] + Jq02 * R[6];
  Ja[1] = Jq00 * R[1] + Jq01 * R[4] + Jq02 * R[7];
  Ja[2] = Jq00 * R[2] + Jq01 * R[5] + Jq02 * R[8];
  Ja[3] = Jq10 * R[0] + Jq11 * R[3] + Jq12 * R[6];
  Ja[4] = Jq10 * R[1] + Jq11 * R[4] + Jq12 * R[7];
  Ja[5] = Jq10 * R[2] + Jq11 * R[5] + Jq12 * R[8];
  Jh[0] = -(Ja[0] * C[0] + Ja[1] * C[1] + Ja[2] * C[2]);
  Jh[1] = -(Ja[3] * C[0] + Ja[4] * C[1] + Ja[5] * C[2]);
  // J_w = -(J_q x b) L,  b = q (Rodrigues branch) or a (first-order branch)
  const double b0 = small ? a0 : q0, b1 = small ? a1 : q1, b2 = small ? a2 : q2;
  const double c00 = Jq01 * b2 - Jq02 * b1, c01 = Jq02 * b0 - Jq00 * b2, c02 = Jq00 * b1 - Jq01 * b0;
  const double c10 = Jq11 * b2 - Jq12 * b1, c11 = Jq12 * b0 - Jq10 * b2, c12 = Jq10 * b1 - Jq11 * b0;
  Jw[0] = -(c00 * L[0] + c01 * L[3] + c02 * L[6]);
  Jw[1] = -(c00 * L[1] + c01 * L[4] + c02 * L[7]);
  Jw[2] = -(c00 * L[2] + c01 * L[5] + c02 * L[8]);
  Jw[3] = -(c10 * L[0] + c11 * L[3] + c12 * L[6]);
  Jw[4] = -(c10 * L[1] + c11 * L[4] + c12 * L[7]);
  Jw[5] = -(c10 * L[2] + c11 * L[5] + c12 * L[8]);
  obs_intr_cols<IMASK>(model, u, v, k, P00, P01, P10, P11, Ji);
  if (uv) { uv[0] = u; uv[1] = v; }
  return true;
}

// ------------------------------------------------------------------ the three other camera models (EXT instantiations)
__host__ __device__ inline void project_pixel_ext(int model, const double* __restrict__ C, const double* __restrict__ R,
                                                  const double* __restrict__ k, const double X0, const double X1, const double X2, const double h,
                                                  double& px, double& py, double& qz, double& a_sq) {
  const double a0 = X0 - h * C[0], a1 = X1 - h * C[1], a2 = X2 - h * C[2];
  a_sq = a0 * a0 + a1 * a1 + a2 * a2;
  double q[3], pix[2];
  q[0] = R[0] * a0 + R[1] * a1 + R[2] * a2;
  q[1] = R[3] * a0 + R[4] * a1 + R[5] * a2;
  q[2] = R[6] * a0 + R[7] * a1 + R[8] * a2;
  qz = q[2];
  camera_to_pixel_ext<double>(model, k, q, pix);
  px = pix[0]; py = pix[1];
}

// linearize_obs for FISHEYE / FOV / DIVISION_UNDISTORTION: d pixel / d (q, k) by forward-mode duals, then the same
// robustification and the same chain J_a = J_q R, J_h = -J_a C, J_w = -(J_q x b) L as above.
template <uint32_t IMASK>
__host__ __device__ inline bool linearize_obs_ext(int model, const double* __restrict__ C, const double* __restrict__ rec,
                                                  const double* __restrict__ k, const double X0, const double X1, const double X2,
                                                  const double h, const double x, const double y, int loss_type, double loss_width,
                                                  double r[2], double& rho0, double Ja[6], double Jw[6], double Jh[2], double* Ji) {
  constexpr int NI = popcount10(IMASK);
  const double* R = rec;
  const double* L = rec + 9;
  const bool small = rec[18] != 0.0;
  const double a0 = X0 - h * C[0], a1 = X1 - h * C[1], a2 = X2 - h * C[2];
  if (a0 * a0 + a1 * a1 + a2 * a2 < 1e-8) return false;
  const double q0 = R[0] * a0 + R[1] * a1 + R[2] * a2;
  const double q1 = R[3] * a0 + R[4] * a1 + R[5] * a2;
  const double q2 = R[6] * a0 + R[7] * a1 + R[8] * a2;
  typedef Dual<13> D;  // partials: 0..2 = q, 3..12 = intrinsics
  D qd[3], kd[10], pix[2];
  const double qv[3] = {q0, q1, q2};
  for (int i = 0; i < 3; ++i) { qd[i].v = qv[i]; for (int j = 0; j < 13; ++j) qd[i].d[j] = 0.0; qd[i].d[i] = 1.0; }
  const int K = model_num_parameters(model);
  for (int i = 0; i < 10; ++i) { kd[i].v = i < K ? k[i] : 0.0; for (int j = 0; j < 13; ++j) kd[i].d[j] = 0.0; if (i < K) kd[i].d[3 + i] = 1.0; }
  camera_to_pixel_ext<D>(model, kd, qd, pix);
  const double rr0 = pix[0].v - x, rr1 = pix[1].v - y;
  const double s = rr0 * rr0 + rr1 * rr1;
  double rho[3];
  loss_evaluate(loss_type, loss_width, s, rho);
  rho0 = rho[0];
  const double sq = sqrt(rho[1]);
  double P00 = sq, P01 = 0.0, P10 = 0.0, P11 = sq, rscale = sq;
  if (!(s == 0.0 || rho[2] <= 0.0)) {
    const double Dd = 1.0 + 2.0 * s * rho[2] / rho[1];
    const double alpha = 1.0 - sqrt(Dd);
    rscale = sq / (1.0 - alpha);
    const double an = alpha / s;
    P00 = sq * (1.0 - an * rr0 * rr0); P01 = -sq * an * rr0 * rr1; P10 = P01; P11 = sq * (1.0 - an * rr1 * rr1);
  }
  r[0] = rr0 * rscale; r[1] = rr1 * rscale;
  const double Jq00 = P00 * pix[0].d[0] + P01 * pix[1].d[0], Jq01 = P00 * pix[0].d[1] + P01 * pix[1].d[1], Jq02 = P00 * pix[0].d[2] + P01 * pix[1].d[2];
  const double Jq10 = P10 * pix[0].d[0] + P11 * pix[1].d[0], Jq11 = P10 * pix[0].d[1] + P11 * pix[1].d[1], Jq12 = P10 * pix[0].d[2] + P11 * pix[1].d[2];
  Ja[0] = Jq00 * R[0] + Jq01 * R[3] + Jq02 * R[6];
  Ja[1] = Jq00 * R[1] + Jq01 * R[4] + Jq02 * R[7];
  Ja[2] = Jq00 * R[2] + Jq01 * R[5] + Jq02 * R[8];
  Ja[3] = Jq10 * R[0] + Jq11 * R[3] + Jq12 * R[6];
  Ja[4] = Jq10 * R[1] + Jq11 * R[4] + Jq12 * R[7];
  Ja[5] = Jq10 * R[2] + Jq11 * R[5] + Jq12 * R[8];
  Jh[0] = -(Ja[0] * C[0] + Ja[1] * C[1] + Ja[2] * C[2]);
  Jh[1] = -(Ja[3] * C[0] + Ja[4] * C[1] + Ja[5] * C[2]);
  const double b0 = small ? a0 : q0, b1 = small ? a1 : q1, b2 = small ? a2 : q2;
  const double c00 = Jq01 * b2 - Jq02 * b1, c01 = Jq02 * b0 - Jq00 * b2, c02 = Jq00 * b1 - Jq01 * b0;
  const double c10 = Jq11 * b2 - Jq12 * b1, c11 = Jq12 * b0 - Jq10 * b2, c12 = Jq10 * b1 - Jq11 * b0;
  Jw[0] = -(c00 * L[0] + c01 * L[3] + c02 * L[6]);
  Jw[1] = -(c00 * L[1] + c01 * L[4] + c02 * L[7]);
  Jw[2] = -(c00 * L[2] + c01 * L[5] + c02 * L[8]);
  Jw[3] = -(c10 * L[0] + c11 * L[3] + c12 * L[6]);
  Jw[4] = -(c10 * L[1] + c11 * L[4] + c12 * L[7]);
  Jw[5] = -(c10 * L[2] + c11 * L[5] + c12 * L[8]);
  if (NI > 0) {
    TBA_UNROLL
    for (int j = 0; j < NI; ++j) {
      constexpr uint32_t M = IMASK;
      const int idx = nth_bit(M, j);
      Ji[j] = P00 * pix[0].d[3 + idx] + P01 * pix[1].d[3 + idx];
      Ji[NI + j] = P10 * pix[0].d[3 + idx] + P11 * pix[1].d[3 + idx];
    }
  }
  return true;
}

// Model dispatch: EXT = false is the PINHOLE / PINHOLE_RADIAL_TANGENTIAL code above and nothing else.
template <bool EXT>
__host__ __device__ inline void project_pixel_any(int model, const double* __restrict__ C, const double* __restrict__ R,
                                                  const double* __restrict__ k, const double X0, const double X1, const double X2, const double h,
                                                  double& px, double& py, double& qz, double& a_sq) {
  if (EXT) {
    if (model >= kModelFisheye) { project_pixel_ext(model, C, R, k, X0, X1, X2, h, px, py, qz, a_sq); return; }
  }
  project_pixel(model, C, R, k, X0, X1, X2, h, px, py, qz, a_sq);
}
template <bool EXT>
__host__ __device__ inline bool reproject_any(int model, const double* __restrict__ C, const double* __restrict__ R,
                                              const double* __restrict__ k, const double X0, const double X1, const double X2,
                                              const double h, const double x, const double y, double& r0, double& r1) {
  if (EXT) {
    if (model >= kModelFisheye) {
      double px, py, qz, a_sq;
      project_pixel_ext(model, C, R, k, X0, X1, X2, h, px, py, qz, a_sq);
      if (a_sq < 1e-8) return false;
      r0 = px - x; r1 = py - y;
      return true;
    }
  }
  return reproject(model, C, R, k, X0, X1, X2, h, x, y, r0, r1);
}
template <uint32_t IMASK, bool EXT>
__host__ __device__ inline bool linearize_obs_any(int model, const double* __restrict__ C, const double* __restrict__ rec,
                                                  const double* __restrict__ k, const double X0, const double X1, const double X2,
                                                  const double h, const double x, const double y, int loss_type, double loss_width,
                                                  double r[2], double& rho0, double Ja[6], double Jw[6], double Jh[2], double* Ji,
                                                  double* uv = nullptr) {
  if (EXT) {
    if (model >= kModelFisheye) return linearize_obs_ext<IMASK>(model, C, rec, k, X0, X1, X2, h, x, y, loss_type, loss_width, r, rho0, Ja, Jw, Jh, Ji);
  }
  return linearize_obs<IMASK>(model, C, rec, k, X0, X1, X2, h, x, y, loss_type, loss_width, r, rho0, Ja, Jw, Jh, Ji, uv);
}

}  // namespace tba
