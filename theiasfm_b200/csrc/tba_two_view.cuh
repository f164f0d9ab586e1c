// tba_two_view.cuh -- BundleAdjustTwoViews (src/theia/sfm/bundle_adjustment/bundle_adjust_two_views.cc:112-191) as a
// self-contained per-pair Levenberg-Marquardt: camera 1 fixed; camera 2's six extrinsics free; each camera's focal length
// free or its whole intrinsics block constant (.cc:71-108); every triangulated point (4-vector) free; two residual blocks per
// point; no robust loss; DENSE_SCHUR; 200 iterations; Ceres' default tolerances (.cc:54-69).
// Host/device: k_two_view_ba runs one instance per WARP (WarpTeam below) -- geometric verification issues one such problem per image pair
// (two_view_match_geometric_verification.cc:268-296), thousands of independent problems of a few hundred points -- and the
// CPU test suite runs the same body against the oracle (tests/host_two_view.cc, tests/test_two_view.py).
//
// Solver semantics = DESIGN.md section 3 with the exact (factorising) linear solver, specialised to this structure: the
// camera-side unknowns are c = [ext2 (6), f1, f2]; per point the 4x4 block C_p = E_p^T E_p + D_p^2 is eliminated, the 8x8
// reduced system S = sum_p (F_p^T F_p - F_p^T E_p C_p^-1 E_p^T F_p) + D_c^2 is solved by Cholesky, points are back-substituted.
// Nothing per point is stored between passes except its Jacobi scale and its candidate value (two scratch 4-vectors): each LM
// iteration makes three passes over the pair's points (assemble, back-substitute + model cost, candidate cost) and a fourth
// one (gradient, column norms) when the step is accepted.
#pragma once
#include <cfloat>
#include <cstdint>

#include "tba_point_lm.cuh"

namespace tba {

struct TwoViewPair {
  const double* ext1;   // [6] constant
  double* ext2;         // [6] in/out
  double* k1;           // [10] in/out (only the focal length can change)
  double* k2;           // [10]
  int model1, model2;
  int free_f1, free_f2; // !constant_cameraN_intrinsics
  int n;                // correspondences
  double* pt;           // [n][4] in/out
  const double* xy1;    // [n][2]
  const double* xy2;    // [n][2]
  double* sp;           // scratch [n][4]: Jacobi scales of the point columns
  double* pt_c;         // scratch [n][4]: candidate points
};

constexpr int kTvC = 8;  // camera-side unknowns: ext2 (6), f1, f2

// A "team" of lanes shares one pair: the loops over the pair's points are strided over the lanes and every sum / flag is
// all-reduced, so that all lanes hold identical scalars and take identical decisions.  SerialTeam (1 lane) is what the host
// tests run and what a thread-per-pair kernel would use; WarpTeam spreads a pair over the 32 lanes of a warp
// (k_two_view_ba: one warp per image pair -- a few hundred correspondences give each lane a handful of points per pass).
struct SerialTeam {
  __host__ __device__ static int rank() { return 0; }
  __host__ __device__ static int size() { return 1; }
  __host__ __device__ static double sum(double v) { return v; }
  __host__ __device__ static double max(double v) { return v; }
  __host__ __device__ static bool all(bool v) { return v; }
  __host__ __device__ static void sync() {}
};
struct WarpTeam {
  __host__ __device__ static int rank() {
#if defined(__CUDA_ARCH__) || defined(TBA_EMULATE)
    return threadIdx.x & 31;
#else
    return 0;
#endif
  }
  __host__ __device__ static int size() {
#if defined(__CUDA_ARCH__) || defined(TBA_EMULATE)
    return 32;
#else
    return 1;
#endif
  }
  __host__ __device__ static double sum(double v) {
#if defined(__CUDA_ARCH__) || defined(TBA_EMULATE)
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);  // butterfly: every lane ends with the same bits
#endif
    return v;
  }
  __host__ __device__ static double max(double v) {
#if defined(__CUDA_ARCH__) || defined(TBA_EMULATE)
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
#endif
    return v;
  }
  __host__ __device__ static bool all(bool v) {
#if defined(__CUDA_ARCH__) || defined(TBA_EMULATE)
    return __all_sync(0xffffffffu, v) != 0;
#else
    return v;
#endif
  }
};

// 8x8 SPD solve S x = b by Cholesky (S row-major, destroyed).
__host__ __device__ inline bool spd8_solve(double* S, const double* b, double* x) {
  for (int i = 0; i < kTvC; ++i)
    for (int j = 0; j <= i; ++j) {
      double acc = S[i * kTvC + j];
      for (int k = 0; k < j; ++k) acc -= S[i * kTvC + k] * S[j * kTvC + k];
      if (i == j) { if (!(acc > 0.0)) return false; S[i * kTvC + i] = sqrt(acc); }
      else S[i * kTvC + j] = acc / S[j * kTvC + j];
    }
  for (int i = 0; i < kTvC; ++i) { double acc = b[i]; for (int k = 0; k < i; ++k) acc -= S[i * kTvC + k] * x[k]; x[i] = acc / S[i * kTvC + i]; }
  for (int i = kTvC - 1; i >= 0; --i) { double acc = x[i]; for (int k = i + 1; k < kTvC; ++k) acc -= S[k * kTvC + i] * x[k]; x[i] = acc / S[i * kTvC + i]; }
  return true;
}

// 4x4 SPD inverse (full symmetric storage) through the Cholesky solve of tba_point_lm.cuh.
__host__ __device__ inline bool spd4_inverse_full(const double A[10], double Cinv[16]) {
  for (int c = 0; c < 4; ++c) {
    double e[4] = {0, 0, 0, 0}, y[4];
    e[c] = 1.0;
    if (!spd4_solve(A, e, y)) return false;
    for (int r = 0; r < 4; ++r) Cinv[r * 4 + c] = y[r];
  }
  return true;
}

// Residuals r[4] and masked, UNSCALED Jacobian rows of one correspondence: Jc[4][8] (camera side), Jp[4][4] (point).
// rows 0,1: the observation in camera 1; rows 2,3: in camera 2.
template <bool EXT>
__host__ __device__ inline bool tv_linearize(const TwoViewPair& P, const double* rec1, const double* ext2, const double* rec2, const double* k1,
                                             const double* k2, const double* X, const double* f1xy, const double* f2xy, int loss_type,
                                             double loss_width, double r[4], double Jc[4][kTvC], double Jp[4][4], double* rho_sum) {
  double Ja[6], Jw[6], Jh[2], Ji[2], rr[2], rho0;
  for (int a = 0; a < 4; ++a) for (int b = 0; b < kTvC; ++b) Jc[a][b] = 0.0;
  if (!linearize_obs_any<0x001u, EXT>(P.model1, P.ext1, rec1, k1, X[0], X[1], X[2], X[3], f1xy[0], f1xy[1], loss_type, loss_width, rr, rho0, Ja, Jw,
                                      Jh, Ji))
    return false;
  *rho_sum = rho0;
  r[0] = rr[0]; r[1] = rr[1];
  for (int row = 0; row < 2; ++row) {
    for (int j = 0; j < 3; ++j) Jp[row][j] = Ja[row * 3 + j];
    Jp[row][3] = Jh[row];
    if (P.free_f1) Jc[row][6] = Ji[row];
  }
  if (!linearize_obs_any<0x001u, EXT>(P.model2, ext2, rec2, k2, X[0], X[1], X[2], X[3], f2xy[0], f2xy[1], loss_type, loss_width, rr, rho0, Ja, Jw, Jh,
                                      Ji))
    return false;
  *rho_sum += rho0;
  r[2] = rr[0]; r[3] = rr[1];
  for (int row = 0; row < 2; ++row) {
    for (int j = 0; j < 3; ++j) { Jp[2 + row][j] = Ja[row * 3 + j]; Jc[2 + row][j] = -X[3] * Ja[row * 3 + j]; Jc[2 + row][3 + j] = Jw[row * 3 + j]; }
    Jp[2 + row][3] = Jh[row];
    if (P.free_f2) Jc[2 + row][7] = Ji[row];
  }
  return true;
}

// Cost, gradient (camera side g_c, max |g| over everything), squared column norms of the camera columns; optionally the
// Jacobi scales (iteration 0).  sc: current camera-side scales (all 1 when init_scale).
template <bool EXT, class Team>
__host__ __device__ inline bool tv_evaluate(const TwoViewPair& P, const double* rec1, const double* rec2, const PointLmOptions& o, bool init_scale,
                                            const double* ext2v, const double* k1v, const double* k2v, double* sc, double* cost, double* gmax,
                                            double* diag_c /*[8] scaled col norms^2*/) {
  double c = 0.0, gm = 0.0, gc[kTvC], cn[kTvC];
  bool ok = true;
  for (int j = 0; j < kTvC; ++j) { gc[j] = 0.0; cn[j] = 0.0; }
  for (int i = Team::rank(); i < P.n; i += Team::size()) {
    double r[4], Jc[4][kTvC], Jp[4][4], rho;
    if (!tv_linearize<EXT>(P, rec1, ext2v, rec2, k1v, k2v, P.pt + (size_t)i * 4, P.xy1 + (size_t)i * 2, P.xy2 + (size_t)i * 2, o.loss_type,
                           o.loss_width, r, Jc, Jp, &rho)) { ok = false; break; }
    c += 0.5 * rho;
    for (int j = 0; j < kTvC; ++j) { double g = 0.0, n2 = 0.0; for (int a = 0; a < 4; ++a) { g += Jc[a][j] * r[a]; n2 += Jc[a][j] * Jc[a][j]; } gc[j] += g; cn[j] += n2; }
    for (int j = 0; j < 4; ++j) {
      double g = 0.0, n2 = 0.0;
      for (int a = 0; a < 4; ++a) { g += Jp[a][j] * r[a]; n2 += Jp[a][j] * Jp[a][j]; }
      gm = fmax(gm, fabs(g));
      if (init_scale) P.sp[(size_t)i * 4 + j] = o.jacobi_scaling ? 1.0 / (1.0 + sqrt(n2)) : 1.0;
    }
  }
  if (!Team::all(ok)) return false;
  c = Team::sum(c); gm = Team::max(gm);
  for (int j = 0; j < kTvC; ++j) { gc[j] = Team::sum(gc[j]); cn[j] = Team::sum(cn[j]); }
  for (int j = 0; j < kTvC; ++j) gm = fmax(gm, fabs(gc[j]));
  if (init_scale) for (int j = 0; j < kTvC; ++j) sc[j] = o.jacobi_scaling ? 1.0 / (1.0 + sqrt(cn[j])) : 1.0;
  for (int j = 0; j < kTvC; ++j) diag_c[j] = cn[j] * sc[j] * sc[j];
  *cost = c; *gmax = gm;
  return true;
}

template <bool EXT, class Team = SerialTeam>
__host__ __device__ inline PointLmResult two_view_lm(const TwoViewPair& P, const PointLmOptions& o) {
  PointLmResult res;
  res.initial_cost = res.final_cost = -1.0; res.iterations = 0; res.termination = 2;
  double rec1[kCamRec], rec2[kCamRec], rec2c[kCamRec];
  // every lane keeps its own copy of the camera-side values (identical in all lanes); lane 0 writes them back at the end
  double ext2v[6], k1v[10], k2v[10];
  for (int j = 0; j < 6; ++j) ext2v[j] = P.ext2[j];
  for (int j = 0; j < 10; ++j) { k1v[j] = P.k1[j]; k2v[j] = P.k2[j]; }
  cam_prep(P.ext1 + 3, rec1);
  cam_prep(ext2v + 3, rec2);
  const bool fr[kTvC] = {true, true, true, true, true, true, P.free_f1 != 0, P.free_f2 != 0};
  double sc[kTvC], diag_c[kTvC], cost, gmax;
  for (int j = 0; j < kTvC; ++j) sc[j] = 1.0;
  if (!tv_evaluate<EXT, Team>(P, rec1, rec2, o, true, ext2v, k1v, k2v, sc, &cost, &gmax, diag_c)) return res;
  res.initial_cost = res.final_cost = cost;
  const int K1 = model_num_parameters(P.model1), K2 = model_num_parameters(P.model2);
  // ||x|| over the non-constant parameter blocks in ambient coordinates (camera 2 extrinsics, an intrinsics block whose focal
  // length is free counts whole, every point)
  auto xnorm2_cam = [&](const double* e2, const double* k1, const double* k2) {
    double s = 0.0;
    for (int j = 0; j < 6; ++j) s += e2[j] * e2[j];
    if (P.free_f1) for (int j = 0; j < K1; ++j) s += k1[j] * k1[j];
    if (P.free_f2) for (int j = 0; j < K2; ++j) s += k2[j] * k2[j];
    return s;
  };
  auto xnorm2_pts = [&]() {
    double s = 0.0;
    for (int i = Team::rank(); i < P.n; i += Team::size()) for (int a = 0; a < 4; ++a) s += P.pt[(size_t)i * 4 + a] * P.pt[(size_t)i * 4 + a];
    return Team::sum(s);
  };
  double xn2 = xnorm2_cam(ext2v, k1v, k2v) + xnorm2_pts();
  double xnorm = sqrt(xn2);
  double radius = o.initial_radius, decrease = 2.0;
  int invalid = 0;
  bool last_successful = true;
  res.termination = 1;
  for (int it = 0;;) {
    if (it >= o.max_num_iterations) { res.termination = 1; break; }
    if (last_successful && gmax <= o.gradient_tolerance) { res.termination = 0; break; }
    if (radius <= o.min_radius) { res.termination = 0; break; }
    ++it;
    res.iterations = it;
    // ---- assemble the reduced system
    double Dc[kTvC];
    for (int j = 0; j < kTvC; ++j) Dc[j] = fr[j] ? sqrt(fmin(fmax(diag_c[j], o.min_diag), o.max_diag) / radius) : 0.0;
    double S[kTvC * kTvC], rhs[kTvC];
    for (int j = 0; j < kTvC * kTvC; ++j) S[j] = 0.0;
    for (int j = 0; j < kTvC; ++j) rhs[j] = 0.0;
    bool valid = true;
    for (int i = Team::rank(); i < P.n && valid; i += Team::size()) {
      double r[4], Jc[4][kTvC], Jp[4][4], rho;
      const double* spi = P.sp + (size_t)i * 4;
      if (!tv_linearize<EXT>(P, rec1, ext2v, rec2, k1v, k2v, P.pt + (size_t)i * 4, P.xy1 + (size_t)i * 2, P.xy2 + (size_t)i * 2, o.loss_type,
                             o.loss_width, r, Jc, Jp, &rho)) { valid = false; break; }
      for (int a = 0; a < 4; ++a) { for (int j = 0; j < kTvC; ++j) Jc[a][j] *= sc[j]; for (int j = 0; j < 4; ++j) Jp[a][j] *= spi[j]; }
      double A[10], Cinv[16];
      int n = 0;
      for (int a = 0; a < 4; ++a) for (int b = a; b < 4; ++b) { double s = 0.0; for (int t = 0; t < 4; ++t) s += Jp[t][a] * Jp[t][b]; A[n++] = s; }
      const int dg[4] = {0, 4, 7, 9};
      for (int a = 0; a < 4; ++a) A[dg[a]] += fmin(fmax(A[dg[a]], o.min_diag), o.max_diag) / radius;  // D_p^2
      if (!spd4_inverse_full(A, Cinv)) { valid = false; break; }
      double etb[4], y2[4], W[4][kTvC];
      for (int a = 0; a < 4; ++a) { double s = 0.0; for (int t = 0; t < 4; ++t) s += Jp[t][a] * r[t]; etb[a] = s; }
      for (int a = 0; a < 4; ++a) { double s = 0.0; for (int b = 0; b < 4; ++b) s += Cinv[a * 4 + b] * etb[b]; y2[a] = s; }
      for (int t = 0; t < 4; ++t) {
        double y3 = r[t];
        for (int a = 0; a < 4; ++a) y3 -= Jp[t][a] * y2[a];
        for (int j = 0; j < kTvC; ++j) rhs[j] += Jc[t][j] * y3;
      }
      for (int a = 0; a < 4; ++a) for (int j = 0; j < kTvC; ++j) { double s = 0.0; for (int t = 0; t < 4; ++t) s += Jp[t][a] * Jc[t][j]; W[a][j] = s; }
      for (int j = 0; j < kTvC; ++j) {
        double cw[4];
        for (int a = 0; a < 4; ++a) { double s = 0.0; for (int b = 0; b < 4; ++b) s += Cinv[a * 4 + b] * W[b][j]; cw[a] = s; }
        for (int l = 0; l < kTvC; ++l) {
          double s = 0.0;
          for (int t = 0; t < 4; ++t) s += Jc[t][l] * Jc[t][j];
          for (int a = 0; a < 4; ++a) s -= W[a][l] * cw[a];
          S[l * kTvC + j] += s;
        }
      }
    }
    double x[kTvC];
    valid = Team::all(valid);
    if (valid) {
      for (int j = 0; j < kTvC * kTvC; ++j) S[j] = Team::sum(S[j]);
      for (int j = 0; j < kTvC; ++j) rhs[j] = Team::sum(rhs[j]);
      for (int j = 0; j < kTvC; ++j) {
        if (fr[j]) S[j * kTvC + j] += Dc[j] * Dc[j];
        else { for (int l = 0; l < kTvC; ++l) { S[j * kTvC + l] = 0.0; S[l * kTvC + j] = 0.0; } S[j * kTvC + j] = 1.0; rhs[j] = 0.0; }
      }
      valid = spd8_solve(S, rhs, x);
    }
    // ---- back-substitution, model cost change, candidate parameters
    double mcc = 0.0, dn2 = 0.0;
    double e2c[6], k1c[10], k2c[10];
    if (valid) {
      for (int j = 0; j < 6; ++j) { const double d = -x[j] * sc[j]; e2c[j] = ext2v[j] + d; dn2 += d * d; if (!isfinite(d)) valid = false; }
      for (int j = 0; j < 10; ++j) { k1c[j] = k1v[j]; k2c[j] = k2v[j]; }
      if (P.free_f1) { const double d = -x[6] * sc[6]; k1c[0] += d; dn2 += d * d; if (!isfinite(d)) valid = false; }
      if (P.free_f2) { const double d = -x[7] * sc[7]; k2c[0] += d; dn2 += d * d; if (!isfinite(d)) valid = false; }
    }
    double dn2_pts = 0.0;
    for (int i = Team::rank(); i < P.n && valid; i += Team::size()) {
      double r[4], Jc[4][kTvC], Jp[4][4], rho;
      const double* spi = P.sp + (size_t)i * 4;
      const double* X = P.pt + (size_t)i * 4;
      if (!tv_linearize<EXT>(P, rec1, ext2v, rec2, k1v, k2v, X, P.xy1 + (size_t)i * 2, P.xy2 + (size_t)i * 2, o.loss_type, o.loss_width, r, Jc, Jp,
                             &rho)) { valid = false; break; }
      for (int a = 0; a < 4; ++a) { for (int j = 0; j < kTvC; ++j) Jc[a][j] *= sc[j]; for (int j = 0; j < 4; ++j) Jp[a][j] *= spi[j]; }
      double A[10], Cinv[16];
      int n = 0;
      for (int a = 0; a < 4; ++a) for (int b = a; b < 4; ++b) { double s = 0.0; for (int t = 0; t < 4; ++t) s += Jp[t][a] * Jp[t][b]; A[n++] = s; }
      const int dg[4] = {0, 4, 7, 9};
      for (int a = 0; a < 4; ++a) A[dg[a]] += fmin(fmax(A[dg[a]], o.min_diag), o.max_diag) / radius;
      if (!spd4_inverse_full(A, Cinv)) { valid = false; break; }
      double fx[4], t4[4], yp[4];
      for (int t = 0; t < 4; ++t) { double s = 0.0; for (int j = 0; j < kTvC; ++j) s += Jc[t][j] * x[j]; fx[t] = s; }
      for (int a = 0; a < 4; ++a) { double s = 0.0; for (int t = 0; t < 4; ++t) s += Jp[t][a] * (r[t] - fx[t]); t4[a] = s; }
      for (int a = 0; a < 4; ++a) { double s = 0.0; for (int b = 0; b < 4; ++b) s += Cinv[a * 4 + b] * t4[b]; yp[a] = s; }
      for (int t = 0; t < 4; ++t) {
        double m = -fx[t];
        for (int a = 0; a < 4; ++a) m -= Jp[t][a] * yp[a];
        mcc -= m * (r[t] + m / 2.0);
      }
      for (int a = 0; a < 4; ++a) {
        const double d = -yp[a] * spi[a];
        if (!isfinite(d)) valid = false;
        P.pt_c[(size_t)i * 4 + a] = X[a] + d;
        dn2_pts += d * d;
      }
    }
    valid = Team::all(valid);
    mcc = Team::sum(mcc);
    dn2 += Team::sum(dn2_pts);
    if (valid) valid = mcc > 0.0;
    if (!valid) {  // HandleInvalidStep
      if (++invalid >= o.max_consecutive_invalid) { res.termination = 2; break; }
      radius /= decrease; decrease *= 2.0;
      last_successful = false;
      continue;
    }
    invalid = 0;
    // ---- candidate cost
    cam_prep(e2c + 3, rec2c);
    double cand = 0.0;
    bool cand_ok = true;
    for (int i = Team::rank(); i < P.n; i += Team::size()) {
      const double* X = P.pt_c + (size_t)i * 4;
      double r0, r1, rho[3];
      if (!reproject_any<EXT>(P.model1, P.ext1, rec1, k1c, X[0], X[1], X[2], X[3], P.xy1[(size_t)i * 2], P.xy1[(size_t)i * 2 + 1], r0, r1)) { cand_ok = false; break; }
      loss_evaluate(o.loss_type, o.loss_width, r0 * r0 + r1 * r1, rho);
      cand += 0.5 * rho[0];
      if (!reproject_any<EXT>(P.model2, e2c, rec2c, k2c, X[0], X[1], X[2], X[3], P.xy2[(size_t)i * 2], P.xy2[(size_t)i * 2 + 1], r0, r1)) { cand_ok = false; break; }
      loss_evaluate(o.loss_type, o.loss_width, r0 * r0 + r1 * r1, rho);
      cand += 0.5 * rho[0];
    }
    cand_ok = Team::all(cand_ok);
    cand = Team::sum(cand);
    if (!cand_ok) cand = DBL_MAX;
    // step norm in ambient coordinates of the non-constant blocks = ||delta|| (constant coordinates do not move)
    if (sqrt(dn2) <= o.parameter_tolerance * (xnorm + o.parameter_tolerance)) { res.termination = 0; break; }
    const double cost_change = cost - cand;
    if (fabs(cost_change) <= o.function_tolerance * cost) { res.termination = 0; break; }
    const double rho_q = cost_change / mcc;
    if (rho_q > o.min_relative_decrease) {  // HandleSuccessfulStep
      for (int j = 0; j < 6; ++j) ext2v[j] = e2c[j];
      k1v[0] = k1c[0]; k2v[0] = k2c[0];
      for (int i = Team::rank(); i < P.n; i += Team::size()) for (int a = 0; a < 4; ++a) P.pt[(size_t)i * 4 + a] = P.pt_c[(size_t)i * 4 + a];
      for (int j = 0; j < kCamRec; ++j) rec2[j] = rec2c[j];
      xn2 = xnorm2_cam(ext2v, k1v, k2v) + xnorm2_pts();
      xnorm = sqrt(xn2);
      if (!tv_evaluate<EXT, Team>(P, rec1, rec2, o, false, ext2v, k1v, k2v, sc, &cost, &gmax, diag_c)) { res.termination = 2; break; }
      res.final_cost = cost;
      const double t = 2.0 * rho_q - 1.0;
      radius = fmin(o.max_radius, radius / fmax(1.0 / 3.0, 1.0 - t * t * t));
      decrease = 2.0;
      last_successful = true;
    } else {  // HandleUnsuccessfulStep
      radius /= decrease; decrease *= 2.0;
      last_successful = false;
    }
  }
  if (Team::rank() == 0) {
    for (int j = 0; j < 6; ++j) P.ext2[j] = ext2v[j];
    P.k1[0] = k1v[0]; P.k2[0] = k2v[0];
  }
  return res;
}

// AcceptableReprojectionError of two_view_match_geometric_verification.cc:72-83 for every correspondence of the pair, with the
// refined cameras and points (the post-BA filter of BundleAdjustRelativePose, :294-312).
template <bool EXT, class Team = SerialTeam>
__host__ __device__ inline void two_view_inliers(const TwoViewPair& P, double sq_max_error, uint8_t* inlier) {
  double rec1[kCamRec], rec2[kCamRec];
  cam_prep(P.ext1 + 3, rec1);
  cam_prep(P.ext2 + 3, rec2);
  for (int i = Team::rank(); i < P.n; i += Team::size()) {
    const double* X = P.pt + (size_t)i * 4;
    double px, py, qz, a_sq;
    bool ok = true;
    project_pixel_any<EXT>(P.model1, P.ext1, rec1, P.k1, X[0], X[1], X[2], X[3], px, py, qz, a_sq);
    const double dx1 = P.xy1[(size_t)i * 2] - px, dy1 = P.xy1[(size_t)i * 2 + 1] - py;
    if (qz / X[3] < 0.0 || !(dx1 * dx1 + dy1 * dy1 < sq_max_error)) ok = false;
    project_pixel_any<EXT>(P.model2, P.ext2, rec2, P.k2, X[0], X[1], X[2], X[3], px, py, qz, a_sq);
    const double dx2 = P.xy2[(size_t)i * 2] - px, dy2 = P.xy2[(size_t)i * 2 + 1] - py;
    if (qz / X[3] < 0.0 || !(dx2 * dx2 + dy2 * dy2 < sq_max_error)) ok = false;
    inlier[i] = ok ? 1 : 0;
  }
}

}  // namespace tba
