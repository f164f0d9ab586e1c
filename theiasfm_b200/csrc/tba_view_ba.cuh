// tba_view_ba.cuh -- BundleAdjustView (src/theia/sfm/bundle_adjustment/bundle_adjustment.cc:83-93) as a self-contained
// per-view Levenberg-Marquardt: one camera's extrinsics and its intrinsics group are the only parameter blocks, with the
// coordinates that SetCameraExtrinsicsParameterization / SetCameraIntrinsicsParameterization leave free (bundle_adjuster.cc:
// 102-139); every point the view observes is constant (SetTrackConstant); one reprojection residual per observation of the
// view; DENSE_QR, no inner iterations.
// Host/device: k_view_ba runs one instance per CTA (CtaTeam below): a localized view carries hundreds to thousands of
// observations, which the CTA's threads stride over.  The CPU test suite runs the same body with one lane and with a team of
// host threads against the oracle (tests/host_view_ba.cc, tests/test_view_ba.py).
//
// Solver semantics = DESIGN.md section 3 restricted to one dense block of at most 16 unknowns (the same rules as
// tba_point_lm.cuh, N <= 16 instead of 4).  The unknowns are kept in ambient coordinates u = [C (3) | w (3) | intrinsics (10)];
// a constant coordinate has a zero Jacobian column and an identity row in the damped system, as in tba_block_lm.h.  Each LM
// iteration makes one pass over the view's observations for J, r, the upper triangle of [J | r]^T [J | r] and the cost, and
// one pass for the candidate cost; a single lane solves the damped 16x16 system in fp64.  Every value the lanes share lives
// in a ViewWork (shared memory on the device), so a thread holds one observation's Jacobian rows and a few accumulators.
#pragma once
#include <cfloat>
#include <cstdint>

#include "tba_two_view.cuh"  // SerialTeam, PointLmOptions / PointLmResult, cam_prep, linearize_obs_any

namespace tba {

constexpr int kVbN = 16;                       // ambient unknowns: extrinsics 6 + intrinsics 10
constexpr int kVbW = kVbN + 1;                 // columns of [J | r]
constexpr int kVbG = kVbW * (kVbW + 1) / 2;    // upper triangle of [J | r]^T [J | r]

__host__ __device__ constexpr int vb_tri(int a, int b) { return a * kVbW - a * (a - 1) / 2 + (b - a); }  // a <= b

// One view of the uploaded problem.  Observation i is slot slot[i] of the packed layout (its point slot_pt[slot[i]], its
// feature at xy[slot / 32][0..1][slot % 32]).
struct ViewBaProblem {
  double* ext;            // [6] the camera's extrinsics, in/out
  double* intr;           // [10] its intrinsics group, in/out
  int model;
  uint32_t free_mask;     // bit j: ambient coordinate j is optimised (0..5 extrinsics, 6..15 intrinsics)
  int n;                  // observations
  const long long* slot;  // [n]
  const int* slot_pt;
  const double* pt;       // [packed point][4], constant
  const double* xy;
};

// Values every lane of a team reads: one instance per view (shared memory on the device).
struct ViewWork {
  double x[kVbN], xc[kVbN];            // current / candidate unknowns
  double rec[kCamRec], recc[kCamRec];  // rotation records of x / xc
  double sc[kVbN];                     // Jacobi scale (fixed at iteration 0)
  double G[kVbG];                      // [J | r]^T [J | r] at x, masked, unscaled: H | g | r.r
  double L[kVbN * kVbN];               // Cholesky factor of the damped system
  double b[kVbN], y[kVbN];
  double mcc, dn2;                     // model cost change, ||xc - x||^2
  int valid;
};

// Team-wide Gram accumulator of the observations' [J | r] rows.  Generic form: every lane accumulates the whole triangle over
// the observations it owns, the team sums it entry by entry at the end.  CtaTeam has its own (k_view_ba, below).
template <class Team>
struct ViewGram {
  double acc[kVbG];
  __host__ __device__ void reset() { for (int e = 0; e < kVbG; ++e) acc[e] = 0.0; }
  __host__ __device__ void add(const double rows[2][kVbW]) {
    int e = 0;
    for (int a = 0; a < kVbW; ++a)
      for (int c = a; c < kVbW; ++c) acc[e++] += rows[0][a] * rows[0][c] + rows[1][a] * rows[1][c];
  }
  __host__ __device__ void total(ViewWork& W) {
    for (int e = 0; e < kVbG; ++e) {
      const double s = Team::sum(acc[e]);
      if (Team::rank() == 0) W.G[e] = s;
    }
    Team::sync();
  }
};

__host__ __device__ inline bool vb_free(uint32_t m, int j) { return ((m >> j) & 1u) != 0; }

// One pass over the view's observations at (x, rec): the cost (sum of 0.5 rho(|r|^2)) and, with derivs, the Gram of the masked,
// robustified [J | r] rows into W.G.  Returns false when a residual functor fails (||X - hC||^2 < 1e-8, reprojection_error.h:75-77)
// in any lane.
template <bool EXT, class Team>
__host__ __device__ inline bool view_pass(const ViewBaProblem& V, ViewWork& W, const double* x, const double* rec, bool derivs, int loss_type,
                                          double loss_width, double* cost) {
  double c = 0.0;
  bool ok = true;
  ViewGram<Team> gram;
  if (derivs) gram.reset();
  const uint32_t fm = V.free_mask;
  for (int base = 0; base < V.n; base += Team::size()) {
    const int i = base + Team::rank();
    double rows[2][kVbW];
    if (derivs)
      for (int a = 0; a < 2; ++a) for (int j = 0; j < kVbW; ++j) rows[a][j] = 0.0;
    if (i < V.n) {
      const long long s = V.slot[i];
      const double* X = V.pt + (size_t)V.slot_pt[s] * 4;
      const long long wq = s >> 5;
      const int l = (int)(s & 31);
      const double ox = V.xy[(size_t)(wq * 2 + 0) * 32 + l], oy = V.xy[(size_t)(wq * 2 + 1) * 32 + l];
      if (derivs) {
        double r[2], rho0, Ja[6], Jw[6], Jh[2], Ji[20];
        if (linearize_obs_any<0x3FFu, EXT>(V.model, x, rec, x + 6, X[0], X[1], X[2], X[3], ox, oy, loss_type, loss_width, r, rho0, Ja, Jw, Jh, Ji)) {
          c += 0.5 * rho0;
          for (int a = 0; a < 2; ++a) {
            for (int j = 0; j < 3; ++j) {
              rows[a][j] = vb_free(fm, j) ? -X[3] * Ja[a * 3 + j] : 0.0;  // d/dC = -h J_a
              rows[a][3 + j] = vb_free(fm, 3 + j) ? Jw[a * 3 + j] : 0.0;
            }
            for (int j = 0; j < 10; ++j) rows[a][6 + j] = vb_free(fm, 6 + j) ? Ji[a * 10 + j] : 0.0;
            rows[a][kVbN] = r[a];
          }
        } else {
          ok = false;
        }
      } else {
        double r0, r1, rho[3];
        if (reproject_any<EXT>(V.model, x, rec, x + 6, X[0], X[1], X[2], X[3], ox, oy, r0, r1)) {
          loss_evaluate(loss_type, loss_width, r0 * r0 + r1 * r1, rho);
          c += 0.5 * rho[0];
        } else {
          ok = false;
        }
      }
    }
    if (derivs) gram.add(rows);
  }
  ok = Team::all(ok);
  *cost = Team::sum(c);
  if (derivs) gram.total(W);
  return ok;
}

// ||u|| over the non-constant parameter blocks (ambient coordinates): the extrinsics when any of them is free, the group's K
// intrinsics when any of them is free.  With y: ||u - y|| over the same blocks.
__host__ __device__ inline double view_xnorm2(const double* u, const double* y, uint32_t fm, int K) {
  double s = 0.0;
  if (fm & 0x3Fu)
    for (int j = 0; j < 6; ++j) { const double d = u[j] - (y ? y[j] : 0.0); s += d * d; }
  if (fm & 0xFFC0u)
    for (int j = 0; j < K; ++j) { const double d = u[6 + j] - (y ? y[6 + j] : 0.0); s += d * d; }
  return s;
}

// The damped, Jacobi-scaled normal equations at (W.G, radius), solved by one lane: W.xc = x + delta on the free coordinates,
// W.mcc, W.dn2 and W.valid (a usable step with a positive model cost change); then the team reads them.
template <class Team>
__host__ __device__ inline void view_step(ViewWork& W, uint32_t fm, int K, double radius, const PointLmOptions& o) {
  Team::sync();  // every lane has read the previous step's W.valid / W.mcc / W.dn2
  if (Team::rank() == 0) {
    double* L = W.L;
    for (int a = 0; a < kVbN; ++a)
      for (int c = 0; c <= a; ++c) {
        const bool f = vb_free(fm, a) && vb_free(fm, c);
        L[a * kVbN + c] = f ? W.sc[c] * W.G[vb_tri(c, a)] * W.sc[a] : (a == c ? 1.0 : 0.0);
      }
    for (int a = 0; a < kVbN; ++a) {
      if (vb_free(fm, a)) { W.b[a] = W.sc[a] * W.G[vb_tri(a, kVbN)]; L[a * kVbN + a] += fmin(fmax(L[a * kVbN + a], o.min_diag), o.max_diag) / radius; }
      else W.b[a] = 0.0;
    }
    bool ok = true;
    for (int i = 0; i < kVbN && ok; ++i)
      for (int j = 0; j <= i; ++j) {
        double acc = L[i * kVbN + j];
        for (int k = 0; k < j; ++k) acc -= L[i * kVbN + k] * L[j * kVbN + k];
        if (i == j) { if (!(acc > 0.0)) { ok = false; break; } L[i * kVbN + i] = sqrt(acc); }
        else L[i * kVbN + j] = acc / L[j * kVbN + j];
      }
    double mcc = 0.0;
    if (ok) {
      double* y = W.y;
      for (int i = 0; i < kVbN; ++i) { double acc = W.b[i]; for (int k = 0; k < i; ++k) acc -= L[i * kVbN + k] * y[k]; y[i] = acc / L[i * kVbN + i]; }
      for (int i = kVbN - 1; i >= 0; --i) { double acc = y[i]; for (int k = i + 1; k < kVbN; ++k) acc -= L[k * kVbN + i] * y[k]; y[i] = acc / L[i * kVbN + i]; }
      // model_cost_change = -(J s).(r + J s / 2) = -(s.b + s^T H~ s / 2),  s = -y (scaled step)
      double sg = 0.0, shs = 0.0;
      for (int a = 0; a < kVbN; ++a) {
        if (!vb_free(fm, a)) { W.xc[a] = W.x[a]; continue; }
        const double sa = -y[a];
        sg += sa * W.b[a];
        for (int c = 0; c < kVbN; ++c)
          if (vb_free(fm, c)) shs += sa * (W.sc[a] * W.G[a <= c ? vb_tri(a, c) : vb_tri(c, a)] * W.sc[c]) * (-y[c]);
        const double d = sa * W.sc[a];
        if (!isfinite(d)) ok = false;
        W.xc[a] = W.x[a] + d;
      }
      mcc = -(sg + 0.5 * shs);
      ok = ok && mcc > 0.0;
    }
    W.mcc = mcc;
    W.valid = ok ? 1 : 0;
    if (ok) {
      W.dn2 = view_xnorm2(W.x, W.xc, fm, K);
      cam_prep(W.xc + 3, W.recc);
    }
  }
  Team::sync();
}

// Minimise over the view's free coordinates.  Mirrors TrustRegionMinimizer::Minimize for one dense block.  iterations: the
// LM iterations Ceres' summary lists (an iteration that ends the solve inside its step -- a tolerance reached, too many invalid
// steps, a failed evaluation -- is not listed).  A view without free coordinates or without observations converges at
// iteration 0 with its cost (Ceres' fixed cost) as initial and final cost.
template <bool EXT, class Team = SerialTeam>
__host__ __device__ inline PointLmResult view_lm(const ViewBaProblem& V, ViewWork& W, const PointLmOptions& o) {
  PointLmResult res;
  res.initial_cost = res.final_cost = -1.0; res.iterations = 0; res.termination = 2;
  const uint32_t fm = V.free_mask;
  const int K = model_num_parameters(V.model);
  if (Team::rank() == 0) {
    for (int j = 0; j < 6; ++j) W.x[j] = V.ext[j];
    for (int j = 0; j < 10; ++j) W.x[6 + j] = V.intr[j];
    cam_prep(W.x + 3, W.rec);
  }
  Team::sync();
  double cost;
  if (!view_pass<EXT, Team>(V, W, W.x, W.rec, true, o.loss_type, o.loss_width, &cost)) return res;  // "Residual and Jacobian evaluation failed."
  res.initial_cost = res.final_cost = cost;
  auto gmax_of = [&]() {
    double m = 0.0;
    for (int j = 0; j < kVbN; ++j) m = fmax(m, fabs(W.G[vb_tri(j, kVbN)]));
    return m;
  };
  if (Team::rank() == 0)
    for (int j = 0; j < kVbN; ++j) W.sc[j] = o.jacobi_scaling ? 1.0 / (1.0 + sqrt(W.G[vb_tri(j, j)])) : 1.0;
  double gmax = gmax_of();
  double xnorm = sqrt(view_xnorm2(W.x, nullptr, fm, K));
  double radius = o.initial_radius, decrease = 2.0;
  int invalid = 0;
  bool last_successful = true;
  for (int it = 0;;) {
    // FinalizeIterationAndCheckIfMinimizerCanContinue: iteration `it` is listed
    res.iterations = it;
    if (it >= o.max_num_iterations) { res.termination = 1; break; }
    if (last_successful && gmax <= o.gradient_tolerance) { res.termination = 0; break; }
    if (radius <= o.min_radius) { res.termination = 0; break; }
    ++it;
    view_step<Team>(W, fm, K, radius, o);
    if (!W.valid) {  // HandleInvalidStep
      if (++invalid >= o.max_consecutive_invalid) { res.termination = 2; break; }
      radius /= decrease; decrease *= 2.0;
      last_successful = false;
      continue;
    }
    invalid = 0;
    double cand;
    if (!view_pass<EXT, Team>(V, W, W.xc, W.recc, false, o.loss_type, o.loss_width, &cand)) cand = DBL_MAX;
    const double mcc = W.mcc;
    if (sqrt(W.dn2) <= o.parameter_tolerance * (xnorm + o.parameter_tolerance)) { res.termination = 0; break; }
    const double cost_change = cost - cand;
    if (fabs(cost_change) <= o.function_tolerance * cost) { res.termination = 0; break; }
    const double rho = cost_change / mcc;
    if (rho > o.min_relative_decrease) {  // HandleSuccessfulStep
      if (Team::rank() == 0) {
        for (int j = 0; j < kVbN; ++j) W.x[j] = W.xc[j];
        for (int j = 0; j < kCamRec; ++j) W.rec[j] = W.recc[j];
      }
      Team::sync();
      xnorm = sqrt(view_xnorm2(W.x, nullptr, fm, K));
      if (!view_pass<EXT, Team>(V, W, W.x, W.rec, true, o.loss_type, o.loss_width, &cost)) { res.termination = 2; break; }
      res.final_cost = cost;
      gmax = gmax_of();
      const double t = 2.0 * rho - 1.0;
      radius = fmin(o.max_radius, radius / fmax(1.0 / 3.0, 1.0 - t * t * t));
      decrease = 2.0;
      last_successful = true;
    } else {  // HandleUnsuccessfulStep
      radius /= decrease; decrease *= 2.0;
      last_successful = false;
    }
  }
  // the minimiser leaves its best point in place: only the blocks with a free coordinate are written
  if (Team::rank() == 0) {
    if (fm & 0x3Fu) for (int j = 0; j < 6; ++j) V.ext[j] = W.x[j];
    if (fm & 0xFFC0u) for (int j = 0; j < 10; ++j) V.intr[j] = W.x[6 + j];
  }
  return res;
}

// ------------------------------------------------------------------------------------------------ device: one CTA per view
#if defined(__CUDACC__) || defined(TBA_EMULATE)
constexpr int kViewThreads = 128;
constexpr int kViewWarps = kViewThreads / 32;
constexpr int kViewGramPerLane = (kVbG + 31) / 32;

// The CTA as a team: every reduction is a butterfly inside each warp, then a fixed-order sum over the warps' partials that
// every thread reads (identical bits in all threads, so all take the same decisions).
struct CtaTeam {
  __host__ __device__ static int rank() {
#if defined(__CUDA_ARCH__) || defined(TBA_EMULATE)
    return threadIdx.x;
#else
    return 0;
#endif
  }
  __host__ __device__ static int size() { return kViewThreads; }
  __host__ __device__ static void sync() {
#if defined(__CUDA_ARCH__) || defined(TBA_EMULATE)
    __syncthreads();
#endif
  }
  __host__ __device__ static double sum(double v) {
#if defined(__CUDA_ARCH__) || defined(TBA_EMULATE)
    __shared__ double red[kViewWarps];
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0.0;
    for (int w = 0; w < kViewWarps; ++w) t += red[w];
    __syncthreads();  // red is reused by the next reduction
    return t;
#else
    return v;
#endif
  }
  __host__ __device__ static bool all(bool v) { return sum(v ? 0.0 : 1.0) == 0.0; }
};

// The CTA's Gram: each warp stages the [J | r] rows of its 32 observations in shared memory, and lane l accumulates the
// triangle entries l, l + 32, ... over them (5 registers instead of 153); at the end the warps' partials are summed in warp
// order.
template <>
struct ViewGram<CtaTeam> {
  double acc[kViewGramPerLane];
  int ea[kViewGramPerLane], eb[kViewGramPerLane];
  __host__ __device__ void reset() {
    const int lane = CtaTeam::rank() & 31;
    for (int k = 0; k < kViewGramPerLane; ++k) {
      acc[k] = 0.0;
      int e = lane + 32 * k, a = 0;
      if (e >= kVbG) { ea[k] = eb[k] = -1; continue; }
      while (e >= kVbW - a) { e -= kVbW - a; ++a; }
      ea[k] = a; eb[k] = a + e;
    }
  }
  __host__ __device__ void add(const double rows[2][kVbW]) {
#if defined(__CUDA_ARCH__) || defined(TBA_EMULATE)
    __shared__ double stage[kViewWarps][64][kVbW];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    for (int j = 0; j < kVbW; ++j) { stage[w][2 * lane][j] = rows[0][j]; stage[w][2 * lane + 1][j] = rows[1][j]; }
    __syncwarp();
    for (int k = 0; k < kViewGramPerLane; ++k) {
      if (ea[k] < 0) continue;
      const int a = ea[k], b = eb[k];
      double s = acc[k];
      for (int r = 0; r < 64; ++r) s += stage[w][r][a] * stage[w][r][b];
      acc[k] = s;
    }
    __syncwarp();
#endif
  }
  __host__ __device__ void total(ViewWork& W) {
#if defined(__CUDA_ARCH__) || defined(TBA_EMULATE)
    __shared__ double part[kViewWarps][kViewGramPerLane * 32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    for (int k = 0; k < kViewGramPerLane; ++k) part[w][lane + 32 * k] = acc[k];
    __syncthreads();
    for (int e = threadIdx.x; e < kVbG; e += kViewThreads) {
      double s = 0.0;
      for (int q = 0; q < kViewWarps; ++q) s += part[q][e];
      W.G[e] = s;
    }
    __syncthreads();
#endif
  }
};

// The batch of tba_adjust_views: view v is camera cam[v] with free-coordinate mask free_mask[v]; the camera's observations are
// the slots cam_slot[cam_off[c] .. cam_off[c + 1]) (the camera-major index of the uploaded problem).
struct ViewBatchDev {
  int n_views;
  const int* cam;
  const uint32_t* free_mask;
  const long long* cam_off;
  const long long* cam_slot;
  double* ext;             // [n_cam][6]
  double* intr;            // [n_group][10]
  const int* cam_group;
  const int* group_model;
  const int* slot_pt;
  const double* pt;
  const double* xy;
};

template <bool EXT>
__global__ void __launch_bounds__(kViewThreads) k_view_ba(ViewBatchDev B, PointLmOptions o, uint8_t* __restrict__ status,
                                                          double* __restrict__ cost2, int* __restrict__ iterations) {
  __shared__ ViewWork W;
  const int v = blockIdx.x;
  const int c = B.cam[v], g = B.cam_group[c];
  ViewBaProblem V;
  V.ext = B.ext + (size_t)c * 6; V.intr = B.intr + (size_t)g * 10; V.model = B.group_model[g]; V.free_mask = B.free_mask[v];
  V.n = (int)(B.cam_off[c + 1] - B.cam_off[c]); V.slot = B.cam_slot + B.cam_off[c];
  V.slot_pt = B.slot_pt; V.pt = B.pt; V.xy = B.xy;
  const PointLmResult r = view_lm<EXT, CtaTeam>(V, W, o);
  if (threadIdx.x == 0) {
    status[v] = (uint8_t)r.termination;
    cost2[2 * v] = r.initial_cost; cost2[2 * v + 1] = r.final_cost;
    iterations[v] = r.iterations;
  }
}
#endif

}  // namespace tba
