// host_view_ba.cc -- runs the PRODUCT's per-view LM (theiasfm_b200/csrc/tba_view_ba.cuh, the body of k_view_ba) on the host, for
// the CPU test suite (tests/test_view_ba.py): with one lane (SerialTeam) and as a 4-lane team of host threads (ThreadTeam).
#define __device__
#define __host__
#define __forceinline__ inline
#define __restrict__
#ifndef _GNU_SOURCE
#define _GNU_SOURCE
#endif
#include <cmath>
#include <vector>
using std::atan; using std::atan2; using std::fabs; using std::fmax; using std::fmin; using std::isfinite; using std::sqrt; using std::tan;

#include <condition_variable>
#include <mutex>
#include <thread>

#include "../include/theia_ba_b200.h"
#include "../theiasfm_b200/csrc/tba_view_ba.cuh"

// A 4-lane team of host threads: the strided observation loops, the reductions (a barrier + a fixed-order sum over the lanes'
// slots, identical bits in every lane) and the lead-lane solve with a barrier before the others read it, as the CTA runs them.
struct ThreadTeam {
  static constexpr int kLanes = 4;
  static thread_local int lane;
  static std::mutex mu; static std::condition_variable cv; static int waiting; static long generation; static double slot[kLanes];
  static void sync() {
    std::unique_lock<std::mutex> lk(mu);
    const long g = generation;
    if (++waiting == kLanes) { waiting = 0; ++generation; cv.notify_all(); }
    else cv.wait(lk, [&] { return generation != g; });
  }
  static int rank() { return lane; }
  static int size() { return kLanes; }
  static double sum(double v) { slot[lane] = v; sync(); double s = 0.0; for (int i = 0; i < kLanes; ++i) s += slot[i]; sync(); return s; }
  static bool all(bool v) { return sum(v ? 0.0 : 1.0) == 0.0; }
};
thread_local int ThreadTeam::lane = 0;
std::mutex ThreadTeam::mu; std::condition_variable ThreadTeam::cv; int ThreadTeam::waiting = 0; long ThreadTeam::generation = 0; double ThreadTeam::slot[ThreadTeam::kLanes];

// One view: ext[6] / intr[10] in/out, its n observations of the (constant) points pt[n][4] at xy[n][2].  out4 = {termination,
// initial cost, final cost, iterations}; use_team: 4 lanes (99 as termination if the lanes disagree).
extern "C" void host_view_ba(const tba_options* opt, double* ext, double* intr, int model, unsigned free_mask, int n, const double* pt, const double* xy,
                             int use_team, double* out4) {
  tba::PointLmOptions o;
  o.loss_type = opt->loss_function_type; o.loss_width = opt->robust_loss_width; o.max_num_iterations = opt->max_num_iterations;
  o.function_tolerance = opt->function_tolerance; o.gradient_tolerance = opt->gradient_tolerance; o.parameter_tolerance = opt->parameter_tolerance;
  o.initial_radius = opt->initial_trust_region_radius; o.max_radius = opt->max_trust_region_radius; o.min_radius = opt->min_trust_region_radius;
  o.min_relative_decrease = opt->min_relative_decrease; o.min_diag = opt->min_lm_diagonal; o.max_diag = opt->max_lm_diagonal;
  o.jacobi_scaling = opt->jacobi_scaling; o.max_consecutive_invalid = opt->max_num_consecutive_invalid_steps;
  // the packed layout the kernel reads: slot i = observation i, xy as [slot / 32][2][32]
  std::vector<long long> slot((size_t)n + 1);
  std::vector<int> slot_pt((size_t)n + 1);
  std::vector<double> xyp((size_t)(n / 32 + 1) * 64);
  for (int i = 0; i < n; ++i) {
    slot[i] = i; slot_pt[i] = i;
    xyp[(size_t)(i / 32) * 64 + (i % 32)] = xy[2 * i]; xyp[(size_t)(i / 32) * 64 + 32 + (i % 32)] = xy[2 * i + 1];
  }
  tba::ViewBaProblem V;
  V.ext = ext; V.intr = intr; V.model = model; V.free_mask = free_mask; V.n = n; V.slot = slot.data(); V.slot_pt = slot_pt.data(); V.pt = pt;
  V.xy = xyp.data();
  tba::ViewWork W;
  tba::PointLmResult r;
  if (use_team) {
    tba::PointLmResult rr[ThreadTeam::kLanes];
    std::vector<std::thread> th;
    for (int l = 0; l < ThreadTeam::kLanes; ++l) th.emplace_back([&, l] { ThreadTeam::lane = l; rr[l] = tba::view_lm<true, ThreadTeam>(V, W, o); });
    for (auto& t : th) t.join();
    r = rr[0];
    for (int l = 1; l < ThreadTeam::kLanes; ++l)
      if (rr[l].termination != r.termination || rr[l].iterations != r.iterations || rr[l].final_cost != r.final_cost) r.termination = 99;
  } else {
    r = tba::view_lm<true>(V, W, o);
  }
  out4[0] = r.termination; out4[1] = r.initial_cost; out4[2] = r.final_cost; out4[3] = r.iterations;
}
