// adapter_views_test.cc -- test driver for adapter/bundle_adjust_views_b200.{h,cc} (built by adapter/Makefile, run by
// tests/test_z_adapter_views_gpu.py).  `adapter_views_test views ORACLE_SO` runs BundleAdjustViewsB200 on a scene and compares
// every view with BundleAdjustView restated view after view: BundleAdjusterB200::AddView's flattening of that one view
// (DENSE_QR, no inner iterations) solved by the CPU oracle (dlopen'ed oracle_solve; test infrastructure only).
#include <dlfcn.h>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <string>

#include "bundle_adjust_views_b200.h"

using namespace theia;

#define EXPECT(cond)                                                                      \
  do {                                                                                    \
    if (!(cond)) { std::fprintf(stderr, "FAILED: %s (%s:%d)\n", #cond, __FILE__, __LINE__); std::exit(1); } \
  } while (0)

typedef int (*oracle_solve_fn)(const tba_options*, tba_problem*, tba_summary*);

// PINHOLE projection for the test data (angle-axis by Rodrigues' formula)
static void Project(const double* e, const double* k, const double* X, double* pix) {
  const double a[3] = {X[0] - e[0], X[1] - e[1], X[2] - e[2]};
  const double* w = e + 3;
  const double th = std::sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
  double q[3] = {a[0], a[1], a[2]};
  if (th > 1e-12) {
    const double c = std::cos(th), s = std::sin(th), kx = w[0] / th, ky = w[1] / th, kz = w[2] / th;
    const double cr[3] = {ky * a[2] - kz * a[1], kz * a[0] - kx * a[2], kx * a[1] - ky * a[0]};
    const double d = (kx * a[0] + ky * a[1] + kz * a[2]) * (1 - c);
    q[0] = a[0] * c + cr[0] * s + kx * d; q[1] = a[1] * c + cr[1] * s + ky * d; q[2] = a[2] * c + cr[2] * s + kz * d;
  }
  const double u = q[0] / q[2], v = q[1] / q[2], r2 = u * u + v * v, d = 1 + r2 * (k[5] + k[6] * r2);
  pix[0] = k[0] * u * d + k[2] * v * d + k[3];
  pix[1] = k[0] * k[1] * v * d + k[4];
}

// n_views cameras looking at a point cloud, poses and focal lengths disturbed; views 0..n_shared-1 share one intrinsics
// group, the others own theirs; every track estimated.  The same seed builds the same scene (Reconstruction copies would share
// their intrinsics objects).
static void BuildScene(Reconstruction* rec, std::vector<ViewId>* views, int n_views, int n_tracks, int n_shared, unsigned seed) {
  std::mt19937 rng(seed);
  std::uniform_real_distribution<double> U(-1.0, 1.0);
  std::normal_distribution<double> N(0.0, 1.0);
  std::vector<std::vector<double>> gt(n_views, std::vector<double>(6));
  const double kgt[7] = {800.0, 1.0, 0.0, 500.0, 500.0, -0.05, 0.01};
  for (int i = 0; i < n_views; ++i) {
    const ViewId id = i < n_shared ? rec->AddView("v" + std::to_string(i), 7) : rec->AddView("v" + std::to_string(i));
    views->push_back(id);
    View* v = rec->MutableView(id);
    v->SetEstimated(true);
    double* e = v->MutableCamera()->mutable_extrinsics();
    for (int j = 0; j < 3; ++j) gt[i][j] = 2.0 * U(rng);
    for (int j = 3; j < 6; ++j) gt[i][j] = 0.1 * U(rng);
    for (int j = 0; j < 6; ++j) e[j] = gt[i][j] + (j < 3 ? 0.05 : 0.005) * N(rng);
    double* k = v->MutableCamera()->mutable_intrinsics();
    { k[0] = 800.0 * (1.0 + 0.01 * U(rng)); k[1] = 1.0; k[2] = 0.0; k[3] = 500.0; k[4] = 500.0; k[5] = 0.0; k[6] = 0.0; }
  }
  for (int t = 0; t < n_tracks; ++t) {
    double X[4] = {1.5 * U(rng), 1.5 * U(rng), 12.0 + 2.0 * U(rng), 1.0};
    std::vector<std::pair<ViewId, Feature>> obs;
    for (int o = 0; o < 5; ++o) {
      const int vi = (t * 3 + o * 5) % n_views;
      bool dup = false;
      for (auto& ob : obs) dup |= ob.first == (*views)[vi];
      if (dup) continue;
      double pix[2];
      Project(gt[vi].data(), kgt, X, pix);
      obs.emplace_back((*views)[vi], Feature(pix[0] + 0.3 * N(rng), pix[1] + 0.3 * N(rng)));
    }
    const TrackId tid = rec->AddTrack(obs);
    Track* tr = rec->MutableTrack(tid);
    for (int j = 0; j < 3; ++j) tr->MutablePoint()->data()[j] = X[j] + 0.01 * N(rng);
    tr->SetEstimated(true);
  }
}

static int TestViews(const char* oracle_path) {
  void* h = dlopen(oracle_path, RTLD_NOW);
  EXPECT(h != nullptr);
  oracle_solve_fn solve = (oracle_solve_fn)dlsym(h, "oracle_solve");
  EXPECT(solve != nullptr);
  for (int variant = 0; variant < 3; ++variant) {
    BundleAdjustmentOptions o;
    o.loss_function_type = variant == 1 ? LossFunctionType::HUBER : LossFunctionType::TRIVIAL;
    o.intrinsics_to_optimize = variant == 2 ? OptimizeIntrinsicsType::NONE : OptimizeIntrinsicsType::FOCAL_LENGTH;
    o.constant_camera_orientation = variant == 1;
    Reconstruction rg, ro;
    std::vector<ViewId> vg, vo;
    BuildScene(&rg, &vg, 14, 600, 4, 31 + variant);
    BuildScene(&ro, &vo, 14, 600, 4, 31 + variant);
    // views 2.. in order: 2 and 3 share a group with a free focal length (variants 0, 1): the second sees the first's intrinsics
    const std::vector<ViewId> batch(vg.begin() + 2, vg.end());
    const std::vector<double> pt_before(rg.MutableTrack(rg.TrackIds()[0])->MutablePoint()->data(),
                                        rg.MutableTrack(rg.TrackIds()[0])->MutablePoint()->data() + 4);
    const std::vector<BundleAdjustmentSummary> sg = BundleAdjustViewsB200(o, batch, &rg);
    EXPECT(sg.size() == batch.size());
    int moved = 0;
    for (size_t i = 0; i < batch.size(); ++i) {
      BundleAdjustmentOptions oo = o; oo.linear_solver_type = ceres::DENSE_QR; oo.use_inner_iterations = false;
      BundleAdjusterB200 ba(oo, &ro);
      ba.AddView(batch[i]);
      BundleAdjusterB200::Flat f; tba_options to;
      ba.Flatten(&f, &to);
      tba_problem p = f.AsProblem();
      tba_summary os; std::memset(&os, 0, sizeof os);
      EXPECT(solve(&to, &p, &os) == 0);
      Camera* c = ro.MutableView(batch[i])->MutableCamera();
      for (int j = 0; j < 6; ++j) c->mutable_extrinsics()[j] = f.ext[j];
      for (int j = 0; j < 7; ++j) c->mutable_intrinsics()[j] = f.intr[j];
      EXPECT(sg[i].success == (os.termination_type != TBA_FAILURE));
      EXPECT(std::fabs(sg[i].initial_cost - os.initial_cost) <= 1e-11 * os.initial_cost);
      EXPECT(std::fabs(sg[i].final_cost - os.final_cost) <= 1e-7 * os.final_cost);
      const double* eg = rg.MutableView(batch[i])->MutableCamera()->extrinsics();
      for (int j = 0; j < 6; ++j) EXPECT(std::fabs(eg[j] - f.ext[j]) <= 1e-8 * (1.0 + std::fabs(f.ext[j])));
      moved += os.final_cost < 0.5 * os.initial_cost;
    }
    EXPECT(moved >= 8);
    // intrinsics at the end: a shared group holds what the last view of the list that frees it made of it
    for (size_t i = 0; i < batch.size(); ++i) {
      const double* kg = rg.MutableView(batch[i])->MutableCamera()->intrinsics();
      const double* ko = ro.MutableView(batch[i])->MutableCamera()->intrinsics();
      for (int j = 0; j < 7; ++j) EXPECT(std::fabs(kg[j] - ko[j]) <= 1e-8 * (1.0 + std::fabs(ko[j])));
    }
    // views outside the batch and every point are untouched
    for (int v = 0; v < 2; ++v)
      for (int j = 0; j < 6; ++j) EXPECT(rg.MutableView(vg[v])->MutableCamera()->extrinsics()[j] == ro.MutableView(vo[v])->MutableCamera()->extrinsics()[j]);
    for (int j = 0; j < 4; ++j) EXPECT(rg.MutableTrack(rg.TrackIds()[0])->MutablePoint()->data()[j] == pt_before[j]);
  }
  std::printf("views ok\n");
  return 0;
}

int main(int argc, char** argv) {
  if (argc >= 3 && std::string(argv[1]) == "views") return TestViews(argv[2]);
  std::fprintf(stderr, "usage: adapter_views_test views ORACLE_SO\n");
  return 2;
}
