// bundle_adjust_two_views_b200.cc -- BundleAdjustTwoViews (bundle_adjust_two_views.cc:112-191) on the H100 engine.
#include "bundle_adjust_two_views_b200.h"

#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>

namespace theia {
namespace {
double Now() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
void Check(bool cond, const char* what) {
  if (!cond) { std::fprintf(stderr, "Check failed: %s (%s)\n", what, __FILE__); std::abort(); }
}
}  // namespace

void FlattenTwoViewProblem(const TwoViewBundleAdjustmentOptions& options, const std::vector<FeatureCorrespondence>& correspondences,
                           Camera* camera1, Camera* camera2, std::vector<TwoViewPoint>* points3d, BundleAdjusterB200::Flat* f,
                           tba_options* o) {
  // SetSolverOptions (.cc:54-69): only these fields come from the caller; everything else is Ceres' default
  tba_options_init(o);
  o->loss_function_type = TBA_LOSS_TRIVIAL;          // residual blocks are added with a NULL loss (.cc:157-170)
  o->linear_solver_type = TBA_DENSE_SCHUR;           // .cc:60
  o->use_inner_iterations = 0;
  o->num_threads = options.ba_options.num_threads;   // .cc:63
  o->max_num_iterations = 200;                       // .cc:64
  o->function_tolerance = 1e-6; o->gradient_tolerance = 1e-10; o->parameter_tolerance = 1e-8;
  o->max_trust_region_radius = 1e16;                 // ceres::Solver::Options default (Theia's 1e12 is not applied here)
  o->max_solver_time_in_seconds = 1e9;
  o->verbose = options.ba_options.verbose;
  Camera* cams[2] = {camera1, camera2};
  const bool const_intr[2] = {options.constant_camera1_intrinsics, options.constant_camera2_intrinsics};
  const bool shared = camera1->mutable_intrinsics() == camera2->mutable_intrinsics();
  for (int i = 0; i < 2; ++i) {
    f->view_of_cam.push_back(static_cast<ViewId>(i));
    for (int j = 0; j < Camera::kExtrinsicsSize; ++j) f->ext.push_back(cams[i]->extrinsics()[j]);
    f->ext_const.push_back(i == 0 ? TBA_EXT_ALL_CONST : 0);  // .cc:141-148
    f->cam_group.push_back(shared ? 0 : i);
    if (i == 1 && shared) break;
    const int K = cams[i]->CameraIntrinsics()->NumParameters();
    f->id_of_group.push_back(static_cast<CameraIntrinsicsGroupId>(i));
    f->group_model.push_back(static_cast<int32_t>(cams[i]->GetCameraIntrinsicsModelType()));
    for (int j = 0; j < TBA_INTR_STRIDE; ++j) f->intr.push_back(j < K ? cams[i]->intrinsics()[j] : 0.0);
    // shared block: AddCameraParametersToProblem runs for both cameras on the SAME parameter block and
    // SetParameterBlockConstant from either call sticks (bundle_adjust_two_views.cc:96-108): constant if EITHER flag is set
    const bool all_const = shared ? (const_intr[0] || const_intr[1]) : const_intr[i];
    const uint32_t all = (1u << K) - 1u;
    f->group_const_mask.push_back(all_const ? all : (all & ~1u));  // focal length (index 0) is the only free one (.cc:96-108)
  }
  if (shared) { f->cam_group.resize(2, 0); }
  for (size_t q = 0; q < points3d->size(); ++q) {
    f->track_of_pt.push_back(static_cast<TrackId>(q));
    for (int j = 0; j < 4; ++j) f->pt.push_back((*points3d)[q].data()[j]);
    f->pt_const.push_back(0);
    f->obs_cam.push_back(0); f->obs_pt.push_back(static_cast<int32_t>(q));
    f->obs_xy.push_back(correspondences[q].feature1.x()); f->obs_xy.push_back(correspondences[q].feature1.y());
    f->obs_cam.push_back(1); f->obs_pt.push_back(static_cast<int32_t>(q));
    f->obs_xy.push_back(correspondences[q].feature2.x()); f->obs_xy.push_back(correspondences[q].feature2.y());
  }
}

BundleAdjustmentSummary BundleAdjustTwoViewsB200(const TwoViewBundleAdjustmentOptions& options,
                                                 const std::vector<FeatureCorrespondence>& correspondences, Camera* camera1, Camera* camera2,
                                                 std::vector<TwoViewPoint>* points3d) {
  Check(camera1 != nullptr, "camera1 != NULL");
  Check(camera2 != nullptr, "camera2 != NULL");
  Check(points3d != nullptr, "points3d != NULL");
  Check(points3d->size() == correspondences.size(), "points3d->size() == correspondences.size()");
  BundleAdjustmentSummary summary;
  const double t0 = Now();
  BundleAdjusterB200::Flat flat;
  tba_options opts;
  FlattenTwoViewProblem(options, correspondences, camera1, camera2, points3d, &flat, &opts);
  tba_problem problem = flat.AsProblem();
  summary.setup_time_in_seconds = Now() - t0;
  std::lock_guard<std::mutex> lock(b200::Mutex());
  tba_context* ctx = b200::AcquireContext();
  if (ctx == nullptr) {
    std::fprintf(stderr, "theia_ba_b200: no usable CUDA device; two-view bundle adjustment not run (there is no CPU fallback)\n");
    return summary;
  }
  ++b200::Generation();
  tba_summary s;
  std::memset(&s, 0, sizeof s);
  const int rc = tba_solve(ctx, &opts, &problem, &s);
  if (rc != TBA_OK) {
    std::fprintf(stderr, "theia_ba_b200: %s\n", tba_last_error(ctx));
    return summary;
  }
  std::memcpy(camera2->mutable_extrinsics(), &flat.ext[6], 6 * sizeof(double));
  Camera* cams[2] = {camera1, camera2};
  for (size_t g = 0; g < flat.id_of_group.size(); ++g)
    std::memcpy(cams[g]->mutable_intrinsics(), &flat.intr[g * TBA_INTR_STRIDE], cams[g]->CameraIntrinsics()->NumParameters() * sizeof(double));
  for (size_t q = 0; q < points3d->size(); ++q) std::memcpy((*points3d)[q].data(), &flat.pt[q * 4], 4 * sizeof(double));
  summary.setup_time_in_seconds += s.setup_time_in_seconds;
  summary.solve_time_in_seconds = s.solve_time_in_seconds;
  summary.initial_cost = s.initial_cost;
  summary.final_cost = s.final_cost;
  summary.success = s.termination_type != TBA_FAILURE;  // .cc:185
  return summary;
}

}  // namespace theia
