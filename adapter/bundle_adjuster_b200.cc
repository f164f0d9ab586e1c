// bundle_adjuster_b200.cc -- the H100 drop-in for src/theia/sfm/bundle_adjustment/bundle_adjuster.cc and
// bundle_adjustment.cc.  Problem construction follows the reference step by step (file:line cited at each step);
// where the reference calls into ceres::Problem to declare blocks constant / sub-parameterised, this adapter
// records the same decision in the flattened tba_problem, and ceres::Solve (bundle_adjuster.cc:205) becomes
// tba_solve().  No CPU fallback: if the engine cannot run, summary.success is false.
#include "bundle_adjuster_b200.h"

#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>

namespace theia {
namespace {

#define B200_CHECK(cond, what)                                                              \
  do {                                                                                      \
    if (!(cond)) { std::fprintf(stderr, "Check failed: %s (%s:%d)\n", what, __FILE__, __LINE__); std::abort(); } \
  } while (0)

double NowSeconds() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

}  // namespace

// One engine context per process (the estimators call BA from a single thread; concurrent callers are serialised).
namespace b200 {
namespace {
std::mutex g_mu;
tba_context* g_ctx = nullptr;
}  // namespace
std::mutex& Mutex() { return g_mu; }
tba_context* AcquireContext() {
  if (g_ctx == nullptr) {
    const char* dev = std::getenv("THEIA_B200_DEVICE");
    if (tba_create(dev ? std::atoi(dev) : 0, 0, 1, nullptr, &g_ctx) != TBA_OK) g_ctx = nullptr;
  }
  return g_ctx;
}
tba_context* CurrentContext() { return g_ctx; }
uint64_t& Generation() { static uint64_t g = 0; return g; }

// 1:1 copy of BundleAdjustmentOptions (SetSolverOptions, bundle_adjuster.cc:57-79)
void ToEngineOptions(const BundleAdjustmentOptions& in, tba_options* o) {
  tba_options_init(o);
  o->loss_function_type = static_cast<int32_t>(in.loss_function_type);
  o->robust_loss_width = in.robust_loss_width;
  o->linear_solver_type = static_cast<int32_t>(in.linear_solver_type);
  o->preconditioner_type = static_cast<int32_t>(in.preconditioner_type);
  o->visibility_clustering_type = static_cast<int32_t>(in.visibility_clustering_type);
  o->verbose = in.verbose;
  o->constant_camera_orientation = in.constant_camera_orientation;
  o->constant_camera_position = in.constant_camera_position;
  o->intrinsics_to_optimize = static_cast<int32_t>(in.intrinsics_to_optimize);
  o->num_threads = in.num_threads;
  o->max_num_iterations = in.max_num_iterations;
  o->max_solver_time_in_seconds = in.max_solver_time_in_seconds;
  o->use_inner_iterations = in.use_inner_iterations;
  o->function_tolerance = in.function_tolerance;
  o->gradient_tolerance = in.gradient_tolerance;
  o->parameter_tolerance = in.parameter_tolerance;
  o->max_trust_region_radius = in.max_trust_region_radius;
}
}  // namespace b200

namespace {
using b200::AcquireContext;
}  // namespace

tba_problem BundleAdjusterB200::Flat::AsProblem() {
  tba_problem p;
  std::memset(&p, 0, sizeof p);
  p.n_cam = static_cast<int32_t>(view_of_cam.size());
  p.ext = ext.data(); p.ext_const = ext_const.data(); p.cam_group = cam_group.data();
  p.n_group = static_cast<int32_t>(id_of_group.size());
  p.group_model = group_model.data(); p.intr = intr.data(); p.group_const_mask = group_const_mask.data();
  p.n_pt = static_cast<int32_t>(track_of_pt.size());
  p.pt = pt.data(); p.pt_const = pt_const.data();
  p.n_obs = static_cast<int64_t>(obs_cam.size());
  p.obs_cam = obs_cam.data(); p.obs_pt = obs_pt.data(); p.obs_xy = obs_xy.data();
  return p;
}

// bundle_adjuster.cc:82-100: loss, problem, solver options; the setup timer starts here.
BundleAdjusterB200::BundleAdjusterB200(const BundleAdjustmentOptions& options, Reconstruction* reconstruction)
    : options_(options), reconstruction_(reconstruction), start_time_(NowSeconds()) {
  B200_CHECK(reconstruction != nullptr, "reconstruction != NULL");
  std::memset(&last_summary_, 0, sizeof last_summary_);
}

BundleAdjusterB200::~BundleAdjusterB200() {}

void BundleAdjusterB200::AddResidual(ViewId view_id, TrackId track_id) { residuals_.emplace_back(view_id, track_id); }

// bundle_adjuster.cc:102-139
void BundleAdjusterB200::AddView(const ViewId view_id) {
  View* view = reconstruction_->MutableView(view_id);
  B200_CHECK(view != nullptr, "view != NULL");
  if (!view->IsEstimated() || optimized_views_.count(view_id)) return;  // :106-108
  optimized_views_.emplace(view_id);                                      // :111
  optimized_camera_intrinsics_groups_.emplace(reconstruction_->CameraIntrinsicsGroupIdFromViewId(view_id));  // :117-119
  for (const TrackId track_id : view->TrackIds()) {                       // :125
    B200_CHECK(view->GetFeature(track_id) != nullptr, "feature != NULL");
    Track* track = reconstruction_->MutableTrack(track_id);
    B200_CHECK(track != nullptr, "track != NULL");
    if (!track->IsEstimated()) continue;                                  // :129-131
    AddResidual(view_id, track_id);                                       // :134
    variable_tracks_.erase(track_id);                                     // SetTrackConstant :137 (re-freezes a track an earlier AddTrack
  }                                                                       // made variable; a later AddTrack makes it variable again)
}

// bundle_adjuster.cc:141-180
void BundleAdjusterB200::AddTrack(const TrackId track_id) {
  Track* track = reconstruction_->MutableTrack(track_id);
  B200_CHECK(track != nullptr, "track != NULL");
  if (!track->IsEstimated() || optimized_tracks_.count(track_id)) return;  // :144-146
  optimized_tracks_.emplace(track_id);                                     // :149
  for (const ViewId view_id : track->ViewIds()) {                          // :152-153
    View* view = reconstruction_->MutableView(view_id);
    B200_CHECK(view != nullptr, "view != NULL");
    if (optimized_views_.count(view_id) || !view->IsEstimated()) continue;  // :156-158
    B200_CHECK(view->GetFeature(track_id) != nullptr, "feature != NULL");
    AddResidual(view_id, track_id);                                         // :164
    constant_extrinsics_views_.emplace(view_id);                            // :168
    potentially_constant_camera_intrinsics_groups_.emplace(reconstruction_->CameraIntrinsicsGroupIdFromViewId(view_id));  // :173-175
  }
  variable_tracks_.emplace(track_id);  // SetTrackVariable :178
}

void BundleAdjusterB200::Flatten(Flat* f, tba_options* o) const {
  b200::ToEngineOptions(options_, o);
  // ---- parameter blocks that appear in residual blocks, in first-use order
  std::unordered_map<ViewId, int32_t> cam_of_view;
  std::unordered_map<TrackId, int32_t> pt_of_track;
  std::unordered_map<CameraIntrinsicsGroupId, int32_t> idx_of_group;
  for (const auto& vt : residuals_) {
    const ViewId view_id = vt.first;
    const TrackId track_id = vt.second;
    View* view = reconstruction_->MutableView(view_id);
    Camera* camera = view->MutableCamera();
    auto cit = cam_of_view.find(view_id);
    if (cit == cam_of_view.end()) {
      const CameraIntrinsicsGroupId gid = reconstruction_->CameraIntrinsicsGroupIdFromViewId(view_id);
      auto git = idx_of_group.find(gid);
      if (git == idx_of_group.end()) {
        git = idx_of_group.emplace(gid, static_cast<int32_t>(f->id_of_group.size())).first;
        f->id_of_group.push_back(gid);
        f->group_model.push_back(static_cast<int32_t>(camera->GetCameraIntrinsicsModelType()));
        const int K = camera->MutableCameraIntrinsics()->NumParameters();
        for (int j = 0; j < TBA_INTR_STRIDE; ++j) f->intr.push_back(j < K ? camera->intrinsics()[j] : 0.0);
        // SetCameraIntrinsicsParameterization, bundle_adjuster.cc:242-287
        uint32_t mask = 0;
        if (optimized_camera_intrinsics_groups_.count(gid)) {
          for (int idx : camera->MutableCameraIntrinsics()->GetSubsetFromOptimizeIntrinsicsType(options_.intrinsics_to_optimize)) mask |= 1u << idx;  // :258-265
        } else {
          mask = (1u << K) - 1u;  // only reached through constant cameras: whole block constant (:270-286)
        }
        f->group_const_mask.push_back(mask);
      }
      cit = cam_of_view.emplace(view_id, static_cast<int32_t>(f->view_of_cam.size())).first;
      f->view_of_cam.push_back(view_id);
      f->cam_group.push_back(git->second);
      for (int j = 0; j < Camera::kExtrinsicsSize; ++j) f->ext.push_back(camera->extrinsics()[j]);
      // SetCameraExtrinsicsParameterization, bundle_adjuster.cc:223-240; constant cameras :166-168
      // (a view that AddTrack reached before AddView stays constant: call order, as in the reference)
      uint8_t c = 0;
      if (constant_extrinsics_views_.count(view_id) || !optimized_views_.count(view_id)) c = TBA_EXT_ALL_CONST;
      else {
        if (options_.constant_camera_position) c |= TBA_EXT_POSITION_CONST;        // SubsetParameterization(6, {0,1,2})
        if (options_.constant_camera_orientation) c |= TBA_EXT_ORIENTATION_CONST;  // SubsetParameterization(6, {3,4,5})
      }
      f->ext_const.push_back(c);
    }
    auto pit = pt_of_track.find(track_id);
    if (pit == pt_of_track.end()) {
      Track* track = reconstruction_->MutableTrack(track_id);
      pit = pt_of_track.emplace(track_id, static_cast<int32_t>(f->track_of_pt.size())).first;
      f->track_of_pt.push_back(track_id);
      for (int j = 0; j < 4; ++j) f->pt.push_back(track->MutablePoint()->data()[j]);
      f->pt_const.push_back(variable_tracks_.count(track_id) ? 0 : 1);  // SetTrackConstant :137 / SetTrackVariable :178, last call wins
    }
    const Feature* feature = view->GetFeature(track_id);
    f->obs_cam.push_back(cit->second);
    f->obs_pt.push_back(pit->second);
    f->obs_xy.push_back(feature->x());
    f->obs_xy.push_back(feature->y());
  }
}

// bundle_adjuster.cc:182-221
BundleAdjustmentSummary BundleAdjusterB200::Optimize() {
  BundleAdjustmentSummary summary;
  Flat flat;
  tba_options opts;
  Flatten(&flat, &opts);
  tba_problem problem = flat.AsProblem();
  const double internal_setup_time = NowSeconds() - start_time_;  // :203
  std::lock_guard<std::mutex> lock(b200::Mutex());
  tba_summary s;
  std::memset(&s, 0, sizeof s);
  int rc;
  const char* ngpu = std::getenv("THEIA_B200_GPUS");  // >1: shard points+observations over that many GPUs of the box
  if (ngpu != nullptr && std::atoi(ngpu) != 1) {
    rc = tba_solve_multi(&opts, &problem, &s, std::atoi(ngpu));  // replaces ceres::Solve, :205
    if (rc != TBA_OK && s.message[0] == 0) std::snprintf(s.message, sizeof s.message, "tba_solve_multi failed with code %d", rc);
  } else {
    tba_context* ctx = AcquireContext();
    if (ctx == nullptr) {
      std::fprintf(stderr, "theia_ba_b200: no usable CUDA device; bundle adjustment not run (there is no CPU fallback)\n");
      std::snprintf(last_summary_.message, sizeof last_summary_.message, "no usable CUDA device");
      return summary;  // success = false
    }
    rc = tba_solve(ctx, &opts, &problem, &s);  // replaces ceres::Solve, :205
    if (rc != TBA_OK) std::snprintf(s.message, sizeof s.message, "%s", tba_last_error(ctx));
    resident_ = rc == TBA_OK;
    generation_ = ++b200::Generation();  // this problem now owns the context's device-resident state
    if (resident_) resident_tracks_ = flat.track_of_pt;
  }
  last_summary_ = s;
  last_summary_.iterations = nullptr;
  if (rc != TBA_OK) {
    std::fprintf(stderr, "theia_ba_b200: %s\n", s.message);
    return summary;  // success = false; parameters untouched
  }
  if (options_.verbose) std::fprintf(stderr, "theia_ba_b200: %s (%d iterations, cost %.6e -> %.6e)\n", s.message, s.num_iterations - 1, s.initial_cost, s.final_cost);
  // Ceres optimises the caller's memory in place (bundle_adjuster.cc:383-385): scatter the result back.
  for (size_t i = 0; i < flat.view_of_cam.size(); ++i) {
    Camera* camera = reconstruction_->MutableView(flat.view_of_cam[i])->MutableCamera();
    std::memcpy(camera->mutable_extrinsics(), &flat.ext[i * 6], 6 * sizeof(double));
  }
  for (size_t g = 0; g < flat.id_of_group.size(); ++g) {
    const auto views = reconstruction_->GetViewsInCameraIntrinsicGroup(flat.id_of_group[g]);  // :289-302
    B200_CHECK(!views.empty(), "!views_in_intrinsics_groups.empty()");
    Camera* camera = reconstruction_->MutableView(*views.begin())->MutableCamera();
    std::memcpy(camera->mutable_intrinsics(), &flat.intr[g * TBA_INTR_STRIDE], camera->MutableCameraIntrinsics()->NumParameters() * sizeof(double));
  }
  for (size_t q = 0; q < flat.track_of_pt.size(); ++q)
    std::memcpy(reconstruction_->MutableTrack(flat.track_of_pt[q])->MutablePoint()->data(), &flat.pt[q * 4], 4 * sizeof(double));
  summary.setup_time_in_seconds = internal_setup_time + s.setup_time_in_seconds;  // :210-211
  summary.solve_time_in_seconds = s.solve_time_in_seconds;                        // :212
  summary.initial_cost = s.initial_cost;
  summary.final_cost = s.final_cost;
  summary.success = s.success != 0;  // IsSolutionUsable(), :218
  return summary;
}

BundleAdjustmentSummary BundleAdjusterB200::OptimizeTracks() {
  BundleAdjustmentSummary summary;
  B200_CHECK(optimized_views_.empty(), "OptimizeTracks() is for problems built with AddTrack only");
  Flat flat;
  tba_options opts;
  Flatten(&flat, &opts);
  opts.use_inner_iterations = 0;                 // bundle_adjustment.cc:101
  opts.linear_solver_type = TBA_DENSE_QR;        // bundle_adjustment.cc:100 (any exact type: a 4x4 solve per track)
  tba_problem problem = flat.AsProblem();
  const double internal_setup_time = NowSeconds() - start_time_;
  std::lock_guard<std::mutex> lock(b200::Mutex());
  tba_context* ctx = AcquireContext();
  std::memset(&last_summary_, 0, sizeof last_summary_);
  if (ctx == nullptr) {
    std::fprintf(stderr, "theia_ba_b200: no usable CUDA device; bundle adjustment not run (there is no CPU fallback)\n");
    std::snprintf(last_summary_.message, sizeof last_summary_.message, "no usable CUDA device");
    return summary;
  }
  const double t0 = NowSeconds();
  resident_ = false;
  ++b200::Generation();
  const size_t n = flat.track_of_pt.size();
  std::vector<uint8_t> status(n + 1);
  std::vector<double> ic(n + 1), fc(n + 1);
  int32_t failed = 0;
  int rc = tba_upload(ctx, &opts, &problem);
  const double t1 = NowSeconds();
  if (rc == TBA_OK) rc = tba_adjust_tracks(ctx, &opts, status.data(), ic.data(), fc.data(), &failed);
  if (rc == TBA_OK) rc = tba_download(ctx, &problem);
  if (rc != TBA_OK) {
    std::snprintf(last_summary_.message, sizeof last_summary_.message, "%s", tba_last_error(ctx));
    std::fprintf(stderr, "theia_ba_b200: %s\n", last_summary_.message);
    return summary;
  }
  for (size_t q = 0; q < n; ++q) {
    if (status[q] == TBA_TRACK_SKIPPED) continue;
    std::memcpy(reconstruction_->MutableTrack(flat.track_of_pt[q])->MutablePoint()->data(), &flat.pt[q * 4], 4 * sizeof(double));
    if (ic[q] >= 0.0) summary.initial_cost += ic[q];
    if (fc[q] >= 0.0) summary.final_cost += fc[q];
  }
  summary.setup_time_in_seconds = internal_setup_time + (t1 - t0);
  summary.solve_time_in_seconds = NowSeconds() - t1;
  summary.success = failed == 0;
  last_summary_.success = summary.success; last_summary_.initial_cost = summary.initial_cost; last_summary_.final_cost = summary.final_cost;
  last_summary_.termination_type = n == 1 ? static_cast<int32_t>(status[0]) : static_cast<int32_t>(failed ? TBA_FAILURE : TBA_CONVERGENCE);
  return summary;
}

int BundleAdjusterB200::SetOutlierTracksToUnestimated(const double max_inlier_reprojection_error,
                                                      const double min_triangulation_angle_degrees) {
  std::lock_guard<std::mutex> lock(b200::Mutex());
  tba_context* g_ctx = b200::CurrentContext();
  if (!resident_ || g_ctx == nullptr || generation_ != b200::Generation()) return -1;
  std::vector<uint8_t> status(resident_tracks_.size() + 1);
  int32_t bad = 0, insufficient = 0;
  if (tba_filter_tracks(g_ctx, max_inlier_reprojection_error, min_triangulation_angle_degrees, status.data(), nullptr, &bad,
                        &insufficient) != TBA_OK) {
    std::fprintf(stderr, "theia_ba_b200: %s\n", tba_last_error(g_ctx));
    return -1;
  }
  int removed = 0;
  for (size_t q = 0; q < resident_tracks_.size(); ++q) {
    // Only tracks added through AddTrack are resident with ALL their estimated views (bundle_adjuster.cc:141-180); a track
    // that came in through AddView alone carries only the observations of the optimised views, so its statistics here would be
    // those of a subset (the reference evaluates a track over all of its estimated views,
    // set_outlier_tracks_to_unestimated.cc:62-136): such tracks are left alone.
    if (optimized_tracks_.count(resident_tracks_[q]) == 0) continue;
    Track* track = reconstruction_->MutableTrack(resident_tracks_[q]);
    if (track == nullptr || !track->IsEstimated()) continue;  // :77-79: only estimated tracks are examined
    if (status[q] != 0) { track->SetEstimated(false); ++removed; }  // :100-101,111-112,121-122
  }
  return removed;  // :135
}

// bundle_adjustment.cc:47-63
BundleAdjustmentSummary BundleAdjustPartialReconstructionB200(const BundleAdjustmentOptions& options,
                                                             const std::unordered_set<ViewId>& view_ids,
                                                             const std::unordered_set<TrackId>& track_ids,
                                                             Reconstruction* reconstruction) {
  B200_CHECK(reconstruction != nullptr, "reconstruction != NULL");
  BundleAdjusterB200 bundle_adjuster(options, reconstruction);
  for (const ViewId view_id : view_ids) bundle_adjuster.AddView(view_id);
  for (const TrackId track_id : track_ids) bundle_adjuster.AddTrack(track_id);
  return bundle_adjuster.Optimize();
}

// bundle_adjustment.cc:82-93
BundleAdjustmentSummary BundleAdjustViewB200(const BundleAdjustmentOptions& options, const ViewId view_id, Reconstruction* reconstruction) {
  BundleAdjustmentOptions ba_options = options;
  ba_options.linear_solver_type = ceres::DENSE_QR;
  ba_options.use_inner_iterations = false;
  BundleAdjusterB200 bundle_adjuster(ba_options, reconstruction);
  bundle_adjuster.AddView(view_id);
  return bundle_adjuster.Optimize();
}

// bundle_adjustment.cc:95-107
BundleAdjustmentSummary BundleAdjustTrackB200(const BundleAdjustmentOptions& options, const TrackId track_id, Reconstruction* reconstruction) {
  BundleAdjustmentOptions ba_options = options;
  ba_options.linear_solver_type = ceres::DENSE_QR;
  ba_options.use_inner_iterations = false;
  BundleAdjusterB200 bundle_adjuster(ba_options, reconstruction);
  bundle_adjuster.AddTrack(track_id);
  return bundle_adjuster.OptimizeTracks();
}

// bundle_adjustment.cc:66-80
BundleAdjustmentSummary BundleAdjustReconstructionB200(const BundleAdjustmentOptions& options, Reconstruction* reconstruction) {
  const auto view_ids = reconstruction->ViewIds();
  const auto track_ids = reconstruction->TrackIds();
  BundleAdjusterB200 bundle_adjuster(options, reconstruction);
  for (const ViewId view_id : view_ids) bundle_adjuster.AddView(view_id);
  for (const TrackId track_id : track_ids) bundle_adjuster.AddTrack(track_id);
  return bundle_adjuster.Optimize();
}

}  // namespace theia
