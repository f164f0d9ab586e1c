// bundle_adjust_views_b200.cc -- batched BundleAdjustView on the H100 engine (tba_adjust_views).
#include "bundle_adjust_views_b200.h"

#include <chrono>
#include <cstdio>
#include <cstring>
#include <unordered_map>
#include <unordered_set>

namespace theia {

std::vector<BundleAdjustmentSummary> BundleAdjustViewsB200(const BundleAdjustmentOptions& options, const std::vector<ViewId>& view_ids,
                                                           Reconstruction* reconstruction) {
  const auto t0 = std::chrono::steady_clock::now();
  std::vector<BundleAdjustmentSummary> summaries(view_ids.size());
  // ---- gather: one camera per estimated view (AddView, bundle_adjuster.cc:102-139), its intrinsics group, one residual per
  // estimated track it sees, every point constant (SetTrackConstant :137)
  std::vector<double> ext, intr, pt, obs_xy;
  std::vector<uint8_t> ext_const, pt_const;
  std::vector<int32_t> cam_group, group_model, obs_cam, obs_pt, cam_of;  // cam_of[i]: camera of view_ids[i], -1 = not adjusted
  std::vector<uint32_t> group_const_mask;
  std::unordered_map<ViewId, int32_t> cam_of_view;
  std::unordered_map<CameraIntrinsicsGroupId, int32_t> idx_of_group;
  std::unordered_map<TrackId, int32_t> pt_of_track;
  std::vector<CameraIntrinsicsGroupId> group_ids;
  bool supported = true;
  for (const ViewId view_id : view_ids) {
    View* view = reconstruction->MutableView(view_id);
    if (view == nullptr) { std::fprintf(stderr, "Check failed: view != NULL (%s:%d)\n", __FILE__, __LINE__); std::abort(); }
    if (!view->IsEstimated() || cam_of_view.count(view_id)) { cam_of.push_back(cam_of_view.count(view_id) ? cam_of_view[view_id] : -1); continue; }
    Camera* camera = view->MutableCamera();
    const CameraIntrinsicsGroupId gid = reconstruction->CameraIntrinsicsGroupIdFromViewId(view_id);
    auto git = idx_of_group.find(gid);
    if (git == idx_of_group.end()) {
      git = idx_of_group.emplace(gid, static_cast<int32_t>(group_model.size())).first;
      group_ids.push_back(gid);
      const int model = static_cast<int>(camera->GetCameraIntrinsicsModelType());
      if (TBA_MODEL_NUM_PARAMETERS(model) < 0) supported = false;
      group_model.push_back(model);
      const int K = camera->MutableCameraIntrinsics()->NumParameters();
      for (int j = 0; j < TBA_INTR_STRIDE; ++j) intr.push_back(j < K ? camera->intrinsics()[j] : 0.0);
      uint32_t mask = 0;  // SetCameraIntrinsicsParameterization, bundle_adjuster.cc:242-265
      for (int idx : camera->MutableCameraIntrinsics()->GetSubsetFromOptimizeIntrinsicsType(options.intrinsics_to_optimize)) mask |= 1u << idx;
      group_const_mask.push_back(mask);
    }
    const int32_t cam = static_cast<int32_t>(cam_group.size());
    cam_of_view.emplace(view_id, cam);
    cam_of.push_back(cam);
    cam_group.push_back(git->second);
    for (int j = 0; j < Camera::kExtrinsicsSize; ++j) ext.push_back(camera->extrinsics()[j]);
    uint8_t c = 0;  // SetCameraExtrinsicsParameterization, bundle_adjuster.cc:223-240
    if (options.constant_camera_position) c |= TBA_EXT_POSITION_CONST;
    if (options.constant_camera_orientation) c |= TBA_EXT_ORIENTATION_CONST;
    ext_const.push_back(c);
    for (const TrackId track_id : view->TrackIds()) {
      Track* track = reconstruction->MutableTrack(track_id);
      if (track == nullptr || !track->IsEstimated()) continue;  // :129-131
      auto pit = pt_of_track.find(track_id);
      if (pit == pt_of_track.end()) {
        pit = pt_of_track.emplace(track_id, static_cast<int32_t>(pt_const.size())).first;
        for (int j = 0; j < 4; ++j) pt.push_back(track->MutablePoint()->data()[j]);
        pt_const.push_back(1);
      }
      const Feature* feature = view->GetFeature(track_id);
      obs_cam.push_back(cam);
      obs_pt.push_back(pit->second);
      obs_xy.push_back(feature->x());
      obs_xy.push_back(feature->y());
    }
  }
  if (!supported) {
    std::fprintf(stderr, "theia_ba_b200: unknown camera intrinsics model type; no view adjusted\n");
    return summaries;
  }
  if (cam_group.empty()) return summaries;
  // ---- calls: consecutive runs of cameras in which every intrinsics group with a free coordinate occurs at most once; a later
  // run sees the intrinsics an earlier one refined (the device-resident problem is updated in place)
  std::vector<std::vector<int32_t>> runs(1);
  {
    std::unordered_set<int32_t> used;
    for (size_t cam = 0; cam < cam_group.size(); ++cam) {
      const int32_t g = cam_group[cam];
      const bool free_group = group_const_mask[g] != (1u << TBA_MODEL_NUM_PARAMETERS(group_model[g])) - 1u;
      if (free_group && used.count(g)) { runs.emplace_back(); used.clear(); }
      if (free_group) used.insert(g);
      runs.back().push_back(static_cast<int32_t>(cam));
    }
  }
  tba_problem p;
  std::memset(&p, 0, sizeof p);
  p.n_cam = static_cast<int32_t>(cam_group.size());
  p.ext = ext.data(); p.ext_const = ext_const.data(); p.cam_group = cam_group.data();
  p.n_group = static_cast<int32_t>(group_model.size());
  p.group_model = group_model.data(); p.intr = intr.data(); p.group_const_mask = group_const_mask.data();
  p.n_pt = static_cast<int32_t>(pt_const.size());
  p.pt = pt.data(); p.pt_const = pt_const.data();
  p.n_obs = static_cast<int64_t>(obs_cam.size());
  p.obs_cam = obs_cam.data(); p.obs_pt = obs_pt.data(); p.obs_xy = obs_xy.data();
  tba_options opts;
  b200::ToEngineOptions(options, &opts);
  opts.linear_solver_type = TBA_DENSE_QR;  // bundle_adjustment.cc:88-89
  opts.use_inner_iterations = 0;
  std::vector<uint8_t> status(cam_group.size(), TBA_FAILURE);
  std::vector<double> ic(cam_group.size(), -1.0), fc(cam_group.size(), -1.0);
  {
    std::lock_guard<std::mutex> lock(b200::Mutex());
    tba_context* ctx = b200::AcquireContext();
    if (ctx == nullptr) {
      std::fprintf(stderr, "theia_ba_b200: no usable CUDA device; views not adjusted (there is no CPU fallback)\n");
      return summaries;
    }
    ++b200::Generation();  // whatever a BundleAdjusterB200 left on the device is gone
    int rc = tba_upload(ctx, &opts, &p);
    for (size_t r = 0; r < runs.size() && rc == TBA_OK; ++r) {
      const std::vector<int32_t>& run = runs[r];
      const size_t b = static_cast<size_t>(run[0]);  // a run is a contiguous range of cameras
      rc = tba_adjust_views(ctx, &opts, run.data(), static_cast<int32_t>(run.size()), status.data() + b, ic.data() + b, fc.data() + b, nullptr);
    }
    if (rc == TBA_OK) rc = tba_download(ctx, &p);
    if (rc != TBA_OK) {
      std::fprintf(stderr, "theia_ba_b200: %s\n", tba_last_error(ctx));
      return summaries;
    }
  }
  const double seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  for (size_t i = 0; i < view_ids.size(); ++i) {
    const int32_t cam = cam_of[i];
    if (cam < 0) continue;
    BundleAdjustmentSummary& s = summaries[i];
    s.success = status[cam] != TBA_FAILURE;
    s.initial_cost = ic[cam]; s.final_cost = fc[cam];
    s.solve_time_in_seconds = seconds;
  }
  // ---- scatter: the free coordinates only
  for (const auto& kv : cam_of_view) {
    const int32_t cam = kv.second, g = cam_group[cam];
    Camera* camera = reconstruction->MutableView(kv.first)->MutableCamera();
    double* e = camera->mutable_extrinsics();
    for (int j = 0; j < Camera::kExtrinsicsSize; ++j)
      if (!(ext_const[cam] & (j < 3 ? TBA_EXT_POSITION_CONST : TBA_EXT_ORIENTATION_CONST))) e[j] = ext[(size_t)cam * 6 + j];
    double* k = camera->mutable_intrinsics();  // the group's shared intrinsics
    const int K = TBA_MODEL_NUM_PARAMETERS(group_model[g]);
    for (int j = 0; j < K; ++j)
      if (!((group_const_mask[g] >> j) & 1u)) k[j] = intr[(size_t)g * TBA_INTR_STRIDE + j];
  }
  return summaries;
}

}  // namespace theia
