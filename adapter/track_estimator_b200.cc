// track_estimator_b200.cc -- TrackEstimator (src/theia/sfm/estimate_track.cc) on the H100 engine: the set of tracks to
// estimate is flattened once (observations in estimated views only, GetObservationsFromTrackViews :59-85), uploaded, and
// every track runs the reference's pipeline on the device in one call.  No CPU fallback.
#include "track_estimator_b200.h"

#include <cstdio>
#include <cstring>
#include <unordered_map>

namespace theia {

// estimate_track.cc:116-131
TrackEstimatorB200::Summary TrackEstimatorB200::EstimateAllTracks() {
  std::unordered_set<TrackId> tracks;
  for (const ViewId view_id : reconstruction_->ViewIds()) {
    View* view = reconstruction_->MutableView(view_id);
    if (view == nullptr || !view->IsEstimated()) continue;
    const auto tracks_in_view = view->TrackIds();
    tracks.insert(tracks_in_view.begin(), tracks_in_view.end());
  }
  return EstimateTracks(tracks);
}

// estimate_track.cc:133-197 with EstimateTrack (:199-264) batched
TrackEstimatorB200::Summary TrackEstimatorB200::EstimateTracks(const std::unordered_set<TrackId>& track_ids) {
  Summary summary;
  for (int j = 0; j < 5; ++j) counts_[j] = 0;
  engine_ok_ = true;
  std::vector<TrackId> tracks_to_estimate;  // :142-150
  tracks_to_estimate.reserve(track_ids.size());
  for (const TrackId track_id : track_ids) {
    Track* track = reconstruction_->MutableTrack(track_id);
    if (track != nullptr && !track->IsEstimated()) tracks_to_estimate.push_back(track_id);
  }
  summary.input_num_estimated_tracks = static_cast<int>(track_ids.size() - tracks_to_estimate.size());
  summary.num_triangulation_attempts = static_cast<int>(tracks_to_estimate.size());
  if (tracks_to_estimate.empty()) return summary;  // :156-158

  // ---- flatten: cameras in first-use order, every block constant but the points
  std::vector<double> ext, intr, pt, obs_xy;
  std::vector<uint8_t> ext_const, pt_const;
  std::vector<int32_t> cam_group, group_model, obs_cam, obs_pt;
  std::vector<uint32_t> group_const_mask;
  std::unordered_map<ViewId, int32_t> cam_of_view;
  std::unordered_map<CameraIntrinsicsGroupId, int32_t> idx_of_group;
  bool supported = true;
  for (size_t q = 0; q < tracks_to_estimate.size(); ++q) {
    const TrackId track_id = tracks_to_estimate[q];
    Track* track = reconstruction_->MutableTrack(track_id);
    for (int j = 0; j < 4; ++j) pt.push_back(track->MutablePoint()->data()[j]);
    pt_const.push_back(0);
    for (const ViewId view_id : track->ViewIds()) {  // :65-84
      View* view = reconstruction_->MutableView(view_id);
      if (view == nullptr || !view->IsEstimated()) continue;
      const Feature* feature = view->GetFeature(track_id);
      if (feature == nullptr) { std::fprintf(stderr, "Check failed: feature != NULL (%s:%d)\n", __FILE__, __LINE__); std::abort(); }
      auto cit = cam_of_view.find(view_id);
      if (cit == cam_of_view.end()) {
        Camera* camera = view->MutableCamera();
        const CameraIntrinsicsGroupId gid = reconstruction_->CameraIntrinsicsGroupIdFromViewId(view_id);
        auto git = idx_of_group.find(gid);
        if (git == idx_of_group.end()) {
          git = idx_of_group.emplace(gid, static_cast<int32_t>(group_model.size())).first;
          const int model = static_cast<int>(camera->GetCameraIntrinsicsModelType());
          if (TBA_MODEL_NUM_PARAMETERS(model) < 0) supported = false;
          group_model.push_back(model);
          const int K = camera->MutableCameraIntrinsics()->NumParameters();
          for (int j = 0; j < TBA_INTR_STRIDE; ++j) intr.push_back(j < K ? camera->intrinsics()[j] : 0.0);
          group_const_mask.push_back((1u << K) - 1u);
        }
        cit = cam_of_view.emplace(view_id, static_cast<int32_t>(cam_group.size())).first;
        cam_group.push_back(git->second);
        for (int j = 0; j < Camera::kExtrinsicsSize; ++j) ext.push_back(camera->extrinsics()[j]);
        ext_const.push_back(TBA_EXT_ALL_CONST);
      }
      obs_cam.push_back(cit->second);
      obs_pt.push_back(static_cast<int32_t>(q));
      obs_xy.push_back(feature->x());
      obs_xy.push_back(feature->y());
    }
  }
  if (!supported) {
    std::fprintf(stderr, "theia_ba_b200: unknown camera intrinsics model type; nothing estimated\n");
    engine_ok_ = false;
    return summary;
  }
  std::vector<uint8_t> status(tracks_to_estimate.size(), TBA_TRACK_BAD_ANGLE);
  if (!obs_cam.empty()) {
    tba_problem p;
    std::memset(&p, 0, sizeof p);
    p.n_cam = static_cast<int32_t>(cam_group.size());
    p.ext = ext.data(); p.ext_const = ext_const.data(); p.cam_group = cam_group.data();
    p.n_group = static_cast<int32_t>(group_model.size());
    p.group_model = group_model.data(); p.intr = intr.data(); p.group_const_mask = group_const_mask.data();
    p.n_pt = static_cast<int32_t>(tracks_to_estimate.size());
    p.pt = pt.data(); p.pt_const = pt_const.data();
    p.n_obs = static_cast<int64_t>(obs_cam.size());
    p.obs_cam = obs_cam.data(); p.obs_pt = obs_pt.data(); p.obs_xy = obs_xy.data();
    tba_options opts;
    b200::ToEngineOptions(options_.ba_options, &opts);
    // BundleAdjustTrack overrides these two (bundle_adjustment.cc:100-101); the per-track solve is an exact 4x4 solve
    // either way, the engine only validates the pair at upload
    opts.linear_solver_type = TBA_ITERATIVE_SCHUR;
    opts.use_inner_iterations = 0;
    std::lock_guard<std::mutex> lock(b200::Mutex());
    tba_context* ctx = b200::AcquireContext();
    if (ctx == nullptr) {
      std::fprintf(stderr, "theia_ba_b200: no usable CUDA device; tracks not estimated (there is no CPU fallback)\n");
      engine_ok_ = false;
      return summary;
    }
    ++b200::Generation();  // whatever a BundleAdjusterB200 left on the device is gone
    int rc = tba_upload(ctx, &opts, &p);
    if (rc == TBA_OK)
      rc = tba_estimate_tracks(ctx, &opts, options_.max_acceptable_reprojection_error_pixels, options_.min_triangulation_angle_degrees,
                               options_.bundle_adjustment ? 1 : 0, status.data(), counts_);
    if (rc == TBA_OK) rc = tba_download(ctx, &p);
    if (rc != TBA_OK) {
      std::fprintf(stderr, "theia_ba_b200: %s\n", tba_last_error(ctx));
      engine_ok_ = false;
      for (int j = 0; j < 5; ++j) counts_[j] = 0;
      return summary;
    }
  } else {
    counts_[TBA_TRACK_BAD_ANGLE] = static_cast<int32_t>(tracks_to_estimate.size());
  }
  // ---- scatter: the reference overwrites Track::MutablePoint as soon as the triangulation succeeds (:232), whatever
  // happens next, and marks the track estimated only when every test passes (:262)
  for (size_t q = 0; q < tracks_to_estimate.size(); ++q) {
    Track* track = reconstruction_->MutableTrack(tracks_to_estimate[q]);
    if (status[q] == TBA_TRACK_ESTIMATED || status[q] == TBA_TRACK_BA_FAILED || status[q] == TBA_TRACK_BAD_REPROJECTION)
      std::memcpy(track->MutablePoint()->data(), &pt[q * 4], 4 * sizeof(double));
    if (status[q] == TBA_TRACK_ESTIMATED) {
      track->SetEstimated(true);
      summary.estimated_tracks.insert(tracks_to_estimate[q]);
    }
  }
  return summary;
}

}  // namespace theia
