// theia_compat/theia/sfm/scene.h -- Eigen-free stand-in for exactly the part of Theia's scene model that
// bundle_adjuster.cc / bundle_adjustment.cc consume (SURVEY.md section 8b), so that the adapter can be compiled
// and tested in an image without Eigen / Ceres / glog.  Same class and method names, same storage semantics
// (parameters are optimised IN PLACE through raw double*):
//   Reconstruction  src/theia/sfm/reconstruction.h:66-181 (ViewIds, TrackIds, MutableView, MutableTrack,
//                   CameraIntrinsicsGroupIdFromViewId, GetViewsInCameraIntrinsicGroup; shared intrinsics wiring
//                   reconstruction.cc:99-139)
//   View            src/theia/sfm/view.h:57-101     Track   src/theia/sfm/track.h:53-89
//   Camera          src/theia/sfm/camera/camera.h:181-200 (extrinsics [C | w], shared_ptr intrinsics)
//   CameraIntrinsicsModel  camera_intrinsics_model.h:206-210, GetSubsetFromOptimizeIntrinsicsType
//                   (pinhole_camera_model.cc:132-162, pinhole_radial_tangential_camera_model.cc:150-188)
// When building inside Theia this directory is NOT on the include path: the adapter includes the real headers.
#ifndef THEIA_COMPAT_SFM_SCENE_H_
#define THEIA_COMPAT_SFM_SCENE_H_

#include <cstdint>
#include <memory>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <vector>

namespace theia {

typedef uint32_t ViewId;
typedef uint32_t TrackId;
typedef uint32_t CameraIntrinsicsGroupId;

enum class OptimizeIntrinsicsType {
  NONE = 0x00, FOCAL_LENGTH = 0x01, ASPECT_RATIO = 0x02, SKEW = 0x04, PRINCIPAL_POINTS = 0x08, RADIAL_DISTORTION = 0x10,
  TANGENTIAL_DISTORTION = 0x20,
  ALL = FOCAL_LENGTH | ASPECT_RATIO | SKEW | PRINCIPAL_POINTS | RADIAL_DISTORTION | TANGENTIAL_DISTORTION,
};
inline OptimizeIntrinsicsType operator|(OptimizeIntrinsicsType a, OptimizeIntrinsicsType b) { return static_cast<OptimizeIntrinsicsType>(static_cast<int>(a) | static_cast<int>(b)); }
inline OptimizeIntrinsicsType operator&(OptimizeIntrinsicsType a, OptimizeIntrinsicsType b) { return static_cast<OptimizeIntrinsicsType>(static_cast<int>(a) & static_cast<int>(b)); }

enum class CameraIntrinsicsModelType { INVALID = -1, PINHOLE = 0, PINHOLE_RADIAL_TANGENTIAL = 1, FISHEYE = 2, FOV = 3, DIVISION_UNDISTORTION = 4 };

// Stand-ins for Eigen::Vector2d / Vector4d (only data() / operator[] are used by the adapter).
struct Vector4d { double v[4] = {0, 0, 0, 1}; double* data() { return v; } const double* data() const { return v; } double& operator[](int i) { return v[i]; } };
struct Feature { double v[2] = {0, 0}; Feature() {} Feature(double x, double y) { v[0] = x; v[1] = y; } double x() const { return v[0]; } double y() const { return v[1]; } };

// matching/feature_correspondence.h:50-63
struct FeatureCorrespondence { Feature feature1, feature2; FeatureCorrespondence() {} FeatureCorrespondence(const Feature& a, const Feature& b) : feature1(a), feature2(b) {} };

class CameraIntrinsicsModel {
 public:
  explicit CameraIntrinsicsModel(CameraIntrinsicsModelType t) : type_(t), parameters_(NumParametersOf(t), 0.0) {
    parameters_[0] = 1.0; parameters_[1] = 1.0;  // focal length 1, aspect ratio 1 (pinhole_camera_model.cc:56-64)
  }
  static int NumParametersOf(CameraIntrinsicsModelType t) {  // NumParameters() of the five models
    switch (t) {
      case CameraIntrinsicsModelType::PINHOLE: return 7;
      case CameraIntrinsicsModelType::PINHOLE_RADIAL_TANGENTIAL: return 10;
      case CameraIntrinsicsModelType::FISHEYE: return 9;
      case CameraIntrinsicsModelType::FOV: return 5;
      case CameraIntrinsicsModelType::DIVISION_UNDISTORTION: return 5;
      default: return 0;
    }
  }
  int NumParameters() const { return static_cast<int>(parameters_.size()); }
  CameraIntrinsicsModelType Type() const { return type_; }
  const double* parameters() const { return parameters_.data(); }
  double* mutable_parameters() { return parameters_.data(); }
  // Indices of the parameters held CONSTANT for the given bitmask.
  std::vector<int> GetSubsetFromOptimizeIntrinsicsType(const OptimizeIntrinsicsType& m) const {
    std::vector<int> c;
    if (m == OptimizeIntrinsicsType::ALL) return c;
    auto off = [&](OptimizeIntrinsicsType f) { return (m & f) == OptimizeIntrinsicsType::NONE; };
    if (type_ == CameraIntrinsicsModelType::FOV || type_ == CameraIntrinsicsModelType::DIVISION_UNDISTORTION) {
      // f, aspect, cx, cy, one distortion term (fov_camera_model.cc / division_undistortion_camera_model.cc)
      if (off(OptimizeIntrinsicsType::FOCAL_LENGTH)) c.push_back(0);
      if (off(OptimizeIntrinsicsType::ASPECT_RATIO)) c.push_back(1);
      if (off(OptimizeIntrinsicsType::PRINCIPAL_POINTS)) { c.push_back(2); c.push_back(3); }
      if (off(OptimizeIntrinsicsType::RADIAL_DISTORTION)) c.push_back(4);
      return c;
    }
    if (type_ == CameraIntrinsicsModelType::FISHEYE) {  // fisheye_camera_model.cc: pinhole layout, four radial terms
      if (off(OptimizeIntrinsicsType::FOCAL_LENGTH)) c.push_back(0);
      if (off(OptimizeIntrinsicsType::ASPECT_RATIO)) c.push_back(1);
      if (off(OptimizeIntrinsicsType::SKEW)) c.push_back(2);
      if (off(OptimizeIntrinsicsType::PRINCIPAL_POINTS)) { c.push_back(3); c.push_back(4); }
      if (off(OptimizeIntrinsicsType::RADIAL_DISTORTION)) { c.push_back(5); c.push_back(6); c.push_back(7); c.push_back(8); }
      return c;
    }
    if (off(OptimizeIntrinsicsType::FOCAL_LENGTH)) c.push_back(0);
    if (off(OptimizeIntrinsicsType::ASPECT_RATIO)) c.push_back(1);
    if (off(OptimizeIntrinsicsType::SKEW)) c.push_back(2);
    if (off(OptimizeIntrinsicsType::PRINCIPAL_POINTS)) { c.push_back(3); c.push_back(4); }
    if (off(OptimizeIntrinsicsType::RADIAL_DISTORTION)) { c.push_back(5); c.push_back(6); if (type_ == CameraIntrinsicsModelType::PINHOLE_RADIAL_TANGENTIAL) c.push_back(7); }
    if (type_ == CameraIntrinsicsModelType::PINHOLE_RADIAL_TANGENTIAL && off(OptimizeIntrinsicsType::TANGENTIAL_DISTORTION)) { c.push_back(8); c.push_back(9); }
    return c;
  }
 private:
  CameraIntrinsicsModelType type_;
  std::vector<double> parameters_;
};

class Camera {
 public:
  enum ExternalParametersIndex { POSITION = 0, ORIENTATION = 3 };
  static const int kExtrinsicsSize = 6;
  explicit Camera(CameraIntrinsicsModelType t = CameraIntrinsicsModelType::PINHOLE) : camera_intrinsics_(new CameraIntrinsicsModel(t)) {}
  const double* extrinsics() const { return camera_parameters_; }
  double* mutable_extrinsics() { return camera_parameters_; }
  const double* intrinsics() const { return camera_intrinsics_->parameters(); }
  double* mutable_intrinsics() { return camera_intrinsics_->mutable_parameters(); }
  CameraIntrinsicsModelType GetCameraIntrinsicsModelType() const { return camera_intrinsics_->Type(); }
  std::shared_ptr<CameraIntrinsicsModel>& MutableCameraIntrinsics() { return camera_intrinsics_; }
  const std::shared_ptr<CameraIntrinsicsModel>& CameraIntrinsics() const { return camera_intrinsics_; }
 private:
  double camera_parameters_[kExtrinsicsSize] = {0, 0, 0, 0, 0, 0};
  std::shared_ptr<CameraIntrinsicsModel> camera_intrinsics_;
};

class View {
 public:
  explicit View(const std::string& name = "") : name_(name) {}
  bool IsEstimated() const { return is_estimated_; }
  void SetEstimated(bool e) { is_estimated_ = e; }
  Camera* MutableCamera() { return &camera_; }
  const Camera& Camera_() const { return camera_; }
  std::vector<TrackId> TrackIds() const { std::vector<TrackId> ids; ids.reserve(features_.size()); for (const auto& kv : features_) ids.push_back(kv.first); return ids; }
  const Feature* GetFeature(TrackId t) const { auto it = features_.find(t); return it == features_.end() ? nullptr : &it->second; }
  void AddFeature(TrackId t, const Feature& f) { features_[t] = f; }
 private:
  std::string name_;
  bool is_estimated_ = false;
  Camera camera_;
  std::unordered_map<TrackId, Feature> features_;
};

class Track {
 public:
  bool IsEstimated() const { return is_estimated_; }
  void SetEstimated(bool e) { is_estimated_ = e; }
  const std::unordered_set<ViewId>& ViewIds() const { return view_ids_; }
  void AddView(ViewId v) { view_ids_.insert(v); }
  Vector4d* MutablePoint() { return &point_; }
  const Vector4d& Point() const { return point_; }
 private:
  bool is_estimated_ = false;
  std::unordered_set<ViewId> view_ids_;
  Vector4d point_;
};

class Reconstruction {
 public:
  // reconstruction.cc:99-139: views added with the same group id share one CameraIntrinsicsModel.
  ViewId AddView(const std::string& name, CameraIntrinsicsGroupId group, CameraIntrinsicsModelType type = CameraIntrinsicsModelType::PINHOLE) {
    const ViewId id = next_view_id_++;
    View v(name);
    *v.MutableCamera() = Camera(type);
    auto& members = groups_[group];
    if (!members.empty()) v.MutableCamera()->MutableCameraIntrinsics() = views_.at(*members.begin()).MutableCamera()->MutableCameraIntrinsics();
    members.insert(id);
    view_group_[id] = group;
    views_.emplace(id, v);
    return id;
  }
  ViewId AddView(const std::string& name) { return AddView(name, next_group_id_++); }
  TrackId AddTrack(const std::vector<std::pair<ViewId, Feature>>& obs) {
    const TrackId id = next_track_id_++;
    Track t;
    for (const auto& o : obs) { t.AddView(o.first); views_.at(o.first).AddFeature(id, o.second); }
    tracks_.emplace(id, t);
    return id;
  }
  std::vector<ViewId> ViewIds() const { std::vector<ViewId> ids; for (const auto& kv : views_) ids.push_back(kv.first); return ids; }
  std::vector<TrackId> TrackIds() const { std::vector<TrackId> ids; for (const auto& kv : tracks_) ids.push_back(kv.first); return ids; }
  View* MutableView(ViewId id) { auto it = views_.find(id); return it == views_.end() ? nullptr : &it->second; }
  Track* MutableTrack(TrackId id) { auto it = tracks_.find(id); return it == tracks_.end() ? nullptr : &it->second; }
  CameraIntrinsicsGroupId CameraIntrinsicsGroupIdFromViewId(ViewId id) const { return view_group_.at(id); }
  std::unordered_set<ViewId> GetViewsInCameraIntrinsicGroup(CameraIntrinsicsGroupId g) const { return groups_.at(g); }
  int NumViews() const { return static_cast<int>(views_.size()); }
  int NumTracks() const { return static_cast<int>(tracks_.size()); }
 private:
  ViewId next_view_id_ = 0; TrackId next_track_id_ = 0; CameraIntrinsicsGroupId next_group_id_ = 1000000;
  std::unordered_map<ViewId, View> views_;
  std::unordered_map<TrackId, Track> tracks_;
  std::unordered_map<ViewId, CameraIntrinsicsGroupId> view_group_;
  std::unordered_map<CameraIntrinsicsGroupId, std::unordered_set<ViewId>> groups_;
};

}  // namespace theia
#endif
