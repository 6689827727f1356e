// rpg_svo_b200/host/svo_host.h -- C++ host classes that keep the reference's call surface for the
// hot path and forward to the C ABI (include/svo_b200.h).  Header-only, depends on nothing but the
// C++17 standard library and libsvo_b200.so.
//
// What is mirrored (names, argument meaning, error behaviour):
//   svo::SparseImgAlign(max_level, min_level, n_iter, method, display, verbose)::run(ref, cur)
//       + getFisherInformation()                      svo/include/svo/sparse_img_align.h:43-57
//   svo::pose_optimizer::optimizeGaussNewton(...)     svo/include/svo/pose_optimizer.h:37-45
//   svo::feature_alignment::align2D / align1D         svo/include/svo/feature_alignment.h:29-44
//   svo::DepthFilter::{addFrame, addKeyframe(seeds), removeKeyframe, reset, getSeeds, updateSeeds}
//       + static updateSeed/computeTau stay host-side in the reference and are not re-exported
//                                                     svo/include/svo/depth_filter.h:101-158
//   svo::Frame / Feature / Point / Seed               svo/include/svo/{frame,feature,point,depth_filter}.h
//   svo::initialization::detectFeatures / trackKlt    svo/src/initialization.cpp:107-169
//   svo::streams::updateSeeds / reprojectMap /        not in the reference: S objects' calls with one launch each;
//     addKeyframes / detect / detectFeatures /        updateSeeds / addKeyframes are for filters without a mapper thread;
//     trackKlt                                        trackKlt builds the streams' LK pyramids with one batched build
// The data model is the reference's pointer graph (std::list<Feature*>, Point*); the wrappers gather it
// into the flat arrays the C ABI takes -- that gather is the cost SURVEY.md row a18 says must be
// counted end to end.  Differences from the reference, all forced by the missing third-party types:
//   * Eigen/Sophus/cv::Mat are replaced by the minimal Vector2d/Vector3d/SE3/Image below;
//   * FramePtr is std::shared_ptr (reference: boost::shared_ptr);
//   * cv::Mat image levels are device-resident: Frame::img_pyr_[l] is an `Image` handle (frame, level), and that
//     handle is what feature_alignment::align2D / align1D take where the reference takes `const cv::Mat& cur_img`;
//   * cameras: vk::PinholeCamera (with the optional radial-tangential coefficients) and vk::ATANCamera, restated;
//   * DepthFilter: updateSeeds is synchronous (the reference's thread_ == NULL branch, depth_filter.cpp:95-96); the
//     mapper thread is the caller's (see FrameHandlerMono below / INTEGRATION.md: one Context per thread), and
//     seeds_updating_halt_ is honoured before the launch and when the results are applied (the reference may stop
//     mid-list; here a halted call leaves the list untouched).
#pragma once
#include <algorithm>
#include <array>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <functional>
#include <atomic>
#include <condition_variable>
#include <limits>
#include <list>
#include <map>
#include <mutex>
#include <memory>
#include <stdexcept>
#include <queue>
#include <set>
#include <string>
#include <thread>
#include <vector>

#include "../../include/svo_b200.h"

namespace svo {

using Vector2d = std::array<double, 2>;
using Vector3d = std::array<double, 3>;
using Matrix6d = std::array<double, 36>;  // row-major

// Minimal rigid transform, row-major [R|t]; only what the wrappers need on the host.
struct SE3 {
  double m[12] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0};
  SE3 operator*(const SE3& o) const {
    SE3 r;
    for (int i = 0; i < 3; ++i) {
      for (int j = 0; j < 3; ++j)
        r.m[i * 4 + j] = m[i * 4] * o.m[j] + m[i * 4 + 1] * o.m[4 + j] + m[i * 4 + 2] * o.m[8 + j];
      r.m[i * 4 + 3] = m[i * 4] * o.m[3] + m[i * 4 + 1] * o.m[7] + m[i * 4 + 2] * o.m[11] + m[i * 4 + 3];
    }
    return r;
  }
  SE3 inverse() const {
    SE3 r;
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) r.m[i * 4 + j] = m[j * 4 + i];
    for (int i = 0; i < 3; ++i) r.m[i * 4 + 3] = -(r.m[i * 4] * m[3] + r.m[i * 4 + 1] * m[7] + r.m[i * 4 + 2] * m[11]);
    return r;
  }
  Vector3d translation() const { return {m[3], m[7], m[11]}; }
};

// [EXT] vk::AbstractCamera and the two models the reference ships parameter files for (svo_ros/param/*.yaml), restated
// from the published rpg_vikit sources; the device runs the same formulas (csrc/svo_math.cuh).
struct AbstractCamera {
  int width_, height_;
  AbstractCamera(int w, int h) : width_(w), height_(h) {}
  virtual ~AbstractCamera() {}
  virtual Vector3d cam2world(const Vector2d& px) const = 0;
  virtual Vector2d world2cam(const Vector3d& xyz_c) const = 0;
  virtual double errorMultiplier2() const = 0;
  virtual svo_b200_camera c_abi() const = 0;
  int width() const { return width_; }
  int height() const { return height_; }
  bool isInFrame(int x, int y, int boundary = 0) const {
    return x >= boundary && x < width_ - boundary && y >= boundary && y < height_ - boundary;
  }
  bool isInFrame(int x, int y, int boundary, int level) const {
    return x >= boundary && x < width_ / (1 << level) - boundary && y >= boundary && y < height_ / (1 << level) - boundary;
  }
};
struct PinholeCamera : AbstractCamera {  // vk::PinholeCamera(width, height, fx, fy, cx, cy, d0..d4)
  double fx_, fy_, cx_, cy_, d_[5];
  bool distortion_;
  PinholeCamera(int w, int h, double fx, double fy, double cx, double cy, double d0 = 0, double d1 = 0, double d2 = 0,
                double d3 = 0, double d4 = 0)
      : AbstractCamera(w, h), fx_(fx), fy_(fy), cx_(cx), cy_(cy), d_{d0, d1, d2, d3, d4}, distortion_(std::fabs(d0) > 0.0000001) {}
  Vector3d cam2world(const Vector2d& px) const override {
    double x, y;
    if (!distortion_) {
      x = (px[0] - cx_) / fx_; y = (px[1] - cy_) / fy_;
    } else {  // cv::undistortPoints on one CV_32FC2 point [EXT OpenCV]
      const double x0 = ((double)(float)px[0] - cx_) * (1.0 / fx_), y0 = ((double)(float)px[1] - cy_) * (1.0 / fy_);
      x = x0; y = y0;
      for (int j = 0; j < 5; ++j) {
        const double r2 = x * x + y * y, icdist = 1.0 / (1.0 + ((d_[4] * r2 + d_[1]) * r2 + d_[0]) * r2);
        const double dX = 2.0 * d_[2] * x * y + d_[3] * (r2 + 2.0 * x * x), dY = d_[2] * (r2 + 2.0 * y * y) + 2.0 * d_[3] * x * y;
        x = (x0 - dX) * icdist; y = (y0 - dY) * icdist;
      }
      x = (double)(float)x; y = (double)(float)y;
    }
    const double n = std::sqrt(x * x + y * y + 1.0);
    return {x / n, y / n, 1.0 / n};
  }
  Vector2d world2cam(const Vector3d& p) const override {
    const double x = p[0] / p[2], y = p[1] / p[2];
    if (!distortion_) return {std::fma(fx_, x, cx_), std::fma(fy_, y, cy_)};
    const double r2 = std::fma(x, x, y * y), r4 = r2 * r2, r6 = r4 * r2;
    const double a1 = 2.0 * x * y, a2 = std::fma(2.0 * x, x, r2), a3 = std::fma(2.0 * y, y, r2);
    const double cdist = std::fma(d_[4], r6, std::fma(d_[1], r4, std::fma(d_[0], r2, 1.0)));
    const double xd = std::fma(d_[3], a2, std::fma(d_[2], a1, x * cdist)), yd = std::fma(d_[3], a1, std::fma(d_[2], a3, y * cdist));
    return {std::fma(xd, fx_, cx_), std::fma(yd, fy_, cy_)};
  }
  double errorMultiplier2() const override { return std::fabs(fx_); }
  svo_b200_camera c_abi() const override {
    return svo_b200_camera{fx_, fy_, cx_, cy_, width_, height_, SVO_B200_CAM_PINHOLE, 0, {d_[0], d_[1], d_[2], d_[3], d_[4]}};
  }
};
struct ATANCamera : AbstractCamera {  // vk::ATANCamera(width, height, fx, fy, cx, cy, s): normalised parameters in
  double fx_, fy_, cx_, cy_, s_, tans_, tans_inv_, s_inv_;
  ATANCamera(double width, double height, double fx, double fy, double cx, double cy, double s)
      : AbstractCamera((int)width, (int)height), fx_(width * fx), fy_(height * fy), cx_(cx * width - 0.5), cy_(cy * height - 0.5),
        s_(s), tans_(s != 0.0 ? 2.0 * std::tan(s / 2.0) : 0.0), tans_inv_(s != 0.0 ? 1.0 / tans_ : 0.0), s_inv_(s != 0.0 ? 1.0 / s : 0.0) {}
  Vector3d cam2world(const Vector2d& px) const override {
    const double dx = (px[0] - cx_) * (1.0 / fx_), dy = (px[1] - cy_) * (1.0 / fy_), dist_r = std::sqrt(dx * dx + dy * dy);
    const double r = s_ != 0.0 ? std::tan(dist_r * s_) * tans_inv_ : dist_r, fac = dist_r > 0.01 ? r / dist_r : 1.0;
    const double x = fac * dx, y = fac * dy, n = std::sqrt(x * x + y * y + 1.0);
    return {x / n, y / n, 1.0 / n};
  }
  Vector2d world2cam(const Vector3d& p) const override {
    const double x = p[0] / p[2], y = p[1] / p[2], r = std::sqrt(std::fma(x, x, y * y));
    const double fac = (r < 0.001 || s_ == 0.0) ? 1.0 : s_inv_ * std::atan(r * tans_) / r;
    return {std::fma(fx_ * fac, x, cx_), std::fma(fy_ * fac, y, cy_)};
  }
  double errorMultiplier2() const override { return std::fabs(fx_); }
  svo_b200_camera c_abi() const override {
    return svo_b200_camera{fx_, fy_, cx_, cy_, width_, height_, SVO_B200_CAM_ATAN, 0, {s_, 0, 0, 0, 0}};
  }
};

// One CUDA context per calling thread, as include/svo_b200.h asks.
class Context {
 public:
  explicit Context(int device = 0) : device_(device) {
    if (svo_b200_create(&ctx_, device) != 0)
      throw std::runtime_error("svo_b200_create failed: no usable CUDA device (there is no CPU fallback)");
  }
  ~Context() { svo_b200_destroy(ctx_); }
  Context(const Context&) = delete;
  Context& operator=(const Context&) = delete;
  svo_b200_ctx* get() const { return ctx_; }
  int device() const { return device_; }
  void check(int rc) const {
    if (rc != 0) throw std::runtime_error(std::string("svo_b200: ") + svo_b200_last_error(ctx_));
  }

 private:
  svo_b200_ctx* ctx_ = nullptr;
  int device_ = 0;
};

class Frame;
struct Feature;
struct Point {  // svo/include/svo/point.h:35-106 (the fields the hot path reads)
  enum PointType { TYPE_DELETED, TYPE_CANDIDATE, TYPE_UNKNOWN, TYPE_GOOD };  // point.h:40-45
  Vector3d pos_;
  std::list<Feature*> obs_;        // references to keyframes which observe the point (point.h:52)
  PointType type_ = TYPE_UNKNOWN;  // point.h:58
  int n_failed_reproj_ = 0;        // point.h:59
  int n_succeeded_reproj_ = 0;     // point.h:60
  explicit Point(const Vector3d& pos) : pos_(pos) {}
  Point(const Vector3d& pos, Feature* ftr) : pos_(pos) { obs_.push_front(ftr); }  // point.cpp:38-50
  void addFrameRef(Feature* ftr) { obs_.push_front(ftr); }                        // point.cpp:55-59
  inline bool getCloseViewObs(const Vector3d& framepos, Feature*& ftr) const;     // point.cpp:97-117
};

struct Feature {  // svo/include/svo/feature.h:25-71
  enum FeatureType { CORNER, EDGELET };
  FeatureType type = CORNER;
  Frame* frame;
  Vector2d px;
  Vector3d f;
  int level;
  Point* point = nullptr;
  Vector2d grad{1.0, 0.0};
  Feature(Frame* _frame, const Vector2d& _px, int _level);
  Feature(Frame* _frame, Point* _point, const Vector2d& _px, const Vector3d& _f, int _level)
      : frame(_frame), px(_px), f(_f), level(_level), point(_point) {}
};
typedef std::list<Feature*> Features;

// svo/include/svo/frame.h:40-139.  The image pyramid lives in HBM (level 0 uploaded once, the other
// levels built on the device with the scalar vk::halfSample rule).
// What the reference passes around as `const cv::Mat&` for one pyramid level: here the level lives in HBM, so the
// handle names (device frame, level); cols / rows as cv::Mat has them.
struct Image {
  const class Frame* frame = nullptr;
  int level = 0, cols = 0, rows = 0;
};
typedef std::vector<Image> ImgPyr;

class Frame {
 public:
  AbstractCamera* cam_;
  SE3 T_f_w_;
  ImgPyr img_pyr_;  // frame.h:52 (device-resident levels)
  Matrix6d Cov_{};
  Features fts_;
  std::vector<Feature*> key_pts_ = std::vector<Feature*>(5, nullptr);  // frame.h:53
  bool is_keyframe_ = false;
  Frame(Context& ctx, AbstractCamera* cam, const uint8_t* img, int n_levels, double /*timestamp*/) : cam_(cam), ctx_(ctx) {
    if (!img) throw std::runtime_error("Frame: provided image is empty");  // frame.cpp:51-52
    ctx_.check(svo_b200_frame_create(ctx_.get(), cam->width_, cam->height_, n_levels, &dev_));
    const uint8_t* lv[1] = {img};
    ctx_.check(svo_b200_frame_upload(ctx_.get(), dev_, lv, 1));  // createImgPyramid on the device (frame.cpp:156-165)
    ctx_.check(svo_b200_synchronize(ctx_.get()));
    for (int l = 0; l < n_levels; ++l) img_pyr_.push_back(Image{this, l, cam->width_ >> l, cam->height_ >> l});
  }
  // A frame whose device pyramid is allocated but not yet uploaded: streams::newFrames uploads many with one call.
  struct NotUploaded {};
  Frame(Context& ctx, AbstractCamera* cam, int n_levels, NotUploaded) : cam_(cam), ctx_(ctx) {
    ctx_.check(svo_b200_frame_create(ctx_.get(), cam->width_, cam->height_, n_levels, &dev_));
    for (int l = 0; l < n_levels; ++l) img_pyr_.push_back(Image{this, l, cam->width_ >> l, cam->height_ >> l});
  }
  ~Frame() {
    for (Feature* f : fts_) delete f;  // frame.cpp:43-46
    svo_b200_klt_pyramid_destroy(ctx_.get(), klt_);
    svo_b200_frame_destroy(ctx_.get(), dev_);
  }
  Frame(const Frame&) = delete;
  void addFeature(Feature* ftr) { fts_.push_back(ftr); }
  inline void setKeyPoints();                 // frame.cpp:71-79
  inline void checkKeyPoints(Feature* ftr);   // frame.cpp:81-124
  void setKeyframe() { is_keyframe_ = true; setKeyPoints(); }  // frame.cpp:60-64
  bool isKeyframe() const { return is_keyframe_; }
  Vector3d pos() const { return T_f_w_.inverse().translation(); }  // frame.h:112
  Vector2d w2c(const Vector3d& xyz_w) const {                        // frame.h:88
    const double* m = T_f_w_.m;
    return cam_->world2cam({m[0] * xyz_w[0] + m[1] * xyz_w[1] + m[2] * xyz_w[2] + m[3], m[4] * xyz_w[0] + m[5] * xyz_w[1] + m[6] * xyz_w[2] + m[7],
                            m[8] * xyz_w[0] + m[9] * xyz_w[1] + m[10] * xyz_w[2] + m[11]});
  }
  size_t nObs() const { return fts_.size(); }
  Vector3d c2f(double x, double y) const { return cam_->cam2world({x, y}); }  // frame.h:94
  svo_b200_frame* device() const { return dev_; }
  Context& context() const { return ctx_; }
  // The LK pyramid cv::calcOpticalFlowPyrLK builds from img_pyr_[0] (initialization::trackKlt), built on first use and
  // kept: the first keyframe's, with derivatives, serves every frame of the initialisation.
  static constexpr int kKltMaxLevel = 4;  // calcOpticalFlowPyrLK's maxLevel in trackKlt (initialization.cpp:136)
  const svo_b200_klt_pyramid* kltPyramid(bool derivatives) {
    if (kltNeedsBuild(derivatives)) {
      ctx_.check(svo_b200_klt_pyramid_build(ctx_.get(), kltHandle(), dev_, kKltMaxLevel, derivatives ? 1 : 0));
      kltBuilt(true, derivatives);
    }
    return klt_;
  }
  // For builds of many frames' LK pyramids in one call (streams::trackKlt): whether kltPyramid(derivatives) would build,
  // the handle such a build fills, and what the build did (ok = it succeeded; a failed one may have left the handle
  // unbuilt, and the next use then builds again).
  bool kltNeedsBuild(bool derivatives) const { return klt_levels_ == 0 || (derivatives && !klt_derivs_); }
  svo_b200_klt_pyramid* kltHandle() {
    if (!klt_) ctx_.check(svo_b200_klt_pyramid_create(ctx_.get(), &klt_));
    return klt_;
  }
  void kltBuilt(bool ok, bool derivatives) {
    klt_levels_ = svo_b200_klt_pyramid_levels(klt_);
    if (ok) klt_derivs_ = derivatives;
    else if (klt_levels_ == 0) klt_derivs_ = false;
  }

 private:
  Context& ctx_;
  svo_b200_frame* dev_ = nullptr;
  svo_b200_klt_pyramid* klt_ = nullptr;
  int klt_levels_ = 0;
  bool klt_derivs_ = false;
};
typedef std::shared_ptr<Frame> FramePtr;

inline Feature::Feature(Frame* _frame, const Vector2d& _px, int _level)
    : frame(_frame), px(_px), f(_frame->cam_->cam2world(_px)), level(_level) {}

inline void Frame::setKeyPoints() {
  for (size_t i = 0; i < 5; ++i)
    if (key_pts_[i] != nullptr && key_pts_[i]->point == nullptr) key_pts_[i] = nullptr;
  for (Feature* ftr : fts_)
    if (ftr->point != nullptr) checkKeyPoints(ftr);
}
inline void Frame::checkKeyPoints(Feature* ftr) {  // including the reference's `px[0] < cv` comparisons (sic, frame.cpp:106,114)
  const int cu = cam_->width() / 2, cv = cam_->height() / 2;
  auto prod = [&](Feature* f) { return (f->px[0] - cu) * (f->px[1] - cv); };
  if (key_pts_[0] == nullptr) key_pts_[0] = ftr;
  else if (std::max(std::fabs(ftr->px[0] - cu), std::fabs(ftr->px[1] - cv)) <
           std::max(std::fabs(key_pts_[0]->px[0] - cu), std::fabs(key_pts_[0]->px[1] - cv)))
    key_pts_[0] = ftr;
  if (ftr->px[0] >= cu && ftr->px[1] >= cv) { if (key_pts_[1] == nullptr || prod(ftr) > prod(key_pts_[1])) key_pts_[1] = ftr; }
  if (ftr->px[0] >= cu && ftr->px[1] < cv) { if (key_pts_[2] == nullptr || prod(ftr) > prod(key_pts_[2])) key_pts_[2] = ftr; }
  if (ftr->px[0] < cv && ftr->px[1] < cv) { if (key_pts_[3] == nullptr || prod(ftr) > prod(key_pts_[3])) key_pts_[3] = ftr; }
  if (ftr->px[0] < cv && ftr->px[1] >= cv) { if (key_pts_[4] == nullptr || prod(ftr) > prod(key_pts_[4])) key_pts_[4] = ftr; }
}

// Point::getCloseViewObs (point.cpp:97-117): the observation with the smallest viewing-angle difference, refused
// beyond 60 degrees.
inline bool Point::getCloseViewObs(const Vector3d& framepos, Feature*& ftr) const {
  Vector3d obs_dir{framepos[0] - pos_[0], framepos[1] - pos_[1], framepos[2] - pos_[2]};
  const double n = std::sqrt(obs_dir[0] * obs_dir[0] + obs_dir[1] * obs_dir[1] + obs_dir[2] * obs_dir[2]);
  for (double& v : obs_dir) v /= n;
  auto min_it = obs_.begin();
  double min_cos_angle = 0;
  for (auto it = obs_.begin(), ite = obs_.end(); it != ite; ++it) {
    const Vector3d fp = (*it)->frame->pos();
    Vector3d dir{fp[0] - pos_[0], fp[1] - pos_[1], fp[2] - pos_[2]};
    const double dn = std::sqrt(dir[0] * dir[0] + dir[1] * dir[1] + dir[2] * dir[2]);
    const double cos_angle = (obs_dir[0] * dir[0] + obs_dir[1] * dir[1] + obs_dir[2] * dir[2]) / dn;
    if (cos_angle > min_cos_angle) { min_cos_angle = cos_angle; min_it = it; }
  }
  if (obs_.empty()) return false;
  ftr = *min_it;
  if (min_cos_angle < 0.5) return false;  // assume that observations larger than 60 degrees are useless
  return true;
}

// ------------------------------------------------------------------------------------------------
// svo::SparseImgAlign (svo/include/svo/sparse_img_align.h:33-81)
// ------------------------------------------------------------------------------------------------
class SparseImgAlign {
 public:
  enum Method { GaussNewton, LevenbergMarquardt };  // [EXT] vk::NLLSSolver::Method; only GaussNewton is used
  // [EXT] vk::NLLSSolver's robust cost, vikit's numbering (= SVO_B200_SCALE_* / SVO_B200_WEIGHT_*)
  enum ScaleEstimatorType { UnitScale, TDistScale, MADScale, NormalScale };
  enum WeightFunctionType { UnitWeight, TDistWeight, TukeyWeight, HuberWeight };
  SparseImgAlign(int max_level, int min_level, int n_iter, Method method, bool /*display*/, bool /*verbose*/)
      : max_level_(max_level), min_level_(min_level), n_iter_(n_iter) {
    if (method != GaussNewton) throw std::invalid_argument("SparseImgAlign: only GaussNewton is implemented");
    H_.fill(0.0);
  }
  // [EXT] NLLSSolver::setRobustCostFunction: every scale estimator but UnitScale turns weights on (UnitScale: plain
  // Gauss-Newton whatever the weight function).  Supported: MADScale with UnitWeight, TukeyWeight or HuberWeight.
  void setRobustCostFunction(ScaleEstimatorType scale_estimator, WeightFunctionType weight_function) {
    if (scale_estimator == TDistScale || scale_estimator == NormalScale)
      throw std::invalid_argument("SparseImgAlign::setRobustCostFunction: only the MAD and unit scale estimators are implemented");
    if (scale_estimator == MADScale && weight_function == TDistWeight)
      throw std::invalid_argument("SparseImgAlign::setRobustCostFunction: the T-distribution weight is not implemented");
    scale_estimator_ = scale_estimator;
    weight_function_ = scale_estimator == UnitScale ? UnitWeight : weight_function;
  }
  // sparse_img_align.cpp:43-75
  size_t run(FramePtr ref_frame, FramePtr cur_frame) {
    if (ref_frame->fts_.empty()) return 0;  // "SparseImgAlign: no features to track!"
    const size_t n = ref_frame->fts_.size();
    std::vector<double> px(2 * n), f(3 * n), pos(3 * n, 0.0);
    std::vector<uint8_t> has_point(n);
    size_t i = 0;
    for (Feature* ft : ref_frame->fts_) {
      px[2 * i] = ft->px[0]; px[2 * i + 1] = ft->px[1];
      for (int k = 0; k < 3; ++k) f[3 * i + k] = ft->f[k];
      has_point[i] = ft->point != nullptr;
      if (ft->point) for (int k = 0; k < 3; ++k) pos[3 * i + k] = ft->point->pos_[k];
      ++i;
    }
    SE3 T_cur_from_ref = cur_frame->T_f_w_ * ref_frame->T_f_w_.inverse();  // :59
    const Vector3d ref_pos = ref_frame->pos();
    const svo_b200_camera cam = ref_frame->cam_->c_abi();
    const svo_b200_sia_options opt = {max_level_, min_level_, n_iter_, 0.000001};  // eps_ (:40)
    svo_b200_sia_stats st;
    visible_fts_.assign(n, 0);
    Context& c = ref_frame->context();
    c.check(svo_b200_sia_robust(c.get(), scale_estimator_, weight_function_));  // this object's mode, set on every call
    c.check(svo_b200_sparse_img_align(c.get(), ref_frame->device(), cur_frame->device(), &cam, &opt, T_cur_from_ref.m,
                                      px.data(), f.data(), pos.data(), has_point.data(), ref_pos.data(), (int)n,
                                      visible_fts_.data(), H_.data(), &st, nullptr, 0, nullptr));
    cur_frame->T_f_w_ = T_cur_from_ref * ref_frame->T_f_w_;  // :70
    return (size_t)st.n_tracked;                              // n_meas_/patch_area_ (:74)
  }
  // sparse_img_align.cpp:77-82
  Matrix6d getFisherInformation() const {
    const double sigma_i_sq = 5e-4 * 255 * 255;
    Matrix6d I;
    for (int k = 0; k < 36; ++k) I[k] = H_[k] / sigma_i_sq;
    return I;
  }
  const std::vector<uint8_t>& visibleFeatures() const { return visible_fts_; }

 private:
  int max_level_, min_level_, n_iter_;
  int scale_estimator_ = UnitScale, weight_function_ = UnitWeight;
  Matrix6d H_;
  std::vector<uint8_t> visible_fts_;
};

// ------------------------------------------------------------------------------------------------
// svo::pose_optimizer (svo/include/svo/pose_optimizer.h:37-45)
// ------------------------------------------------------------------------------------------------
namespace pose_optimizer {
inline void optimizeGaussNewton(const double reproj_thresh, const size_t n_iter, const bool /*verbose*/, FramePtr& frame,
                                double& estimated_scale, double& error_init, double& error_final, size_t& num_obs) {
  const size_t n = frame->fts_.size();
  std::vector<double> f(3 * n), pos(3 * n, 0.0);
  std::vector<int> level(n);
  std::vector<uint8_t> has_point(n);
  size_t i = 0;
  for (Feature* ft : frame->fts_) {
    for (int k = 0; k < 3; ++k) f[3 * i + k] = ft->f[k];
    level[i] = ft->level;
    has_point[i] = ft->point != nullptr;
    if (ft->point) for (int k = 0; k < 3; ++k) pos[3 * i + k] = ft->point->pos_[k];
    ++i;
  }
  size_t n_with_point = 0;
  for (uint8_t h : has_point) n_with_point += h;
  if (n_with_point == 0) return;  // errors.empty(): outputs untouched (pose_optimizer.cpp:57-58)
  svo_b200_pose_opt_result out;
  Context& c = frame->context();
  c.check(svo_b200_pose_optimize(c.get(), reproj_thresh, (int)n_iter, frame->cam_->errorMultiplier2(), frame->T_f_w_.m,
                                 f.data(), pos.data(), level.data(), has_point.data(), (int)n, &out));
  i = 0;
  for (Feature* ft : frame->fts_) {  // culled observations lose their point (:139-143)
    if (ft->point && !has_point[i]) ft->point = nullptr;
    ++i;
  }
  for (int k = 0; k < 36; ++k) frame->Cov_[k] = out.cov[k];
  estimated_scale = out.estimated_scale;
  error_init = out.error_init;
  error_final = out.error_final;
  num_obs = (size_t)out.num_obs;
}
}  // namespace pose_optimizer

// ------------------------------------------------------------------------------------------------
// svo::feature_alignment (svo/include/svo/feature_alignment.h:29-44): the reference's argument lists, with the
// device-resident `Image` handle (frame->img_pyr_[level]) where the reference has `const cv::Mat& cur_img`.
// ------------------------------------------------------------------------------------------------
namespace feature_alignment {
inline bool align1D(const Image& cur_img, const std::array<float, 2>& dir, uint8_t* ref_patch_with_border, uint8_t* ref_patch,
                    const int n_iter, Vector2d& cur_px_estimate, double& h_inv) {
  uint8_t conv = 0;
  Context& c = cur_img.frame->context();
  c.check(svo_b200_align1d_batch(c.get(), cur_img.frame->device(), 1, &cur_img.level, dir.data(), ref_patch_with_border, ref_patch,
                                 n_iter, cur_px_estimate.data(), &conv, &h_inv));
  return conv != 0;
}
inline bool align2D(const Image& cur_img, uint8_t* ref_patch_with_border, uint8_t* ref_patch, const int n_iter,
                    Vector2d& cur_px_estimate, bool /*no_simd*/ = false) {
  uint8_t conv = 0;
  Context& c = cur_img.frame->context();
  c.check(svo_b200_align2d_batch(c.get(), cur_img.frame->device(), 1, &cur_img.level, ref_patch_with_border, ref_patch, n_iter,
                                 cur_px_estimate.data(), &conv));
  return conv != 0;
}
}  // namespace feature_alignment

// ------------------------------------------------------------------------------------------------
// svo::Matcher (svo/include/svo/matcher.h:69-130): the two entry points the hot path calls, and the public scratch
// members their callers read afterwards (reprojector.cpp:182-193, depth_filter.cpp:257).  Each call is one device
// launch for one candidate; the batched paths (Reprojector, DepthFilter) use the batch entry points directly.
// ------------------------------------------------------------------------------------------------
class Matcher {
 public:
  static const int halfpatch_size_ = 4;
  static const int patch_size_ = 8;
  struct Options {
    bool align_1d = false;
    int align_max_iter = 10;
    double max_epi_length_optim = 2.0;
    size_t max_epi_search_steps = 1000;
    bool subpix_refinement = true;
    bool epi_search_edgelet_filtering = true;
    double epi_search_edgelet_max_angle = 0.7;
    int n_pyr_levels = 3;  // Config::nPyrLevels() (config.cpp:30)
  } options_;
  // The options findEpipolarMatchDirect reads besides the iteration limits, as the C ABI's context setting
  // (svo_b200_set_epipolar_options); max_epi_length_optim is never read (matcher.cpp:226 uses the literal 2.0).
  svo_b200_epipolar_options abiEpipolarOptions() const {
    return {options_.align_1d ? 1 : 0, options_.subpix_refinement ? 1 : 0, options_.epi_search_edgelet_filtering ? 1 : 0,
            options_.epi_search_edgelet_max_angle};
  }
  std::array<double, 4> A_cur_ref_{};  // affine warp matrix, row-major
  double epi_length_ = 0.0;
  double h_inv_ = 0.0;
  int search_level_ = 0;
  bool reject_ = false;
  Feature* ref_ftr_ = nullptr;
  Vector2d px_cur_{};

  // matcher.cpp:135-177.  px_cur must hold an estimate within ~2-3 px of the result.
  bool findMatchDirect(const Point& pt, const Frame& cur_frame, Vector2d& px_cur) {
    if (!pt.getCloseViewObs(cur_frame.pos(), ref_ftr_)) return false;
    const Frame& rf = *ref_ftr_->frame;
    if (!rf.cam_->isInFrame((int)ref_ftr_->px[0] / (1 << ref_ftr_->level), (int)ref_ftr_->px[1] / (1 << ref_ftr_->level),
                            halfpatch_size_ + 2, ref_ftr_->level))
      return false;
    const svo_b200_frame* ref_dev = rf.device();
    const svo_b200_camera cam = cur_frame.cam_->c_abi();
    const svo_b200_match_options opt = {options_.n_pyr_levels - 1, options_.align_max_iter};
    const int ref_index = 0, type = ref_ftr_->type;
    uint8_t ok = 0;
    Context& c = cur_frame.context();
    c.check(svo_b200_find_match_direct(c.get(), &ref_dev, rf.T_f_w_.m, 1, cur_frame.device(), cur_frame.T_f_w_.m, &cam, &opt, 1,
                                       &ref_index, ref_ftr_->px.data(), ref_ftr_->f.data(), &ref_ftr_->level, &type,
                                       ref_ftr_->grad.data(), pt.pos_.data(), px_cur.data(), &ok, &search_level_,
                                       A_cur_ref_.data(), &h_inv_));
    return ok != 0;
  }
  // matcher.cpp:179-321.  Sets the context's epipolar options from options_ first, every call: a context may be shared
  // with a DepthFilter or another Matcher.  h_inv_ changes only where align1D ran (it sets h_inv_ on entry).
  bool findEpipolarMatchDirect(const Frame& ref_frame, const Frame& cur_frame, const Feature& ref_ftr, const double d_estimate,
                               const double d_min, const double d_max, double& depth) {
    const svo_b200_epipolar_options eo = abiEpipolarOptions();
    const svo_b200_frame* ref_dev = ref_frame.device();
    const svo_b200_camera cam = cur_frame.cam_->c_abi();
    const svo_b200_depth_options opt = {3, 200.0, options_.n_pyr_levels - 1, options_.align_max_iter, (int)options_.max_epi_search_steps};
    const int ref_index = 0, type = ref_ftr.type;
    uint8_t ok = 0, rej = 0;
    double z = 0.0;
    Context& c = cur_frame.context();
    c.check(svo_b200_set_epipolar_options(c.get(), &eo));
    c.check(svo_b200_find_epipolar_match_direct(c.get(), &ref_dev, ref_frame.T_f_w_.m, 1, cur_frame.device(), cur_frame.T_f_w_.m, &cam,
                                                &opt, 1, &ref_index, ref_ftr.px.data(), ref_ftr.f.data(), &ref_ftr.level, &type,
                                                ref_ftr.grad.data(), &d_estimate, &d_min, &d_max, &ok, &z, px_cur_.data(),
                                                &search_level_, &epi_length_, &rej, A_cur_ref_.data(), nullptr));
    double h_inv = 0.0;
    uint8_t ran_1d = 0;
    c.check(svo_b200_epipolar_last_h_inv(c.get(), 1, &h_inv, &ran_1d));
    if (ran_1d) h_inv_ = h_inv;
    reject_ = rej != 0;
    if (ok) depth = z;
    return ok != 0;
  }
};

// ------------------------------------------------------------------------------------------------
// svo::DepthFilter (svo/include/svo/depth_filter.h:35-51,53-158)
// ------------------------------------------------------------------------------------------------
// ------------------------------------------------------------------------------------------------
// svo::feature_detection (svo/include/svo/feature_detection.h:28-125): grid bookkeeping on the host, FAST-10 + score +
// non-maximum suppression + Shi-Tomasi + per-cell selection in one device launch (svo_b200_fast_detect).
// ------------------------------------------------------------------------------------------------
namespace feature_detection {
class AbstractDetector {
 public:
  AbstractDetector(int img_width, int img_height, int cell_size, int n_pyr_levels)
      : cell_size_(cell_size), n_pyr_levels_(n_pyr_levels), grid_n_cols_((int)std::ceil((double)img_width / cell_size)),
        grid_n_rows_((int)std::ceil((double)img_height / cell_size)), grid_occupancy_((size_t)grid_n_cols_ * grid_n_rows_, 0) {}
  virtual ~AbstractDetector() {}
  // img_pyr = the frame's device pyramid; `ctx` = the calling thread's context (default: the frame's)
  virtual void detect(Frame* frame, const double detection_threshold, Features& fts, Context* ctx = nullptr) = 0;
  void setGridOccpuancy(const Vector2d& px) {  // feature_detection.cpp:51-56 (spelling as in the reference)
    grid_occupancy_.at((size_t)((int)(px[1] / cell_size_) * grid_n_cols_ + (int)(px[0] / cell_size_))) = 1;
  }
  void setExistingFeatures(const Features& fts) { for (Feature* f : fts) setGridOccpuancy(f->px); }  // :42-49

 protected:
  const int cell_size_, n_pyr_levels_, grid_n_cols_, grid_n_rows_;
  std::vector<uint8_t> grid_occupancy_;
  void resetGrid() { std::fill(grid_occupancy_.begin(), grid_occupancy_.end(), 0); }
};
typedef std::shared_ptr<AbstractDetector> DetectorPtr;

class FastDetector : public AbstractDetector {
 public:
  FastDetector(int img_width, int img_height, int cell_size, int n_pyr_levels)
      : AbstractDetector(img_width, img_height, cell_size, n_pyr_levels) {}
  void detect(Frame* frame, const double detection_threshold, Features& fts, Context* ctx = nullptr) override {  // feature_detection.cpp:66-115
    Call k;
    const svo_b200_detect_stream a = gather(frame, detection_threshold, k);
    Context& c = ctx ? *ctx : frame->context();
    c.check(svo_b200_fast_detect(c.get(), a.frame, a.opt, a.grid_occupancy, a.cap, a.x_out, a.y_out, a.level_out, a.score_out,
                                 a.n_out));
    apply(frame, k, fts);
  }

  // The two host halves of detect around the device call, for streams::detect: the C-ABI arguments (the grid as it
  // stands; the buffers in `k`), and the new features appended to fts with the grid reset.
  struct Call {
    svo_b200_detect_options opt;
    std::vector<int> x, y, level;
    int n = 0;
  };
  svo_b200_detect_stream gather(Frame* frame, double detection_threshold, Call& k) {
    k.opt = {cell_size_, n_pyr_levels_, 20, 0, detection_threshold};
    const int cap = (int)grid_occupancy_.size();  // at most one corner per cell
    k.x.resize(cap); k.y.resize(cap); k.level.resize(cap);
    return {frame->device(), &k.opt, grid_occupancy_.data(), cap, k.x.data(), k.y.data(), k.level.data(), nullptr, &k.n};
  }
  void apply(Frame* frame, const Call& k, Features& fts) {
    for (int i = 0; i < k.n; ++i) fts.push_back(new Feature(frame, Vector2d{(double)k.x[i], (double)k.y[i]}, k.level[i]));
    resetGrid();
  }
};
}  // namespace feature_detection

// ------------------------------------------------------------------------------------------------
// svo::initialization (svo/src/initialization.cpp:107-169): the per-frame work of KltHomographyInit.  cv::Point2f is
// restated as Point2f; the KLT tracker runs on the device (svo_b200_klt_track).
// ------------------------------------------------------------------------------------------------
struct Point2f {
  float x, y;
};
struct Config {  // the values of svo/src/config.cpp that the initialisation reads
  static int gridSize() { return 30; }
  static int nPyrLevels() { return 3; }
  static double triangMinCornerScore() { return 20.0; }
};

namespace initialization {
// the detected features as pixel and bearing vectors; the features are freed (:114-124)
inline void takeFeatures(Features& new_features, std::vector<Point2f>& px_vec, std::vector<Vector3d>& f_vec) {
  px_vec.clear(); px_vec.reserve(new_features.size());
  f_vec.clear(); f_vec.reserve(new_features.size());
  for (Feature* ftr : new_features) {
    px_vec.push_back(Point2f{(float)ftr->px[0], (float)ftr->px[1]});
    f_vec.push_back(ftr->f);
    delete ftr;
  }
}
inline void detectFeatures(const FramePtr& frame, std::vector<Point2f>& px_vec, std::vector<Vector3d>& f_vec) {  // :107-125
  Features new_features;
  feature_detection::FastDetector detector(frame->img_pyr_[0].cols, frame->img_pyr_[0].rows, Config::gridSize(), Config::nPyrLevels());
  detector.detect(frame.get(), Config::triangMinCornerScore(), new_features);
  takeFeatures(new_features, px_vec, f_vec);
}

}  // namespace initialization

// Many camera streams per GPU: S streams' new frames with one batched upload, and S streams' initialization::trackKlt with one
// pyramid build and one tracking launch.
namespace streams {

// new Frame(ctx, cams[s], imgs[s], n_levels, timestamps[s]) of every stream: S frames whose device pyramids equal the
// constructor's, uploaded and built with one svo_b200_frame_upload_streams call and one synchronisation for all S.  Vectors
// of different lengths and a NULL camera throw std::invalid_argument, a NULL image throws as the constructor does
// (frame.cpp:51-52), before any frame is created.
inline std::vector<FramePtr> newFrames(Context& ctx, const std::vector<AbstractCamera*>& cams, const std::vector<const uint8_t*>& imgs,
                                       int n_levels, const std::vector<double>& timestamps) {
  const size_t S = cams.size();
  if (imgs.size() != S || timestamps.size() != S)
    throw std::invalid_argument("streams::newFrames: one camera, image and timestamp per stream");
  for (size_t s = 0; s < S; ++s) {
    if (!cams[s]) throw std::invalid_argument("streams::newFrames: NULL camera");
    if (!imgs[s]) throw std::runtime_error("Frame: provided image is empty");
  }
  std::vector<FramePtr> frames;
  std::vector<svo_b200_frame_upload_entry> e(S);
  for (size_t s = 0; s < S; ++s) {
    frames.emplace_back(new Frame(ctx, cams[s], n_levels, Frame::NotUploaded{}));
    e[s] = {frames[s]->device(), imgs[s]};
  }
  ctx.check(svo_b200_frame_upload_streams(ctx.get(), (int)S, e.data()));  // createImgPyramid of every frame on the device
  ctx.check(svo_b200_synchronize(ctx.get()));
  return frames;
}

// initialization::trackKlt(frames_ref[s], frames_cur[s], px_ref[s], px_cur[s], f_ref[s], f_cur[s], disparities[s]) of
// every stream: every LK pyramid a frame does not yet hold is built in one batched build (svo_b200_klt_pyramid_build_streams;
// the reference frames with derivatives, the current frames without, kept by the frames as Frame::kltPyramid keeps them),
// all streams are tracked with one launch (svo_b200_klt_track_streams), and then, stream by stream, the lost points are
// erased and f_cur (through the stream's own camera) and the disparities computed as the single function does.  Streams may
// share frames (e.g. one first keyframe).  The device work runs on `ctx`, by default the context of frames_cur[0].  Vectors
// of different lengths, a NULL frame, or a frame on another device than that context throw std::invalid_argument before
// any object or vector changes.
inline void trackKlt(const std::vector<FramePtr>& frames_ref, const std::vector<FramePtr>& frames_cur,
                     std::vector<std::vector<Point2f>>& px_ref, std::vector<std::vector<Point2f>>& px_cur,
                     std::vector<std::vector<Vector3d>>& f_ref, std::vector<std::vector<Vector3d>>& f_cur,
                     std::vector<std::vector<double>>& disparities, Context* ctx = nullptr) {
  const size_t S = frames_ref.size();
  if (frames_cur.size() != S || px_ref.size() != S || px_cur.size() != S || f_ref.size() != S || f_cur.size() != S ||
      disparities.size() != S)
    throw std::invalid_argument("streams::trackKlt: one frame pair and one set of vectors per stream");
  if (S == 0) return;
  for (size_t s = 0; s < S; ++s)
    if (!frames_ref[s] || !frames_cur[s]) throw std::invalid_argument("streams::trackKlt: NULL frame");
  Context& c = ctx ? *ctx : frames_cur[0]->context();
  for (size_t s = 0; s < S; ++s)
    if (frames_ref[s]->context().device() != c.device() || frames_cur[s]->context().device() != c.device())
      throw std::invalid_argument("streams::trackKlt: a frame lives on another device than the context");
  // 1. the pyramids no frame holds yet, each frame once (with derivatives where any stream tracks from it)
  std::vector<Frame*> todo;
  std::vector<bool> der;
  auto want = [&](Frame* f, bool d) {
    if (!f->kltNeedsBuild(d)) return;
    for (size_t k = 0; k < todo.size(); ++k)
      if (todo[k] == f) { der[k] = der[k] || d; return; }
    todo.push_back(f);
    der.push_back(d);
  };
  for (size_t s = 0; s < S; ++s) { want(frames_ref[s].get(), true); want(frames_cur[s].get(), false); }
  if (!todo.empty()) {
    std::vector<svo_b200_klt_build> b(todo.size());
    for (size_t k = 0; k < todo.size(); ++k) b[k] = {todo[k]->kltHandle(), todo[k]->device(), Frame::kKltMaxLevel, der[k] ? 1 : 0};
    const int rc = svo_b200_klt_pyramid_build_streams(c.get(), (int)b.size(), b.data());
    for (size_t k = 0; k < todo.size(); ++k) todo[k]->kltBuilt(rc == 0, der[k]);
    c.check(rc);
  }
  // 2. one tracking launch: calcOpticalFlowPyrLK(ref, cur, px_ref, px_cur, ..., Size(30, 30), 4, (COUNT + EPS, 30, 0.001),
  // OPTFLOW_USE_INITIAL_FLOW) of every stream
  const svo_b200_klt_options opt = {30, Frame::kKltMaxLevel, 30, 0.001};
  std::vector<std::vector<uint8_t>> status(S);
  std::vector<svo_b200_klt_stream> a(S);
  for (size_t s = 0; s < S; ++s) {
    status[s].resize(px_ref[s].size());
    px_cur[s].resize(px_ref[s].size());  // the reference requires the initial flow to have px_ref's size
    a[s] = {frames_ref[s]->kltPyramid(true), frames_cur[s]->kltPyramid(false), &opt, (int)px_ref[s].size(),
            reinterpret_cast<const float*>(px_ref[s].data()), reinterpret_cast<float*>(px_cur[s].data()), status[s].data(), nullptr};
  }
  c.check(svo_b200_klt_track_streams(c.get(), (int)S, a.data()));
  // 3. per stream, in order: lost points erased from px_ref, px_cur and f_ref; f_cur and the disparities of the rest
  // (initialization.cpp:146-168)
  for (size_t s = 0; s < S; ++s) {
    auto px_ref_it = px_ref[s].begin();
    auto px_cur_it = px_cur[s].begin();
    auto f_ref_it = f_ref[s].begin();
    f_cur[s].clear(); f_cur[s].reserve(px_cur[s].size());
    disparities[s].clear(); disparities[s].reserve(px_cur[s].size());
    for (size_t i = 0; px_ref_it != px_ref[s].end(); ++i) {
      if (!status[s][i]) {
        px_ref_it = px_ref[s].erase(px_ref_it);
        px_cur_it = px_cur[s].erase(px_cur_it);
        f_ref_it = f_ref[s].erase(f_ref_it);
        continue;
      }
      f_cur[s].push_back(frames_cur[s]->c2f(px_cur_it->x, px_cur_it->y));
      const double dx = px_ref_it->x - px_cur_it->x, dy = px_ref_it->y - px_cur_it->y;  // float differences, widened
      disparities[s].push_back(std::sqrt(dx * dx + dy * dy));
      ++px_ref_it;
      ++px_cur_it;
      ++f_ref_it;
    }
  }
}

}  // namespace streams

namespace initialization {
// calcOpticalFlowPyrLK(ref, cur, px_ref, px_cur, ..., Size(30, 30), 4, (COUNT + EPS, 30, 0.001), OPTFLOW_USE_INITIAL_FLOW),
// then lost points erased from px_ref, px_cur and f_ref in order; f_cur and the disparities of the rest (:127-169).
// streams::trackKlt of one stream.
inline void trackKlt(const FramePtr& frame_ref, const FramePtr& frame_cur, std::vector<Point2f>& px_ref, std::vector<Point2f>& px_cur,
                     std::vector<Vector3d>& f_ref, std::vector<Vector3d>& f_cur, std::vector<double>& disparities) {
  std::vector<std::vector<Point2f>> pr(1), pc(1);
  std::vector<std::vector<Vector3d>> fr(1), fc(1);
  std::vector<std::vector<double>> d(1);
  auto swap_all = [&] { pr[0].swap(px_ref); pc[0].swap(px_cur); fr[0].swap(f_ref); fc[0].swap(f_cur); d[0].swap(disparities); };
  swap_all();
  try {
    streams::trackKlt({frame_ref}, {frame_cur}, pr, pc, fr, fc, d, frame_cur ? &frame_cur->context() : nullptr);
  } catch (...) {
    swap_all();
    throw;
  }
  swap_all();
}
}  // namespace initialization

// Many camera streams per GPU: S detectors' FastDetector::detect, and S frames' initialization::detectFeatures, with one
// device launch (svo_b200_fast_detect_streams).  The device work runs on `ctx`, by default the context of frames[0];
// every frame must live on that context's device.
namespace streams {

// FastDetector::detect(frames[s], thresholds[s], fts[s]) of every detectors[s]: fts[s] gets the features the detector's
// own call would append, and every detector's grid is reset afterwards, as detect resets it.  A detector listed twice is
// refused (std::invalid_argument) before anything changes.
inline void detect(const std::vector<feature_detection::FastDetector*>& detectors, const std::vector<FramePtr>& frames,
                   const std::vector<double>& thresholds, std::vector<Features>& fts, Context* ctx = nullptr) {
  const size_t S = detectors.size();
  if (frames.size() != S || thresholds.size() != S || fts.size() != S)
    throw std::invalid_argument("streams::detect: one frame, threshold and feature list per detector");
  if (S == 0) return;
  for (size_t s = 0; s < S; ++s) {
    if (!detectors[s] || !frames[s]) throw std::invalid_argument("streams::detect: NULL detector or frame");
    for (size_t t = 0; t < s; ++t)
      if (detectors[t] == detectors[s]) throw std::invalid_argument("streams::detect: a detector is listed twice");
  }
  std::vector<feature_detection::FastDetector::Call> k(S);
  std::vector<svo_b200_detect_stream> a(S);
  for (size_t s = 0; s < S; ++s) a[s] = detectors[s]->gather(frames[s].get(), thresholds[s], k[s]);
  Context& c = ctx ? *ctx : frames[0]->context();
  c.check(svo_b200_fast_detect_streams(c.get(), (int)S, a.data()));
  for (size_t s = 0; s < S; ++s) detectors[s]->apply(frames[s].get(), k[s], fts[s]);
}

// initialization::detectFeatures(frames[s], px_vecs[s], f_vecs[s]) of every frame.
inline void detectFeatures(const std::vector<FramePtr>& frames, std::vector<std::vector<Point2f>>& px_vecs,
                           std::vector<std::vector<Vector3d>>& f_vecs) {
  const size_t S = frames.size();
  if (px_vecs.size() != S || f_vecs.size() != S) throw std::invalid_argument("streams::detectFeatures: one output pair per frame");
  std::vector<std::unique_ptr<feature_detection::FastDetector>> owned;
  std::vector<feature_detection::FastDetector*> detectors;
  for (const FramePtr& frame : frames) {
    if (!frame) throw std::invalid_argument("streams::detectFeatures: NULL frame");
    owned.emplace_back(new feature_detection::FastDetector(frame->img_pyr_[0].cols, frame->img_pyr_[0].rows, Config::gridSize(),
                                                           Config::nPyrLevels()));
    detectors.push_back(owned.back().get());
  }
  std::vector<Features> fts(S);
  detect(detectors, frames, std::vector<double>(S, Config::triangMinCornerScore()), fts);
  for (size_t s = 0; s < S; ++s) initialization::takeFeatures(fts[s], px_vecs[s], f_vecs[s]);
}

}  // namespace streams

class DepthFilter;
class Reprojector;
// Many camera streams per GPU: S objects' updateSeeds / reprojectMap with one device launch each (defined after the
// classes, see there).
namespace streams {
void updateSeeds(const std::vector<DepthFilter*>& filters, const std::vector<FramePtr>& frames);
void addKeyframes(const std::vector<DepthFilter*>& filters, const std::vector<FramePtr>& frames,
                  const std::vector<double>& depth_mean, const std::vector<double>& depth_min);
void reprojectMap(const std::vector<Reprojector*>& reprojectors, const std::vector<FramePtr>& frames,
                  std::vector<std::vector<std::pair<FramePtr, size_t>>>& overlap_kfs);
}  // namespace streams

struct Seed {
  static int& batch_counter() { static int c = 0; return c; }
  static int& seed_counter() { static int c = 0; return c; }
  int batch_id, id;
  Feature* ftr;
  float a, b, mu, z_range, sigma2;
  Seed(Feature* _ftr, float depth_mean, float depth_min)  // depth_filter.cpp:37-46
      : batch_id(batch_counter()), id(seed_counter()++), ftr(_ftr), a(10), b(10), mu(1.0 / depth_mean),
        z_range(1.0 / depth_min), sigma2(z_range * z_range / 36) {}
};

class DepthFilter {
 public:
  typedef std::function<void(Point*, double)> callback_t;
  struct Options {
    int max_n_kfs = 3;
    double seed_convergence_sigma2_thresh = 200.0;
    int max_search_level = 2;  // Config::nPyrLevels()-1 with the non-ROS default n_pyr_levels = 3
  } options_;
  explicit DepthFilter(callback_t seed_converged_cb) : seed_converged_cb_(seed_converged_cb) {}
  DepthFilter(feature_detection::DetectorPtr feature_detector, callback_t seed_converged_cb)  // depth_filter.h:88-90
      : seed_converged_cb_(seed_converged_cb), feature_detector_(feature_detector) {}
  virtual ~DepthFilter() { stopThread(); }
  // The mapper thread issues its device work on a context (= CUDA stream + staging buffers) of its own, as
  // include/svo_b200.h asks; without one the filter borrows the context of the frame it is handed.
  void setContext(Context* ctx) { ctx_ = ctx; }
  // depth_filter.cpp:64-86: the reference's mapper boost::thread
  void startThread() { thread_.reset(new std::thread(&DepthFilter::updateSeedsLoop, this)); }
  void stopThread() {
    if (!thread_) return;
    seeds_updating_halt_ = true;
    { std::lock_guard<std::mutex> lock(frame_queue_mut_); quit_ = true; }
    frame_queue_cond_.notify_one();
    thread_->join();
    thread_.reset();
    quit_ = false;
  }
  // depth_filter.cpp:88-99
  void addFrame(FramePtr frame) {
    if (thread_) {
      {
        std::lock_guard<std::mutex> lock(frame_queue_mut_);
        if (frame_queue_.size() > 2) frame_queue_.pop();
        frame_queue_.push(frame);
      }
      seeds_updating_halt_ = false;
      frame_queue_cond_.notify_one();
    } else {
      updateSeeds(frame);
    }
  }
  // depth_filter.cpp:101-114 + initializeSeeds :116-132: detect new corners away from the frame's features
  void addKeyframe(FramePtr frame, double depth_mean, double depth_min) {
    if (!feature_detector_) throw std::runtime_error("DepthFilter: no feature detector (use the overload that takes the features)");
    new_keyframe_min_depth_ = depth_min;
    new_keyframe_mean_depth_ = depth_mean;
    if (thread_) {
      { std::lock_guard<std::mutex> lock(frame_queue_mut_); new_keyframe_ = frame; new_keyframe_set_ = true; }
      seeds_updating_halt_ = true;
      frame_queue_cond_.notify_one();
    } else {
      initializeSeeds(frame);
    }
  }
  // the same with the detector's output passed in (synchronous)
  void addKeyframe(FramePtr frame, const std::vector<Feature*>& new_features, double depth_mean, double depth_min) {
    seeds_updating_halt_ = true;
    std::lock_guard<std::mutex> lock(seeds_mut_);
    keyframes_.push_back(frame);
    ++Seed::batch_counter();
    for (Feature* ftr : new_features) seeds_.push_back(Seed(ftr, (float)depth_mean, (float)depth_min));
    seeds_updating_halt_ = false;
  }
  bool idle() {  // test helper: the mapper has drained its queue
    std::lock_guard<std::mutex> lock(frame_queue_mut_);
    return frame_queue_.empty() && !new_keyframe_set_ && !busy_;
  }
  void removeKeyframe(FramePtr frame) {                  // :134-151
    seeds_updating_halt_ = true;
    std::lock_guard<std::mutex> lock(seeds_mut_);
    seeds_.remove_if([&](const Seed& s) { return s.ftr->frame == frame.get(); });
    keyframes_.remove(frame);
    seeds_updating_halt_ = false;
  }
  void reset() { seeds_updating_halt_ = true; { std::lock_guard<std::mutex> lock(seeds_mut_); seeds_.clear(); } keyframes_.clear(); seeds_updating_halt_ = false; }
  std::list<Seed>& getSeeds() { return seeds_; }
  // depth_filter.cpp:182-195: copy of the seeds that belong to `frame`
  void getSeedsCopy(const FramePtr& frame, std::list<Seed>& seeds) {
    std::lock_guard<std::mutex> lock(seeds_mut_);
    for (const Seed& s : seeds_)
      if (s.ftr->frame == frame.get()) seeds.push_back(s);
  }
  std::atomic<bool> seeds_updating_halt_{false};  // depth_filter.h:140: set while the seed list is being edited elsewhere
  size_t n_failed_matches_ = 0, n_updates_ = 0;

  // One updateSeeds call between the gather and the apply: the seed list flattened in list order, the keyframe table
  // its ref_index points into, and the buffers the C ABI writes.
  struct SeedGather {
    std::vector<FramePtr> refs;
    std::vector<const svo_b200_frame*> ref_dev;
    std::vector<double> ref_T;
    std::vector<int> ref_index, level, type, batch;
    std::vector<double> px, f, grad, px_cur, z;
    std::vector<float> a, b, mu, zr, s2;
    std::vector<uint8_t> status;
  };

  // depth_filter.cpp:197-291: one launch for all seeds, then the list side effects in list order
  virtual void updateSeeds(FramePtr frame) {
    std::lock_guard<std::mutex> lock(seeds_mut_);  // lock_t lock(seeds_mut_)  (:202)
    SeedGather g;
    if (!gatherSeeds(g)) return;
    const size_t M = g.ref_index.size();
    const svo_b200_camera cam = frame->cam_->c_abi();
    const svo_b200_depth_options opt = abiOptions();
    const svo_b200_epipolar_options eo = matcher_.abiEpipolarOptions();
    Context& c = ctx_ ? *ctx_ : frame->context();
    c.check(svo_b200_set_epipolar_options(c.get(), &eo));
    c.check(svo_b200_depth_filter_update(c.get(), g.ref_dev.data(), g.ref_T.data(), (int)g.refs.size(), frame->device(),
                                         frame->T_f_w_.m, &cam, &opt, (int)M, g.ref_index.data(), g.px.data(), g.f.data(),
                                         g.level.data(), g.type.data(), g.grad.data(), g.batch.data(), Seed::batch_counter(),
                                         g.a.data(), g.b.data(), g.mu.data(), g.zr.data(), g.s2.data(), g.status.data(),
                                         g.px_cur.data(), g.z.data(), nullptr));
    applySeeds(frame, g);
  }

 protected:
  friend void streams::updateSeeds(const std::vector<DepthFilter*>&, const std::vector<FramePtr>&);
  friend void streams::addKeyframes(const std::vector<DepthFilter*>&, const std::vector<FramePtr>&, const std::vector<double>&,
                                    const std::vector<double>&);
  // depth_filter.h:152: the Matcher whose findEpipolarMatchDirect updateSeeds calls; a subclass may set its options_
  // (align_1d, subpix_refinement, the edgelet filter, align_max_iter, max_epi_search_steps), which every launch reads.
  Matcher matcher_;
  svo_b200_depth_options abiOptions() const {
    return {options_.max_n_kfs, options_.seed_convergence_sigma2_thresh, options_.max_search_level,
            matcher_.options_.align_max_iter, (int)matcher_.options_.max_epi_search_steps};
  }
  // The gather of updateSeeds (seeds_mut_ held).  false: nothing to launch -- halted (:212) or no seeds.
  bool gatherSeeds(SeedGather& g) {
    if (seeds_updating_halt_) return false;  // (:212) checked before the launch ...
    const size_t M = seeds_.size();
    if (M == 0) return false;
    g.refs.assign(keyframes_.begin(), keyframes_.end());
    g.ref_dev.resize(g.refs.size());
    g.ref_T.resize(12 * g.refs.size());
    for (size_t r = 0; r < g.refs.size(); ++r) { g.ref_dev[r] = g.refs[r]->device(); std::memcpy(&g.ref_T[12 * r], g.refs[r]->T_f_w_.m, sizeof(double) * 12); }
    g.ref_index.resize(M); g.level.resize(M); g.type.resize(M); g.batch.resize(M);
    g.px.resize(2 * M); g.f.resize(3 * M); g.grad.resize(2 * M); g.px_cur.resize(2 * M); g.z.resize(M);
    g.a.resize(M); g.b.resize(M); g.mu.resize(M); g.zr.resize(M); g.s2.resize(M);
    g.status.resize(M);
    size_t i = 0;
    for (const Seed& s : seeds_) {
      size_t r = 0;
      while (r < g.refs.size() && g.refs[r].get() != s.ftr->frame) ++r;
      if (r == g.refs.size()) throw std::runtime_error("DepthFilter: seed references a frame that is not a keyframe");
      g.ref_index[i] = (int)r; g.level[i] = s.ftr->level; g.type[i] = s.ftr->type; g.batch[i] = s.batch_id;
      g.px[2 * i] = s.ftr->px[0]; g.px[2 * i + 1] = s.ftr->px[1];
      g.grad[2 * i] = s.ftr->grad[0]; g.grad[2 * i + 1] = s.ftr->grad[1];
      for (int k = 0; k < 3; ++k) g.f[3 * i + k] = s.ftr->f[k];
      g.a[i] = s.a; g.b[i] = s.b; g.mu[i] = s.mu; g.zr[i] = s.z_range; g.s2[i] = s.sigma2;
      ++i;
    }
    return true;
  }
  // The apply of updateSeeds (seeds_mut_ held): the list side effects in list order.
  void applySeeds(const FramePtr& frame, const SeedGather& g) {
    if (seeds_updating_halt_) return;  // ... and before the results are applied: a halted call changes nothing
    const std::vector<float>&a = g.a, &b = g.b, &mu = g.mu, &s2 = g.s2;
    const std::vector<uint8_t>& status = g.status;
    const std::vector<double>& px_cur = g.px_cur;
    size_t i = 0;
    for (auto it = seeds_.begin(); it != seeds_.end(); ++i) {
      it->a = a[i]; it->b = b[i]; it->mu = mu[i]; it->sigma2 = s2[i];
      // the feature detector should not initialise new seeds close to a seed that was just matched in a keyframe (:254-258)
      if (frame->isKeyframe() && feature_detector_ &&
          (status[i] == SVO_B200_SEED_UPDATED || status[i] == SVO_B200_SEED_CONVERGED || status[i] == SVO_B200_SEED_NAN))
        feature_detector_->setGridOccpuancy(Vector2d{px_cur[2 * i], px_cur[2 * i + 1]});
      switch (status[i]) {
        case SVO_B200_SEED_TOO_OLD: it = seeds_.erase(it); continue;                       // :216-219
        case SVO_B200_SEED_NO_MATCH: ++n_failed_matches_; break;                           // :240-244
        case SVO_B200_SEED_CONVERGED: {                                                    // :261-282
          ++n_updates_;
          const SE3 T_w_f = it->ftr->frame->T_f_w_.inverse();
          const double d = 1.0 / it->mu;
          const Vector3d p{it->ftr->f[0] * d, it->ftr->f[1] * d, it->ftr->f[2] * d};
          Vector3d xyz_world;
          for (int r = 0; r < 3; ++r) xyz_world[r] = T_w_f.m[r * 4] * p[0] + T_w_f.m[r * 4 + 1] * p[1] + T_w_f.m[r * 4 + 2] * p[2] + T_w_f.m[r * 4 + 3];
          Point* point = new Point(xyz_world, it->ftr);  // (:265) the seed's feature is the point's first observation
          it->ftr->point = point;
          seed_converged_cb_(point, it->sigma2);
          it = seeds_.erase(it);
          continue;
        }
        case SVO_B200_SEED_NAN: ++n_updates_; it = seeds_.erase(it); continue;             // :283-287
        case SVO_B200_SEED_UPDATED: ++n_updates_; break;
        default: break;  // behind the camera / not in frame: untouched
      }
      ++it;
    }
  }

  // depth_filter.cpp:116-132
  void initializeSeeds(FramePtr frame) {
    Features new_features;
    feature_detector_->setExistingFeatures(frame->fts_);
    feature_detector_->detect(frame.get(), triang_min_corner_score_, new_features, ctx_);
    addKeyframe(frame, std::vector<Feature*>(new_features.begin(), new_features.end()), new_keyframe_mean_depth_,
                new_keyframe_min_depth_);
  }
  // depth_filter.cpp:153-180: the mapper thread; a pending keyframe takes precedence over queued frames
  void updateSeedsLoop() {
    for (;;) {
      FramePtr frame;
      bool is_new_kf = false;
      {
        std::unique_lock<std::mutex> lock(frame_queue_mut_);
        frame_queue_cond_.wait(lock, [&] { return quit_ || new_keyframe_set_ || !frame_queue_.empty(); });
        if (quit_) return;
        if (new_keyframe_set_) {
          new_keyframe_set_ = false;
          seeds_updating_halt_ = false;
          while (!frame_queue_.empty()) frame_queue_.pop();  // clear_frame_queue (:166)
          frame = new_keyframe_;
          is_new_kf = true;
        } else {
          frame = frame_queue_.front();
          frame_queue_.pop();
        }
        busy_ = true;
      }
      updateSeeds(frame);
      if (is_new_kf) initializeSeeds(frame);  // frame->isKeyframe() (:176-177)
      { std::lock_guard<std::mutex> lock(frame_queue_mut_); busy_ = false; }
    }
  }
  callback_t seed_converged_cb_;
  feature_detection::DetectorPtr feature_detector_;
  std::list<Seed> seeds_;
  std::mutex seeds_mut_;
  std::list<FramePtr> keyframes_;
  Context* ctx_ = nullptr;
  std::unique_ptr<std::thread> thread_;
  std::queue<FramePtr> frame_queue_;
  std::mutex frame_queue_mut_;
  std::condition_variable frame_queue_cond_;
  FramePtr new_keyframe_;
  bool new_keyframe_set_ = false, quit_ = false, busy_ = false;
  double new_keyframe_min_depth_ = 0.0, new_keyframe_mean_depth_ = 0.0;

 public:
  double triang_min_corner_score_ = 20.0;  // Config::triangMinCornerScore() (config.cpp:44)
};

// ------------------------------------------------------------------------------------------------
// svo::Map / MapPointCandidates (svo/include/svo/map.h:32-129): the parts Reprojector::reprojectMap touches.
// ------------------------------------------------------------------------------------------------
class MapPointCandidates {
 public:
  typedef std::pair<Point*, Feature*> PointCandidate;
  std::list<PointCandidate> candidates_;
  std::list<Point*> trash_points_;
  std::mutex mut_;  // map.h:47: the depth filter (mapper thread) appends while the tracker reads
  ~MapPointCandidates() { reset(); }
  void newCandidatePoint(Point* point, double /*depth_sigma2*/) {  // map.cpp:213-218
    point->type_ = Point::TYPE_CANDIDATE;
    std::lock_guard<std::mutex> lock(mut_);
    candidates_.push_back(PointCandidate(point, point->obs_.front()));
  }
  void addCandidatePointToFrame(const std::shared_ptr<Frame>& frame);  // map.cpp:220-237
  void deleteCandidate(PointCandidate& c) {  // map.cpp:280-287
    delete c.second; c.second = nullptr;
    c.first->type_ = Point::TYPE_DELETED;
    trash_points_.push_back(c.first);
  }
  bool deleteCandidatePoint(Point* point) {  // map.cpp:239-252
    for (auto it = candidates_.begin(); it != candidates_.end(); ++it)
      if (it->first == point) { deleteCandidate(*it); candidates_.erase(it); return true; }
    return false;
  }
  void emptyTrash() { for (Point* p : trash_points_) delete p; trash_points_.clear(); }
  void reset() { for (auto& c : candidates_) { delete c.first; delete c.second; } candidates_.clear(); }
};

class Map {
 public:
  std::list<FramePtr> keyframes_;
  std::list<Point*> trash_points_;
  MapPointCandidates point_candidates_;
  void addKeyframe(FramePtr kf) { keyframes_.push_back(kf); }
  void safeDeletePoint(Point* pt) {  // map.cpp:82-99
    for (Feature* ftr : pt->obs_) {
      ftr->point = nullptr;
      for (Feature*& k : ftr->frame->key_pts_) if (k == ftr) k = nullptr;  // Frame::removeKeyPoint without re-selection
    }
    pt->obs_.clear();
    pt->type_ = Point::TYPE_DELETED;
    trash_points_.push_back(pt);
  }
  void emptyTrash() { for (Point* p : trash_points_) delete p; trash_points_.clear(); point_candidates_.emptyTrash(); }
};

// ------------------------------------------------------------------------------------------------
// svo::Reprojector (svo/include/svo/reprojector.h:37-99): reprojectMap gathers the pointer graph into a flat
// svo_b200_map_view, makes ONE device call (projection + speculative alignment of every in-frame point), and applies
// the results the C ABI replayed in the reference's cell order: new Features on the frame, point counters / types,
// safeDeletePoint / deleteCandidatePoint.
// ------------------------------------------------------------------------------------------------
struct ReprojectorOptions {
  size_t max_n_kfs = 10;          // reprojector.h:44
  bool find_match_direct = true;  // reprojector.h:45
  int grid_size = 30, max_fts = 120, n_pyr_levels = 3;  // Config::gridSize(), maxFts(), nPyrLevels()
};
class Reprojector {
 public:
  typedef ReprojectorOptions Options;
  Options options_;
  size_t n_matches_ = 0, n_trials_ = 0;

  Reprojector(AbstractCamera* cam, Map& map, Options opt = Options(), unsigned shuffle_seed = 1) : options_(opt), map_(map) {
    // initializeGrid (reprojector.cpp:47-58); the reference shuffles with rand(), here a seeded LCG Fisher-Yates
    const int cols = (cam->width_ + options_.grid_size - 1) / options_.grid_size, rows = (cam->height_ + options_.grid_size - 1) / options_.grid_size;
    cell_order_.resize((size_t)cols * rows);
    for (size_t i = 0; i < cell_order_.size(); ++i) cell_order_[i] = (int)i;
    uint64_t s = shuffle_seed;
    for (size_t i = cell_order_.size(); i > 1; --i) {
      s = s * 6364136223846793005ULL + 1442695040888963407ULL;
      std::swap(cell_order_[i - 1], cell_order_[(size_t)((s >> 33) % i)]);
    }
  }
  std::vector<int>& cellOrder() { return cell_order_; }

  // One reprojectMap call between the gather and the apply: the map's pointer graph as the flat svo_b200_map_view
  // arrays, and the buffers the C ABI writes.  `view` points into the vectors, so a MapGather is never copied or moved.
  struct MapGather {
    MapGather() = default;
    MapGather(const MapGather&) = delete;
    MapGather& operator=(const MapGather&) = delete;
    std::vector<FramePtr> kfs;
    std::vector<Feature*> ftrs;
    std::vector<Point*> pts;
    std::vector<int> kf_fts_offset, kf_fts, cand_point, pt_obs_offset, pt_obs, ftr_kf, ftr_level, ftr_type, ftr_point, pt_type,
        pt_failed, pt_succ;
    std::vector<double> kf_T, keypt_pos, ftr_px, ftr_f, ftr_grad, pt_pos;
    std::vector<uint8_t> keypt_valid, action;
    std::vector<const svo_b200_frame*> kf_dev;
    std::vector<int> ov_kf, new_point, new_level, new_type;
    std::vector<int64_t> ov_count;
    std::vector<double> new_px, new_grad;
    svo_b200_map_view view;
    svo_b200_reproject_options opt;
    svo_b200_camera cam;
    svo_b200_reproject_stats st;
  };

  void reprojectMap(FramePtr frame, std::vector<std::pair<FramePtr, size_t>>& overlap_kfs) {
    MapGather g;
    gatherMap(frame, g);
    Context& c = frame->context();
    c.check(svo_b200_reproject_map(c.get(), &g.view, g.kf_dev.data(), frame->device(), frame->T_f_w_.m, &g.cam, &g.opt,
                                   cell_order_.data(), g.pt_type.data(), g.pt_failed.data(), g.pt_succ.data(), g.action.data(),
                                   g.ov_kf.data(), g.ov_count.data(), g.new_point.data(), g.new_px.data(), g.new_level.data(),
                                   g.new_type.data(), g.new_grad.data(), &g.st));
    applyMap(frame, g, overlap_kfs);
  }

 private:
  friend void streams::reprojectMap(const std::vector<Reprojector*>&, const std::vector<FramePtr>&,
                                    std::vector<std::vector<std::pair<FramePtr, size_t>>>&);
  // The gather of reprojectMap: Map::keyframes_ (pose, device pyramid, key_pts_ positions, fts_), every Feature reachable
  // through fts_ / Point::obs_, every Point, point_candidates_.candidates_, and the options.
  void gatherMap(const FramePtr& frame, MapGather& g) {
    n_matches_ = n_trials_ = 0;
    g.kfs.assign(map_.keyframes_.begin(), map_.keyframes_.end());
    std::vector<FramePtr>& kfs = g.kfs;
    std::map<const Frame*, int> kf_index;
    for (size_t k = 0; k < kfs.size(); ++k) kf_index[kfs[k].get()] = (int)k;
    std::map<Feature*, int> ftr_index;
    std::map<Point*, int> pt_index;
    std::vector<Feature*>& ftrs = g.ftrs;
    std::vector<Point*>& pts = g.pts;
    auto ftr_id = [&](Feature* f) { auto it = ftr_index.find(f); if (it != ftr_index.end()) return it->second; ftr_index[f] = (int)ftrs.size(); ftrs.push_back(f); return (int)ftrs.size() - 1; };
    auto pt_id = [&](Point* p) { auto it = pt_index.find(p); if (it != pt_index.end()) return it->second; pt_index[p] = (int)pts.size(); pts.push_back(p); return (int)pts.size() - 1; };
    g.kf_fts_offset.assign(kfs.size() + 1, 0);
    g.kf_T.resize(12 * kfs.size());
    g.keypt_pos.assign(15 * kfs.size(), 0.0);
    g.keypt_valid.assign(5 * kfs.size(), 0);
    g.kf_dev.resize(kfs.size());
    for (size_t k = 0; k < kfs.size(); ++k) {
      g.kf_dev[k] = kfs[k]->device();
      std::memcpy(&g.kf_T[12 * k], kfs[k]->T_f_w_.m, sizeof(double) * 12);
      for (Feature* f : kfs[k]->fts_) { g.kf_fts.push_back(ftr_id(f)); if (f->point) pt_id(f->point); }
      g.kf_fts_offset[k + 1] = (int)g.kf_fts.size();
      for (int i = 0; i < 5; ++i) {
        Feature* kp = kfs[k]->key_pts_[i];
        if (!kp || !kp->point) continue;
        g.keypt_valid[5 * k + i] = 1;
        for (int c = 0; c < 3; ++c) g.keypt_pos[3 * (5 * k + i) + c] = kp->point->pos_[c];
      }
    }
    for (auto& c : map_.point_candidates_.candidates_) g.cand_point.push_back(pt_id(c.first));
    g.pt_obs_offset.assign(1, 0);
    for (size_t p = 0; p < pts.size(); ++p) {  // obs_ may reach features outside any fts_ list (candidates) -> extends ftrs
      for (Feature* f : pts[p]->obs_) g.pt_obs.push_back(ftr_id(f));
      g.pt_obs_offset.push_back((int)g.pt_obs.size());
    }
    const size_t F = ftrs.size(), P = pts.size();
    g.ftr_kf.resize(F); g.ftr_level.resize(F); g.ftr_type.resize(F); g.ftr_point.resize(F);
    g.pt_type.resize(P); g.pt_failed.resize(P); g.pt_succ.resize(P);
    g.ftr_px.resize(2 * F); g.ftr_f.resize(3 * F); g.ftr_grad.resize(2 * F); g.pt_pos.resize(3 * P);
    for (size_t i = 0; i < F; ++i) {
      const Feature* f = ftrs[i];
      auto it = kf_index.find(f->frame);
      if (it == kf_index.end()) throw std::runtime_error("Reprojector: a point is observed from a frame that is not a map keyframe");
      g.ftr_kf[i] = it->second; g.ftr_level[i] = f->level; g.ftr_type[i] = f->type;
      g.ftr_point[i] = f->point ? pt_index.at(f->point) : -1;
      g.ftr_px[2 * i] = f->px[0]; g.ftr_px[2 * i + 1] = f->px[1];
      g.ftr_grad[2 * i] = f->grad[0]; g.ftr_grad[2 * i + 1] = f->grad[1];
      for (int c = 0; c < 3; ++c) g.ftr_f[3 * i + c] = f->f[c];
    }
    for (size_t p = 0; p < P; ++p) {
      g.pt_type[p] = pts[p]->type_; g.pt_failed[p] = pts[p]->n_failed_reproj_; g.pt_succ[p] = pts[p]->n_succeeded_reproj_;
      for (int c = 0; c < 3; ++c) g.pt_pos[3 * p + c] = pts[p]->pos_[c];
    }
    g.view = {(int)kfs.size(), g.kf_T.data(), g.keypt_pos.data(), g.keypt_valid.data(), g.kf_fts_offset.data(),
              g.kf_fts.data(), (int)F, g.ftr_kf.data(), g.ftr_px.data(), g.ftr_f.data(), g.ftr_level.data(),
              g.ftr_type.data(), g.ftr_grad.data(), g.ftr_point.data(), (int)P, g.pt_pos.data(),
              g.pt_obs_offset.data(), g.pt_obs.data(), (int)g.cand_point.size(), g.cand_point.data()};
    g.opt = {options_.grid_size, options_.max_fts, (int)options_.max_n_kfs, options_.find_match_direct ? 1 : 0,
             options_.n_pyr_levels - 1, 10};
    const size_t cap = (size_t)options_.max_fts + 1;
    g.action.resize(P);
    g.ov_kf.resize(options_.max_n_kfs); g.ov_count.resize(options_.max_n_kfs);
    g.new_point.resize(cap); g.new_level.resize(cap); g.new_type.resize(cap);
    g.new_px.resize(2 * cap); g.new_grad.resize(2 * cap);
    g.cam = frame->cam_->c_abi();
  }

  // The apply of reprojectMap (reprojector.cpp:183-196 and the point bookkeeping): overlap keyframes, the new features on
  // the frame, point counters and types, safeDeletePoint / deleteCandidatePoint.
  void applyMap(const FramePtr& frame, const MapGather& g, std::vector<std::pair<FramePtr, size_t>>& overlap_kfs) {
    n_matches_ = (size_t)g.st.n_matches;
    n_trials_ = (size_t)g.st.n_trials;
    overlap_kfs.reserve(options_.max_n_kfs);
    for (int i = 0; i < g.st.n_overlap; ++i) overlap_kfs.push_back(std::make_pair(g.kfs[g.ov_kf[i]], (size_t)g.ov_count[i]));
    for (int q = 0; q < g.st.n_new; ++q) {  // reprojector.cpp:183-196
      Feature* nf = new Feature(frame.get(), Vector2d{g.new_px[2 * q], g.new_px[2 * q + 1]}, g.new_level[q]);
      nf->point = g.pts[g.new_point[q]];
      if (g.new_type[q]) { nf->type = Feature::EDGELET; nf->grad = Vector2d{g.new_grad[2 * q], g.new_grad[2 * q + 1]}; }
      frame->addFeature(nf);
    }
    for (size_t p = 0; p < g.pts.size(); ++p) {
      g.pts[p]->n_failed_reproj_ = g.pt_failed[p];
      g.pts[p]->n_succeeded_reproj_ = g.pt_succ[p];
      switch (g.action[p]) {
        case SVO_B200_PT_SAFE_DELETE: map_.safeDeletePoint(g.pts[p]); break;
        case SVO_B200_PT_DELETE_CANDIDATE:
        case SVO_B200_PT_CANDIDATE_ERASED: map_.point_candidates_.deleteCandidatePoint(g.pts[p]); break;
        default: g.pts[p]->type_ = (Point::PointType)g.pt_type[p];
      }
    }
  }

  Map& map_;
  std::vector<int> cell_order_;
};

// ------------------------------------------------------------------------------------------------
// svo::streams: S independent camera streams (one DepthFilter / Reprojector and one frame each) with ONE device launch
// per stage (svo_b200_depth_filter_update_streams, svo_b200_reproject_map_streams).  Each object's gather and apply are
// the code of its own updateSeeds / reprojectMap, run in list order per object, so every object ends exactly as after
// its own call: seed erasures, convergence callbacks, keyframe grid occupancy; point counters, deletions, new features.
// The device work runs on the context of frames[0] (of filters[0]'s own context, if it has one); every frame must live
// on that context's device.
// ------------------------------------------------------------------------------------------------
namespace streams {

// DepthFilter::updateSeeds(frames[s]) of every filters[s], for filters WITHOUT a thread of their own: the reference's
// synchronous mode, where addFrame falls through to updateSeeds (depth_filter.cpp:95-96).  The filters must be distinct
// and share their options, their matcher_'s included (one svo_b200_depth_options and one epipolar setting per launch;
// std::invalid_argument before any launch otherwise); a halted filter is skipped as its own call skips.
inline void updateSeeds(const std::vector<DepthFilter*>& filters, const std::vector<FramePtr>& frames) {
  const size_t S = filters.size();
  if (frames.size() != S) throw std::invalid_argument("streams::updateSeeds: one frame per filter");
  if (S == 0) return;
  for (size_t s = 0; s < S; ++s) {
    if (!filters[s] || !frames[s]) throw std::invalid_argument("streams::updateSeeds: NULL filter or frame");
    if (filters[s]->thread_) throw std::invalid_argument("streams::updateSeeds: a filter runs its own mapper thread");
    for (size_t t = 0; t < s; ++t)
      if (filters[t] == filters[s]) throw std::invalid_argument("streams::updateSeeds: a filter is listed twice");
  }
  const svo_b200_depth_options opt = filters[0]->abiOptions();
  const svo_b200_epipolar_options eo = filters[0]->matcher_.abiEpipolarOptions();
  for (DepthFilter* df : filters) {
    const svo_b200_depth_options o = df->abiOptions();
    const svo_b200_epipolar_options e = df->matcher_.abiEpipolarOptions();
    if (o.max_n_kfs != opt.max_n_kfs || o.seed_convergence_sigma2_thresh != opt.seed_convergence_sigma2_thresh ||
        o.max_search_level != opt.max_search_level)
      throw std::invalid_argument("streams::updateSeeds: the filters' options differ");
    if (o.align_max_iter != opt.align_max_iter || o.max_epi_search_steps != opt.max_epi_search_steps ||
        e.align_1d != eo.align_1d || e.subpix_refinement != eo.subpix_refinement ||
        e.epi_search_edgelet_filtering != eo.epi_search_edgelet_filtering ||
        std::memcmp(&e.epi_search_edgelet_max_angle, &eo.epi_search_edgelet_max_angle, sizeof(double)) != 0)
      throw std::invalid_argument("streams::updateSeeds: the filters' matcher_.options_ differ");
  }
  std::vector<std::unique_lock<std::mutex>> locks;
  for (DepthFilter* df : filters) locks.emplace_back(df->seeds_mut_);
  std::vector<DepthFilter::SeedGather> g(S);
  std::vector<char> active(S, 0);
  for (size_t s = 0; s < S; ++s) active[s] = filters[s]->gatherSeeds(g[s]) ? 1 : 0;
  // concatenation: one keyframe table (each filter's keyframes in turn), the seeds of stream s at seed_offset[s]
  std::vector<const svo_b200_frame*> cur(S), ref_dev;
  std::vector<double> cur_T(12 * S), ref_T;
  std::vector<svo_b200_camera> cam(S);
  std::vector<int> counter(S, Seed::batch_counter()), seed_offset(S + 1, 0), ref_index, level, type, batch;
  std::vector<double> px, f, grad;
  std::vector<float> a, b, mu, zr, s2;
  for (size_t s = 0; s < S; ++s) {
    cur[s] = frames[s]->device();
    std::memcpy(&cur_T[12 * s], frames[s]->T_f_w_.m, sizeof(double) * 12);
    cam[s] = frames[s]->cam_->c_abi();
    seed_offset[s + 1] = seed_offset[s];
    if (!active[s]) continue;
    const DepthFilter::SeedGather& x = g[s];
    const int base = (int)ref_dev.size();
    ref_dev.insert(ref_dev.end(), x.ref_dev.begin(), x.ref_dev.end());
    ref_T.insert(ref_T.end(), x.ref_T.begin(), x.ref_T.end());
    for (int r : x.ref_index) ref_index.push_back(base + r);
    level.insert(level.end(), x.level.begin(), x.level.end());
    type.insert(type.end(), x.type.begin(), x.type.end());
    batch.insert(batch.end(), x.batch.begin(), x.batch.end());
    px.insert(px.end(), x.px.begin(), x.px.end());
    f.insert(f.end(), x.f.begin(), x.f.end());
    grad.insert(grad.end(), x.grad.begin(), x.grad.end());
    a.insert(a.end(), x.a.begin(), x.a.end());
    b.insert(b.end(), x.b.begin(), x.b.end());
    mu.insert(mu.end(), x.mu.begin(), x.mu.end());
    zr.insert(zr.end(), x.zr.begin(), x.zr.end());
    s2.insert(s2.end(), x.s2.begin(), x.s2.end());
    seed_offset[s + 1] += (int)x.ref_index.size();
  }
  const size_t M = (size_t)seed_offset[S];
  if (M == 0) return;
  std::vector<uint8_t> status(M);
  std::vector<double> px_cur(2 * M), z(M);
  Context& c = filters[0]->ctx_ ? *filters[0]->ctx_ : frames[0]->context();
  c.check(svo_b200_set_epipolar_options(c.get(), &eo));
  c.check(svo_b200_depth_filter_update_streams(c.get(), (int)S, cur.data(), cur_T.data(), cam.data(), counter.data(),
                                               seed_offset.data(), ref_dev.data(), ref_T.data(), (int)ref_dev.size(), &opt,
                                               ref_index.data(), px.data(), f.data(), level.data(), type.data(), grad.data(),
                                               batch.data(), a.data(), b.data(), mu.data(), zr.data(), s2.data(),
                                               status.data(), px_cur.data(), z.data(), nullptr));
  for (size_t s = 0; s < S; ++s) {
    if (!active[s]) continue;
    DepthFilter::SeedGather& x = g[s];
    const size_t o = (size_t)seed_offset[s], n = x.ref_index.size();
    std::copy(a.begin() + o, a.begin() + o + n, x.a.begin());
    std::copy(b.begin() + o, b.begin() + o + n, x.b.begin());
    std::copy(mu.begin() + o, mu.begin() + o + n, x.mu.begin());
    std::copy(s2.begin() + o, s2.begin() + o + n, x.s2.begin());
    std::copy(status.begin() + o, status.begin() + o + n, x.status.begin());
    std::copy(px_cur.begin() + 2 * o, px_cur.begin() + 2 * (o + n), x.px_cur.begin());
    std::copy(z.begin() + o, z.begin() + o + n, x.z.begin());
    filters[s]->applySeeds(frames[s], x);
  }
}

// DepthFilter::addKeyframe(frames[s], depth_mean[s], depth_min[s]) of every filters[s] -- initializeSeeds with one
// detection launch -- for filters WITHOUT a thread of their own (the reference's synchronous mode, depth_filter.cpp:110-113).
// Every filter's grid is filled from its keyframe's features, all keyframes are detected in one launch, and then each
// filter takes its new seeds in stream order: Seed::batch_counter() and Seed::seed_counter() are process-wide, and only
// that order leaves batch and seed ids as S sequential calls leave them.  Refused with std::invalid_argument before any
// object changes: a filter listed twice, one with a thread, one without a detector or with one that is not a
// FastDetector, and two filters sharing one detector (sequential calls would fill, detect and reset its grid once per
// filter, which one launch cannot reproduce).
inline void addKeyframes(const std::vector<DepthFilter*>& filters, const std::vector<FramePtr>& frames,
                         const std::vector<double>& depth_mean, const std::vector<double>& depth_min) {
  const size_t S = filters.size();
  if (frames.size() != S || depth_mean.size() != S || depth_min.size() != S)
    throw std::invalid_argument("streams::addKeyframes: one frame and one depth pair per filter");
  if (S == 0) return;
  std::vector<feature_detection::FastDetector*> detectors(S);
  for (size_t s = 0; s < S; ++s) {
    if (!filters[s] || !frames[s]) throw std::invalid_argument("streams::addKeyframes: NULL filter or frame");
    if (filters[s]->thread_) throw std::invalid_argument("streams::addKeyframes: a filter runs its own mapper thread");
    if (!filters[s]->feature_detector_) throw std::invalid_argument("streams::addKeyframes: a filter has no feature detector");
    detectors[s] = dynamic_cast<feature_detection::FastDetector*>(filters[s]->feature_detector_.get());
    if (!detectors[s]) throw std::invalid_argument("streams::addKeyframes: a filter's detector is not a FastDetector");
    for (size_t t = 0; t < s; ++t) {
      if (filters[t] == filters[s]) throw std::invalid_argument("streams::addKeyframes: a filter is listed twice");
      if (detectors[t] == detectors[s]) throw std::invalid_argument("streams::addKeyframes: two filters share one detector");
    }
  }
  std::vector<double> thresholds(S);
  for (size_t s = 0; s < S; ++s) {  // addKeyframe (:103-104), then initializeSeeds up to the detection (:119-120)
    DepthFilter& df = *filters[s];
    df.new_keyframe_min_depth_ = depth_min[s];
    df.new_keyframe_mean_depth_ = depth_mean[s];
    df.feature_detector_->setExistingFeatures(frames[s]->fts_);
    thresholds[s] = df.triang_min_corner_score_;
  }
  std::vector<Features> fts(S);
  detect(detectors, frames, thresholds, fts, filters[0]->ctx_);
  for (size_t s = 0; s < S; ++s) {
    DepthFilter& df = *filters[s];
    df.addKeyframe(frames[s], std::vector<Feature*>(fts[s].begin(), fts[s].end()), df.new_keyframe_mean_depth_,
                   df.new_keyframe_min_depth_);
  }
}

// Reprojector::reprojectMap(frames[s], overlap_kfs[s]) of every reprojectors[s].  The reprojectors must be distinct, and
// so must their maps (the replay of one stream must not see another's changes to a shared map).
inline void reprojectMap(const std::vector<Reprojector*>& reprojectors, const std::vector<FramePtr>& frames,
                         std::vector<std::vector<std::pair<FramePtr, size_t>>>& overlap_kfs) {
  const size_t S = reprojectors.size();
  if (frames.size() != S || overlap_kfs.size() != S)
    throw std::invalid_argument("streams::reprojectMap: one frame and one overlap list per reprojector");
  if (S == 0) return;
  for (size_t s = 0; s < S; ++s) {
    if (!reprojectors[s] || !frames[s]) throw std::invalid_argument("streams::reprojectMap: NULL reprojector or frame");
    for (size_t t = 0; t < s; ++t)
      if (reprojectors[t] == reprojectors[s] || &reprojectors[t]->map_ == &reprojectors[s]->map_)
        throw std::invalid_argument("streams::reprojectMap: a reprojector or a map is listed twice");
  }
  std::vector<std::unique_ptr<Reprojector::MapGather>> g;
  std::vector<svo_b200_reproject_stream> rs(S);
  for (size_t s = 0; s < S; ++s) {
    g.emplace_back(new Reprojector::MapGather);
    Reprojector::MapGather& x = *g.back();
    reprojectors[s]->gatherMap(frames[s], x);
    rs[s] = {&x.view, x.kf_dev.data(), frames[s]->device(), frames[s]->T_f_w_.m, &x.cam, &x.opt,
             reprojectors[s]->cell_order_.data(), x.pt_type.data(), x.pt_failed.data(), x.pt_succ.data(), x.action.data(),
             x.ov_kf.data(), x.ov_count.data(), x.new_point.data(), x.new_px.data(), x.new_level.data(), x.new_type.data(),
             x.new_grad.data(), &x.st};
  }
  Context& c = frames[0]->context();
  c.check(svo_b200_reproject_map_streams(c.get(), (int)S, rs.data()));
  for (size_t s = 0; s < S; ++s) reprojectors[s]->applyMap(frames[s], *g[s], overlap_kfs[s]);
}

}  // namespace streams

inline void MapPointCandidates::addCandidatePointToFrame(const FramePtr& frame) {
  std::lock_guard<std::mutex> lock(mut_);
  for (auto it = candidates_.begin(); it != candidates_.end();) {
    if (it->first->obs_.front()->frame == frame.get()) {
      it->first->type_ = Point::TYPE_UNKNOWN;
      it->first->n_failed_reproj_ = 0;
      it->second->frame->addFeature(it->second);
      it = candidates_.erase(it);
    } else {
      ++it;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// svo::FrameHandlerMono (svo/include/svo/frame_handler_mono.h:34-61), the per-frame driver of the hot path:
//   addImage -> processFrame (frame_handler_mono.cpp:129-245): SparseImgAlign::run -> Reprojector::reprojectMap ->
//   pose_optimizer::optimizeGaussNewton -> optimizeStructure (Point::optimize) -> DepthFilter::addFrame / addKeyframe,
// with the depth filter on a mapper thread that owns a second device context, as the reference's two threads do.
// Outside the hot path and therefore the caller's job here (SURVEY.md 2): the two-view initialisation (KLT +
// homography; setFirstFrame takes the keyframe that processSecondFrame would leave behind), relocalisation, bundle
// adjustment and the keyframe-removal policy.
// ------------------------------------------------------------------------------------------------
struct FrameHandlerMonoOptions {  // svo/src/config.cpp:56-84 defaults
  int n_pyr_levels = 3, klt_max_level = 4, klt_min_level = 2, grid_size = 30, max_fts = 120, quality_min_fts = 50,
      quality_max_drop_fts = 40, poseoptim_num_iter = 10, structureoptim_max_pts = 20, structureoptim_num_iter = 5;
  double poseoptim_thresh = 2.0, kfselect_mindist = 0.12, triang_min_corner_score = 20.0;
  bool mapper_thread = true;
};
class FrameHandlerMono {
 public:
  enum Stage { STAGE_PAUSED, STAGE_FIRST_FRAME, STAGE_DEFAULT_FRAME };
  enum UpdateResult { RESULT_NO_KEYFRAME, RESULT_IS_KEYFRAME, RESULT_FAILURE };
  enum TrackingQuality { TRACKING_INSUFFICIENT, TRACKING_BAD, TRACKING_GOOD };
  typedef FrameHandlerMonoOptions Options;
  struct FrameLog { size_t img_align_n_tracked = 0, repr_n_matches = 0, repr_n_trials = 0, sfba_n_edges_final = 0; double sfba_error_init = 0, sfba_error_final = 0; };

  FrameHandlerMono(AbstractCamera* cam, Options opt = Options(), int device = 0)
      : cam_(cam), opt_(opt), tracking_ctx_(device), mapping_ctx_(device),
        reprojector_(cam, map_, make_reprojector_options(opt)),
        depth_filter_(feature_detection::DetectorPtr(new feature_detection::FastDetector(cam->width_, cam->height_, opt.grid_size, opt.n_pyr_levels)),
                      std::bind(&MapPointCandidates::newCandidatePoint, &map_.point_candidates_, std::placeholders::_1, std::placeholders::_2)) {
    depth_filter_.options_.max_search_level = opt.n_pyr_levels - 1;
    depth_filter_.triang_min_corner_score_ = opt.triang_min_corner_score;
    depth_filter_.setContext(&mapping_ctx_);
    if (opt.mapper_thread) depth_filter_.startThread();
  }
  ~FrameHandlerMono() { depth_filter_.stopThread(); }
  Context& trackingContext() { return tracking_ctx_; }
  // The first keyframe, with its features and map points already attached (what the two-view initialisation produces).
  void setFirstFrame(const FramePtr& first_frame) {
    new_frame_ = first_frame;
    new_frame_->setKeyframe();
    double depth_mean = 0, depth_min = 0;
    getSceneDepth(*new_frame_, depth_mean, depth_min);
    for (Feature* f : new_frame_->fts_)
      if (f->point && std::find(f->point->obs_.begin(), f->point->obs_.end(), f) == f->point->obs_.end()) f->point->addFrameRef(f);
    depth_filter_.addKeyframe(new_frame_, depth_mean, 0.5 * depth_min);
    map_.addKeyframe(new_frame_);
    last_frame_ = new_frame_;
    num_obs_last_ = last_frame_->nObs();
    new_frame_.reset();
    stage_ = STAGE_DEFAULT_FRAME;
  }
  // frame_handler_mono.cpp:62-86
  UpdateResult addImage(const uint8_t* img, const double timestamp) {
    if (stage_ != STAGE_DEFAULT_FRAME) return RESULT_FAILURE;
    core_kfs_.clear();
    overlap_kfs_.clear();
    new_frame_.reset(new Frame(tracking_ctx_, cam_, img, std::max(opt_.n_pyr_levels, opt_.klt_max_level + 1), timestamp));
    const UpdateResult res = processFrame();
    last_frame_ = new_frame_;  // finishFrameProcessing (frame_handler_base.cpp:104-106)
    new_frame_.reset();
    num_obs_last_ = last_frame_->nObs();
    return res;
  }
  FramePtr lastFrame() { return last_frame_; }
  DepthFilter* depthFilter() { return &depth_filter_; }
  Map& map() { return map_; }
  const FrameLog& log() const { return log_; }
  TrackingQuality trackingQuality() const { return tracking_quality_; }

  static bool getSceneDepth(const Frame& frame, double& depth_mean, double& depth_min) {  // frame.cpp:167-188
    std::vector<double> depth_vec;
    depth_min = std::numeric_limits<double>::max();
    const double* m = frame.T_f_w_.m;
    for (Feature* f : frame.fts_) {
      if (!f->point) continue;
      const double z = m[8] * f->point->pos_[0] + m[9] * f->point->pos_[1] + m[10] * f->point->pos_[2] + m[11];
      depth_vec.push_back(z);
      depth_min = std::fmin(z, depth_min);
    }
    if (depth_vec.empty()) return false;
    std::nth_element(depth_vec.begin(), depth_vec.begin() + depth_vec.size() / 2, depth_vec.end());  // vk::getMedian [EXT]
    depth_mean = depth_vec[depth_vec.size() / 2];
    return true;
  }

 protected:
  static Reprojector::Options make_reprojector_options(const Options& o) {
    Reprojector::Options r;
    r.grid_size = o.grid_size; r.max_fts = o.max_fts; r.n_pyr_levels = o.n_pyr_levels;
    return r;
  }
  // frame_handler_mono.cpp:129-245
  UpdateResult processFrame() {
    new_frame_->T_f_w_ = last_frame_->T_f_w_;  // set initial pose
    SparseImgAlign img_align(opt_.klt_max_level, opt_.klt_min_level, 30, SparseImgAlign::GaussNewton, false, false);
    log_ = FrameLog();
    log_.img_align_n_tracked = img_align.run(last_frame_, new_frame_);
    reprojector_.reprojectMap(new_frame_, overlap_kfs_);
    log_.repr_n_matches = reprojector_.n_matches_;
    log_.repr_n_trials = reprojector_.n_trials_;
    if ((int)log_.repr_n_matches < opt_.quality_min_fts) {
      new_frame_->T_f_w_ = last_frame_->T_f_w_;  // reset to avoid crazy pose jumps
      tracking_quality_ = TRACKING_INSUFFICIENT;
      return RESULT_FAILURE;
    }
    double sfba_thresh = 0;
    pose_optimizer::optimizeGaussNewton(opt_.poseoptim_thresh, (size_t)opt_.poseoptim_num_iter, false, new_frame_, sfba_thresh,
                                        log_.sfba_error_init, log_.sfba_error_final, log_.sfba_n_edges_final);
    if (log_.sfba_n_edges_final < 20) return RESULT_FAILURE;
    optimizeStructure(new_frame_, (size_t)opt_.structureoptim_max_pts, opt_.structureoptim_num_iter);
    core_kfs_.insert(new_frame_);
    setTrackingQuality(log_.sfba_n_edges_final);
    if (tracking_quality_ == TRACKING_INSUFFICIENT) {
      new_frame_->T_f_w_ = last_frame_->T_f_w_;
      return RESULT_FAILURE;
    }
    double depth_mean = 0, depth_min = 0;
    getSceneDepth(*new_frame_, depth_mean, depth_min);
    if (!needNewKf(depth_mean) || tracking_quality_ == TRACKING_BAD) {
      depth_filter_.addFrame(new_frame_);
      return RESULT_NO_KEYFRAME;
    }
    new_frame_->setKeyframe();
    for (Feature* f : new_frame_->fts_)
      if (f->point) f->point->addFrameRef(f);
    map_.point_candidates_.addCandidatePointToFrame(new_frame_);
    depth_filter_.addKeyframe(new_frame_, depth_mean, 0.5 * depth_min);
    map_.addKeyframe(new_frame_);
    return RESULT_IS_KEYFRAME;
  }
  // frame_handler_base.cpp:157-171
  void setTrackingQuality(const size_t num_observations) {
    tracking_quality_ = TRACKING_GOOD;
    if ((int)num_observations < opt_.quality_min_fts) tracking_quality_ = TRACKING_INSUFFICIENT;
    const int feature_drop = (int)std::min(num_obs_last_, (size_t)opt_.max_fts) - (int)num_observations;
    if (feature_drop > opt_.quality_max_drop_fts) tracking_quality_ = TRACKING_INSUFFICIENT;
  }
  // frame_handler_mono.cpp:304-315
  bool needNewKf(double scene_depth_mean) {
    for (auto& kf : overlap_kfs_) {
      const Vector3d p = kf.first->pos();
      const double* m = new_frame_->T_f_w_.m;
      const double rx = m[0] * p[0] + m[1] * p[1] + m[2] * p[2] + m[3], ry = m[4] * p[0] + m[5] * p[1] + m[6] * p[2] + m[7],
                   rz = m[8] * p[0] + m[9] * p[1] + m[10] * p[2] + m[11];
      if (std::fabs(rx) / scene_depth_mean < opt_.kfselect_mindist && std::fabs(ry) / scene_depth_mean < opt_.kfselect_mindist * 0.8 &&
          std::fabs(rz) / scene_depth_mean < opt_.kfselect_mindist * 1.3)
        return false;
    }
    return true;
  }
  // frame_handler_base.cpp:178-196: Point::optimize on the points optimised longest ago, one batched device call
  void optimizeStructure(FramePtr frame, size_t max_n_pts, int max_iter) {
    std::vector<Point*> pts;
    for (Feature* f : frame->fts_)
      if (f->point) pts.push_back(f->point);
    max_n_pts = std::min(max_n_pts, pts.size());
    if (max_n_pts == 0) return;
    std::nth_element(pts.begin(), pts.begin() + max_n_pts, pts.end(),
                     [&](Point* a, Point* b) { return last_structure_optim_[a] < last_structure_optim_[b]; });
    std::vector<int> obs_offset(1, 0), obs_frame;
    std::vector<double> obs_f, frame_T, pos;
    std::map<const Frame*, int> fidx;
    for (size_t k = 0; k < max_n_pts; ++k) {
      for (Feature* o : pts[k]->obs_) {
        auto it = fidx.find(o->frame);
        if (it == fidx.end()) {
          it = fidx.emplace(o->frame, (int)fidx.size()).first;
          frame_T.insert(frame_T.end(), o->frame->T_f_w_.m, o->frame->T_f_w_.m + 12);
        }
        obs_frame.push_back(it->second);
        obs_f.insert(obs_f.end(), o->f.begin(), o->f.end());
      }
      obs_offset.push_back((int)obs_frame.size());
      pos.insert(pos.end(), pts[k]->pos_.begin(), pts[k]->pos_.end());
    }
    if (obs_frame.empty()) return;
    tracking_ctx_.check(svo_b200_point_optimize_batch(tracking_ctx_.get(), (int)max_n_pts, max_iter, obs_offset.data(), obs_frame.data(),
                                                      obs_f.data(), frame_T.data(), (int)fidx.size(), pos.data()));
    for (size_t k = 0; k < max_n_pts; ++k) {
      for (int c = 0; c < 3; ++c) pts[k]->pos_[c] = pos[3 * k + c];
      last_structure_optim_[pts[k]] = frame_counter_;
    }
    ++frame_counter_;
  }

  AbstractCamera* cam_;
  Options opt_;
  Context tracking_ctx_, mapping_ctx_;  // one device context per host thread (include/svo_b200.h)
  Map map_;
  Reprojector reprojector_;
  DepthFilter depth_filter_;
  FramePtr new_frame_, last_frame_;
  std::set<FramePtr> core_kfs_;
  std::vector<std::pair<FramePtr, size_t>> overlap_kfs_;
  std::map<Point*, int> last_structure_optim_;
  int frame_counter_ = 0;
  size_t num_obs_last_ = 0;
  Stage stage_ = STAGE_PAUSED;
  TrackingQuality tracking_quality_ = TRACKING_INSUFFICIENT;
  FrameLog log_;
};

}  // namespace svo
