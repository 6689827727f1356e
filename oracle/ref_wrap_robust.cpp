// oracle/ref_wrap_robust.cpp -- TEST INFRASTRUCTURE ONLY: the reference's own svo::SparseImgAlign with the robust cost of
// [EXT] vk::NLLSSolver set (MADScale with unit, Tukey or Huber weights), so that the weighted lines of sparse_img_align.cpp
// (:162-164, 213-230, 238-240) run against the oracle.  Compiled with the reference's sources and oracle/ref_wrap*.cpp into
// oracle/_ref/libsvo_ref_robust.so by oracle/robust.mk.
#include "ref_wrap.cpp"

#include <limits>

namespace {
// [EXT] vk::robust_cost weights the stand-in robust_cost.h does not restate: unit and Huber (k = 1.345, f32)
struct UnitWeightFn : vk::robust_cost::WeightFunction {
  float value(const float&) const override { return 1.0f; }
};
struct HuberWeightFn : vk::robust_cost::WeightFunction {
  float value(const float& t) const override {
    const float k = 1.345f, t_abs = std::fabs(t);
    if (t_abs < k) return 1.0f;
    return k / t_abs;
  }
};

// setRobustCostFunction(MADScale, weight) [EXT]: a MAD scale estimator turns use_weights_ on; weight 0 unit, 2 Tukey,
// 3 Huber.  A derived class records scale_ after every pre-call computeResiduals(model, false, true).
struct SIARobust : public SparseImgAlign {
  float* scales = nullptr;
  SIARobust(int a, int b, int c, int weight) : SparseImgAlign(a, b, c, GaussNewton, false, false) {
    use_weights_ = true;
    scale_estimator_.reset(new vk::robust_cost::MADScaleEstimator());
    if (weight == 2) weight_function_.reset(new vk::robust_cost::TukeyWeightFunction());
    else if (weight == 3) weight_function_.reset(new HuberWeightFn());
    else weight_function_.reset(new UnitWeightFn());
  }
  double computeResiduals(const SE3& model, bool linearize_system, bool compute_weight_scale) override {
    const double chi2 = SparseImgAlign::computeResiduals(model, linearize_system, compute_weight_scale);
    if (compute_weight_scale && scales) scales[level_] = scale_;
    return chi2;
  }
  const std::vector<bool>& visible() const { return visible_fts_; }
  const Matrix<double, 6, 6>& H() const { return H_; }
};
}  // namespace

extern "C" {

// ref_sparse_img_align with the robust cost on; scales_out[level] (8 floats, NaN for the levels not run).
long long ref_sparse_img_align_robust(const uint8_t* ref_l0, const uint8_t* cur_l0, int w, int h, int n_levels, const double* cam4,
                                      const double* T_ref_w, double* T_cur_w_io, const double* px, const double* f, const double* pos,
                                      const uint8_t* has_point, int N, int max_level, int min_level, int n_iter, int weight,
                                      uint8_t* visible_out, double* H_out, float* scales_out) {
  std::unique_ptr<vk::AbstractCamera> cam_owner(ref_make_camera(w, h, cam4));
  vk::AbstractCamera& cam = *cam_owner;
  FramePtr ref = make_frame(&cam, ref_l0, w, h, n_levels, T_ref_w);
  FramePtr cur = make_frame(&cam, cur_l0, w, h, n_levels, T_cur_w_io);
  std::vector<std::unique_ptr<Point>> pts;
  for (int i = 0; i < N; ++i) {
    Point* p = nullptr;
    if (has_point[i]) { pts.emplace_back(new Point(Vector3d(pos[3 * i], pos[3 * i + 1], pos[3 * i + 2]))); p = pts.back().get(); }
    ref->addFeature(new Feature(ref.get(), p, Vector2d(px[2 * i], px[2 * i + 1]), Vector3d(f[3 * i], f[3 * i + 1], f[3 * i + 2]), 0));
  }
  for (int l = 0; l < 8; ++l) scales_out[l] = std::numeric_limits<float>::quiet_NaN();
  SIARobust sia(max_level, min_level, n_iter, weight);
  sia.scales = scales_out;
  const size_t ret = sia.run(ref, cur);
  se3_to12(cur->T_f_w_, T_cur_w_io);
  if (visible_out) for (int i = 0; i < N && i < (int)sia.visible().size(); ++i) visible_out[i] = sia.visible()[i];
  if (H_out) for (int a = 0; a < 6; ++a) for (int b = 0; b < 6; ++b) H_out[a * 6 + b] = sia.H()(a, b);
  return (long long)ret;
}

}  // extern "C"
