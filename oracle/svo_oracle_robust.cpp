// oracle/svo_oracle_robust.cpp -- TEST INFRASTRUCTURE ONLY: svo::SparseImgAlign with the robust cost of [EXT]
// vk::NLLSSolver::setRobustCostFunction(MADScale, weight) restated on top of the oracle's SparseImgAlign (svo_oracle.cpp,
// compiled into this library unchanged).  sparse_img_align.cpp:162-164, 213-230, 238-240: every pixel residual of a pass is
// weighted by weight_function_->value(res / scale_), and the pre-call computeResiduals(model, false, true) that starts each
// level's Gauss-Newton loop sets scale_ = 1.48 * median(|res|) when iter_ is 0.
//
// The residuals are the base class's own: its computeResiduals(T, false) evaluates every in-image patch in feature order and
// leaves the residuals in last_res_ (NaN where not evaluated) and the count in n_meas_.  This class weights them and forms
// chi2, H_ and Jres_ from them and the base's Jacobian cache in the same serial order as the reference.
#include "svo_oracle.cpp"

namespace {

// [EXT] vk::robust_cost weight functions, f32 as in vikit: 0 unit, 2 Tukey (b = 4.6851), 3 Huber (k = 1.345).  Tukey of +-inf
// or NaN is 0; Huber of NaN (0 / 0 with scale_ 0) is NaN.
float robust_weight(int fn, float x) {
  if (fn == 2) {
    const float b = 4.6851f, b_square = b * b;
    const float x_square = x * x;
    if (x_square <= b_square) { const float tmp = 1.0f - x_square / b_square; return tmp * tmp; }
    return 0.0f;
  }
  if (fn == 3) {
    const float k = 1.345f, t_abs = std::fabs(x);
    return t_abs < k ? 1.0f : k / t_abs;
  }
  return 1.0f;
}

struct RobustSparseImgAlign : SparseImgAlign {
  int weight_fn_ = 0;
  float scale_ = 0.0f;          // NLLSSolver() initialises it to 0 [EXT]
  float* scales_out = nullptr;  // scale_ after each level's pre-call, indexed by level

  using SparseImgAlign::SparseImgAlign;

  // sparse_img_align.cpp:147-243 with use_weights_ == true
  double computeResidualsWeighted(const SE3& T_cur_from_ref, bool linearize_system, bool compute_weight_scale) {
    SparseImgAlign::computeResiduals(T_cur_from_ref, false);  // residuals of the in-image patches -> last_res_, n_meas_
    std::vector<float> errors;
    float chi2 = 0.0f;
    for (int i = 0; i < N; ++i) {
      if (!last_in_img_[i]) continue;
      for (int p = 0; p < patch_area_; ++p) {
        const float res = last_res_[size_t(i) * patch_area_ + p];
        if (compute_weight_scale) errors.push_back(std::fabs(res));  // :213-214
        const float weight = robust_weight(weight_fn_, res / scale_);  // :216-220
        chi2 = std::fmaf(res * res, weight, chi2);                      // :222
        if (linearize_system) {                                         // :228-230
          const double* J = jacobian_cache_.data() + 6 * (size_t(i) * patch_area_ + p);
          const double w = weight, r = res;
          for (int a = 0; a < 6; ++a) {
            for (int b = 0; b < 6; ++b) H_[a][b] += J[a] * J[b] * w;
            Jres_[a] -= J[a] * r * w;
          }
        }
      }
    }
    // :238-240 MADScaleEstimator: 1.48f * vk::getMedian (nth_element at floor(n / 2)).  With no errors the reference's
    // getMedian is undefined behaviour; scale_ is kept here (not pinned).
    if (compute_weight_scale && iter_ == 0 && !errors.empty()) {
      auto it = errors.begin() + errors.size() / 2;
      std::nth_element(errors.begin(), it, errors.end());
      scale_ = 1.48f * *it;
    }
    return chi2 / n_meas_;  // float / size_t -> float; NaN when n_meas_ == 0
  }

  // [EXT] vk::NLLSSolver<6,SE3>::optimizeGaussNewton with use_weights_: the pre-call counts n_meas_ (only the loop resets it)
  // and recomputes scale_ when iter_ == 0, which still holds the previous level's value
  void optimizeGaussNewtonWeighted(SE3& model) {
    computeResidualsWeighted(model, false, true);
    if (scales_out) scales_out[level_] = scale_;
    SE3 old_model = model;
    for (iter_ = 0; iter_ < n_iter_; ++iter_) {
      std::memset(H_, 0, sizeof(H_));
      std::memset(Jres_, 0, sizeof(Jres_));
      n_meas_ = 0;
      const double new_chi2 = computeResidualsWeighted(model, true, false);
      if (!solve()) stop_ = true;
      const bool reject = (iter_ > 0 && new_chi2 > chi2_) || stop_;
      if (reject) {
        model = old_model;  // rollback
        record(new_chi2, 0, model);
        break;
      }
      SE3 new_model;
      update(model, new_model);
      old_model = model;
      model = new_model;
      chi2_ = new_chi2;
      record(new_chi2, 1, model);
      if (norm_max6(x_) <= eps_) break;
    }
  }

  // sparse_img_align.cpp:43-75 (as SparseImgAlign::run, with the weighted driver)
  size_t runWeighted(SE3& T_cur_from_ref) {
    reset();
    if (N == 0) return 0;
    ref_patch_cache_.assign(size_t(N) * patch_area_, 0.f);
    jacobian_cache_.assign(size_t(N) * patch_area_ * 6, 0.0);
    visible_fts_.assign(N, 0);
    last_res_.assign(size_t(N) * patch_area_, 0.f);
    last_in_img_.assign(N, 0);
    for (level_ = max_level_; level_ >= min_level_; --level_) {
      std::fill(jacobian_cache_.begin(), jacobian_cache_.end(), 0.0);
      have_ref_patch_cache_ = false;
      optimizeGaussNewtonWeighted(T_cur_from_ref);
    }
    return n_meas_ / patch_area_;
  }
};

}  // namespace

extern "C" {

// orc_sparse_img_align_run with the robust cost on: setRobustCostFunction(MADScale, weight_fn), weight_fn 0 = unit,
// 2 = Tukey, 3 = Huber.  scales_out[level] (ORC_MAX_LEVELS floats, NaN for the levels not run): scale_ after the pre-call of
// that level.
int64_t orc_sparse_img_align_robust(const uint8_t* const* ref_levels, const uint8_t* const* cur_levels, const int* cols,
                                    const int* rows, int n_levels, const orc_camera* cam, double* T_io, const double* px,
                                    const double* f, const double* point_pos, const uint8_t* has_point, const double* ref_pos,
                                    int N, int max_level, int min_level, int n_iter, double eps, int weight_fn,
                                    uint8_t* visible_out, double* H_out, float* scales_out, orc_sia_iter* trace, int trace_cap,
                                    int* n_trace) {
  Img rp[ORC_MAX_LEVELS], cp[ORC_MAX_LEVELS];
  for (int l = 0; l < n_levels && l < ORC_MAX_LEVELS; ++l) {
    rp[l] = Img{ref_levels[l], cols[l], rows[l], cols[l]};
    cp[l] = Img{cur_levels[l], cols[l], rows[l], cols[l]};
  }
  RobustSparseImgAlign sia(max_level, min_level, n_iter, eps);
  sia.ref_pyr = rp;
  sia.cur_pyr = cp;
  sia.cam = make_cam(cam);
  sia.N = N;
  sia.px = px;
  sia.f = f;
  sia.pos = point_pos;
  sia.has_point = has_point;
  sia.ref_pos = V3{ref_pos[0], ref_pos[1], ref_pos[2]};
  sia.trace = trace;
  sia.trace_cap = trace_cap;
  sia.weight_fn_ = weight_fn;
  sia.scales_out = scales_out;
  if (scales_out)
    for (int l = 0; l < ORC_MAX_LEVELS; ++l) scales_out[l] = std::numeric_limits<float>::quiet_NaN();
  std::memset(sia.H_, 0, sizeof(sia.H_));
  SE3 T = se3_from_rt12(T_io);
  const size_t ret = sia.runWeighted(T);
  se3_to_rt12(T, T_io);
  if (visible_out)
    for (int i = 0; i < N; ++i) visible_out[i] = sia.visible_fts_[i];
  if (H_out)
    for (int a = 0; a < 6; ++a)
      for (int b = 0; b < 6; ++b) H_out[a * 6 + b] = sia.H_[a][b];
  if (n_trace) *n_trace = sia.n_trace;
  return int64_t(ret);
}

}  // extern "C"
