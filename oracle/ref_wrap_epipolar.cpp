// oracle/ref_wrap_epipolar.cpp -- TEST INFRASTRUCTURE ONLY: the reference's own svo::Matcher::findEpipolarMatchDirect and
// svo::DepthFilter::updateSeeds with Matcher::options_ set (align_1d, subpix_refinement, epi_search_edgelet_filtering,
// epi_search_edgelet_max_angle; matcher.h:74-91), on the standalone Matcher and on the filter's own matcher_.  Compiled with
// the reference's sources and oracle/ref_wrap*.cpp into oracle/_ref/libsvo_ref_epipolar.so by oracle/epipolar.mk.
#include "ref_wrap.cpp"

#include <cstdint>

namespace {
struct epi_options {  // the layout of svo_b200_epipolar_options
  int align_1d, subpix_refinement, epi_search_edgelet_filtering;
  double epi_search_edgelet_max_angle;
};
void set_options(Matcher::Options& o, const epi_options* e) {
  o.align_1d = e->align_1d != 0;
  o.subpix_refinement = e->subpix_refinement != 0;
  o.epi_search_edgelet_filtering = e->epi_search_edgelet_filtering != 0;
  o.epi_search_edgelet_max_angle = e->epi_search_edgelet_max_angle;
}
// h_inv_ before the call: a value align1D cannot set (1 / H * 64 of a float H), so that the call's h_inv_ tells whether it ran
const uint64_t kHinvUnset = 0x7ff4dead0000beefull;  // a signalling-NaN payload no arithmetic produces
double unset_h_inv() { double d; std::memcpy(&d, &kHinvUnset, 8); return d; }
bool is_unset(double d) { uint64_t u; std::memcpy(&u, &d, 8); return u == kHinvUnset; }

// DepthFilter whose matcher_ (protected, depth_filter.h:152) is configured before updateSeeds, as a subclass can
struct RefDFOpt : public RefDF {
  RefDFOpt(callback_t cb, const epi_options* e) : RefDF(cb) { set_options(matcher_.options_, e); }
};
}  // namespace

extern "C" {

// ref_matcher(mode 1) with Matcher::options_ set from `opt`; *ran_1d_out: align1D ran (it set h_inv_), out->h_inv its value
// (0 when it did not run).
void ref_matcher_epipolar(const uint8_t* ref_l0, const uint8_t* cur_l0, int w, int h, int n_levels, const double* cam4,
                          const double* T_ref_w, const double* T_cur_w, const double* ref_px, const double* ref_f, int ref_level,
                          int ftr_type, const double* ref_grad, double d_est, double d_min, double d_max, int n_pyr_levels,
                          const epi_options* opt, ref_match_out* out, int* ran_1d_out) {
  std::unique_ptr<vk::AbstractCamera> cam_owner(ref_make_camera(w, h, cam4));
  vk::AbstractCamera& cam = *cam_owner;
  FramePtr ref = make_frame(&cam, ref_l0, w, h, n_levels, T_ref_w);
  FramePtr cur = make_frame(&cam, cur_l0, w, h, n_levels, T_cur_w);
  Config::nPyrLevels() = n_pyr_levels;
  Feature* ft = new Feature(ref.get(), Vector2d(ref_px[0], ref_px[1]), Vector3d(ref_f[0], ref_f[1], ref_f[2]), ref_level);
  ft->type = ftr_type ? Feature::EDGELET : Feature::CORNER;
  ft->grad = Vector2d(ref_grad[0], ref_grad[1]);
  ref->addFeature(ft);
  Matcher m;
  set_options(m.options_, opt);
  memset(m.patch_, 0, sizeof(m.patch_));
  memset(m.patch_with_border_, 0, sizeof(m.patch_with_border_));
  m.search_level_ = 0; m.h_inv_ = unset_h_inv(); m.epi_length_ = 0; m.reject_ = false;
  m.px_cur_ = Vector2d(0, 0); m.A_cur_ref_.setZero();
  memset(out, 0, sizeof(*out));
  double depth = 0;
  out->success = m.findEpipolarMatchDirect(*ref, *cur, *ft, d_est, d_min, d_max, depth);
  out->px_cur[0] = m.px_cur_[0]; out->px_cur[1] = m.px_cur_[1];
  out->depth = depth;
  out->search_level = m.search_level_; out->reject = m.reject_;
  out->A[0] = m.A_cur_ref_(0, 0); out->A[1] = m.A_cur_ref_(0, 1); out->A[2] = m.A_cur_ref_(1, 0); out->A[3] = m.A_cur_ref_(1, 1);
  *ran_1d_out = is_unset(m.h_inv_) ? 0 : 1;
  out->h_inv = *ran_1d_out ? m.h_inv_ : 0.0;
  out->epi_length = m.epi_length_;
}

// ref_depth_filter_update with DepthFilter::matcher_.options_ set from `opt`.
void ref_depth_filter_update_epipolar(const uint8_t* ref_l0s, const double* ref_T_f_w, int n_ref, const uint8_t* cur_l0,
                                      const double* cur_T_f_w, int w, int h, int n_levels, const double* cam4, int M,
                                      const int* ref_index, const double* ftr_px, const double* ftr_f, const int* ftr_level,
                                      const int* ftr_type, const double* ftr_grad, const int* batch_id, int batch_counter,
                                      int n_pyr_levels, const epi_options* opt, float* a, float* b, float* mu, float* z_range,
                                      float* sigma2, uint8_t* status_out, double* xyz_world_out) {
  std::unique_ptr<vk::AbstractCamera> cam_owner(ref_make_camera(w, h, cam4));
  vk::AbstractCamera& cam = *cam_owner;
  std::vector<FramePtr> refs;
  for (int r = 0; r < n_ref; ++r) refs.push_back(make_frame(&cam, ref_l0s + (size_t)r * w * h, w, h, n_levels, ref_T_f_w + 12 * r));
  FramePtr cur = make_frame(&cam, cur_l0, w, h, n_levels, cur_T_f_w);
  Config::nPyrLevels() = n_pyr_levels;
  std::vector<Feature*> fts(M);
  std::vector<Point*> made;
  std::vector<double> conv_sigma2;
  RefDFOpt df([&](Point* p, double s2) { made.push_back(p); conv_sigma2.push_back(s2); }, opt);
  for (int i = 0; i < M; ++i) {
    Frame* fr = refs[ref_index[i]].get();
    Feature* ft = new Feature(fr, Vector2d(ftr_px[2 * i], ftr_px[2 * i + 1]), Vector3d(ftr_f[3 * i], ftr_f[3 * i + 1], ftr_f[3 * i + 2]), ftr_level[i]);
    ft->type = ftr_type[i] ? Feature::EDGELET : Feature::CORNER;
    ft->grad = Vector2d(ftr_grad[2 * i], ftr_grad[2 * i + 1]);
    fr->addFeature(ft);
    fts[i] = ft;
    Seed s(ft, 1.0f, 0.5f);
    s.id = i; s.batch_id = batch_id[i];
    s.a = a[i]; s.b = b[i]; s.mu = mu[i]; s.z_range = z_range[i]; s.sigma2 = sigma2[i];
    df.getSeeds().push_back(s);
  }
  Seed::batch_counter = batch_counter;
  df.update(cur);
  for (int i = 0; i < M; ++i) status_out[i] = 2;
  for (auto& s : df.getSeeds()) {
    const int i = s.id;
    status_out[i] = 0;
    a[i] = s.a; b[i] = s.b; mu[i] = s.mu; z_range[i] = s.z_range; sigma2[i] = s.sigma2;
  }
  for (int i = 0; i < M; ++i) {
    if (fts[i]->point == NULL) continue;
    status_out[i] = 1;
    for (size_t k = 0; k < made.size(); ++k)
      if (made[k] == fts[i]->point) sigma2[i] = (float)conv_sigma2[k];
    for (int k = 0; k < 3; ++k) xyz_world_out[3 * i + k] = fts[i]->point->pos_[k];
  }
  for (Point* p : made) delete p;
}

}  // extern "C"
