// oracle/svo_oracle_epipolar.cpp -- TEST INFRASTRUCTURE ONLY: svo::Matcher::findEpipolarMatchDirect (matcher.cpp:179-321)
// under every Matcher::Options setting it reads (matcher.h:74-91): align_1d, subpix_refinement,
// epi_search_edgelet_filtering and epi_search_edgelet_max_angle, and DepthFilter::updateSeeds (depth_filter.cpp:197-291) with
// its matcher_ so configured.  The oracle of svo_oracle.cpp is compiled into this library unchanged; at the defaults the
// functions here compute what its findEpipolarMatchDirect / orc_depth_filter_update compute.
#include "svo_oracle.cpp"

extern "C" {
typedef struct {  // the layout of svo_b200_epipolar_options
  int align_1d;
  int subpix_refinement;
  int epi_search_edgelet_filtering;
  double epi_search_edgelet_max_angle;
} orc_epipolar_options;
}

namespace {

struct EpiOptions {  // Matcher::Options (matcher.h:74-91), the fields findEpipolarMatchDirect reads besides the two iteration limits
  bool align_1d = false;
  bool subpix_refinement = true;
  bool edgelet_filtering = true;
  double edgelet_max_angle = 0.7;
};

EpiOptions epi_options(const orc_epipolar_options* o) {
  EpiOptions e;
  if (o) {
    e.align_1d = o->align_1d != 0;
    e.subpix_refinement = o->subpix_refinement != 0;
    e.edgelet_filtering = o->epi_search_edgelet_filtering != 0;
    e.edgelet_max_angle = o->epi_search_edgelet_max_angle;
  }
  return e;
}

// svo/src/matcher.cpp:179-321.  *ran_1d: align1D ran (and set m.h_inv_).
bool findEpipolarMatchDirectOpt(MatcherState& m, const Img* ref_pyr, const Img* cur_pyr, const Cam& cam, const SE3& T_cur_ref,
                                const RefFeature& ref_ftr, const double d_estimate, const double d_min, const double d_max,
                                int max_search_level, int align_max_iter, size_t max_epi_search_steps, const EpiOptions& opt,
                                double& depth, bool* ran_1d) {
  *ran_1d = false;
  int zmssd_best = ZMSSD::threshold();
  V2 uv_best{0, 0};
  m.n_zmssd_ = 0;
  const V3 pA = T_cur_ref * (ref_ftr.f * d_min);
  const V3 pB = T_cur_ref * (ref_ftr.f * d_max);
  const V2 A{pA.x / pA.z, pA.y / pA.z};  // vk::project2d
  const V2 B{pB.x / pB.z, pB.y / pB.z};
  m.epi_dir_ = A - B;
  getWarpMatrixAffine(cam, cam, ref_ftr.px, ref_ftr.f, d_estimate, T_cur_ref, ref_ftr.level, m.A_cur_ref_);
  m.reject_ = false;
  if (ref_ftr.type == 1 && opt.edgelet_filtering) {  // :204-212
    V2 g{m.A_cur_ref_[0][0] * ref_ftr.grad.x + m.A_cur_ref_[0][1] * ref_ftr.grad.y,
         m.A_cur_ref_[1][0] * ref_ftr.grad.x + m.A_cur_ref_[1][1] * ref_ftr.grad.y};
    const double gn = norm(g), en = norm(m.epi_dir_);
    const double cosangle = std::fabs((g.x / gn) * (m.epi_dir_.x / en) + (g.y / gn) * (m.epi_dir_.y / en));
    if (cosangle < opt.edgelet_max_angle) {
      m.reject_ = true;
      return false;
    }
  }
  m.search_level_ = getBestSearchLevel(m.A_cur_ref_, max_search_level);
  const V2 px_A = cam.world2cam_uv(A);
  const V2 px_B = cam.world2cam_uv(B);
  m.epi_length_ = norm(px_A - px_B) / (1 << m.search_level_);
  warpAffine(m.A_cur_ref_, ref_pyr[ref_ftr.level], ref_ftr.px, ref_ftr.level, m.search_level_, 4 + 1, m.patch_with_border_);
  createPatchFromPatchWithBorder(m.patch_with_border_, m.patch_);

  auto refine = [&](V2 px_start) -> bool {  // :228-245 / :297-314
    m.px_cur_ = px_start;
    double px_scaled[2] = {m.px_cur_.x / (1 << m.search_level_), m.px_cur_.y / (1 << m.search_level_)};
    bool res;
    if (opt.align_1d) {
      // (px_A-px_B).cast<float>().normalized(): divided by the norm without a guard, so a zero-length line is a NaN direction
      const float dx = float(px_A.x - px_B.x), dy = float(px_A.y - px_B.y);
      const float n = std::sqrt(std::fmaf(dx, dx, dy * dy));
      const float dirf[2] = {dx / n, dy / n};
      res = align1D(cur_pyr[m.search_level_], dirf, m.patch_with_border_, m.patch_, align_max_iter, px_scaled, m.h_inv_);
      *ran_1d = true;
    } else {
      res = align2D(cur_pyr[m.search_level_], m.patch_with_border_, m.patch_, align_max_iter, px_scaled);
    }
    if (res) {
      m.px_cur_ = V2{px_scaled[0] * (1 << m.search_level_), px_scaled[1] * (1 << m.search_level_)};
      if (depthFromTriangulation(T_cur_ref, ref_ftr.f, cam.cam2world(m.px_cur_.x, m.px_cur_.y), depth)) return true;
    }
    return false;
  };

  if (m.epi_length_ < 2.0) return refine((px_A + px_B) * (1.0 / 2.0));  // whatever subpix_refinement says

  size_t n_steps = m.epi_length_ / 0.7;
  const V2 step{m.epi_dir_.x / n_steps, m.epi_dir_.y / n_steps};
  if (n_steps > max_epi_search_steps) return false;

  ZMSSD patch_score(m.patch_);
  V2 uv = B - step;
  int last_x = 0, last_y = 0;
  ++n_steps;
  const Img& img = cur_pyr[m.search_level_];
  for (size_t i = 0; i < n_steps; ++i, uv = uv + step) {
    const V2 px = cam.world2cam_uv(uv);
    const int pxi_x = int(px.x / (1 << m.search_level_) + 0.5);
    const int pxi_y = int(px.y / (1 << m.search_level_) + 0.5);
    if (pxi_x == last_x && pxi_y == last_y) continue;
    last_x = pxi_x;
    last_y = pxi_y;
    if (!cam.isInFrame(pxi_x, pxi_y, 8, m.search_level_)) continue;
    const uint8_t* cur_patch_ptr = img.data + (pxi_y - 4) * img.cols + (pxi_x - 4);
    const int zmssd = patch_score.computeScore(cur_patch_ptr, img.cols);
    ++m.n_zmssd_;
    if (zmssd < zmssd_best) {
      zmssd_best = zmssd;
      uv_best = uv;
    }
  }
  if (zmssd_best < ZMSSD::threshold()) {
    if (opt.subpix_refinement) return refine(cam.world2cam_uv(uv_best));
    // :316-318.  vk::unproject2d(uv_best).normalized(): the reference's build fuses the squared norm's sum as
    // (u*u + v*v) + 1*1 with two fused multiply-adds
    m.px_cur_ = cam.world2cam_uv(uv_best);
    const double n = std::sqrt(std::fma(1.0, 1.0, std::fma(uv_best.y, uv_best.y, uv_best.x * uv_best.x)));
    if (depthFromTriangulation(T_cur_ref, ref_ftr.f, V3{uv_best.x / n, uv_best.y / n, 1.0 / n}, depth)) return true;
  }
  return false;
}

}  // namespace

extern "C" {

// orc_find_epipolar_match_direct under Matcher::Options `opt` (NULL = the defaults); *ran_1d_out: align1D ran and
// out->h_inv is the h_inv_ it set (a fresh Matcher's 0 otherwise).
void orc_find_epipolar_match_direct_opt(const uint8_t* const* ref_levels, const uint8_t* const* cur_levels, const int* cols,
                                        const int* rows, int n_levels, const orc_camera* cam, const double* T_cur_ref,
                                        const double* ref_px, const double* ref_f, int ref_level, int ftr_type,
                                        const double* ref_grad, double d_estimate, double d_min, double d_max,
                                        int max_search_level, int align_max_iter, int max_epi_search_steps,
                                        const orc_epipolar_options* opt, orc_epi_result* out, int* ran_1d_out) {
  Img rp[ORC_MAX_LEVELS], cp[ORC_MAX_LEVELS];
  fill_pyr(rp, ref_levels, cols, rows, n_levels);
  fill_pyr(cp, cur_levels, cols, rows, n_levels);
  MatcherState m;
  RefFeature rf{V2{ref_px[0], ref_px[1]}, V3{ref_f[0], ref_f[1], ref_f[2]}, ref_level, ftr_type, V2{ref_grad[0], ref_grad[1]}};
  double depth = 0;
  bool ran_1d = false;
  const bool ok = findEpipolarMatchDirectOpt(m, rp, cp, make_cam(cam), se3_from_rt12(T_cur_ref), rf, d_estimate, d_min, d_max,
                                             max_search_level, align_max_iter, size_t(max_epi_search_steps), epi_options(opt),
                                             depth, &ran_1d);
  out->success = ok;
  out->reject = m.reject_;
  out->search_level = m.search_level_;
  out->n_zmssd_evals = m.n_zmssd_;
  out->n_align_iter = -1;
  out->epi_length = m.epi_length_;
  out->px_cur[0] = m.px_cur_.x;
  out->px_cur[1] = m.px_cur_.y;
  out->depth = depth;
  out->h_inv = m.h_inv_;
  out->A_cur_ref[0] = m.A_cur_ref_[0][0]; out->A_cur_ref[1] = m.A_cur_ref_[0][1];
  out->A_cur_ref[2] = m.A_cur_ref_[1][0]; out->A_cur_ref[3] = m.A_cur_ref_[1][1];
  if (ran_1d_out) *ran_1d_out = ran_1d ? 1 : 0;
}

// orc_depth_filter_update (svo_oracle_depth.inc) with DepthFilter::matcher_.options_ = `opt` (NULL = the defaults).
void orc_depth_filter_update_opt(const uint8_t* const* ref_levels, const double* ref_T_f_w, int n_ref,
                                 const uint8_t* const* cur_levels, const double* cur_T_f_w, const int* cols, const int* rows,
                                 int n_levels, const orc_camera* cam_c, int M, const int* ref_index, const double* ftr_px,
                                 const double* ftr_f, const int* ftr_level, const int* ftr_type, const double* ftr_grad,
                                 const int* batch_id, int batch_counter, int max_n_kfs, double seed_convergence_sigma2_thresh,
                                 int max_search_level, int align_max_iter, int max_epi_search_steps,
                                 const orc_epipolar_options* opt, float* a, float* b, float* mu, float* z_range, float* sigma2,
                                 uint8_t* status_out, double* px_cur_out, double* z_out, int* n_zmssd_out) {
  const EpiOptions eo = epi_options(opt);
  const Cam cam = make_cam(cam_c);
  Img cp[ORC_MAX_LEVELS];
  fill_pyr(cp, cur_levels, cols, rows, n_levels);
  const SE3 T_cur_w = se3_from_rt12(cur_T_f_w);
  const double px_error_angle = std::atan(1.0 / (2.0 * cam.errorMultiplier2())) * 2.0;  // :205-207
  MatcherState matcher;  // DepthFilter::matcher_, reused for all seeds (depth_filter.h:152)
  for (int i = 0; i < M; ++i) {
    if (px_cur_out) px_cur_out[2 * i] = px_cur_out[2 * i + 1] = 0;
    if (z_out) z_out[i] = 0;
    if (n_zmssd_out) n_zmssd_out[i] = 0;
    if ((batch_counter - batch_id[i]) > max_n_kfs) {  // :216-219
      status_out[i] = ORC_SEED_TOO_OLD;
      continue;
    }
    const int r = ref_index[i];
    Img rp[ORC_MAX_LEVELS];
    fill_pyr(rp, ref_levels + size_t(r) * n_levels, cols, rows, n_levels);
    const SE3 T_ref_w = se3_from_rt12(ref_T_f_w + 12 * size_t(r));
    const SE3 T_ref_cur = T_ref_w * inverse(T_cur_w);  // :222
    const V3 fv{ftr_f[3 * i], ftr_f[3 * i + 1], ftr_f[3 * i + 2]};
    const V3 xyz_f = inverse(T_ref_cur) * (fv * (1.0 / mu[i]));  // :223
    if (xyz_f.z < 0.0) {
      status_out[i] = ORC_SEED_BEHIND;
      continue;
    }
    const V2 c = cam.world2cam(xyz_f);
    if (!cam.isInFrame(int(c.x), int(c.y), 0)) {
      status_out[i] = ORC_SEED_NOT_IN_FRAME;
      continue;
    }
    float z_inv_min = mu[i] + std::sqrt(sigma2[i]);
    float z_inv_max = std::max(mu[i] - std::sqrt(sigma2[i]), 0.00000001f);
    double z = 0;
    RefFeature rf{V2{ftr_px[2 * i], ftr_px[2 * i + 1]}, fv, ftr_level[i], ftr_type[i], V2{ftr_grad[2 * i], ftr_grad[2 * i + 1]}};
    const SE3 T_cur_ref = T_cur_w * inverse(T_ref_w);  // matcher.cpp:188
    bool ran_1d = false;
    const bool ok = findEpipolarMatchDirectOpt(matcher, rp, cp, cam, T_cur_ref, rf, 1.0 / mu[i], 1.0 / z_inv_min,
                                               1.0 / z_inv_max, max_search_level, align_max_iter,
                                               size_t(max_epi_search_steps), eo, z, &ran_1d);
    if (n_zmssd_out) n_zmssd_out[i] = matcher.n_zmssd_;
    if (!ok) {
      b[i]++;  // :240
      status_out[i] = ORC_SEED_NO_MATCH;
      continue;
    }
    double tau = computeTau(T_ref_cur, fv, z, px_error_angle);
    double tau_inverse = 0.5 * (1.0 / std::max(0.0000001, z - tau) - 1.0 / (z + tau));
    updateSeed(float(1. / z), float(tau_inverse * tau_inverse), SeedRef{a[i], b[i], mu[i], z_range[i], sigma2[i]});
    if (px_cur_out) {  // matcher_.px_cur_, what setGridOccpuancy reads (:255-259)
      px_cur_out[2 * i] = matcher.px_cur_.x;
      px_cur_out[2 * i + 1] = matcher.px_cur_.y;
    }
    if (z_out) z_out[i] = z;
    if (double(std::sqrt(sigma2[i])) < double(z_range[i]) / seed_convergence_sigma2_thresh)
      status_out[i] = ORC_SEED_CONVERGED;  // :261-282
    else if (std::isnan(z_inv_min))
      status_out[i] = ORC_SEED_NAN;  // :283-287
    else
      status_out[i] = ORC_SEED_UPDATED;
  }
  (void)n_ref;
}

}  // extern "C"
