// rpg_svo_b200/csrc/align.cu -- batched feature alignment on sm_90a: one warp per feature.
//
//   svo_b200_align2d_batch / svo_b200_align1d_batch  <- feature_alignment::align2D / align1D
//                                                       (svo/src/feature_alignment.cpp:149-277, 30-147)
//   svo_b200_find_match_direct                       <- Matcher::findMatchDirect (svo/src/matcher.cpp:135-177)
//
// The reference calls these once per map point inside Reprojector::reprojectCell
// (svo/src/reprojector.cpp:151-204); here the host gathers the candidates of a frame into flat arrays
// and one launch aligns them all.  Per-feature state (10x10 template, gradients, residuals) lives in a
// per-warp slice of shared memory; see warp_align.cuh for the arithmetic contract.
#include <cstring>
#include <vector>

#include "ctx.h"
#include "warp_align.cuh"

namespace svo {

constexpr int kWarpsPerCta = 4;

__global__ void __launch_bounds__(kWarpsPerCta * 32) align_batch_kernel(
    FrameDesc cur, int M, const int* __restrict__ level, const float* __restrict__ dir /*NULL -> 2D*/,
    const uint8_t* __restrict__ pwb, const uint8_t* __restrict__ patch, int n_iter, double* __restrict__ px_io,
    uint8_t* __restrict__ converged_out, double* __restrict__ h_inv_out) {
  __shared__ WarpAlignScratch scratch[kWarpsPerCta];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m = blockIdx.x * kWarpsPerCta + warp;
  if (m >= M) return;
  WarpAlignScratch& S = scratch[warp];
  for (int i = lane; i < 100; i += 32) S.pwb[i] = pwb[(size_t)m * 100 + i];
  for (int i = lane; i < 64; i += 32) S.patch[i] = patch[(size_t)m * 64 + i];
  __syncwarp();
  const int L = level[m];
  ImgView img = {cur.lvl[L], cur.w[L], cur.h[L]};
  double u = px_io[2 * m], v = px_io[2 * m + 1], h_inv = 0.0;
  bool nan_exit = false, ok;
  if (dir) ok = warp_align1d(img, S, dir[2 * m], dir[2 * m + 1], n_iter, u, v, h_inv, &nan_exit);
  else ok = warp_align2d(img, S, n_iter, u, v, &nan_exit);
  if (lane == 0) {
    if (!nan_exit) { px_io[2 * m] = u; px_io[2 * m + 1] = v; }
    converged_out[m] = ok ? 1 : 0;
    if (h_inv_out) h_inv_out[m] = h_inv;
  }
}

struct MatchIn {  // device pointers to the flat candidate arrays
  const int* ref_index;
  const double* ref_px;
  const double* ref_f;
  const int* ref_level;
  const int* ftr_type;
  const double* ref_grad;
  const double* point_pos;
  const double* ref_T_f_w;  // n_ref * 12
  const FrameDesc* ref_frames;
};
struct MatchOut {
  double* px_cur;
  uint8_t* success;
  int* search_level;
  double* A_cur_ref;
  double* h_inv;
};

// Matcher::findMatchDirect (matcher.cpp:135-177) for M candidates whose reference observation has
// been selected by Point::getCloseViewObs on the host.
__global__ void __launch_bounds__(kWarpsPerCta * 32) find_match_direct_kernel(
    FrameDesc cur, Cam cam, int M, MatchIn in, MatchOut out, int max_search_level, int align_max_iter,
    const double* __restrict__ cur_T_f_w) {
  __shared__ WarpAlignScratch scratch[kWarpsPerCta];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m = blockIdx.x * kWarpsPerCta + warp;
  if (m >= M) return;
  WarpAlignScratch& S = scratch[warp];
  const int r = in.ref_index[m];
  const double ref_px[2] = {in.ref_px[2 * m], in.ref_px[2 * m + 1]};
  const double f_ref[3] = {in.ref_f[3 * m], in.ref_f[3 * m + 1], in.ref_f[3 * m + 2]};
  const double grad[2] = {in.ref_grad[2 * m], in.ref_grad[2 * m + 1]};
  const double pos[3] = {in.point_pos[3 * m], in.point_pos[3 * m + 1], in.point_pos[3 * m + 2]};
  int search_level = 0;
  double A[4] = {0, 0, 0, 0}, h_inv = 0.0;
  double pu = out.px_cur[2 * m], pv = out.px_cur[2 * m + 1];
  const int success = warp_find_match_direct(cur, cam, in.ref_frames[r], pose_from_rt12(in.ref_T_f_w + 12 * (size_t)r),
                                             pose_from_rt12(cur_T_f_w), ref_px, f_ref, in.ref_level[m], in.ftr_type[m], grad,
                                             pos, max_search_level, align_max_iter, S, pu, pv, search_level, A, h_inv)
                          ? 1 : 0;
  if (lane == 0) {
    out.px_cur[2 * m] = pu;
    out.px_cur[2 * m + 1] = pv;
    out.success[m] = (uint8_t)success;
    if (out.search_level) out.search_level[m] = search_level;
    if (out.A_cur_ref) { for (int k = 0; k < 4; ++k) out.A_cur_ref[4 * m + k] = A[k]; }
    if (out.h_inv) out.h_inv[m] = h_inv;
  }
}

static int align_batch(svo_b200_ctx* ctx, const svo_b200_frame* cur, int M, const int* level, const float* dir,
                       const uint8_t* pwb, const uint8_t* patch, int n_iter, double* px_io, uint8_t* converged_out,
                       double* h_inv_out) {
  if (!ctx || !cur || M < 0 || (M > 0 && (!level || !pwb || !patch || !px_io || !converged_out)))
    return set_err(ctx, SVO_B200_EINVAL, "align_batch: bad arguments");
  if (M == 0) return 0;
  for (int m = 0; m < M; ++m)
    if (level[m] < 0 || level[m] >= cur->n_levels)
      return set_err(ctx, SVO_B200_EINVAL, "align_batch: level[%d]=%d outside the pyramid", m, level[m]);
  cudaSetDevice(ctx->device);
  Staging st(ctx);
  const int* d_level;
  const float* d_dir = nullptr;  // 2D: no direction
  const uint8_t *d_pwb, *d_patch;
  double *d_px, *d_h_inv = nullptr;
  uint8_t* d_conv;
  st.in(level, M, &d_level);
  if (dir) st.in(dir, 2 * (size_t)M, &d_dir);
  st.in(pwb, 100 * (size_t)M, &d_pwb);
  st.in(patch, 64 * (size_t)M, &d_patch);
  st.inout(px_io, 2 * (size_t)M, &d_px);
  st.out(converged_out, M, &d_conv);
  if (h_inv_out) st.out(h_inv_out, M, &d_h_inv);
  int rc;
  if ((rc = st.open()) || (rc = st.send())) return rc;
  const int blocks = (M + kWarpsPerCta - 1) / kWarpsPerCta;
  if ((rc = launch_kernels(ctx, 1, [&] {
         align_batch_kernel<<<blocks, kWarpsPerCta * 32, 0, ctx->stream>>>(make_desc(cur), M, d_level, d_dir, d_pwb, d_patch, n_iter,
                                                                           d_px, d_conv, d_h_inv);
       })))
    return rc;
  return st.receive();
}

}  // namespace svo

using namespace svo;

extern "C" {

int svo_b200_align2d_batch(svo_b200_ctx* ctx, const svo_b200_frame* cur, int M, const int* level,
                           const uint8_t* ref_patch_with_border, const uint8_t* ref_patch, int n_iter,
                           double* px_io, uint8_t* converged_out) {
  return align_batch(ctx, cur, M, level, nullptr, ref_patch_with_border, ref_patch, n_iter, px_io, converged_out, nullptr);
}

int svo_b200_align1d_batch(svo_b200_ctx* ctx, const svo_b200_frame* cur, int M, const int* level, const float* dir,
                           const uint8_t* ref_patch_with_border, const uint8_t* ref_patch, int n_iter,
                           double* px_io, uint8_t* converged_out, double* h_inv_out) {
  if (M > 0 && !dir) return set_err(ctx, SVO_B200_EINVAL, "align1d_batch: dir is NULL");
  return align_batch(ctx, cur, M, level, dir, ref_patch_with_border, ref_patch, n_iter, px_io, converged_out, h_inv_out);
}

int svo_b200_find_match_direct(svo_b200_ctx* ctx, const svo_b200_frame* const* ref_frames, const double* ref_T_f_w,
                               int n_ref, const svo_b200_frame* cur, const double* cur_T_f_w,
                               const svo_b200_camera* cam, const svo_b200_match_options* opt, int M,
                               const int* ref_index, const double* ref_px, const double* ref_f, const int* ref_level,
                               const int* ftr_type, const double* ref_grad, const double* point_pos,
                               double* px_cur_io, uint8_t* success_out, int* search_level_out,
                               double* A_cur_ref_out, double* h_inv_out) {
  if (!ctx || !cur || !cur_T_f_w || !cam || !opt || M < 0)
    return set_err(ctx, SVO_B200_EINVAL, "find_match_direct: bad arguments");
  if (M == 0) return 0;  // no candidates: nothing to read, whatever the reference frames
  if (!ref_frames || !ref_T_f_w || n_ref <= 0)
    return set_err(ctx, SVO_B200_EINVAL, "find_match_direct: no reference frames");
  for (int r = 0; r < n_ref; ++r)
    if (!ref_frames[r]) return set_err(ctx, SVO_B200_EINVAL, "find_match_direct: ref_frames[%d] is NULL", r);
  if (!ref_index || !ref_px || !ref_f || !ref_level || !ftr_type || !ref_grad || !point_pos || !px_cur_io || !success_out)
    return set_err(ctx, SVO_B200_EINVAL, "find_match_direct: NULL candidate arrays");
  int rc = check_ref_table(ctx, "find_match_direct", "ref_level", ref_frames, n_ref, M, ref_index, ref_level, cur, cam,
                           opt->max_search_level);
  if (rc) return rc;
  Cam cm;
  if ((rc = cam_to_dev(ctx, cam, cm))) return rc;
  cudaSetDevice(ctx->device);
  std::vector<FrameDesc> frames((size_t)n_ref);
  for (int r = 0; r < n_ref; ++r) frames[r] = make_desc(ref_frames[r]);
  Staging st(ctx);
  MatchIn in;
  MatchOut out;
  const double* d_cur_T;
  st.in(ref_index, M, &in.ref_index);
  st.in(ref_px, 2 * (size_t)M, &in.ref_px);
  st.in(ref_f, 3 * (size_t)M, &in.ref_f);
  st.in(ref_level, M, &in.ref_level);
  st.in(ftr_type, M, &in.ftr_type);
  st.in(ref_grad, 2 * (size_t)M, &in.ref_grad);
  st.in(point_pos, 3 * (size_t)M, &in.point_pos);
  st.in(ref_T_f_w, 12 * (size_t)n_ref, &in.ref_T_f_w);
  st.in(cur_T_f_w, 12, &d_cur_T);
  st.in(frames.data(), n_ref, &in.ref_frames);
  st.inout(px_cur_io, 2 * (size_t)M, &out.px_cur);
  st.out(success_out, M, &out.success);
  st.out(search_level_out, M, &out.search_level);
  st.out(A_cur_ref_out, 4 * (size_t)M, &out.A_cur_ref);
  st.out(h_inv_out, M, &out.h_inv);
  if ((rc = st.open()) || (rc = st.send())) return rc;
  const int blocks = (M + kWarpsPerCta - 1) / kWarpsPerCta;
  if ((rc = launch_kernels(ctx, 1, [&] {
         find_match_direct_kernel<<<blocks, kWarpsPerCta * 32, 0, ctx->stream>>>(make_desc(cur), cm, M, in, out, opt->max_search_level,
                                                                                 opt->align_max_iter, d_cur_T);
       })))
    return rc;
  return st.receive();
}

}  // extern "C"
