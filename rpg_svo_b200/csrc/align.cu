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
  Carver c;
  const size_t o_lvl = c.take(sizeof(int) * M), o_dir = c.take(dir ? sizeof(float) * 2 * M : 0),
               o_pwb = c.take((size_t)100 * M), o_pat = c.take((size_t)64 * M), o_px = c.take(sizeof(double) * 2 * M);
  const size_t in_bytes = c.off;
  const size_t o_conv = c.take(M), o_h = c.take(sizeof(double) * M);
  int rc;
  if ((rc = ensure_host(ctx, ctx->h_in, c.off))) return rc;
  if ((rc = ensure_dev(ctx, ctx->d_in, c.off))) return rc;
  SVO_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
  uint8_t* h = static_cast<uint8_t*>(ctx->h_in.p);
  uint8_t* d = static_cast<uint8_t*>(ctx->d_in.p);
  memcpy(h + o_lvl, level, sizeof(int) * M);
  if (dir) memcpy(h + o_dir, dir, sizeof(float) * 2 * M);
  memcpy(h + o_pwb, pwb, (size_t)100 * M);
  memcpy(h + o_pat, patch, (size_t)64 * M);
  memcpy(h + o_px, px_io, sizeof(double) * 2 * M);
  SVO_CUDA_CHECK(ctx, cudaMemcpyAsync(d, h, in_bytes, cudaMemcpyHostToDevice, ctx->stream));
  const int blocks = (M + kWarpsPerCta - 1) / kWarpsPerCta;
  kt_begin(ctx);
  align_batch_kernel<<<blocks, kWarpsPerCta * 32, 0, ctx->stream>>>(
      make_desc(cur), M, reinterpret_cast<const int*>(d + o_lvl), dir ? reinterpret_cast<const float*>(d + o_dir) : nullptr,
      d + o_pwb, d + o_pat, n_iter, reinterpret_cast<double*>(d + o_px), d + o_conv,
      h_inv_out ? reinterpret_cast<double*>(d + o_h) : nullptr);
  ctx->launches++;
  kt_end(ctx);
  SVO_CUDA_CHECK(ctx, cudaGetLastError());
  SVO_CUDA_CHECK(ctx, cudaMemcpyAsync(h + o_px, d + o_px, c.off - o_px, cudaMemcpyDeviceToHost, ctx->stream));
  SVO_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
  memcpy(px_io, h + o_px, sizeof(double) * 2 * M);
  memcpy(converged_out, h + o_conv, M);
  if (h_inv_out) memcpy(h_inv_out, h + o_h, sizeof(double) * M);
  return 0;
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
  for (int m = 0; m < M; ++m) {
    if (ref_index[m] < 0 || ref_index[m] >= n_ref)
      return set_err(ctx, SVO_B200_EINVAL, "find_match_direct: ref_index[%d] out of range", m);
    if (ref_level[m] < 0 || ref_level[m] >= ref_frames[ref_index[m]]->n_levels)
      return set_err(ctx, SVO_B200_EINVAL, "find_match_direct: ref_level[%d] outside the pyramid", m);
  }
  if (opt->max_search_level >= cur->n_levels)
    return set_err(ctx, SVO_B200_EINVAL, "find_match_direct: max_search_level %d >= %d pyramid levels",
                   opt->max_search_level, cur->n_levels);
  if (const int rc_sz = cam_check_frames(ctx, "find_match_direct", cam, &cur, 1)) return rc_sz;
  if (const int rc_sz = cam_check_frames(ctx, "find_match_direct", cam, ref_frames, n_ref)) return rc_sz;
  cudaSetDevice(ctx->device);
  Carver c;
  const size_t o_ri = c.take(sizeof(int) * M), o_px = c.take(sizeof(double) * 2 * M), o_f = c.take(sizeof(double) * 3 * M),
               o_lv = c.take(sizeof(int) * M), o_ty = c.take(sizeof(int) * M), o_gr = c.take(sizeof(double) * 2 * M),
               o_pp = c.take(sizeof(double) * 3 * M), o_rT = c.take(sizeof(double) * 12 * n_ref),
               o_cT = c.take(sizeof(double) * 12), o_fr = c.take(sizeof(FrameDesc) * n_ref),
               o_pc = c.take(sizeof(double) * 2 * M);
  const size_t in_bytes = c.off;
  const size_t o_su = c.take(M), o_sl = c.take(sizeof(int) * M), o_A = c.take(sizeof(double) * 4 * M),
               o_h = c.take(sizeof(double) * M);
  int rc;
  if ((rc = ensure_host(ctx, ctx->h_in, c.off))) return rc;
  if ((rc = ensure_dev(ctx, ctx->d_in, c.off))) return rc;
  SVO_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
  uint8_t* h = static_cast<uint8_t*>(ctx->h_in.p);
  uint8_t* d = static_cast<uint8_t*>(ctx->d_in.p);
  memcpy(h + o_ri, ref_index, sizeof(int) * M);
  memcpy(h + o_px, ref_px, sizeof(double) * 2 * M);
  memcpy(h + o_f, ref_f, sizeof(double) * 3 * M);
  memcpy(h + o_lv, ref_level, sizeof(int) * M);
  memcpy(h + o_ty, ftr_type, sizeof(int) * M);
  memcpy(h + o_gr, ref_grad, sizeof(double) * 2 * M);
  memcpy(h + o_pp, point_pos, sizeof(double) * 3 * M);
  memcpy(h + o_rT, ref_T_f_w, sizeof(double) * 12 * n_ref);
  memcpy(h + o_cT, cur_T_f_w, sizeof(double) * 12);
  for (int r = 0; r < n_ref; ++r) reinterpret_cast<FrameDesc*>(h + o_fr)[r] = make_desc(ref_frames[r]);
  memcpy(h + o_pc, px_cur_io, sizeof(double) * 2 * M);
  SVO_CUDA_CHECK(ctx, cudaMemcpyAsync(d, h, in_bytes, cudaMemcpyHostToDevice, ctx->stream));
  MatchIn in = {reinterpret_cast<const int*>(d + o_ri), reinterpret_cast<const double*>(d + o_px),
                reinterpret_cast<const double*>(d + o_f), reinterpret_cast<const int*>(d + o_lv),
                reinterpret_cast<const int*>(d + o_ty), reinterpret_cast<const double*>(d + o_gr),
                reinterpret_cast<const double*>(d + o_pp), reinterpret_cast<const double*>(d + o_rT),
                reinterpret_cast<const FrameDesc*>(d + o_fr)};
  MatchOut out = {reinterpret_cast<double*>(d + o_pc), d + o_su, reinterpret_cast<int*>(d + o_sl),
                  reinterpret_cast<double*>(d + o_A), reinterpret_cast<double*>(d + o_h)};
  Cam cm;
  { const int rc_cam = cam_to_dev(ctx, cam, cm); if (rc_cam) return rc_cam; }
  const int blocks = (M + kWarpsPerCta - 1) / kWarpsPerCta;
  kt_begin(ctx);
  find_match_direct_kernel<<<blocks, kWarpsPerCta * 32, 0, ctx->stream>>>(
      make_desc(cur), cm, M, in, out, opt->max_search_level, opt->align_max_iter, reinterpret_cast<const double*>(d + o_cT));
  ctx->launches++;
  kt_end(ctx);
  SVO_CUDA_CHECK(ctx, cudaGetLastError());
  SVO_CUDA_CHECK(ctx, cudaMemcpyAsync(h + o_pc, d + o_pc, c.off - o_pc, cudaMemcpyDeviceToHost, ctx->stream));
  SVO_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
  memcpy(px_cur_io, h + o_pc, sizeof(double) * 2 * M);
  memcpy(success_out, h + o_su, M);
  if (search_level_out) memcpy(search_level_out, h + o_sl, sizeof(int) * M);
  if (A_cur_ref_out) memcpy(A_cur_ref_out, h + o_A, sizeof(double) * 4 * M);
  if (h_inv_out) memcpy(h_inv_out, h + o_h, sizeof(double) * M);
  return 0;
}

}  // extern "C"
