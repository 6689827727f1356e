// rpg_svo_b200/csrc/warp_align.cuh -- warp-cooperative device routines shared by align.cu,
// depth_filter.cu and reproject.cu: one warp owns one feature / seed / point.
//
//   warp_align2d / warp_align1d  <- feature_alignment::align2D / align1D   svo/src/feature_alignment.cpp:149-277, 30-147
//   warp_get_warp_matrix_affine  <- warp::getWarpMatrixAffine              svo/src/matcher.cpp:33-55
//   best_search_level            <- warp::getBestSearchLevel               svo/src/matcher.cpp:57-70
//   warp_warp_affine             <- warp::warpAffine + createPatchFromPatchWithBorder   svo/src/matcher.cpp:72-105,124-133
//   depth_from_triangulation     <- depthFromTriangulation                 svo/src/matcher.cpp:109-122
//
// The 64 pixel residuals of an 8x8 patch are computed two per lane; the three Jres sums are then
// accumulated in the reference's pixel order (every lane runs the same 64-step chain on shared
// memory), so the float arithmetic is the reference's operation for operation and the results are
// bit-identical to the CPU oracle, not merely close.
#pragma once
#include <cstring>

#include "ctx.h"
#include "svo_math.cuh"

namespace svo {

// level pointers + geometry of one frame, passed to kernels by value or in arrays
struct FrameDesc {
  const uint8_t* lvl[SVO_B200_MAX_LEVELS];
  int w[SVO_B200_MAX_LEVELS], h[SVO_B200_MAX_LEVELS];
  int n_levels;
};
static inline FrameDesc make_desc(const svo_b200_frame* f) {
  FrameDesc d;
  memset(&d, 0, sizeof(d));
  d.n_levels = f->n_levels;
  for (int l = 0; l < f->n_levels; ++l) { d.lvl[l] = f->lvl(l); d.w[l] = f->w[l]; d.h[l] = f->h[l]; }
  return d;
}

// The stream that owns item i of a launch over n_streams streams' concatenated items, stream s owning items offset[s] ..
// offset[s + 1] - 1: the last s with offset[s] <= i (streams without items are skipped over).
__device__ __forceinline__ int stream_of(const int* __restrict__ offset, int n_streams, int i) {
  int lo = 0, hi = n_streams - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(offset + mid) <= i) lo = mid; else hi = mid - 1;
  }
  return lo;
}


struct ImgView {
  const uint8_t* data;
  int cols, rows;  // row pitch == cols
};

using Cam = CamDev;  // [EXT] vk::AbstractCamera: pinhole (+ radial-tangential distortion) or ATAN, see ctx.h / svo_math.cuh

struct __align__(16) WarpAlignScratch {  // one per warp, shared memory
  float dx[64];
  float dy[64];
  float res[64];
  uint8_t pwb[112];    // 10x10 reference patch with border (100 used)
  uint8_t patch[64];   // 8x8 reference patch
};

// [EXT] Eigen compute_inverse_size3 for Matrix3f (same formula as oracle/svo_oracle_align.inc).
__device__ __forceinline__ float cof3(const float (&m)[3][3], int i, int j) {
  const int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
  return fmaf(m[i1][j1], m[i2][j2], -__fmul_rn(m[i1][j2], m[i2][j1]));
}
__device__ __forceinline__ void inverse3f(const float (&m)[3][3], float (&r)[3][3]) {
  const float c0 = cof3(m, 0, 0), c1 = cof3(m, 1, 0), c2 = cof3(m, 2, 0);
  const float det = fmaf(c2, m[2][0], fmaf(c0, m[0][0], __fmul_rn(c1, m[1][0])));
  const float invdet = __fdiv_rn(1.0f, det);
  r[0][0] = __fmul_rn(c0, invdet); r[0][1] = __fmul_rn(c1, invdet); r[0][2] = __fmul_rn(c2, invdet);
  r[1][0] = __fmul_rn(cof3(m, 0, 1), invdet); r[1][1] = __fmul_rn(cof3(m, 1, 1), invdet); r[1][2] = __fmul_rn(cof3(m, 2, 1), invdet);
  r[2][0] = __fmul_rn(cof3(m, 0, 2), invdet); r[2][1] = __fmul_rn(cof3(m, 1, 2), invdet); r[2][2] = __fmul_rn(cof3(m, 2, 2), invdet);
}
__device__ __forceinline__ void inverse2f(const float (&m)[2][2], float (&r)[2][2]) {
  const float det = fmaf(m[0][0], m[1][1], -__fmul_rn(m[1][0], m[0][1]));
  const float invdet = __fdiv_rn(1.0f, det);
  r[0][0] = __fmul_rn(m[1][1], invdet);
  r[1][0] = __fmul_rn(-m[1][0], invdet);
  r[0][1] = __fmul_rn(-m[0][1], invdet);
  r[1][1] = __fmul_rn(m[0][0], invdet);
}

// One residual pass: lane l fills res[l] and res[l+32].
__device__ __forceinline__ void warp_patch_residuals(const ImgView& img, WarpAlignScratch& S, int u_r, int v_r,
                                                     float wTL, float wTR, float wBL, float wBR, float mean_diff) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int p = lane + 32 * h, y = p >> 3, x = p & 7;
    const uint8_t* it = img.data + (size_t)(v_r + y - 4) * img.cols + (u_r + x - 4);
    const float search_pixel = bilin(wTL, wTR, wBL, wBR, (float)__ldg(it), (float)__ldg(it + 1),
                                     (float)__ldg(it + img.cols), (float)__ldg(it + img.cols + 1));
    S.res[p] = __fadd_rn(__fsub_rn(search_pixel, (float)S.patch[p]), mean_diff);
  }
  __syncwarp();
}

// feature_alignment::align2D (float path).  All lanes call with the same arguments; the return value
// and (u, v) are warp-uniform.  *nan_exit is set when the reference would `return false` without
// writing cur_px_estimate (feature_alignment.cpp:209).
__device__ inline bool warp_align2d(const ImgView& img, WarpAlignScratch& S, int n_iter, double& px_u,
                                    double& px_v, bool* nan_exit, int* iters_done = nullptr) {
  const int lane = threadIdx.x & 31;
  // template gradients (:176-189): J = [0.5*(I[+1]-I[-1]), 0.5*(I[+10]-I[-10]), 1]
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int p = lane + 32 * h, y = p >> 3, x = p & 7;
    const uint8_t* it = S.pwb + (y + 1) * 10 + 1 + x;
    S.dx[p] = 0.5f * (float)((int)it[1] - (int)it[-1]);
    S.dy[p] = 0.5f * (float)((int)it[10] - (int)it[-10]);
  }
  __syncwarp();
  float H[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
  for (int p = 0; p < 64; ++p) {
    const float J[3] = {S.dx[p], S.dy[p], 1.0f};
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
      for (int b = 0; b < 3; ++b) H[a][b] = fmaf(J[a], J[b], H[a][b]);
  }
  float Hinv[3][3];
  inverse3f(H, Hinv);
  float mean_diff = 0.f;
  float u = (float)px_u, v = (float)px_v;
  const float min_update_squared = (float)(0.03 * 0.03);
  bool converged = false;
  *nan_exit = false;
  int iter = 0;
  for (; iter < n_iter; ++iter) {
    const bool bad = !(fabsf(u) < 1e9f) || !(fabsf(v) < 1e9f);  // NaN / out of int range: x86 yields INT_MIN
    const int u_r = bad ? -1 : (int)floorf(u), v_r = bad ? -1 : (int)floorf(v);
    if (u_r < 4 || v_r < 4 || u_r >= img.cols - 4 || v_r >= img.rows - 4) break;  // (:206-207)
    if (isnan(u) || isnan(v)) {  // unreachable after the border test, kept for fidelity (:209)
      *nan_exit = true;
      return false;
    }
    float wTL, wTR, wBL, wBR;
    bilin_weights(__fsub_rn(u, (float)u_r), __fsub_rn(v, (float)v_r), wTL, wTR, wBL, wBR);
    warp_patch_residuals(img, S, u_r, v_r, wTL, wTR, wBL, wBR, mean_diff);
    float J0 = 0.f, J1 = 0.f, J2 = 0.f;
    for (int p = 0; p < 64; ++p) {  // reference pixel order (:226-238)
      const float r = S.res[p];
      J0 = fmaf(-r, S.dx[p], J0);
      J1 = fmaf(-r, S.dy[p], J1);
      J2 = __fsub_rn(J2, r);
    }
    __syncwarp();
    const float up0 = fmaf(Hinv[0][2], J2, fmaf(Hinv[0][0], J0, __fmul_rn(Hinv[0][1], J1)));
    const float up1 = fmaf(Hinv[1][2], J2, fmaf(Hinv[1][0], J0, __fmul_rn(Hinv[1][1], J1)));
    const float up2 = fmaf(Hinv[2][2], J2, fmaf(Hinv[2][0], J0, __fmul_rn(Hinv[2][1], J1)));
    u = __fadd_rn(u, up0);
    v = __fadd_rn(v, up1);
    mean_diff = __fadd_rn(mean_diff, up2);
    if (fmaf(up0, up0, __fmul_rn(up1, up1)) < min_update_squared) {
      converged = true;
      ++iter;
      break;
    }
  }
  if (iters_done) *iters_done = iter;
  px_u = (double)u;
  px_v = (double)v;
  return converged;
}

// feature_alignment::align1D.
__device__ inline bool warp_align1d(const ImgView& img, WarpAlignScratch& S, float dir0, float dir1, int n_iter,
                                    double& px_u, double& px_v, double& h_inv, bool* nan_exit) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int p = lane + 32 * h, y = p >> 3, x = p & 7;
    const uint8_t* it = S.pwb + (y + 1) * 10 + 1 + x;
    // J[0] = 0.5*(dir[0]*(it[1]-it[-1]) + dir[1]*(it[ref_step]-it[-ref_step]))  (:56)
    S.dx[p] = 0.5f * fmaf(dir0, (float)((int)it[1] - (int)it[-1]), __fmul_rn(dir1, (float)((int)it[10] - (int)it[-10])));
  }
  __syncwarp();
  float H[2][2] = {{0, 0}, {0, 0}};
  for (int p = 0; p < 64; ++p) {
    const float J[2] = {S.dx[p], 1.0f};
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
      for (int b = 0; b < 2; ++b) H[a][b] = fmaf(J[a], J[b], H[a][b]);
  }
  h_inv = 1.0 / (double)H[0][0] * 8 * 8;  // (:63)
  float Hinv[2][2];
  inverse2f(H, Hinv);
  float mean_diff = 0.f;
  float u = (float)px_u, v = (float)px_v;
  const float min_update_squared = (float)(0.03 * 0.03);
  float chi2 = 0.f, up0 = 0.f, up1 = 0.f;
  bool converged = false;
  *nan_exit = false;
  for (int iter = 0; iter < n_iter; ++iter) {
    const bool bad = !(fabsf(u) < 1e9f) || !(fabsf(v) < 1e9f);
    const int u_r = bad ? -1 : (int)floorf(u), v_r = bad ? -1 : (int)floorf(v);
    if (u_r < 4 || v_r < 4 || u_r >= img.cols - 4 || v_r >= img.rows - 4) break;
    if (isnan(u) || isnan(v)) {
      *nan_exit = true;
      return false;
    }
    float wTL, wTR, wBL, wBR;
    bilin_weights(__fsub_rn(u, (float)u_r), __fsub_rn(v, (float)v_r), wTL, wTR, wBL, wBR);
    warp_patch_residuals(img, S, u_r, v_r, wTL, wTR, wBL, wBR, mean_diff);
    float J0 = 0.f, J1 = 0.f, new_chi2 = 0.f;
    for (int p = 0; p < 64; ++p) {
      const float r = S.res[p];
      J0 = fmaf(-r, S.dx[p], J0);
      J1 = __fsub_rn(J1, r);
      new_chi2 = fmaf(r, r, new_chi2);
    }
    __syncwarp();
    if (iter > 0 && new_chi2 > chi2) {  // (:112-120) rollback subtracts the raw update (sic)
      u = __fsub_rn(u, up0);
      v = __fsub_rn(v, up1);
      break;
    }
    chi2 = new_chi2;
    up0 = fmaf(Hinv[0][1], J1, __fmul_rn(Hinv[0][0], J0));  // fusion order as the compiled reference (oracle/_ref)
    up1 = fmaf(Hinv[1][1], J1, __fmul_rn(Hinv[1][0], J0));
    u = fmaf(up0, dir0, u);
    v = fmaf(up0, dir1, v);
    mean_diff = __fadd_rn(mean_diff, up1);
    if (fmaf(up0, up0, __fmul_rn(up1, up1)) < min_update_squared) {
      converged = true;
      break;
    }
  }
  px_u = (double)u;
  px_v = (double)v;
  return converged;
}

// ------------------------------------------------------------------------------------------ geometry
__device__ __forceinline__ void cam2world(const Cam& c, double u, double v, double* out) {  // [EXT] normalised bearing
  double f[3];
  cam_cam2world(c, u, v, f);
  out[0] = f[0]; out[1] = f[1]; out[2] = f[2];
}
__device__ __forceinline__ void world2cam(const Cam& c, const double* p, double& u, double& v) {  // [EXT] world2cam(project2d(xyz))
  cam_world2cam(c, p[0] / p[2], p[1] / p[2], u, v);
}
__device__ __forceinline__ void pose_apply(const Pose& T, const double* p, double* out) {
  qrotate(T.q, p, out);
  out[0] += T.t[0]; out[1] += T.t[1]; out[2] += T.t[2];
}

// warp::getWarpMatrixAffine (matcher.cpp:33-55); A row-major [a00 a01 a10 a11]
__device__ inline void get_warp_matrix_affine(const Cam& cam, double pxu, double pxv, const double* f_ref,
                                              double depth_ref, const Pose& T_cur_ref, int level_ref, double* A) {
  const int halfpatch_size = 5;
  const double xyz_ref[3] = {f_ref[0] * depth_ref, f_ref[1] * depth_ref, f_ref[2] * depth_ref};
  double du[3], dv[3];
  cam2world(cam, pxu + (double)halfpatch_size * (double)(1 << level_ref), pxv, du);
  cam2world(cam, pxu, pxv + (double)halfpatch_size * (double)(1 << level_ref), dv);
  const double su = xyz_ref[2] / du[2], sv = xyz_ref[2] / dv[2];
  du[0] *= su; du[1] *= su; du[2] *= su;
  dv[0] *= sv; dv[1] *= sv; dv[2] *= sv;
  double p0[3], p1[3], p2[3], cu, cv, uu, uv, vu, vv;
  pose_apply(T_cur_ref, xyz_ref, p0);
  pose_apply(T_cur_ref, du, p1);
  pose_apply(T_cur_ref, dv, p2);
  world2cam(cam, p0, cu, cv);
  world2cam(cam, p1, uu, uv);
  world2cam(cam, p2, vu, vv);
  A[0] = (uu - cu) / halfpatch_size;
  A[2] = (uv - cv) / halfpatch_size;
  A[1] = (vu - cu) / halfpatch_size;
  A[3] = (vv - cv) / halfpatch_size;
}

// warp::getBestSearchLevel (matcher.cpp:57-70)
__device__ __forceinline__ int best_search_level(const double* A, int max_level) {
  int search_level = 0;
  double D = A[0] * A[3] - A[2] * A[1];
  while (D > 3.0 && search_level < max_level) {
    search_level += 1;
    D *= 0.25;
  }
  return search_level;
}

// [EXT] vk::interpolateMat_8u
__device__ __forceinline__ float interpolate_mat_8u(const ImgView& img, float u, float v) {
  const int x = (int)floorf(u), y = (int)floorf(v);
  const float sx = __fsub_rn(u, (float)x), sy = __fsub_rn(v, (float)y);
  const float w00 = __fmul_rn(__fsub_rn(1.0f, sx), __fsub_rn(1.0f, sy));
  const float w01 = __fmul_rn(__fsub_rn(1.0f, sx), sy);
  const float w10 = __fmul_rn(sx, __fsub_rn(1.0f, sy));
  const float w11 = __fsub_rn(__fsub_rn(__fsub_rn(1.0f, w00), w01), w10);
  const uint8_t* ptr = img.data + (size_t)y * img.cols + x;
  return fmaf(w11, (float)__ldg(ptr + img.cols + 1),
              fmaf(w10, (float)__ldg(ptr + 1), fmaf(w00, (float)__ldg(ptr), __fmul_rn(w01, (float)__ldg(ptr + img.cols)))));
}

// warp::warpAffine for the 10x10 patch + createPatchFromPatchWithBorder.  Lanes stride over the 100
// samples.  On the NaN path the reference leaves the (reused) patch untouched; the caller passes
// what that stale content would be (zeros for a fresh Matcher).
__device__ inline bool warp_warp_affine(const double* A_cur_ref, const ImgView& img_ref, double pxu, double pxv,
                                        int level_ref, int search_level, WarpAlignScratch& S) {
  const int lane = threadIdx.x & 31;
  const double det = A_cur_ref[0] * A_cur_ref[3] - A_cur_ref[2] * A_cur_ref[1];
  const double invdet = 1.0 / det;  // [EXT] Eigen 2x2 inverse
  const float A00 = (float)(A_cur_ref[3] * invdet), A01 = (float)(-A_cur_ref[1] * invdet);
  const float A10 = (float)(-A_cur_ref[2] * invdet), A11 = (float)(A_cur_ref[0] * invdet);
  const bool ok = !isnan(A00);
  if (ok) {
    const float prx = __fdiv_rn((float)pxu, (float)(1 << level_ref));
    const float pry = __fdiv_rn((float)pxv, (float)(1 << level_ref));
    const float sc = (float)(1 << search_level);
    for (int i = lane; i < 100; i += 32) {
      const int y = i / 10, x = i - 10 * y;
      const float ppx = __fmul_rn((float)(x - 5), sc), ppy = __fmul_rn((float)(y - 5), sc);
      const float qx = __fadd_rn(fmaf(A00, ppx, __fmul_rn(A01, ppy)), prx);
      const float qy = __fadd_rn(fmaf(A10, ppx, __fmul_rn(A11, ppy)), pry);
      uint8_t val = 0;
      if (!(qx < 0 || qy < 0 || qx >= (float)(img_ref.cols - 1) || qy >= (float)(img_ref.rows - 1)))
        val = (uint8_t)interpolate_mat_8u(img_ref, qx, qy);  // truncation
      S.pwb[i] = val;
    }
  }
  __syncwarp();
  for (int i = lane; i < 64; i += 32) S.patch[i] = S.pwb[((i >> 3) + 1) * 10 + 1 + (i & 7)];
  __syncwarp();
  return ok;
}

// depthFromTriangulation (matcher.cpp:109-122)
__device__ inline bool depth_from_triangulation(const Pose& T_search_ref, const double* f_ref, const double* f_cur,
                                                double& depth) {
  double a0[3];
  {
    double R[9];
    qmatrix(T_search_ref.q, R);
    a0[0] = R[0] * f_ref[0] + R[1] * f_ref[1] + R[2] * f_ref[2];
    a0[1] = R[3] * f_ref[0] + R[4] * f_ref[1] + R[5] * f_ref[2];
    a0[2] = R[6] * f_ref[0] + R[7] * f_ref[1] + R[8] * f_ref[2];
  }
  const double* a1 = f_cur;
  const double m00 = a0[0] * a0[0] + a0[1] * a0[1] + a0[2] * a0[2];
  const double m01 = a0[0] * a1[0] + a0[1] * a1[1] + a0[2] * a1[2];
  const double m11 = a1[0] * a1[0] + a1[1] * a1[1] + a1[2] * a1[2];
  const double det = m00 * m11 - m01 * m01;
  if (det < 0.000001) return false;
  const double invdet = 1.0 / det;
  const double i00 = m11 * invdet, i01 = -m01 * invdet;
  const double* t = T_search_ref.t;
  const double b0 = a0[0] * t[0] + a0[1] * t[1] + a0[2] * t[2];
  const double b1 = a1[0] * t[0] + a1[1] * t[1] + a1[2] * t[2];
  depth = fabs(-(i00 * b0 + i01 * b1));
  return true;
}

// Matcher::findMatchDirect (matcher.cpp:135-177) for one candidate, after Point::getCloseViewObs picked the reference
// observation: one warp, S = its scratch slice.  px_cur (pu, pv) is the initial guess in level-0 pixels and receives the
// refined position; search_level / A / h_inv are the Matcher members the callers read afterwards.
__device__ inline bool warp_find_match_direct(const FrameDesc& cur, const Cam& cam, const FrameDesc& rf, const Pose& T_ref_w,
                                              const Pose& T_cur_w, const double* ref_px, const double* f_ref, int lvl,
                                              int ftr_type, const double* ref_grad, const double* point_pos,
                                              int max_search_level, int align_max_iter, WarpAlignScratch& S, double& pu,
                                              double& pv, int& search_level, double* A, double& h_inv) {
  const int lane = threadIdx.x & 31;
  for (int i = lane; i < 112; i += 32) S.pwb[i] = 0;  // a fresh Matcher's patch_with_border_
  __syncwarp();
  const double pxu = ref_px[0], pxv = ref_px[1];
  // isInFrame(px.cast<int>()/(1<<level), halfpatch_size_+2, level)  (:143-145)
  const int xi = (int)pxu / (1 << lvl), yi = (int)pxv / (1 << lvl);
  const bool in_frame = xi >= 6 && xi < cam.width / (1 << lvl) - 6 && yi >= 6 && yi < cam.height / (1 << lvl) - 6;
  if (!in_frame) return false;
  const Pose T_ref_w_inv = pose_inv(T_ref_w);
  const Pose T_cur_ref = pose_mul(T_cur_w, T_ref_w_inv);
  // depth = (ref_frame.pos() - pt.pos_).norm()
  const double dxp = T_ref_w_inv.t[0] - point_pos[0], dyp = T_ref_w_inv.t[1] - point_pos[1], dzp = T_ref_w_inv.t[2] - point_pos[2];
  const double depth = sqrt(dxp * dxp + dyp * dyp + dzp * dzp);
  get_warp_matrix_affine(cam, pxu, pxv, f_ref, depth, T_cur_ref, lvl, A);
  search_level = best_search_level(A, max_search_level);
  ImgView ref_img = {rf.lvl[lvl], rf.w[lvl], rf.h[lvl]};
  warp_warp_affine(A, ref_img, pxu, pxv, lvl, search_level, S);
  ImgView cur_img = {cur.lvl[search_level], cur.w[search_level], cur.h[search_level]};
  double su = pu / (double)(1 << search_level), sv = pv / (double)(1 << search_level);
  bool nan_exit = false, ok;
  if (ftr_type == 1) {  // EDGELET: dir = normalize(A * grad)  (:158-164)
    const double gx = ref_grad[0], gy = ref_grad[1];
    const double dx = A[0] * gx + A[1] * gy, dy = A[2] * gx + A[3] * gy;
    const double n = sqrt(dx * dx + dy * dy);
    ok = warp_align1d(cur_img, S, (float)(dx / n), (float)(dy / n), align_max_iter, su, sv, h_inv, &nan_exit);
  } else {
    ok = warp_align2d(cur_img, S, align_max_iter, su, sv, &nan_exit);
  }
  // px_cur = px_scaled * (1<<search_level_) -- px_scaled keeps its input value on the NaN exit
  pu = su * (double)(1 << search_level);
  pv = sv * (double)(1 << search_level);
  return ok;
}

}  // namespace svo
