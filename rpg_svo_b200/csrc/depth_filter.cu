// rpg_svo_b200/csrc/depth_filter.cu -- DepthFilter::updateSeeds on sm_90a: one warp per seed.
//
// Replaces svo/src/depth_filter.cpp:197-291 (updateSeeds), :309-332 (updateSeed), :334-350
// (computeTau) and the Matcher::findEpipolarMatchDirect call inside it (svo/src/matcher.cpp:179-321).
// The reference walks a std::list<Seed> on the mapper thread; seeds are independent given the two
// frames, so here the host flattens the list to SoA, one launch updates every seed, and a status
// byte per seed tells the host which list operations (erase, converged callback, b++) to replay in
// list order.
//
// Per seed (warp): geometry in f64 on all lanes (uniform), the 10x10 affine warp of the reference
// patch with lanes striding the 100 samples, the epipolar ZMSSD scan with lanes striding the <= 1001
// steps (integer score via dp4a on 8-byte rows fetched as aligned words; warp arg-min with the
// reference's "first strict minimum wins" tie rule on the packed (score, step) key), then the
// warp-cooperative align2D, triangulation, computeTau and the f32 Bayesian update.
#include <cstring>
#include <vector>

#include "ctx.h"
#include "warp_align.cuh"

namespace svo {

constexpr int kDfWarps = 4;

// What differs between the streams of one launch, in a per-launch device table: the current frame, its pose, the camera
// and Seed::batch_counter.
struct DepthStream {
  FrameDesc cur;
  Cam cam;
  double cur_T_f_w[12];
  int batch_counter;
};

struct DepthParams {
  const FrameDesc* ref_frames;
  const double* ref_T_f_w;
  int M;
  const int* ref_index;
  const double* ftr_px;
  const double* ftr_f;
  const int* ftr_level;
  const int* ftr_type;
  const double* ftr_grad;
  const int* batch_id;
  int max_n_kfs;
  double sigma2_thresh;
  int max_search_level, align_max_iter, max_epi_search_steps;
  float *a, *b, *mu, *z_range, *sigma2;
  uint8_t* status;
  double* px_cur;
  double* z;
  int* n_zmssd;
  // standalone Matcher::findEpipolarMatchDirect (svo_b200_find_epipolar_match_direct): explicit depth range per
  // candidate instead of seeds, no Bayesian update, the Matcher's public scratch members as outputs
  int match_only;
  const double *d_est, *d_min, *d_max;
  int* search_level_out;
  double* epi_length_out;
  uint8_t* reject_out;
  double* A_out;
  // Matcher::Options of svo_b200_set_epipolar_options, read only by the general instantiation; with match_only it also
  // returns h_inv_ and whether align1D ran (svo_b200_epipolar_last_h_inv)
  svo_b200_epipolar_options epi;
  double* h_inv_out;
  uint8_t* ran_1d_out;
};

// [EXT] vk::patch_score::ZMSSD<4>::computeScore on the 8x8 block whose top-left pixel is at byte
// offset `off` of an image with row pitch `cols`; ref = the 16 words of the warped reference patch.
__device__ __forceinline__ int zmssd_score(const uint8_t* img, int off, int cols, const uint32_t* ref, int sumA,
                                           int sumAA) {
  unsigned sumB = 0, sumBB = 0, sumAB = 0;
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    const int o = off + r * cols;
    const int a = o & ~3;
    const unsigned sh = (unsigned)(o & 3) * 8u;
    const uint32_t w0 = __ldg(reinterpret_cast<const uint32_t*>(img + a));
    const uint32_t w1 = __ldg(reinterpret_cast<const uint32_t*>(img + a + 4));
    const uint32_t w2 = __ldg(reinterpret_cast<const uint32_t*>(img + a + 8));
    const uint32_t lo = __funnelshift_r(w0, w1, sh), hi = __funnelshift_r(w1, w2, sh);
    sumB = __dp4a(lo, 0x01010101u, sumB);
    sumB = __dp4a(hi, 0x01010101u, sumB);
    sumBB = __dp4a(lo, lo, sumBB);
    sumBB = __dp4a(hi, hi, sumBB);
    sumAB = __dp4a(lo, ref[2 * r], sumAB);
    sumAB = __dp4a(hi, ref[2 * r + 1], sumAB);
  }
  const int iB = (int)sumB, iBB = (int)sumBB, iAB = (int)sumAB;
  return sumAA - 2 * iAB + iBB - (sumA * sumA - 2 * sumA * iB + iB * iB) / 64;
}

// [EXT] boost::math::pdf(normal_distribution<float>(mean, sd), x)
__device__ __forceinline__ float normal_pdf_f(float mean, float sd, float x) {
  if (isinf(x)) return 0.f;
  float exponent = __fsub_rn(x, mean);
  exponent = __fmul_rn(exponent, -exponent);
  exponent = __fdiv_rn(exponent, __fmul_rn(__fmul_rn(2.f, sd), sd));
  float result = expf(exponent);
  result = __fdiv_rn(result, __fmul_rn(sd, sqrtf(2.f * 3.14159265358979323846264338327950288f)));
  return result;
}

// DepthFilter::updateSeed (depth_filter.cpp:309-332); float/double promotions as the literals dictate.
__device__ inline void update_seed(float x, float tau2, float& a, float& b, float& mu, float z_range, float& sigma2) {
  const float norm_scale = sqrtf(__fadd_rn(sigma2, tau2));
  if (isnan(norm_scale)) return;
  const float s2 = (float)(1. / (1. / (double)sigma2 + 1. / (double)tau2));
  const float m = __fmul_rn(s2, __fadd_rn(__fdiv_rn(mu, sigma2), __fdiv_rn(x, tau2)));
  float C1 = __fmul_rn(__fdiv_rn(a, __fadd_rn(a, b)), normal_pdf_f(mu, norm_scale, x));
  float C2 = (float)((double)__fdiv_rn(b, __fadd_rn(a, b)) * 1. / (double)z_range);
  const float normalization_constant = __fadd_rn(C1, C2);
  C1 = __fdiv_rn(C1, normalization_constant);
  C2 = __fdiv_rn(C2, normalization_constant);
  const double ab = (double)__fadd_rn(a, b);
  const float f = (float)((double)C1 * ((double)a + 1.) / (ab + 1.) + (double)__fmul_rn(C2, a) / (ab + 1.));
  const float e = (float)((double)C1 * ((double)a + 1.) * ((double)a + 2.) / ((ab + 1.) * (ab + 2.)) +
                          (double)__fdiv_rn(__fmul_rn(__fmul_rn(C2, a), __fadd_rn(a, 1.0f)),
                                            __fmul_rn(__fadd_rn(__fadd_rn(a, b), 1.0f), __fadd_rn(__fadd_rn(a, b), 2.0f))));
  const float mu_new = fmaf(C1, m, __fmul_rn(C2, mu));
  sigma2 = fmaf(-mu_new, mu_new, fmaf(C1, fmaf(m, m, s2), __fmul_rn(C2, fmaf(mu, mu, sigma2))));
  mu = mu_new;
  a = __fdiv_rn(__fsub_rn(e, f), __fsub_rn(f, __fdiv_rn(e, f)));
  b = __fdiv_rn(__fmul_rn(a, __fsub_rn(1.0f, f)), f);
}

// DepthFilter::computeTau (depth_filter.cpp:334-350), PI truncated as svo/include/svo/global.h:78
__device__ inline double compute_tau(const Pose& T_ref_cur, const double* f, double z, double px_error_angle) {
  const double PI = 3.14159265;
  const double* t = T_ref_cur.t;
  const double ax = f[0] * z - t[0], ay = f[1] * z - t[1], az = f[2] * z - t[2];
  const double t_norm = sqrt(t[0] * t[0] + t[1] * t[1] + t[2] * t[2]);
  const double a_norm = sqrt(ax * ax + ay * ay + az * az);
  const double alpha = acos((f[0] * t[0] + f[1] * t[1] + f[2] * t[2]) / t_norm);
  const double beta = acos((ax * -t[0] + ay * -t[1] + az * -t[2]) / (t_norm * a_norm));
  const double beta_plus = beta + px_error_angle;
  const double gamma_plus = PI - alpha - beta_plus;
  const double z_plus = t_norm * sin(beta_plus) / sin(gamma_plus);
  return z_plus - z;
}

// One warp per seed of n_streams streams' concatenated seeds.  Seed i belongs to stream stream_of(seed_offset, .., i)
// and reads that stream's current frame, pose, camera and batch counter from `streams`; `ref_index` points into one
// keyframe table shared by all streams.  The pose products (T_ref_cur, T_cur_ref) are formed per warp: a per-stream table
// built on the host would round differently from the device's code, and one built on the device would cost a second
// launch.  <= 128 registers: the 500 CTAs of C2 (2000 seeds) are resident at once.
// kGeneral = false is Matcher::Options at its defaults (edgelet filter at 0.7, align2D, sub-pixel refinement); true reads
// P.epi and follows every branch of matcher.cpp:204-212, 226-246 and 293-320 that the options select.
template <bool kGeneral>
__global__ void __launch_bounds__(kDfWarps * 32, 4) depth_filter_kernel(const DepthParams P,
                                                                         const DepthStream* __restrict__ streams,
                                                                         const int* __restrict__ seed_offset, int n_streams) {
  __shared__ WarpAlignScratch scratch[kDfWarps];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i = blockIdx.x * kDfWarps + warp;
  if (i >= P.M) return;
  WarpAlignScratch& S = scratch[warp];
  for (int k = lane; k < 112; k += 32) S.pwb[k] = 0;
  __syncwarp();

  int status = 0, n_zm = 0;
  double out_pu = 0, out_pv = 0, out_z = 0;
  float sa = 0.f, sb = 0.f, smu = 1.f, ssig = 0.f, szr = 1.f;
  if (!P.match_only) { sa = P.a[i]; sb = P.b[i]; smu = P.mu[i]; ssig = P.sigma2[i]; szr = P.z_range[i]; }
  const DepthStream& st = streams[stream_of(seed_offset, n_streams, i)];
  const Cam& cam = st.cam;

  do {
    if (!P.match_only && (st.batch_counter - P.batch_id[i]) > P.max_n_kfs) { status = SVO_B200_SEED_TOO_OLD; break; }  // :216-219
    const int r = P.ref_index[i];
    const Pose T_ref_w = pose_from_rt12(P.ref_T_f_w + 12 * (size_t)r);
    const Pose T_cur_w = pose_from_rt12(st.cur_T_f_w);
    const Pose T_ref_cur = pose_mul(T_ref_w, pose_inv(T_cur_w));  // :222
    const double fv[3] = {P.ftr_f[3 * i], P.ftr_f[3 * i + 1], P.ftr_f[3 * i + 2]};
    float z_inv_min = 0.f;
    double d_estimate, d_min, d_max;
    if (!P.match_only) {
      const double inv_mu = 1.0 / (double)smu;
      const double p[3] = {fv[0] * inv_mu, fv[1] * inv_mu, fv[2] * inv_mu};
      double xyz_f[3];
      pose_apply(pose_inv(T_ref_cur), p, xyz_f);  // :223
      if (xyz_f[2] < 0.0) { status = SVO_B200_SEED_BEHIND; break; }
      double cu, cv;
      world2cam(cam, xyz_f, cu, cv);
      // isInFrame(f2c(xyz_f).cast<int>()), boundary 0; non-finite projections cannot be in frame
      const bool fin = fabs(cu) < 1e9 && fabs(cv) < 1e9;
      const int xi = fin ? (int)cu : -1, yi = fin ? (int)cv : -1;
      if (!(xi >= 0 && xi < cam.width && yi >= 0 && yi < cam.height)) { status = SVO_B200_SEED_NOT_IN_FRAME; break; }
      const float sq = sqrtf(ssig);
      z_inv_min = __fadd_rn(smu, sq);
      const float z_inv_max = fmaxf(__fsub_rn(smu, sq), 0.00000001f);
      d_estimate = 1.0 / (double)smu; d_min = 1.0 / (double)z_inv_min; d_max = 1.0 / (double)z_inv_max;
    } else {
      d_estimate = P.d_est[i]; d_min = P.d_min[i]; d_max = P.d_max[i];
    }

    // ---------------- Matcher::findEpipolarMatchDirect (matcher.cpp:179-321) -----------------
    bool ok = false;
    double depth = 0.0;
    const Pose T_cur_ref = pose_mul(T_cur_w, pose_inv(T_ref_w));  // :188
    const int lvl = P.ftr_level[i];
    const double pxu = P.ftr_px[2 * i], pxv = P.ftr_px[2 * i + 1];
    double pA[3], pB[3];
    {
      const double a3[3] = {fv[0] * d_min, fv[1] * d_min, fv[2] * d_min};
      const double b3[3] = {fv[0] * d_max, fv[1] * d_max, fv[2] * d_max};
      pose_apply(T_cur_ref, a3, pA);
      pose_apply(T_cur_ref, b3, pB);
    }
    const double Ax = pA[0] / pA[2], Ay = pA[1] / pA[2], Bx = pB[0] / pB[2], By = pB[1] / pB[2];  // project2d
    const double epi_x = Ax - Bx, epi_y = Ay - By;
    double Aff[4];
    get_warp_matrix_affine(cam, pxu, pxv, fv, d_estimate, T_cur_ref, lvl, Aff);
    bool reject = false;
    int out_level = 0;
    double out_epi_length = 0.0;
    double h_inv = 0.0;
    bool ran_1d = false;
    if (P.ftr_type[i] == 1 && (!kGeneral || P.epi.epi_search_edgelet_filtering)) {  // edgelet filtering (:204-212)
      const double gx0 = P.ftr_grad[2 * i], gy0 = P.ftr_grad[2 * i + 1];
      const double gx = Aff[0] * gx0 + Aff[1] * gy0, gy = Aff[2] * gx0 + Aff[3] * gy0;
      const double gn = sqrt(gx * gx + gy * gy), en = sqrt(epi_x * epi_x + epi_y * epi_y);
      const double cosangle = fabs((gx / gn) * (epi_x / en) + (gy / gn) * (epi_y / en));
      if (cosangle < (kGeneral ? P.epi.epi_search_edgelet_max_angle : 0.7)) reject = true;  // NaN on either side: kept
    }
    if (!reject) {
      const int L = best_search_level(Aff, P.max_search_level);
      double pAu, pAv, pBu, pBv;
      cam_world2cam(cam, Ax, Ay, pAu, pAv);  // cam_->world2cam(A), world2cam(B)  (:217-218)
      cam_world2cam(cam, Bx, By, pBu, pBv);
      const double ddx = pAu - pBu, ddy = pAv - pBv;
      const double epi_length = sqrt(ddx * ddx + ddy * ddy) / (double)(1 << L);
      out_level = L; out_epi_length = epi_length;
      const FrameDesc& rf = P.ref_frames[r];
      ImgView ref_img = {rf.lvl[lvl], rf.w[lvl], rf.h[lvl]};
      warp_warp_affine(Aff, ref_img, pxu, pxv, lvl, L, S);
      ImgView cur_img = {st.cur.lvl[L], st.cur.w[L], st.cur.h[L]};
      const double sc = (double)(1 << L), inv_sc = 1.0 / sc;  // a power of two: x * inv_sc == x / sc exactly
      bool have_start = false, from_scan = false;
      double start_u = 0, start_v = 0, uv_best_u = 0, uv_best_v = 0;
      if (epi_length < 2.0) {  // :226-246
        start_u = (pAu + pBu) * 0.5;
        start_v = (pAv + pBv) * 0.5;
        have_start = true;
      } else if (epi_length >= 2.0) {  // (NaN lengths fall through: the reference's size_t cast overflows -> skip)
        const unsigned long long n0 = (unsigned long long)(epi_length / 0.7);
        if (n0 <= (unsigned long long)P.max_epi_search_steps) {
          const double step_x = epi_x / (double)n0, step_y = epi_y / (double)n0;
          const double u0 = Bx - step_x, v0 = By - step_y;  // uv = B - step
          const int n_steps = (int)n0 + 1;
          // reference patch words + sums for the score
          uint32_t refw[16];
#pragma unroll
          for (int k = 0; k < 16; ++k) refw[k] = reinterpret_cast<const uint32_t*>(S.patch)[k];
          unsigned sA = 0, sAA = 0;
#pragma unroll
          for (int k = 0; k < 16; ++k) { sA = __dp4a(refw[k], 0x01010101u, sA); sAA = __dp4a(refw[k], refw[k], sAA); }
          const int lim_x = cam.width / (1 << L) - 8, lim_y = cam.height / (1 << L) - 8;
          long long best_key = (long long)(2000 * 64) * 4294967296LL;  // PatchScore::threshold(), strict '<'
          for (int k = lane; k < n_steps; k += 32) {
            // uv_k = (B - step) + k*step  (the reference accumulates uv += step; same value to ~1 ulp)
            const double uk = fma((double)k, step_x, u0), vk = fma((double)k, step_y, v0);
            double wu, wv;
            cam_world2cam(cam, uk, vk, wu, wv);  // cam_->world2cam(uv)  (:272)
            const int qx = (int)(wu * inv_sc + 0.5), qy = (int)(wv * inv_sc + 0.5);
            int px_prev = 0, py_prev = 0;  // last_checked_pxi starts at (0,0)
            if (k > 0) {
              const double up = fma((double)(k - 1), step_x, u0), vp = fma((double)(k - 1), step_y, v0);
              cam_world2cam(cam, up, vp, wu, wv);
              px_prev = (int)(wu * inv_sc + 0.5);
              py_prev = (int)(wv * inv_sc + 0.5);
            }
            if (qx == px_prev && qy == py_prev) continue;                 // :273-275
            if (!(qx >= 8 && qx < lim_x && qy >= 8 && qy < lim_y)) continue;  // isInFrame(pxi, 8, level)
            const int score = zmssd_score(cur_img.data, (qy - 4) * cur_img.cols + (qx - 4), cur_img.cols, refw, (int)sA, (int)sAA);
            ++n_zm;
            const long long key = (long long)score * 4294967296LL + (long long)k;
            if (key < best_key && score < 2000 * 64) best_key = key;
          }
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) {
            const long long other = __shfl_xor_sync(0xffffffffu, best_key, o);
            best_key = other < best_key ? other : best_key;
            n_zm += __shfl_xor_sync(0xffffffffu, n_zm, o);
          }
          if (best_key < (long long)(2000 * 64) * 4294967296LL) {
            const int kb = (int)(best_key & 0xffffffffLL);
            const double ub = fma((double)kb, step_x, u0), vb = fma((double)kb, step_y, v0);
            cam_world2cam(cam, ub, vb, start_u, start_v);  // px_cur_ = world2cam(uv_best)  (:297, :316)
            have_start = true;
            if (kGeneral) { from_scan = true; uv_best_u = ub; uv_best_v = vb; }
          }
        }
      }
      if (kGeneral && from_scan && !P.epi.subpix_refinement) {
        // no refinement (:316-318): the scan's best step, triangulated along unproject2d(uv_best).normalized() with the
        // squared norm summed and fused as the reference's build does ((u*u + v*v) + 1*1, two fused multiply-adds)
        out_pu = start_u; out_pv = start_v;
        const double n = sqrt(fma(1.0, 1.0, fma(uv_best_v, uv_best_v, uv_best_u * uv_best_u)));
        const double f_cur[3] = {uv_best_u / n, uv_best_v / n, 1.0 / n};
        ok = depth_from_triangulation(T_cur_ref, fv, f_cur, depth);
      } else if (have_start) {  // subpixel refinement + triangulation (:295-315 / :229-245)
        double su = start_u / sc, sv = start_v / sc;
        bool nan_exit = false, res;
        if (kGeneral && P.epi.align_1d) {
          // align1D along (px_A - px_B).cast<float>().normalized() (:231-234, :300-303): no guard on the norm, so a
          // zero-length line gives a NaN direction, which align1D then runs with
          const float dx = (float)ddx, dy = (float)ddy;
          const float n = sqrtf(fmaf(dx, dx, __fmul_rn(dy, dy)));
          res = warp_align1d(cur_img, S, __fdiv_rn(dx, n), __fdiv_rn(dy, n), P.align_max_iter, su, sv, h_inv, &nan_exit);
          ran_1d = true;
        } else {
          res = warp_align2d(cur_img, S, P.align_max_iter, su, sv, &nan_exit);
        }
        out_pu = start_u; out_pv = start_v;
        if (res) {
          out_pu = su * sc; out_pv = sv * sc;
          double f_cur[3];
          cam2world(cam, out_pu, out_pv, f_cur);
          ok = depth_from_triangulation(T_cur_ref, fv, f_cur, depth);
        }
      }
    }
    if (P.match_only) {  // Matcher's public members after the call (matcher.h:92-101)
      if (lane == 0) {
        if (P.search_level_out) P.search_level_out[i] = out_level;
        if (P.epi_length_out) P.epi_length_out[i] = out_epi_length;
        if (P.reject_out) P.reject_out[i] = reject ? 1 : 0;
        if (P.A_out) { P.A_out[4 * i] = Aff[0]; P.A_out[4 * i + 1] = Aff[1]; P.A_out[4 * i + 2] = Aff[2]; P.A_out[4 * i + 3] = Aff[3]; }
        if (kGeneral) { P.h_inv_out[i] = h_inv; P.ran_1d_out[i] = ran_1d ? 1 : 0; }
      }
      status = ok ? SVO_B200_SEED_UPDATED : SVO_B200_SEED_NO_MATCH;
      out_z = ok ? depth : 0.0;
      break;
    }
    if (!ok) {
      sb = __fadd_rn(sb, 1.0f);  // it->b++  (:240)
      status = SVO_B200_SEED_NO_MATCH;
      out_pu = out_pv = 0.0;
      break;
    }
    // ---------------- computeTau + updateSeed (:247-252) ---------------------------------------
    const double px_error_angle = atan(1.0 / (2.0 * fabs(cam.fx))) * 2.0;  // :205-207
    const double z = depth;
    const double tau = compute_tau(T_ref_cur, fv, z, px_error_angle);
    const double tau_inverse = 0.5 * (1.0 / fmax(0.0000001, z - tau) - 1.0 / (z + tau));
    update_seed((float)(1. / z), (float)(tau_inverse * tau_inverse), sa, sb, smu, szr, ssig);
    out_z = z;
    if ((double)sqrtf(ssig) < (double)szr / P.sigma2_thresh) status = SVO_B200_SEED_CONVERGED;  // :261
    else if (isnan(z_inv_min)) status = SVO_B200_SEED_NAN;                                       // :283
    else status = SVO_B200_SEED_UPDATED;
  } while (false);

  if (lane == 0) {
    if (!P.match_only) { P.a[i] = sa; P.b[i] = sb; P.mu[i] = smu; P.sigma2[i] = ssig; }
    P.status[i] = (uint8_t)status;
    if (P.px_cur) { P.px_cur[2 * i] = out_pu; P.px_cur[2 * i + 1] = out_pv; }
    if (P.z) P.z[i] = out_z;
    if (P.n_zmssd) P.n_zmssd[i] = n_zm;
  }
}

}  // namespace svo

using namespace svo;

namespace {

// Matcher::Options() (svo/include/svo/matcher.h:83-91): the setting that runs the default instantiation
bool epi_is_default(const svo_b200_epipolar_options& o) {
  return !o.align_1d && o.subpix_refinement && o.epi_search_edgelet_filtering && o.epi_search_edgelet_max_angle == 0.7;
}

// The current frame, pose, camera and batch counter of one stream, as the kernel reads them.
int depth_stream(svo_b200_ctx* ctx, const svo_b200_frame* cur, const double* cur_T_f_w, const svo_b200_camera* cam,
                 int batch_counter, DepthStream& st) {
  memset(&st, 0, sizeof(st));
  st.cur = make_desc(cur);
  memcpy(st.cur_T_f_w, cur_T_f_w, sizeof(double) * 12);
  st.batch_counter = batch_counter;
  return cam_to_dev(ctx, cam, st.cam);
}

// One depth filter launch over the M seeds of S streams, or with H.match_only over M epipolar-match candidates.  H holds
// the caller's host arrays in the fields the kernel reads their device copies from (NULL optional outputs are not copied
// back; with match_only, H.status receives success flags).  The arrays, the keyframe table, the stream table and the seed
// offsets go to the device in one copy; the kernel runs once and the results come back in one copy.
int depth_run(svo_b200_ctx* ctx, const DepthParams& H, const svo_b200_frame* const* ref_frames, const double* ref_T_f_w,
              int n_ref, const svo_b200_depth_options* opt, const DepthStream* streams, const int* seed_offset, int S) {
  const int M = H.M;
  const bool mo = H.match_only != 0;
  const bool general = !epi_is_default(ctx->epi);
  cudaSetDevice(ctx->device);
  std::vector<FrameDesc> frames((size_t)n_ref);
  for (int r = 0; r < n_ref; ++r) frames[r] = make_desc(ref_frames[r]);
  Staging st(ctx);
  DepthParams P;
  memset(&P, 0, sizeof(P));
  const DepthStream* d_streams;
  const int* d_seed_offset;
  st.in(H.ref_index, M, &P.ref_index);
  st.in(H.ftr_px, 2 * (size_t)M, &P.ftr_px);
  st.in(H.ftr_f, 3 * (size_t)M, &P.ftr_f);
  st.in(H.ftr_level, M, &P.ftr_level);
  st.in(H.ftr_type, M, &P.ftr_type);
  st.in(H.ftr_grad, 2 * (size_t)M, &P.ftr_grad);
  st.in(ref_T_f_w, 12 * (size_t)n_ref, &P.ref_T_f_w);
  st.in(frames.data(), n_ref, &P.ref_frames);
  st.in(streams, S, &d_streams);
  st.in(seed_offset, S + 1, &d_seed_offset);
  if (mo) {  // the candidates' depth ranges in; the status flags are converted on the way out
    st.in(H.d_est, M, &P.d_est);
    st.in(H.d_min, M, &P.d_min);
    st.in(H.d_max, M, &P.d_max);
    st.out<uint8_t>(nullptr, M, &P.status);
  } else {   // batch ids and z_range in, the seeds both ways
    st.in(H.batch_id, M, &P.batch_id);
    st.in(H.z_range, M, &P.z_range);
    st.inout(H.a, M, &P.a);
    st.inout(H.b, M, &P.b);
    st.inout(H.mu, M, &P.mu);
    st.inout(H.sigma2, M, &P.sigma2);
    st.out(H.status, M, &P.status);
  }
  st.out(H.px_cur, 2 * (size_t)M, &P.px_cur);
  st.out(H.z, M, &P.z);
  st.out(H.n_zmssd, M, &P.n_zmssd);
  if (mo) {  // the Matcher's scratch members
    st.out(H.search_level_out, M, &P.search_level_out);
    st.out(H.epi_length_out, M, &P.epi_length_out);
    st.out(H.reject_out, M, &P.reject_out);
    st.out(H.A_out, 4 * (size_t)M, &P.A_out);
    if (general) {  // h_inv_ (align1D runs only here)
      st.out<double>(nullptr, M, &P.h_inv_out);
      st.out<uint8_t>(nullptr, M, &P.ran_1d_out);
    }
  }
  int rc;
  if ((rc = st.open()) || (rc = st.send())) return rc;
  if (mo) SVO_CUDA_CHECK(ctx, cudaMemsetAsync(st.tail(), 0, st.tail_bytes(), ctx->stream));
  P.M = M;
  P.max_n_kfs = opt->max_n_kfs;
  P.sigma2_thresh = opt->seed_convergence_sigma2_thresh;
  P.max_search_level = opt->max_search_level;
  P.align_max_iter = opt->align_max_iter;
  P.max_epi_search_steps = opt->max_epi_search_steps;
  P.match_only = H.match_only;
  if (general) P.epi = ctx->epi;
  const int blocks = (M + kDfWarps - 1) / kDfWarps;
  if ((rc = launch_kernels(ctx, 1, [&] {
         if (general) depth_filter_kernel<true><<<blocks, kDfWarps * 32, 0, ctx->stream>>>(P, d_streams, d_seed_offset, S);
         else depth_filter_kernel<false><<<blocks, kDfWarps * 32, 0, ctx->stream>>>(P, d_streams, d_seed_offset, S);
       })))
    return rc;
  if ((rc = st.receive())) return rc;
  if (mo) {
    const uint8_t* status = st.host(P.status);
    for (int m = 0; m < M; ++m) H.status[m] = status[m] == SVO_B200_SEED_UPDATED;
    ctx->epi_h_inv.assign((size_t)M, 0.0);
    ctx->epi_ran_1d.assign((size_t)M, 0);
    if (general) {
      memcpy(ctx->epi_h_inv.data(), st.host(P.h_inv_out), sizeof(double) * M);
      memcpy(ctx->epi_ran_1d.data(), st.host(P.ran_1d_out), M);
    }
    ctx->epi_last_valid = true;
  }
  return 0;
}

}  // namespace

extern "C" int svo_b200_depth_filter_update(svo_b200_ctx* ctx, const svo_b200_frame* const* ref_frames,
                                            const double* ref_T_f_w, int n_ref, const svo_b200_frame* cur,
                                            const double* cur_T_f_w, const svo_b200_camera* cam,
                                            const svo_b200_depth_options* opt, int M, const int* ref_index,
                                            const double* ftr_px, const double* ftr_f, const int* ftr_level,
                                            const int* ftr_type, const double* ftr_grad, const int* batch_id,
                                            int batch_counter, float* a, float* b, float* mu, float* z_range,
                                            float* sigma2, uint8_t* status_out, double* px_cur_out, double* z_out,
                                            int* n_zmssd_out) {
  if (!ctx || !ref_frames || !ref_T_f_w || n_ref <= 0 || !cur || !cur_T_f_w || !cam || !opt || M < 0)
    return set_err(ctx, SVO_B200_EINVAL, "depth_filter_update: bad arguments");
  if (M == 0) return 0;
  if (!ref_index || !ftr_px || !ftr_f || !ftr_level || !ftr_type || !ftr_grad || !batch_id || !a || !b || !mu ||
      !z_range || !sigma2 || !status_out)
    return set_err(ctx, SVO_B200_EINVAL, "depth_filter_update: NULL seed arrays");
  if (const int rc = check_ref_table(ctx, "depth_filter_update", "ftr_level", ref_frames, n_ref, M, ref_index, ftr_level, cur, cam,
                                     opt->max_search_level))
    return rc;
  DepthStream st;
  if (const int rc = depth_stream(ctx, cur, cur_T_f_w, cam, batch_counter, st)) return rc;
  const int seed_offset[2] = {0, M};
  DepthParams H;
  memset(&H, 0, sizeof(H));
  H.M = M; H.ref_index = ref_index; H.ftr_px = ftr_px; H.ftr_f = ftr_f; H.ftr_level = ftr_level; H.ftr_type = ftr_type;
  H.ftr_grad = ftr_grad; H.batch_id = batch_id; H.a = a; H.b = b; H.mu = mu; H.z_range = z_range; H.sigma2 = sigma2;
  H.status = status_out; H.px_cur = px_cur_out; H.z = z_out; H.n_zmssd = n_zmssd_out;
  return depth_run(ctx, H, ref_frames, ref_T_f_w, n_ref, opt, &st, seed_offset, 1);
}

extern "C" int svo_b200_depth_filter_update_streams(svo_b200_ctx* ctx, int S, const svo_b200_frame* const* cur,
                                                    const double* cur_T_f_w, const svo_b200_camera* cam,
                                                    const int* batch_counter, const int* seed_offset,
                                                    const svo_b200_frame* const* ref_frames, const double* ref_T_f_w,
                                                    int n_ref, const svo_b200_depth_options* opt, const int* ref_index,
                                                    const double* ftr_px, const double* ftr_f, const int* ftr_level,
                                                    const int* ftr_type, const double* ftr_grad, const int* batch_id,
                                                    float* a, float* b, float* mu, float* z_range, float* sigma2,
                                                    uint8_t* status_out, double* px_cur_out, double* z_out,
                                                    int* n_zmssd_out) {
  if (!ctx || S < 0) return set_err(ctx, SVO_B200_EINVAL, "depth_filter_update_streams: bad arguments (S %d)", S);
  if (S == 0) return 0;
  if (!cur || !cur_T_f_w || !cam || !batch_counter || !seed_offset || !opt || n_ref < 0)
    return set_err(ctx, SVO_B200_EINVAL, "depth_filter_update_streams: bad arguments");
  if (seed_offset[0] != 0) return set_err(ctx, SVO_B200_EINVAL, "depth_filter_update_streams: seed_offset[0] != 0");
  for (int s = 0; s < S; ++s) {
    if (seed_offset[s + 1] < seed_offset[s])
      return set_err(ctx, SVO_B200_EINVAL, "depth_filter_update_streams: seed_offset not monotone at stream %d", s);
    if (!cur[s]) return set_err(ctx, SVO_B200_EINVAL, "depth_filter_update_streams: cur[%d] is NULL", s);
    if (opt->max_search_level >= cur[s]->n_levels)
      return set_err(ctx, SVO_B200_EINVAL, "depth_filter_update_streams: max_search_level %d >= %d pyramid levels of cur[%d]",
                     opt->max_search_level, cur[s]->n_levels, s);
  }
  const int M = seed_offset[S];
  if (M == 0) return 0;
  if (!ref_frames || !ref_T_f_w || !ref_index || !ftr_px || !ftr_f || !ftr_level || !ftr_type || !ftr_grad || !batch_id ||
      !a || !b || !mu || !z_range || !sigma2 || !status_out)
    return set_err(ctx, SVO_B200_EINVAL, "depth_filter_update_streams: NULL keyframe table or seed arrays");
  for (int r = 0; r < n_ref; ++r)
    if (!ref_frames[r]) return set_err(ctx, SVO_B200_EINVAL, "depth_filter_update_streams: ref_frames[%d] is NULL", r);
  if (const int rc = check_ref_levels(ctx, "depth_filter_update_streams", "ftr_level", ref_frames, n_ref, M, ref_index, ftr_level))
    return rc;
  // each stream's camera against its current frame and the keyframes its seeds refer to (the table is shared by streams
  // of different cameras)
  for (int s = 0; s < S; ++s) {
    if (const int rc = cam_check_frames(ctx, "depth_filter_update_streams", cam + s, cur + s, 1)) return rc;
    for (int m = seed_offset[s]; m < seed_offset[s + 1]; ++m)
      if (const int rc = cam_check_frames(ctx, "depth_filter_update_streams", cam + s, ref_frames + ref_index[m], 1)) return rc;
  }
  std::vector<DepthStream> st((size_t)S);
  for (int s = 0; s < S; ++s)
    if (const int rc = depth_stream(ctx, cur[s], cur_T_f_w + 12 * (size_t)s, cam + s, batch_counter[s], st[s])) return rc;
  DepthParams H;
  memset(&H, 0, sizeof(H));
  H.M = M; H.ref_index = ref_index; H.ftr_px = ftr_px; H.ftr_f = ftr_f; H.ftr_level = ftr_level; H.ftr_type = ftr_type;
  H.ftr_grad = ftr_grad; H.batch_id = batch_id; H.a = a; H.b = b; H.mu = mu; H.z_range = z_range; H.sigma2 = sigma2;
  H.status = status_out; H.px_cur = px_cur_out; H.z = z_out; H.n_zmssd = n_zmssd_out;
  return depth_run(ctx, H, ref_frames, ref_T_f_w, n_ref, opt, st.data(), seed_offset, S);
}

// Matcher::findEpipolarMatchDirect (svo/src/matcher.cpp:179-321) for M independent candidates: the same device code as
// inside DepthFilter::updateSeeds, with the depth range given explicitly and the Matcher's scratch members returned.
extern "C" int svo_b200_find_epipolar_match_direct(svo_b200_ctx* ctx, const svo_b200_frame* const* ref_frames,
                                                   const double* ref_T_f_w, int n_ref, const svo_b200_frame* cur,
                                                   const double* cur_T_f_w, const svo_b200_camera* cam,
                                                   const svo_b200_depth_options* opt, int M, const int* ref_index,
                                                   const double* ftr_px, const double* ftr_f, const int* ftr_level,
                                                   const int* ftr_type, const double* ftr_grad, const double* d_estimate,
                                                   const double* d_min, const double* d_max, uint8_t* success_out,
                                                   double* depth_out, double* px_cur_out, int* search_level_out,
                                                   double* epi_length_out, uint8_t* reject_out, double* A_cur_ref_out,
                                                   int* n_zmssd_out) {
  if (!ctx || !ref_frames || !ref_T_f_w || n_ref <= 0 || !cur || !cur_T_f_w || !cam || !opt || M < 0)
    return set_err(ctx, SVO_B200_EINVAL, "find_epipolar_match_direct: bad arguments");
  if (M == 0) {
    ctx->epi_h_inv.clear(); ctx->epi_ran_1d.clear(); ctx->epi_last_valid = true;
    return 0;
  }
  if (!ref_index || !ftr_px || !ftr_f || !ftr_level || !ftr_type || !ftr_grad || !d_estimate || !d_min || !d_max || !success_out)
    return set_err(ctx, SVO_B200_EINVAL, "find_epipolar_match_direct: NULL candidate arrays");
  if (const int rc = check_ref_table(ctx, "find_epipolar_match_direct", "ftr_level", ref_frames, n_ref, M, ref_index, ftr_level, cur, cam,
                                     opt->max_search_level))
    return rc;
  DepthStream st;
  if (const int rc = depth_stream(ctx, cur, cur_T_f_w, cam, 0, st)) return rc;
  const int seed_offset[2] = {0, M};
  DepthParams H;
  memset(&H, 0, sizeof(H));
  H.match_only = 1;
  H.M = M; H.ref_index = ref_index; H.ftr_px = ftr_px; H.ftr_f = ftr_f; H.ftr_level = ftr_level; H.ftr_type = ftr_type;
  H.ftr_grad = ftr_grad; H.d_est = d_estimate; H.d_min = d_min; H.d_max = d_max;
  H.status = success_out; H.px_cur = px_cur_out; H.z = depth_out; H.n_zmssd = n_zmssd_out;
  H.search_level_out = search_level_out; H.epi_length_out = epi_length_out; H.reject_out = reject_out; H.A_out = A_cur_ref_out;
  return depth_run(ctx, H, ref_frames, ref_T_f_w, n_ref, opt, &st, seed_offset, 1);
}

extern "C" int svo_b200_set_epipolar_options(svo_b200_ctx* ctx, const svo_b200_epipolar_options* opt) {
  if (!ctx) return SVO_B200_EINVAL;
  if (!opt) {
    ctx->epi = svo_b200_epipolar_options{0, 1, 1, 0.7};
    return 0;
  }
  const auto flag = [](int v) { return v == 0 || v == 1; };
  if (!flag(opt->align_1d) || !flag(opt->subpix_refinement) || !flag(opt->epi_search_edgelet_filtering))
    return set_err(ctx, SVO_B200_EINVAL, "set_epipolar_options: flags must be 0 or 1 (align_1d %d, subpix_refinement %d, "
                   "epi_search_edgelet_filtering %d)", opt->align_1d, opt->subpix_refinement, opt->epi_search_edgelet_filtering);
  ctx->epi = *opt;
  return 0;
}

extern "C" int svo_b200_get_epipolar_options(const svo_b200_ctx* ctx, svo_b200_epipolar_options* out) {
  if (!ctx || !out) return SVO_B200_EINVAL;
  *out = ctx->epi;
  return 0;
}

extern "C" int svo_b200_epipolar_last_h_inv(const svo_b200_ctx* ctx, int M, double* h_inv_out, uint8_t* ran_1d_out) {
  if (!ctx || M < 0 || !ctx->epi_last_valid || (size_t)M > ctx->epi_h_inv.size() || (M > 0 && (!h_inv_out || !ran_1d_out)))
    return SVO_B200_EINVAL;
  if (M > 0) {
    memcpy(h_inv_out, ctx->epi_h_inv.data(), sizeof(double) * M);
    memcpy(ran_1d_out, ctx->epi_ran_1d.data(), M);
  }
  return 0;
}
