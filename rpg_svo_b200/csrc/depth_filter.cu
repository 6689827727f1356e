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

struct DepthParams {
  const FrameDesc* ref_frames;
  const double* ref_T_f_w;
  FrameDesc cur;
  double cur_T_f_w[12];
  Cam cam;
  int M;
  const int* ref_index;
  const double* ftr_px;
  const double* ftr_f;
  const int* ftr_level;
  const int* ftr_type;
  const double* ftr_grad;
  const int* batch_id;
  int batch_counter, max_n_kfs;
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

__global__ void __launch_bounds__(kDfWarps * 32, 4) depth_filter_kernel(const DepthParams P) {  // <= 128 registers: the 500 CTAs of C2 (2000 seeds) are resident at once
#define DF_CUR P.cur
#define DF_CUR_T_F_W P.cur_T_f_w
#define DF_CAM P.cam
#define DF_BATCH_COUNTER P.batch_counter
#define DF_STREAM_LOOKUP
#include "depth_filter_seed.inc"
#undef DF_CUR
#undef DF_CUR_T_F_W
#undef DF_CAM
#undef DF_BATCH_COUNTER
#undef DF_STREAM_LOOKUP
}

// One stream of svo_b200_depth_filter_update_streams: what the single-stream call passes by value in DepthParams, read
// from a per-launch device table instead.
struct DepthStream {
  FrameDesc cur;
  Cam cam;
  double cur_T_f_w[12];
  int batch_counter;
};

// The stream that owns seed i: the last s with seed_offset[s] <= i (streams without seeds are skipped over).
__device__ __forceinline__ int stream_of(const int* __restrict__ seed_offset, int n_streams, int i) {
  int lo = 0, hi = n_streams - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(seed_offset + mid) <= i) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// svo_b200_depth_filter_update_streams: the seeds of n_streams streams in one launch.  P holds the concatenated seed
// arrays and the shared keyframe table, `streams` what differs per stream.  The pose products (T_ref_cur, T_cur_ref) are
// formed per warp as in the single-stream kernel: a per-stream table built on the host would round differently from the
// device's code, and one built on the device would cost a second launch.
__global__ void __launch_bounds__(kDfWarps * 32, 4) depth_filter_streams_kernel(const DepthParams P,
                                                                                 const DepthStream* __restrict__ streams,
                                                                                 const int* __restrict__ seed_offset,
                                                                                 int n_streams) {
#define DF_CUR st.cur
#define DF_CUR_T_F_W st.cur_T_f_w
#define DF_CAM st.cam
#define DF_BATCH_COUNTER st.batch_counter
#define DF_STREAM_LOOKUP const DepthStream& st = streams[stream_of(seed_offset, n_streams, i)];
#include "depth_filter_seed.inc"
#undef DF_CUR
#undef DF_CUR_T_F_W
#undef DF_CAM
#undef DF_BATCH_COUNTER
#undef DF_STREAM_LOOKUP
}

}  // namespace svo

using namespace svo;

namespace {

// Stages the M seeds (and, for S > 0 streams, the stream table and seed offsets), runs one depth filter launch and copies
// the results back.  S == 0: one stream, whose frame, pose, camera and batch counter the caller has put into P.
int depth_update_run(svo_b200_ctx* ctx, DepthParams& P, const svo_b200_frame* const* ref_frames, const double* ref_T_f_w,
                     int n_ref, const svo_b200_frame* cur, const double* cur_T_f_w, const svo_b200_camera* cam, int S,
                     const DepthStream* streams, const int* seed_offset, const svo_b200_depth_options* opt, int M,
                     const int* ref_index, const double* ftr_px, const double* ftr_f, const int* ftr_level,
                     const int* ftr_type, const double* ftr_grad, const int* batch_id, int batch_counter, float* a,
                     float* b, float* mu, float* z_range, float* sigma2, uint8_t* status_out, double* px_cur_out,
                     double* z_out, int* n_zmssd_out) {
  cudaSetDevice(ctx->device);
  Carver c;
  const size_t o_ri = c.take(sizeof(int) * M), o_px = c.take(sizeof(double) * 2 * M), o_f = c.take(sizeof(double) * 3 * M),
               o_lv = c.take(sizeof(int) * M), o_ty = c.take(sizeof(int) * M), o_gr = c.take(sizeof(double) * 2 * M),
               o_bi = c.take(sizeof(int) * M), o_rT = c.take(sizeof(double) * 12 * n_ref),
               o_fr = c.take(sizeof(FrameDesc) * n_ref), o_zr = c.take(sizeof(float) * M);
  const size_t o_st_tab = S ? c.take(sizeof(DepthStream) * S) : 0, o_so = S ? c.take(sizeof(int) * (S + 1)) : 0;
  // in/out block (copied both ways)
  const size_t o_a = c.take(sizeof(float) * M), o_b = c.take(sizeof(float) * M), o_mu = c.take(sizeof(float) * M),
               o_s2 = c.take(sizeof(float) * M);
  const size_t in_bytes = c.off;
  const size_t o_st = c.take(M), o_pc = c.take(sizeof(double) * 2 * M), o_z = c.take(sizeof(double) * M),
               o_nz = c.take(sizeof(int) * M);
  int rc;
  if ((rc = ensure_host(ctx, ctx->h_in, c.off))) return rc;
  if ((rc = ensure_dev(ctx, ctx->d_in, c.off))) return rc;
  SVO_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
  uint8_t* h = static_cast<uint8_t*>(ctx->h_in.p);
  uint8_t* d = static_cast<uint8_t*>(ctx->d_in.p);
  memcpy(h + o_ri, ref_index, sizeof(int) * M);
  memcpy(h + o_px, ftr_px, sizeof(double) * 2 * M);
  memcpy(h + o_f, ftr_f, sizeof(double) * 3 * M);
  memcpy(h + o_lv, ftr_level, sizeof(int) * M);
  memcpy(h + o_ty, ftr_type, sizeof(int) * M);
  memcpy(h + o_gr, ftr_grad, sizeof(double) * 2 * M);
  memcpy(h + o_bi, batch_id, sizeof(int) * M);
  memcpy(h + o_rT, ref_T_f_w, sizeof(double) * 12 * n_ref);
  for (int r = 0; r < n_ref; ++r) reinterpret_cast<FrameDesc*>(h + o_fr)[r] = make_desc(ref_frames[r]);
  memcpy(h + o_zr, z_range, sizeof(float) * M);
  if (S) {
    memcpy(h + o_st_tab, streams, sizeof(DepthStream) * S);
    memcpy(h + o_so, seed_offset, sizeof(int) * (S + 1));
  }
  memcpy(h + o_a, a, sizeof(float) * M);
  memcpy(h + o_b, b, sizeof(float) * M);
  memcpy(h + o_mu, mu, sizeof(float) * M);
  memcpy(h + o_s2, sigma2, sizeof(float) * M);
  SVO_CUDA_CHECK(ctx, cudaMemcpyAsync(d, h, in_bytes, cudaMemcpyHostToDevice, ctx->stream));
  P.ref_frames = reinterpret_cast<const FrameDesc*>(d + o_fr);
  P.ref_T_f_w = reinterpret_cast<const double*>(d + o_rT);
  if (!S) {
    P.cur = make_desc(cur);
    memcpy(P.cur_T_f_w, cur_T_f_w, sizeof(double) * 12);
    if ((rc = cam_to_dev(ctx, cam, P.cam))) return rc;
    P.batch_counter = batch_counter;
  }
  P.M = M;
  P.ref_index = reinterpret_cast<const int*>(d + o_ri);
  P.ftr_px = reinterpret_cast<const double*>(d + o_px);
  P.ftr_f = reinterpret_cast<const double*>(d + o_f);
  P.ftr_level = reinterpret_cast<const int*>(d + o_lv);
  P.ftr_type = reinterpret_cast<const int*>(d + o_ty);
  P.ftr_grad = reinterpret_cast<const double*>(d + o_gr);
  P.batch_id = reinterpret_cast<const int*>(d + o_bi);
  P.max_n_kfs = opt->max_n_kfs;
  P.sigma2_thresh = opt->seed_convergence_sigma2_thresh;
  P.max_search_level = opt->max_search_level;
  P.align_max_iter = opt->align_max_iter;
  P.max_epi_search_steps = opt->max_epi_search_steps;
  P.a = reinterpret_cast<float*>(d + o_a);
  P.b = reinterpret_cast<float*>(d + o_b);
  P.mu = reinterpret_cast<float*>(d + o_mu);
  P.z_range = reinterpret_cast<float*>(d + o_zr);
  P.sigma2 = reinterpret_cast<float*>(d + o_s2);
  P.status = d + o_st;
  P.px_cur = reinterpret_cast<double*>(d + o_pc);
  P.z = reinterpret_cast<double*>(d + o_z);
  P.n_zmssd = reinterpret_cast<int*>(d + o_nz);
  const int blocks = (M + kDfWarps - 1) / kDfWarps;
  kt_begin(ctx);
  if (S)
    depth_filter_streams_kernel<<<blocks, kDfWarps * 32, 0, ctx->stream>>>(
        P, reinterpret_cast<const DepthStream*>(d + o_st_tab), reinterpret_cast<const int*>(d + o_so), S);
  else
    depth_filter_kernel<<<blocks, kDfWarps * 32, 0, ctx->stream>>>(P);
  ctx->launches++;
  kt_end(ctx);
  SVO_CUDA_CHECK(ctx, cudaGetLastError());
  SVO_CUDA_CHECK(ctx, cudaMemcpyAsync(h + o_a, d + o_a, c.off - o_a, cudaMemcpyDeviceToHost, ctx->stream));
  SVO_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
  memcpy(a, h + o_a, sizeof(float) * M);
  memcpy(b, h + o_b, sizeof(float) * M);
  memcpy(mu, h + o_mu, sizeof(float) * M);
  memcpy(sigma2, h + o_s2, sizeof(float) * M);
  memcpy(status_out, h + o_st, M);
  if (px_cur_out) memcpy(px_cur_out, h + o_pc, sizeof(double) * 2 * M);
  if (z_out) memcpy(z_out, h + o_z, sizeof(double) * M);
  if (n_zmssd_out) memcpy(n_zmssd_out, h + o_nz, sizeof(int) * M);
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
  for (int m = 0; m < M; ++m) {
    if (ref_index[m] < 0 || ref_index[m] >= n_ref)
      return set_err(ctx, SVO_B200_EINVAL, "depth_filter_update: ref_index[%d] out of range", m);
    if (ftr_level[m] < 0 || ftr_level[m] >= ref_frames[ref_index[m]]->n_levels)
      return set_err(ctx, SVO_B200_EINVAL, "depth_filter_update: ftr_level[%d] outside the pyramid", m);
  }
  if (opt->max_search_level >= cur->n_levels)
    return set_err(ctx, SVO_B200_EINVAL, "depth_filter_update: max_search_level %d >= %d pyramid levels",
                   opt->max_search_level, cur->n_levels);
  DepthParams P;
  memset(&P, 0, sizeof(P));
  return depth_update_run(ctx, P, ref_frames, ref_T_f_w, n_ref, cur, cur_T_f_w, cam, 0, nullptr, nullptr, opt, M, ref_index,
                          ftr_px, ftr_f, ftr_level, ftr_type, ftr_grad, batch_id, batch_counter, a, b, mu, z_range, sigma2,
                          status_out, px_cur_out, z_out, n_zmssd_out);
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
  for (int m = 0; m < M; ++m) {
    if (ref_index[m] < 0 || ref_index[m] >= n_ref)
      return set_err(ctx, SVO_B200_EINVAL, "depth_filter_update_streams: ref_index[%d] out of range", m);
    if (ftr_level[m] < 0 || ftr_level[m] >= ref_frames[ref_index[m]]->n_levels)
      return set_err(ctx, SVO_B200_EINVAL, "depth_filter_update_streams: ftr_level[%d] outside the pyramid", m);
  }
  std::vector<DepthStream> st((size_t)S);
  for (int s = 0; s < S; ++s) {
    memset(&st[s], 0, sizeof(DepthStream));
    st[s].cur = make_desc(cur[s]);
    memcpy(st[s].cur_T_f_w, cur_T_f_w + 12 * (size_t)s, sizeof(double) * 12);
    const int rc = cam_to_dev(ctx, cam + s, st[s].cam);
    if (rc) return rc;
    st[s].batch_counter = batch_counter[s];
  }
  DepthParams P;
  memset(&P, 0, sizeof(P));
  return depth_update_run(ctx, P, ref_frames, ref_T_f_w, n_ref, nullptr, nullptr, nullptr, S, st.data(), seed_offset, opt, M,
                          ref_index, ftr_px, ftr_f, ftr_level, ftr_type, ftr_grad, batch_id, 0, a, b, mu, z_range, sigma2,
                          status_out, px_cur_out, z_out, n_zmssd_out);
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
  if (M == 0) return 0;
  if (!ref_index || !ftr_px || !ftr_f || !ftr_level || !ftr_type || !ftr_grad || !d_estimate || !d_min || !d_max || !success_out)
    return set_err(ctx, SVO_B200_EINVAL, "find_epipolar_match_direct: NULL candidate arrays");
  for (int m = 0; m < M; ++m) {
    if (ref_index[m] < 0 || ref_index[m] >= n_ref)
      return set_err(ctx, SVO_B200_EINVAL, "find_epipolar_match_direct: ref_index[%d] out of range", m);
    if (ftr_level[m] < 0 || ftr_level[m] >= ref_frames[ref_index[m]]->n_levels)
      return set_err(ctx, SVO_B200_EINVAL, "find_epipolar_match_direct: ftr_level[%d] outside the pyramid", m);
  }
  if (opt->max_search_level >= cur->n_levels)
    return set_err(ctx, SVO_B200_EINVAL, "find_epipolar_match_direct: max_search_level %d >= %d pyramid levels",
                   opt->max_search_level, cur->n_levels);
  cudaSetDevice(ctx->device);
  Carver c;
  const size_t o_ri = c.take(sizeof(int) * M), o_px = c.take(sizeof(double) * 2 * M), o_f = c.take(sizeof(double) * 3 * M),
               o_lv = c.take(sizeof(int) * M), o_ty = c.take(sizeof(int) * M), o_gr = c.take(sizeof(double) * 2 * M),
               o_de = c.take(sizeof(double) * M), o_dn = c.take(sizeof(double) * M), o_dx = c.take(sizeof(double) * M),
               o_rT = c.take(sizeof(double) * 12 * n_ref), o_fr = c.take(sizeof(FrameDesc) * n_ref);
  const size_t in_bytes = c.off;
  const size_t o_st = c.take(M), o_pc = c.take(sizeof(double) * 2 * M), o_z = c.take(sizeof(double) * M),
               o_nz = c.take(sizeof(int) * M), o_sl = c.take(sizeof(int) * M), o_el = c.take(sizeof(double) * M),
               o_rj = c.take(M), o_A = c.take(sizeof(double) * 4 * M);
  int rc;
  if ((rc = ensure_host(ctx, ctx->h_in, c.off))) return rc;
  if ((rc = ensure_dev(ctx, ctx->d_in, c.off))) return rc;
  SVO_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
  uint8_t* h = static_cast<uint8_t*>(ctx->h_in.p);
  uint8_t* d = static_cast<uint8_t*>(ctx->d_in.p);
  memcpy(h + o_ri, ref_index, sizeof(int) * M);
  memcpy(h + o_px, ftr_px, sizeof(double) * 2 * M);
  memcpy(h + o_f, ftr_f, sizeof(double) * 3 * M);
  memcpy(h + o_lv, ftr_level, sizeof(int) * M);
  memcpy(h + o_ty, ftr_type, sizeof(int) * M);
  memcpy(h + o_gr, ftr_grad, sizeof(double) * 2 * M);
  memcpy(h + o_de, d_estimate, sizeof(double) * M);
  memcpy(h + o_dn, d_min, sizeof(double) * M);
  memcpy(h + o_dx, d_max, sizeof(double) * M);
  memcpy(h + o_rT, ref_T_f_w, sizeof(double) * 12 * n_ref);
  for (int r = 0; r < n_ref; ++r) reinterpret_cast<FrameDesc*>(h + o_fr)[r] = make_desc(ref_frames[r]);
  SVO_CUDA_CHECK(ctx, cudaMemcpyAsync(d, h, in_bytes, cudaMemcpyHostToDevice, ctx->stream));
  SVO_CUDA_CHECK(ctx, cudaMemsetAsync(d + o_st, 0, c.off - o_st, ctx->stream));
  DepthParams P;
  memset(&P, 0, sizeof(P));
  P.match_only = 1;
  P.ref_frames = reinterpret_cast<const FrameDesc*>(d + o_fr);
  P.ref_T_f_w = reinterpret_cast<const double*>(d + o_rT);
  P.cur = make_desc(cur);
  memcpy(P.cur_T_f_w, cur_T_f_w, sizeof(double) * 12);
  if ((rc = cam_to_dev(ctx, cam, P.cam))) return rc;
  P.M = M;
  P.ref_index = reinterpret_cast<const int*>(d + o_ri);
  P.ftr_px = reinterpret_cast<const double*>(d + o_px);
  P.ftr_f = reinterpret_cast<const double*>(d + o_f);
  P.ftr_level = reinterpret_cast<const int*>(d + o_lv);
  P.ftr_type = reinterpret_cast<const int*>(d + o_ty);
  P.ftr_grad = reinterpret_cast<const double*>(d + o_gr);
  P.d_est = reinterpret_cast<const double*>(d + o_de);
  P.d_min = reinterpret_cast<const double*>(d + o_dn);
  P.d_max = reinterpret_cast<const double*>(d + o_dx);
  P.max_search_level = opt->max_search_level;
  P.align_max_iter = opt->align_max_iter;
  P.max_epi_search_steps = opt->max_epi_search_steps;
  P.status = d + o_st;
  P.px_cur = reinterpret_cast<double*>(d + o_pc);
  P.z = reinterpret_cast<double*>(d + o_z);
  P.n_zmssd = reinterpret_cast<int*>(d + o_nz);
  P.search_level_out = reinterpret_cast<int*>(d + o_sl);
  P.epi_length_out = reinterpret_cast<double*>(d + o_el);
  P.reject_out = d + o_rj;
  P.A_out = reinterpret_cast<double*>(d + o_A);
  const int blocks = (M + kDfWarps - 1) / kDfWarps;
  kt_begin(ctx);
  depth_filter_kernel<<<blocks, kDfWarps * 32, 0, ctx->stream>>>(P);
  ctx->launches++;
  kt_end(ctx);
  SVO_CUDA_CHECK(ctx, cudaGetLastError());
  SVO_CUDA_CHECK(ctx, cudaMemcpyAsync(h + o_st, d + o_st, c.off - o_st, cudaMemcpyDeviceToHost, ctx->stream));
  SVO_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
  for (int m = 0; m < M; ++m) success_out[m] = h[o_st + m] == SVO_B200_SEED_UPDATED;
  if (depth_out) memcpy(depth_out, h + o_z, sizeof(double) * M);
  if (px_cur_out) memcpy(px_cur_out, h + o_pc, sizeof(double) * 2 * M);
  if (search_level_out) memcpy(search_level_out, h + o_sl, sizeof(int) * M);
  if (epi_length_out) memcpy(epi_length_out, h + o_el, sizeof(double) * M);
  if (reject_out) memcpy(reject_out, h + o_rj, M);
  if (A_cur_ref_out) memcpy(A_cur_ref_out, h + o_A, sizeof(double) * 4 * M);
  if (n_zmssd_out) memcpy(n_zmssd_out, h + o_nz, sizeof(int) * M);
  return 0;
}
