// rpg_svo_b200/csrc/klt.cu -- the two-view initialisation's KLT tracking (initialization::trackKlt,
// svo/src/initialization.cpp:127-169, over cv::calcOpticalFlowPyrLK) on the device.
//
// [EXT] OpenCV's pyramidal Lucas-Kanade (modules/video/src/lkpyramid.cpp), restated from its published algorithm; the
// oracle (oracle/svo_oracle_klt.cpp) restates it the same way and DESIGN.md section 4.2d lists the rules.
//   * LK pyramid: every level is stored with a 30-pixel border on each side, as OpenCV keeps it: the image's border is
//     its reflect-101 continuation, the derivatives' border is zero.  The tracker's window reads (corner >= -30,
//     corner < size, 31 x 31 pixels with the bilinear neighbour) then never leave the allocation.
//   * Tracker: one warp per point.  Lane l owns window pixels l, l + 32, ... (900 = 28 * 32 + 4); the reference window
//     (intensity and derivatives) sits in the warp's shared memory for the whole level.  Every float sum is the lane's
//     partial in increasing pixel order followed by an xor-butterfly over the lanes: the order the oracle uses, so the
//     kernel and the oracle agree bit for bit (-fmad=false keeps every product and sum rounded on its own, as OpenCV's
//     scalar code does).  All lanes hold the same sums, so the per-point control flow is warp-uniform.
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstring>

#include "ctx.h"

struct svo_b200_klt_pyramid {
  int n_levels = 0, width = 0, height = 0;
  bool derivs = false;
  int w[SVO_B200_MAX_LEVELS] = {0}, h[SVO_B200_MAX_LEVELS] = {0};
  uint8_t* img[SVO_B200_MAX_LEVELS] = {nullptr};  // (w + 2B) x (h + 2B), pitch w + 2B
  int* der[SVO_B200_MAX_LEVELS] = {nullptr};      // same geometry, one (dx, dy) int16 pair per int; null without derivatives
  void* mem = nullptr;
  size_t bytes = 0;
};

namespace svo {
namespace {

constexpr int kWin = 30;               // the only window size the reference uses (initialization.cpp:136)
constexpr int kB = kWin;               // border of every stored level
constexpr int kWinPx = kWin * kWin;    // 900
constexpr int kPxPerLane = (kWinPx + 31) / 32;
constexpr int kWarps = 4;              // points per CTA
constexpr float kMinEig = 1e-4f;       // calcOpticalFlowPyrLK's default minEigThreshold

__device__ __forceinline__ int reflect101(int p, int len) {  // cv::borderInterpolate(p, len, BORDER_REFLECT_101)
  if (len == 1) return 0;
  while (p < 0 || p >= len) p = p < 0 ? -p : 2 * len - p - 2;
  return p;
}

// level 0 of the frame (pitch == width) into the bordered layout
__global__ void klt_level0_kernel(const uint8_t* __restrict__ src, int w, int h, uint8_t* __restrict__ dst) {
  const int S = w + 2 * kB, R = h + 2 * kB;
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= S || y >= R) return;
  dst[(size_t)y * S + x] = src[(size_t)reflect101(y - kB, h) * w + reflect101(x - kB, w)];
}

// pyrDown of the bordered level (sw, sh) into the bordered level (dw, dh): the border pixels are the filter's values at
// their reflect-101 source, so the whole bordered level is written by one pass.  The source's 5 x 5 taps around
// (2x, 2y) stay inside its border (2 pixels beyond the level at most) and read its reflect-101 continuation.
__global__ void klt_down_kernel(const uint8_t* __restrict__ src, int sw, uint8_t* __restrict__ dst, int dw, int dh) {
  const int S = dw + 2 * kB, R = dh + 2 * kB, SS = sw + 2 * kB;
  const int X = blockIdx.x * blockDim.x + threadIdx.x, Y = blockIdx.y * blockDim.y + threadIdx.y;
  if (X >= S || Y >= R) return;
  const int x = reflect101(X - kB, dw), y = reflect101(Y - kB, dh);
  const int k[5] = {1, 4, 6, 4, 1};
  int s = 0;
#pragma unroll
  for (int i = 0; i < 5; ++i) {
    const uint8_t* row = src + (size_t)(2 * y + i - 2 + kB) * SS + (2 * x - 2 + kB);
    s += k[i] * (row[0] + 4 * row[1] + 6 * row[2] + 4 * row[3] + row[4]);
  }
  dst[(size_t)Y * S + X] = (uint8_t)((s + 128) >> 8);
}

// Scharr derivatives of a bordered level: [3 10 3] x [-1 0 1], reflect-101 neighbours (the image's border), zero outside
// the level.
__global__ void klt_scharr_kernel(const uint8_t* __restrict__ img, int w, int h, int* __restrict__ der) {
  const int S = w + 2 * kB, R = h + 2 * kB;
  const int X = blockIdx.x * blockDim.x + threadIdx.x, Y = blockIdx.y * blockDim.y + threadIdx.y;
  if (X >= S || Y >= R) return;
  int v = 0;
  if (X >= kB && X < kB + w && Y >= kB && Y < kB + h) {
    const uint8_t* c = img + (size_t)Y * S + X;
    const int t0m = (c[-S - 1] + c[S - 1]) * 3 + c[-1] * 10, t0p = (c[-S + 1] + c[S + 1]) * 3 + c[1] * 10;
    const int t1m = c[S - 1] - c[-S - 1], t1c = c[S] - c[-S], t1p = c[S + 1] - c[-S + 1];
    const int dx = t0p - t0m, dy = (t1p + t1m) * 3 + t1c * 10;
    v = (int)(uint16_t)(int16_t)dx | ((int)(int16_t)dy << 16);
  }
  der[(size_t)Y * S + X] = v;
}

struct KltLevels {
  const uint8_t* I[SVO_B200_MAX_LEVELS];
  const int* D[SVO_B200_MAX_LEVELS];
  const uint8_t* J[SVO_B200_MAX_LEVELS];
  int w[SVO_B200_MAX_LEVELS], h[SVO_B200_MAX_LEVELS];
  int n_levels;
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  return v;
}
__device__ __forceinline__ int descale(int x, int n) { return (x + (1 << (n - 1))) >> n; }
__device__ __forceinline__ void weights(float a, float b, int& w00, int& w01, int& w10, int& w11) {
  w00 = __float2int_rn((1.f - a) * (1.f - b) * (float)(1 << 14));
  w01 = __float2int_rn(a * (1.f - b) * (float)(1 << 14));
  w10 = __float2int_rn((1.f - a) * b * (float)(1 << 14));
  w11 = (1 << 14) - w00 - w01 - w10;
}
// The window corner (ix, iy) = floor of (x, y), converted with cvt.rzi, which saturates +-inf and values beyond int's range
// (those fail the bounds) but turns NaN into 0.  OpenCV's cvFloor gives INT_MIN for NaN, so a NaN corner is out of bounds.
__device__ __forceinline__ bool out_of_bounds(float x, float y, int ix, int iy, int w, int h) {
  return ix < -kWin || ix >= w || iy < -kWin || iy >= h || isnan(x) || isnan(y);
}

__global__ void __launch_bounds__(kWarps * 32) klt_track_kernel(KltLevels L, int max_iter, double eps2, int n,
                                                               const float2* __restrict__ prev_pts, float2* __restrict__ next_pts,
                                                               uint8_t* __restrict__ status, svo_b200_klt_exit* __restrict__ ex) {
  __shared__ int16_t s_I[kWarps][kWinPx];
  __shared__ int s_D[kWarps][kWinPx];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i = blockIdx.x * kWarps + warp;
  if (i >= n) return;
  int16_t* sI = s_I[warp];
  int* sD = s_D[warp];
  const float hw = (kWin - 1) * 0.5f;
  const float2 p0 = prev_pts[i];
  float2 nxt = next_pts[i];  // nextPts[ptidx]
  bool st = true;
  svo_b200_klt_exit e;
  e.reason = -1;
  for (int l = 0; l < SVO_B200_MAX_LEVELS; ++l) { e.level_reason[l] = -1; e.iters[l] = 0; }
  const int maxL = L.n_levels - 1;
  for (int level = maxL; level >= 0; --level) {
    const int w = L.w[level], h = L.h[level], S = w + 2 * kB;
    const float sc = (float)(1. / (1 << level));
    float px = p0.x * sc, py = p0.y * sc;
    float nx, ny;
    if (level == maxL) { nx = nxt.x * sc; ny = nxt.y * sc; }
    else { nx = nxt.x * 2.f; ny = nxt.y * 2.f; }
    nxt = make_float2(nx, ny);
    px -= hw; py -= hw;
    const int ipx = (int)floorf(px), ipy = (int)floorf(py);
    if (out_of_bounds(px, py, ipx, ipy, w, h)) {
      e.level_reason[level] = SVO_B200_KLT_OUT_OF_BOUNDS;
      if (level == 0) st = false;
      continue;
    }
    int w00, w01, w10, w11;
    weights(px - ipx, py - ipy, w00, w01, w10, w11);
    const uint8_t* I = L.I[level] + (size_t)(ipy + kB) * S + (ipx + kB);
    const int* D = L.D[level] + (size_t)(ipy + kB) * S + (ipx + kB);
    float a11 = 0.f, a12 = 0.f, a22 = 0.f;
#pragma unroll 4
    for (int k = 0; k < kPxPerLane; ++k) {
      const int p = lane + 32 * k;
      if (p < kWinPx) {
        const int y = p / kWin, x = p - y * kWin;
        const uint8_t* s = I + y * S + x;
        const int* d = D + y * S + x;
        const int ival = descale(s[0] * w00 + s[1] * w01 + s[S] * w10 + s[S + 1] * w11, 9);
        const int d00 = d[0], d01 = d[1], d10 = d[S], d11 = d[S + 1];
        const int ix = descale((int16_t)d00 * w00 + (int16_t)d01 * w01 + (int16_t)d10 * w10 + (int16_t)d11 * w11, 14);
        const int iy = descale((d00 >> 16) * w00 + (d01 >> 16) * w01 + (d10 >> 16) * w10 + (d11 >> 16) * w11, 14);
        sI[p] = (int16_t)ival;
        sD[p] = (int)(uint16_t)(int16_t)ix | ((int)(int16_t)iy << 16);
        a11 += (float)(ix * ix);
        a12 += (float)(ix * iy);
        a22 += (float)(iy * iy);
      }
    }
    const float FLT_SCALE = 1.f / (1 << 20);
    const float A11 = warp_sum(a11) * FLT_SCALE, A12 = warp_sum(a12) * FLT_SCALE, A22 = warp_sum(a22) * FLT_SCALE;
    float Dt = A11 * A22 - A12 * A12;
    const float minEig = (A22 + A11 - sqrtf((A11 - A22) * (A11 - A22) + 4.f * A12 * A12)) / (float)(2 * kWinPx);
    if (minEig < kMinEig || Dt < FLT_EPSILON) {
      e.level_reason[level] = SVO_B200_KLT_SMALL_EIG;
      if (level == 0) st = false;
      continue;
    }
    Dt = 1.f / Dt;
    nx -= hw; ny -= hw;
    float pdx = 0.f, pdy = 0.f;
    int why = SVO_B200_KLT_MAX_ITER;
    for (int j = 0; j < max_iter; ++j) {
      const int inx = (int)floorf(nx), iny = (int)floorf(ny);
      if (out_of_bounds(nx, ny, inx, iny, w, h)) {
        why = SVO_B200_KLT_OUT_OF_BOUNDS;
        if (level == 0) st = false;
        break;
      }
      weights(nx - inx, ny - iny, w00, w01, w10, w11);
      const uint8_t* J = L.J[level] + (size_t)(iny + kB) * S + (inx + kB);
      float b1 = 0.f, b2 = 0.f;
#pragma unroll 4
      for (int k = 0; k < kPxPerLane; ++k) {
        const int p = lane + 32 * k;
        if (p < kWinPx) {
          const int y = p / kWin, x = p - y * kWin;
          const uint8_t* s = J + y * S + x;
          const int diff = descale(s[0] * w00 + s[1] * w01 + s[S] * w10 + s[S + 1] * w11, 9) - sI[p];
          const int d = sD[p];
          b1 += (float)(diff * (int)(int16_t)d);
          b2 += (float)(diff * (d >> 16));
        }
      }
      b1 = warp_sum(b1) * FLT_SCALE;
      b2 = warp_sum(b2) * FLT_SCALE;
      const float dx = (A12 * b2 - A22 * b1) * Dt, dy = (A12 * b1 - A11 * b2) * Dt;
      nx += dx; ny += dy;
      nxt = make_float2(nx + hw, ny + hw);
      e.iters[level] = j + 1;
      if ((double)dx * dx + (double)dy * dy <= eps2) { why = SVO_B200_KLT_CONVERGED; break; }
      if (j > 0 && (double)fabsf(dx + pdx) < 0.01 && (double)fabsf(dy + pdy) < 0.01) {
        nxt.x -= dx * 0.5f; nxt.y -= dy * 0.5f;
        why = SVO_B200_KLT_HALF_STEP;
        break;
      }
      pdx = dx; pdy = dy;
    }
    e.level_reason[level] = why;
  }
  if (lane == 0) {
    next_pts[i] = nxt;
    status[i] = st ? 1 : 0;
    if (ex) { e.reason = e.level_reason[0]; ex[i] = e; }
  }
}

inline dim3 grid2d(int S, int R) { return dim3((S + 31) / 32, (R + 7) / 8); }

}  // namespace
}  // namespace svo

using namespace svo;

extern "C" int svo_b200_klt_pyramid_create(svo_b200_ctx* ctx, svo_b200_klt_pyramid** pyr_out) {
  if (!ctx || !pyr_out) return set_err(ctx, SVO_B200_EINVAL, "klt_pyramid_create: bad arguments");
  *pyr_out = new svo_b200_klt_pyramid();
  return 0;
}

extern "C" void svo_b200_klt_pyramid_destroy(svo_b200_ctx* ctx, svo_b200_klt_pyramid* pyr) {
  if (!pyr) return;
  if (pyr->mem) {
    if (ctx) cudaSetDevice(ctx->device);
    cudaFree(pyr->mem);
  }
  delete pyr;
}

extern "C" int svo_b200_klt_pyramid_levels(const svo_b200_klt_pyramid* pyr) { return pyr ? pyr->n_levels : 0; }

extern "C" int svo_b200_klt_pyramid_build(svo_b200_ctx* ctx, svo_b200_klt_pyramid* pyr, const svo_b200_frame* frame, int max_level,
                                          int with_derivatives) {
  if (!ctx || !pyr || !frame || max_level < 0 || (with_derivatives != 0 && with_derivatives != 1))
    return set_err(ctx, SVO_B200_EINVAL, "klt_pyramid_build: bad arguments");
  int w[SVO_B200_MAX_LEVELS], h[SVO_B200_MAX_LEVELS], n = 0;
  for (int level = 0, cw = frame->width, ch = frame->height; level <= max_level; ++level) {
    if (level == SVO_B200_MAX_LEVELS)  // OpenCV would build another level: refuse rather than track from a finer start
      return set_err(ctx, SVO_B200_EINVAL, "klt_pyramid_build: %dx%d at max_level %d needs more than %d levels", frame->width,
                     frame->height, max_level, SVO_B200_MAX_LEVELS);
    w[level] = cw; h[level] = ch;  // buildOpticalFlowPyramid's level cut
    n = level + 1;
    cw = (cw + 1) / 2; ch = (ch + 1) / 2;
    if (cw <= kWin || ch <= kWin) break;
  }
  size_t off[SVO_B200_MAX_LEVELS], doff[SVO_B200_MAX_LEVELS];
  Carver c;
  for (int l = 0; l < n; ++l) off[l] = c.take((size_t)(w[l] + 2 * kB) * (h[l] + 2 * kB));
  for (int l = 0; l < n; ++l) doff[l] = with_derivatives ? c.take((size_t)(w[l] + 2 * kB) * (h[l] + 2 * kB) * 4) : 0;
  cudaSetDevice(ctx->device);
  if (c.off > pyr->bytes) {
    if (pyr->mem) SVO_CUDA_CHECK(ctx, cudaFree(pyr->mem));
    pyr->mem = nullptr;
    pyr->bytes = 0;
    if (cudaMalloc(&pyr->mem, c.off) != cudaSuccess) {
      cudaGetLastError();
      return set_err(ctx, SVO_B200_ENOMEM, "klt_pyramid_build: cudaMalloc(%zu) failed", c.off);
    }
    pyr->bytes = c.off;
  }
  uint8_t* base = static_cast<uint8_t*>(pyr->mem);
  pyr->n_levels = n;
  pyr->width = frame->width;
  pyr->height = frame->height;
  pyr->derivs = with_derivatives != 0;
  for (int l = 0; l < SVO_B200_MAX_LEVELS; ++l) {
    pyr->w[l] = l < n ? w[l] : 0;
    pyr->h[l] = l < n ? h[l] : 0;
    pyr->img[l] = l < n ? base + off[l] : nullptr;
    pyr->der[l] = l < n && with_derivatives ? reinterpret_cast<int*>(base + doff[l]) : nullptr;
  }
  kt_begin(ctx);
  const dim3 blk(32, 8);
  klt_level0_kernel<<<grid2d(w[0] + 2 * kB, h[0] + 2 * kB), blk, 0, ctx->stream>>>(frame->lvl(0), w[0], h[0], pyr->img[0]);
  ctx->launches++;
  for (int l = 1; l < n; ++l) {
    klt_down_kernel<<<grid2d(w[l] + 2 * kB, h[l] + 2 * kB), blk, 0, ctx->stream>>>(pyr->img[l - 1], w[l - 1], pyr->img[l], w[l], h[l]);
    ctx->launches++;
  }
  if (with_derivatives)
    for (int l = 0; l < n; ++l) {
      klt_scharr_kernel<<<grid2d(w[l] + 2 * kB, h[l] + 2 * kB), blk, 0, ctx->stream>>>(pyr->img[l], w[l], h[l], pyr->der[l]);
      ctx->launches++;
    }
  kt_end(ctx);
  SVO_CUDA_CHECK(ctx, cudaGetLastError());
  return 0;
}

extern "C" int svo_b200_klt_pyramid_download(svo_b200_ctx* ctx, const svo_b200_klt_pyramid* pyr, int level, uint8_t* img_out,
                                             int16_t* deriv_out) {
  if (!ctx || !pyr || level < 0 || level >= pyr->n_levels || (deriv_out && !pyr->derivs))
    return set_err(ctx, SVO_B200_EINVAL, "klt_pyramid_download: bad arguments");
  cudaSetDevice(ctx->device);
  const int w = pyr->w[level], h = pyr->h[level], S = w + 2 * kB;
  ctx->sia_chain = false;
  if (img_out)
    SVO_CUDA_CHECK(ctx, cudaMemcpy2DAsync(img_out, w, pyr->img[level] + (size_t)kB * S + kB, S, w, h, cudaMemcpyDeviceToHost, ctx->stream));
  if (deriv_out)
    SVO_CUDA_CHECK(ctx, cudaMemcpy2DAsync(deriv_out, (size_t)w * 4, pyr->der[level] + (size_t)kB * S + kB, (size_t)S * 4, (size_t)w * 4, h,
                                          cudaMemcpyDeviceToHost, ctx->stream));
  SVO_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
  return 0;
}

extern "C" int svo_b200_klt_track(svo_b200_ctx* ctx, const svo_b200_klt_pyramid* prev, const svo_b200_klt_pyramid* next,
                                  const svo_b200_klt_options* opt, int N, const float* prev_pts, float* next_pts_io,
                                  uint8_t* status_out, svo_b200_klt_exit* exit_out) {
  if (!ctx || !prev || !next || !opt || N < 0) return set_err(ctx, SVO_B200_EINVAL, "klt_track: bad arguments");
  if (opt->win_size != kWin)
    return set_err(ctx, SVO_B200_EINVAL, "klt_track: window size %d (only %d is supported)", opt->win_size, kWin);
  if (opt->max_level < 0 || !(opt->eps >= 0.0))
    return set_err(ctx, SVO_B200_EINVAL, "klt_track: bad options (max_level %d, eps %g)", opt->max_level, opt->eps);
  if (prev->n_levels == 0 || next->n_levels == 0 || !prev->derivs)
    return set_err(ctx, SVO_B200_EINVAL, "klt_track: the previous pyramid needs a build with derivatives, the next one a build");
  if (prev->width != next->width || prev->height != next->height)
    return set_err(ctx, SVO_B200_EINVAL, "klt_track: images of different sizes (%dx%d, %dx%d)", prev->width, prev->height,
                   next->width, next->height);
  if (N == 0) return 0;
  if (!prev_pts || !next_pts_io || !status_out) return set_err(ctx, SVO_B200_EINVAL, "klt_track: bad arguments");
  KltLevels L;
  std::memset(&L, 0, sizeof(L));
  L.n_levels = std::min(std::min(prev->n_levels, next->n_levels), opt->max_level + 1);
  for (int l = 0; l < L.n_levels; ++l) {
    L.I[l] = prev->img[l]; L.D[l] = prev->der[l]; L.J[l] = next->img[l];
    L.w[l] = prev->w[l]; L.h[l] = prev->h[l];
  }
  const int max_iter = std::min(std::max(opt->max_iter, 0), 100);  // calcOpticalFlowPyrLK's clamps
  const double eps = std::min(opt->eps, 10.0);
  cudaSetDevice(ctx->device);
  Carver ci, co;
  const size_t i_prev = ci.take((size_t)N * 8), i_next = ci.take((size_t)N * 8);
  const size_t o_next = co.take((size_t)N * 8), o_st = co.take((size_t)N), o_ex = co.take(exit_out ? (size_t)N * sizeof(svo_b200_klt_exit) : 0);
  int rc;
  if ((rc = ensure_host(ctx, ctx->h_in, ci.off)) || (rc = ensure_dev(ctx, ctx->d_in, ci.off)) ||
      (rc = ensure_host(ctx, ctx->h_out, co.off)) || (rc = ensure_dev(ctx, ctx->d_out, co.off)))
    return rc;
  SVO_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
  uint8_t* hi = static_cast<uint8_t*>(ctx->h_in.p);
  uint8_t* di = static_cast<uint8_t*>(ctx->d_in.p);
  uint8_t* ho = static_cast<uint8_t*>(ctx->h_out.p);
  uint8_t* dout = static_cast<uint8_t*>(ctx->d_out.p);
  std::memcpy(hi + i_prev, prev_pts, (size_t)N * 8);
  std::memcpy(hi + i_next, next_pts_io, (size_t)N * 8);
  SVO_CUDA_CHECK(ctx, cudaMemcpyAsync(di, hi, ci.off, cudaMemcpyHostToDevice, ctx->stream));
  // the kernel reads the initial guess and writes the result through one array: the output slot starts as the guess
  SVO_CUDA_CHECK(ctx, cudaMemcpyAsync(dout + o_next, di + i_next, (size_t)N * 8, cudaMemcpyDeviceToDevice, ctx->stream));
  kt_begin(ctx);
  klt_track_kernel<<<(N + kWarps - 1) / kWarps, kWarps * 32, 0, ctx->stream>>>(
      L, max_iter, eps * eps, N, reinterpret_cast<const float2*>(di + i_prev), reinterpret_cast<float2*>(dout + o_next), dout + o_st,
      exit_out ? reinterpret_cast<svo_b200_klt_exit*>(dout + o_ex) : nullptr);
  ctx->launches++;
  kt_end(ctx);
  SVO_CUDA_CHECK(ctx, cudaGetLastError());
  SVO_CUDA_CHECK(ctx, cudaMemcpyAsync(ho, dout, co.off, cudaMemcpyDeviceToHost, ctx->stream));
  SVO_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
  std::memcpy(next_pts_io, ho + o_next, (size_t)N * 8);
  std::memcpy(status_out, ho + o_st, (size_t)N);
  if (exit_out) std::memcpy(exit_out, ho + o_ex, (size_t)N * sizeof(svo_b200_klt_exit));
  return 0;
}
