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
//   * Many streams: one tracking launch and one pyramid build serve S streams (svo_b200_klt_track_streams,
//     svo_b200_klt_pyramid_build_streams; DESIGN.md section 4.2e).  Each stream's levels, options and point offset sit in
//     a table in global memory; a CTA finds its stream with stream_of.  The single calls are one stream of these.
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstring>
#include <vector>

#include "ctx.h"
#include "warp_align.cuh"

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

// One image of a batched pyramid build launch (S pyramids' stage in one launch): CTA i of the launch is tile
// i - cta_offset[j] of job j = stream_of(cta_offset, n_jobs, i), tiles of 32 x 8 pixels of the bordered level, row by row.
//   level 0:  src = the frame's level 0 (pitch == w), dst = the bordered level 0
//   pyrDown:  src = the bordered level above (sw wide), dst = the bordered level (w x h)
//   Scharr:   src = the bordered level (w x h), der = its derivatives
struct KltJob {
  const uint8_t* src;
  uint8_t* dst;
  int* der;
  int sw, w, h, tiles_x;
};

// the job of this CTA and the bordered pixel (X, Y) of this thread
__device__ __forceinline__ const KltJob& klt_job(const KltJob* __restrict__ jobs, const int* __restrict__ cta_offset, int n_jobs,
                                                 int& X, int& Y) {
  const int j = stream_of(cta_offset, n_jobs, (int)blockIdx.x);
  const KltJob& jb = jobs[j];
  const int t = (int)blockIdx.x - __ldg(cta_offset + j);
  const int ty = t / jb.tiles_x, tx = t - ty * jb.tiles_x;
  X = tx * 32 + (int)threadIdx.x;
  Y = ty * 8 + (int)threadIdx.y;
  return jb;
}

// level 0 of the frame (pitch == width) into the bordered layout
__global__ void __launch_bounds__(256) klt_level0_kernel(const KltJob* __restrict__ jobs, const int* __restrict__ cta_offset, int n_jobs) {
  int X, Y;
  const KltJob& jb = klt_job(jobs, cta_offset, n_jobs, X, Y);
  const int w = jb.w, h = jb.h;
  const int S = w + 2 * kB, R = h + 2 * kB;
  if (X >= S || Y >= R) return;
  jb.dst[(size_t)Y * S + X] = jb.src[(size_t)reflect101(Y - kB, h) * w + reflect101(X - kB, w)];
}

// pyrDown of the bordered level (sw, sh) into the bordered level (dw, dh): the border pixels are the filter's values at
// their reflect-101 source, so the whole bordered level is written by one pass.  The source's 5 x 5 taps around
// (2x, 2y) stay inside its border (2 pixels beyond the level at most) and read its reflect-101 continuation.
__global__ void __launch_bounds__(256) klt_down_kernel(const KltJob* __restrict__ jobs, const int* __restrict__ cta_offset, int n_jobs) {
  int X, Y;
  const KltJob& jb = klt_job(jobs, cta_offset, n_jobs, X, Y);
  const int dw = jb.w, dh = jb.h;
  const int S = dw + 2 * kB, R = dh + 2 * kB, SS = jb.sw + 2 * kB;
  if (X >= S || Y >= R) return;
  const uint8_t* __restrict__ src = jb.src;
  const int x = reflect101(X - kB, dw), y = reflect101(Y - kB, dh);
  const int k[5] = {1, 4, 6, 4, 1};
  int s = 0;
#pragma unroll
  for (int i = 0; i < 5; ++i) {
    const uint8_t* row = src + (size_t)(2 * y + i - 2 + kB) * SS + (2 * x - 2 + kB);
    s += k[i] * (row[0] + 4 * row[1] + 6 * row[2] + 4 * row[3] + row[4]);
  }
  jb.dst[(size_t)Y * S + X] = (uint8_t)((s + 128) >> 8);
}

// Scharr derivatives of a bordered level: [3 10 3] x [-1 0 1], reflect-101 neighbours (the image's border), zero outside
// the level.
__global__ void __launch_bounds__(256) klt_scharr_kernel(const KltJob* __restrict__ jobs, const int* __restrict__ cta_offset, int n_jobs) {
  int X, Y;
  const KltJob& jb = klt_job(jobs, cta_offset, n_jobs, X, Y);
  const int w = jb.w, h = jb.h;
  const int S = w + 2 * kB, R = h + 2 * kB;
  if (X >= S || Y >= R) return;
  int v = 0;
  if (X >= kB && X < kB + w && Y >= kB && Y < kB + h) {
    const uint8_t* c = jb.src + (size_t)Y * S + X;
    const int t0m = (c[-S - 1] + c[S - 1]) * 3 + c[-1] * 10, t0p = (c[-S + 1] + c[S + 1]) * 3 + c[1] * 10;
    const int t1m = c[S - 1] - c[-S - 1], t1c = c[S] - c[-S], t1p = c[S + 1] - c[-S + 1];
    const int dx = t0p - t0m, dy = (t1p + t1m) * 3 + t1c * 10;
    v = (int)(uint16_t)(int16_t)dx | ((int)(int16_t)dy << 16);
  }
  jb.der[(size_t)Y * S + X] = v;
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

// One stream of a tracking launch: its levels (after the max_level cut), its clamped options, and where its points sit in
// the launch's concatenated arrays (ex_off < 0: no exit records).
struct KltStream {
  KltLevels L;
  double eps2;
  int max_iter, n, pt_off, ex_off;
};

// One point, tracked by one warp: p0 = prevPts[ptidx], nxt = the initial guess nextPts[ptidx]; sI / sD the warp's window.
// Lane 0 writes the point, its status and (ex non-null) its exit record.
__device__ __forceinline__ void klt_track_point(const KltLevels& L, int max_iter, double eps2, float2 p0, float2 nxt, int lane,
                                                int16_t* sI, int* sD, float2* next_out, uint8_t* status_out,
                                                svo_b200_klt_exit* ex) {
  const float hw = (kWin - 1) * 0.5f;
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
    *next_out = nxt;
    *status_out = st ? 1 : 0;
    if (ex) { e.reason = e.level_reason[0]; *ex = e; }
  }
}

// One warp per point of n_streams streams' concatenated points: CTA i holds points (i - cta_offset[s]) * kWarps ... of
// stream s = stream_of(cta_offset, n_streams, i) (stream s has ceil(n / kWarps) CTAs, so a CTA never spans two streams).
// The initial guesses come in through `guess`, the results go out through next_pts.
__global__ void __launch_bounds__(kWarps * 32) klt_track_kernel(const KltStream* __restrict__ streams, const int* __restrict__ cta_offset,
                                                               int n_streams, const float2* __restrict__ prev_pts,
                                                               const float2* __restrict__ guess, float2* __restrict__ next_pts,
                                                               uint8_t* __restrict__ status, svo_b200_klt_exit* __restrict__ ex) {
  __shared__ int16_t s_I[kWarps][kWinPx];
  __shared__ int s_D[kWarps][kWinPx];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int s = stream_of(cta_offset, n_streams, (int)blockIdx.x);
  const KltStream& st = streams[s];
  const int k = ((int)blockIdx.x - __ldg(cta_offset + s)) * kWarps + warp;
  if (k >= st.n) return;
  const int i = st.pt_off + k;
  klt_track_point(st.L, st.max_iter, st.eps2, prev_pts[i], guess[i], lane, s_I[warp], s_D[warp], next_pts + i, status + i,
                  st.ex_off < 0 ? nullptr : ex + st.ex_off + k);
}

// S = 1: the same body with the stream's levels and options passed by value, from the parameter space.  A single stream's
// launch is latency-bound (350 points at 752 x 480 are 88 CTAs), and there the table-driven launch measured about 7 %
// slower (DESIGN.md section 4.2e).
__global__ void __launch_bounds__(kWarps * 32) klt_track_one_kernel(const KltStream st, const float2* __restrict__ prev_pts,
                                                                   const float2* __restrict__ guess, float2* __restrict__ next_pts,
                                                                   uint8_t* __restrict__ status, svo_b200_klt_exit* __restrict__ ex) {
  __shared__ int16_t s_I[kWarps][kWinPx];
  __shared__ int s_D[kWarps][kWinPx];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i = blockIdx.x * kWarps + warp;
  if (i >= st.n) return;
  klt_track_point(st.L, st.max_iter, st.eps2, prev_pts[i], guess[i], lane, s_I[warp], s_D[warp], next_pts + i, status + i,
                  st.ex_off < 0 ? nullptr : ex + i);
}

}  // namespace
}  // namespace svo

using namespace svo;


namespace {

// The single build's argument checks and level cut (every entry's, for the batched build); nothing is written.
int klt_build_check(svo_b200_ctx* ctx, const svo_b200_klt_build& b, int w[SVO_B200_MAX_LEVELS], int h[SVO_B200_MAX_LEVELS], int& n) {
  const svo_b200_frame* frame = b.frame;
  if (!ctx || !b.pyr || !frame || b.max_level < 0 || (b.with_derivatives != 0 && b.with_derivatives != 1))
    return set_err(ctx, SVO_B200_EINVAL, "klt_pyramid_build: bad arguments");
  n = 0;
  for (int level = 0, cw = frame->width, ch = frame->height; level <= b.max_level; ++level) {
    if (level == SVO_B200_MAX_LEVELS)  // OpenCV would build another level: refuse rather than track from a finer start
      return set_err(ctx, SVO_B200_EINVAL, "klt_pyramid_build: %dx%d at max_level %d needs more than %d levels", frame->width,
                     frame->height, b.max_level, SVO_B200_MAX_LEVELS);
    w[level] = cw; h[level] = ch;  // buildOpticalFlowPyramid's level cut
    n = level + 1;
    cw = (cw + 1) / 2; ch = (ch + 1) / 2;
    if (cw <= kWin || ch <= kWin) break;
  }
  return 0;
}

// One checked build entry: its level sizes and the offsets of its levels and derivatives in the handle's block.
struct KltBuild {
  int w[SVO_B200_MAX_LEVELS], h[SVO_B200_MAX_LEVELS], n = 0;
  size_t off[SVO_B200_MAX_LEVELS], doff[SVO_B200_MAX_LEVELS], bytes = 0;
};

inline int tiles_x(int w) { return (w + 2 * kB + 31) / 32; }
inline int64_t tiles(int w, int h) { return (int64_t)tiles_x(w) * ((h + 2 * kB + 7) / 8); }

// A handle whose block is about to be freed: 0 levels, so that a track refuses it rather than read freed memory.
void klt_unbuild(svo_b200_klt_pyramid* p) {
  p->n_levels = 0;
  p->width = p->height = 0;
  p->derivs = false;
  for (int l = 0; l < SVO_B200_MAX_LEVELS; ++l) { p->w[l] = p->h[l] = 0; p->img[l] = nullptr; p->der[l] = nullptr; }
}

// Every entry checked before anything is allocated or launched; then the handles that need a larger block get one (a
// failed allocation returns before any launch, its handle left unbuilt); then one copy of the job tables to the device
// and one launch per stage: level 0 of every entry, pyrDown of each level 1 .. L_max - 1 of every entry that has it, and
// the Scharr derivatives of every level of every entry that asks for them.  The handles' levels are set last.
int klt_build_run(svo_b200_ctx* ctx, int S, const svo_b200_klt_build* builds, const char* name) {
  std::vector<KltBuild> bs((size_t)S);
  int L_max = 0;
  bool any_der = false;
  for (int s = 0; s < S; ++s) {
    KltBuild& r = bs[s];
    if (const int rc = klt_build_check(ctx, builds[s], r.w, r.h, r.n)) return entry_err(ctx, rc, name, "build", s);
    for (int t = 0; t < s; ++t)
      if (builds[t].pyr == builds[s].pyr) return set_err(ctx, SVO_B200_EINVAL, "%s: builds %d and %d name one handle", name, t, s);
    Carver c;
    for (int l = 0; l < r.n; ++l) r.off[l] = c.take((size_t)(r.w[l] + 2 * kB) * (r.h[l] + 2 * kB));
    for (int l = 0; l < r.n; ++l) r.doff[l] = builds[s].with_derivatives ? c.take((size_t)(r.w[l] + 2 * kB) * (r.h[l] + 2 * kB) * 4) : 0;
    r.bytes = c.off;
    L_max = std::max(L_max, r.n);
    any_der = any_der || builds[s].with_derivatives;
  }
  // one table per launch: level 0, levels 1 .. L_max - 1, Scharr; the jobs' addresses are set once the blocks are allocated
  const int n_launch = L_max + (any_der ? 1 : 0);
  std::vector<LaunchTable<KltJob>> tabs((size_t)n_launch);
  for (int s = 0; s < S; ++s) {
    const KltBuild& r = bs[s];
    for (int l = 0; l < r.n; ++l) {
      const int64_t n = tiles(r.w[l], r.h[l]);
      tabs[l].add(KltJob{nullptr, nullptr, nullptr, l == 0 ? r.w[0] : r.w[l - 1], r.w[l], r.h[l], tiles_x(r.w[l])}, n, 1);
      if (builds[s].with_derivatives) tabs[L_max].add(KltJob{nullptr, nullptr, nullptr, r.w[l], r.w[l], r.h[l], tiles_x(r.w[l])}, n, 1);
    }
  }
  for (const auto& t : tabs)
    if (t.over)
      return set_err(ctx, SVO_B200_ELIMIT, "%s: %lld CTAs exceed one launch's grid", name ? name : "klt_pyramid_build", t.ctas);
  if (S == 0) return 0;
  Staging st(ctx, Staging::Pageable{});
  for (auto& t : tabs) t.stage(st);
  cudaSetDevice(ctx->device);
  int rc;
  if ((rc = st.open())) return rc;
  for (int s = 0; s < S; ++s) {
    svo_b200_klt_pyramid* p = builds[s].pyr;
    if (bs[s].bytes <= p->bytes) continue;
    klt_unbuild(p);
    if (p->mem) {
      void* old = p->mem;
      p->mem = nullptr;
      p->bytes = 0;
      SVO_CUDA_CHECK(ctx, cudaFree(old));
    }
    if (cudaMalloc(&p->mem, bs[s].bytes) != cudaSuccess) {
      cudaGetLastError();
      p->mem = nullptr;
      return set_err(ctx, SVO_B200_ENOMEM, "klt_pyramid_build: cudaMalloc(%zu) failed", bs[s].bytes);
    }
    p->bytes = bs[s].bytes;
  }
  std::vector<int> next((size_t)n_launch, 0);  // jobs of each table addressed so far, in the order they were added
  for (int s = 0; s < S; ++s) {
    const KltBuild& r = bs[s];
    uint8_t* base = static_cast<uint8_t*>(builds[s].pyr->mem);
    for (int l = 0; l < r.n; ++l) {
      KltJob& j = st.host(tabs[l].jobs_at)[next[l]++];
      j.src = l == 0 ? builds[s].frame->lvl(0) : base + r.off[l - 1];
      j.dst = base + r.off[l];
      if (builds[s].with_derivatives) {
        KltJob& d = st.host(tabs[L_max].jobs_at)[next[L_max]++];
        d.src = base + r.off[l];
        d.der = reinterpret_cast<int*>(base + r.doff[l]);
      }
    }
  }
  if ((rc = st.send())) return rc;
  if ((rc = launch_kernels(ctx, n_launch, [&] {
         const dim3 blk(32, 8);
         for (int k = 0; k < n_launch; ++k) {
           const LaunchTable<KltJob>& t = tabs[k];
           if (k == 0) klt_level0_kernel<<<(unsigned)t.ctas, blk, 0, ctx->stream>>>(t.jobs_at, t.off_at, t.n());
           else if (k < L_max) klt_down_kernel<<<(unsigned)t.ctas, blk, 0, ctx->stream>>>(t.jobs_at, t.off_at, t.n());
           else klt_scharr_kernel<<<(unsigned)t.ctas, blk, 0, ctx->stream>>>(t.jobs_at, t.off_at, t.n());
         }
       })))
    return rc;
  for (int s = 0; s < S; ++s) {
    const KltBuild& r = bs[s];
    svo_b200_klt_pyramid* p = builds[s].pyr;
    uint8_t* base = static_cast<uint8_t*>(p->mem);
    const bool der = builds[s].with_derivatives != 0;
    p->n_levels = r.n;
    p->width = builds[s].frame->width;
    p->height = builds[s].frame->height;
    p->derivs = der;
    for (int l = 0; l < SVO_B200_MAX_LEVELS; ++l) {
      p->w[l] = l < r.n ? r.w[l] : 0;
      p->h[l] = l < r.n ? r.h[l] : 0;
      p->img[l] = l < r.n ? base + r.off[l] : nullptr;
      p->der[l] = l < r.n && der ? reinterpret_cast<int*>(base + r.doff[l]) : nullptr;
    }
  }
  return 0;
}

// The single track's argument checks (every stream's, for the streams call); nothing is written.
int klt_track_check(svo_b200_ctx* ctx, const svo_b200_klt_stream& a) {
  const svo_b200_klt_pyramid *prev = a.prev, *next = a.next;
  const svo_b200_klt_options* opt = a.opt;
  if (!ctx || !prev || !next || !opt || a.N < 0) return set_err(ctx, SVO_B200_EINVAL, "klt_track: bad arguments");
  if (opt->win_size != kWin)
    return set_err(ctx, SVO_B200_EINVAL, "klt_track: window size %d (only %d is supported)", opt->win_size, kWin);
  if (opt->max_level < 0 || !(opt->eps >= 0.0))
    return set_err(ctx, SVO_B200_EINVAL, "klt_track: bad options (max_level %d, eps %g)", opt->max_level, opt->eps);
  if (prev->n_levels == 0 || next->n_levels == 0 || !prev->derivs)
    return set_err(ctx, SVO_B200_EINVAL, "klt_track: the previous pyramid needs a build with derivatives, the next one a build");
  if (prev->width != next->width || prev->height != next->height)
    return set_err(ctx, SVO_B200_EINVAL, "klt_track: images of different sizes (%dx%d, %dx%d)", prev->width, prev->height,
                   next->width, next->height);
  if (a.N > 0 && (!a.prev_pts || !a.next_pts_io || !a.status_out)) return set_err(ctx, SVO_B200_EINVAL, "klt_track: bad arguments");
  return 0;
}

// The table entry of one checked stream (point and exit offsets filled in by the caller).
KltStream klt_stream_entry(const svo_b200_klt_stream& a) {
  KltStream t;
  std::memset(&t, 0, sizeof(t));
  KltLevels& L = t.L;
  L.n_levels = std::min(std::min(a.prev->n_levels, a.next->n_levels), a.opt->max_level + 1);
  for (int l = 0; l < L.n_levels; ++l) {
    L.I[l] = a.prev->img[l]; L.D[l] = a.prev->der[l]; L.J[l] = a.next->img[l];
    L.w[l] = a.prev->w[l]; L.h[l] = a.prev->h[l];
  }
  t.max_iter = std::min(std::max(a.opt->max_iter, 0), 100);  // calcOpticalFlowPyrLK's clamps
  const double eps = std::min(a.opt->eps, 10.0);
  t.eps2 = eps * eps;
  t.n = a.N;
  return t;
}

// Every stream checked before anything is written; then one host-to-device copy (table, CTA offsets, every stream's
// points and guesses), one launch, one copy back of every stream's points, statuses and exit records, and each stream's
// share copied into its own outputs.
int klt_track_run(svo_b200_ctx* ctx, int S, const svo_b200_klt_stream* streams, const char* name) {
  LaunchTable<KltStream> tab;
  int64_t n_pts = 0, n_ex = 0;
  for (int s = 0; s < S; ++s) {
    if (const int rc = klt_track_check(ctx, streams[s])) return entry_err(ctx, rc, name, "stream", s);
    KltStream e = klt_stream_entry(streams[s]);
    e.pt_off = (int)std::min<int64_t>(n_pts, INT32_MAX);
    e.ex_off = streams[s].exit_out ? (int)std::min<int64_t>(n_ex, INT32_MAX) : -1;
    tab.add(e, streams[s].N, kWarps);
    n_pts += streams[s].N;
    if (streams[s].exit_out) n_ex += streams[s].N;
  }
  if (n_pts > INT32_MAX)
    return set_err(ctx, SVO_B200_ELIMIT, "%s: %lld points exceed one launch", name ? name : "klt_track", (long long)n_pts);
  if (n_pts == 0) return 0;  // S == 0 included: no copy, no launch
  cudaSetDevice(ctx->device);
  Staging st(ctx);
  const float2 *d_prev, *d_guess;
  float2* d_next;
  uint8_t* d_status;
  svo_b200_klt_exit* d_ex;
  tab.stage(st);
  st.in(nullptr, n_pts, &d_prev);  // every stream's points and guesses, back to back
  st.in(nullptr, n_pts, &d_guess);
  st.out(nullptr, n_pts, &d_next);
  st.out(nullptr, n_pts, &d_status);
  st.out(nullptr, n_ex, &d_ex);
  int rc;
  if ((rc = st.open())) return rc;
  for (int s = 0; s < S; ++s) {
    const svo_b200_klt_stream& a = streams[s];
    if (a.N == 0) continue;
    std::memcpy(st.host(d_prev + tab.jobs[s].pt_off), a.prev_pts, (size_t)a.N * 8);
    std::memcpy(st.host(d_guess + tab.jobs[s].pt_off), a.next_pts_io, (size_t)a.N * 8);
  }
  if ((rc = st.send())) return rc;
  if ((rc = launch_kernels(ctx, 1, [&] {
         if (S == 1)  // the table's entry by value (see klt_track_one_kernel); the staged table is then not read
           klt_track_one_kernel<<<(unsigned)tab.ctas, kWarps * 32, 0, ctx->stream>>>(tab.jobs[0], d_prev, d_guess, d_next, d_status, d_ex);
         else
           klt_track_kernel<<<(unsigned)tab.ctas, kWarps * 32, 0, ctx->stream>>>(tab.jobs_at, tab.off_at, S, d_prev, d_guess, d_next,
                                                                                d_status, d_ex);
       })))
    return rc;
  if ((rc = st.receive())) return rc;
  for (int s = 0; s < S; ++s) {
    const svo_b200_klt_stream& a = streams[s];
    if (a.N == 0) continue;
    std::memcpy(a.next_pts_io, st.host(d_next + tab.jobs[s].pt_off), (size_t)a.N * 8);
    std::memcpy(a.status_out, st.host(d_status + tab.jobs[s].pt_off), (size_t)a.N);
    if (a.exit_out) std::memcpy(a.exit_out, st.host(d_ex + tab.jobs[s].ex_off), (size_t)a.N * sizeof(svo_b200_klt_exit));
  }
  return 0;
}

}  // namespace

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
  const svo_b200_klt_build b = {pyr, frame, max_level, with_derivatives};
  return klt_build_run(ctx, 1, &b, nullptr);
}

extern "C" int svo_b200_klt_pyramid_build_streams(svo_b200_ctx* ctx, int S, const svo_b200_klt_build* builds) {
  if (!ctx || S < 0 || (S > 0 && !builds))
    return set_err(ctx, SVO_B200_EINVAL, "klt_pyramid_build_streams: bad arguments (S %d)", S);
  return klt_build_run(ctx, S, builds, "klt_pyramid_build_streams");
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
  const svo_b200_klt_stream a = {prev, next, opt, N, prev_pts, next_pts_io, status_out, exit_out};
  return klt_track_run(ctx, 1, &a, nullptr);
}

extern "C" int svo_b200_klt_track_streams(svo_b200_ctx* ctx, int S, const svo_b200_klt_stream* streams) {
  if (!ctx || S < 0 || (S > 0 && !streams))
    return set_err(ctx, SVO_B200_EINVAL, "klt_track_streams: bad arguments (S %d)", S);
  return klt_track_run(ctx, S, streams, "klt_track_streams");
}
