// rpg_svo_b200/csrc/detect.cu -- C ABI entry point
//   svo_b200_fast_detect  <- feature_detection::FastDetector::detect (svo/src/feature_detection.cpp:66-115)
//
// "Next" row f4 of SURVEY.md 8f: the seed-initialisation detector that runs after DepthFilter::updateSeeds on keyframes
// (depth_filter.cpp:114-132).  The reference runs, per pyramid level, the `fast` library's segment test (FAST-10, b=20),
// its score bisection and 3x3 non-maximum suppression [EXT], then vk::shiTomasiScore [EXT] per surviving corner and keeps
// the best corner per 30-px grid cell across levels.  Here ONE launch covers all levels: a CTA owns a 32x8 pixel tile
// (+5 px halo in shared memory), evaluates the segment test with two 16-bit ring masks, scores the few corners in closed
// form (score = max over the 16 arcs of the minimum ring contrast, minus one = what the bisection converges to),
// suppresses non-maxima inside the tile (+1 halo of scores), computes the Shi-Tomasi score from the same tile and
// competes for its grid cell with one 64-bit atomicMax on (score bits, reverse scan order) -- which reproduces the
// reference's "first strictly greater score in (level, row, column) order wins".  Integer work throughout; the only
// floating-point step (the eigenvalue formula) uses the oracle's operation order, so results are bit-identical.
#include <cmath>
#include <cstring>
#include <vector>

#include "ctx.h"
#include "warp_align.cuh"

namespace svo {

constexpr int kTileW = 32, kTileH = 8, kHalo = 5;
constexpr int kImgW = kTileW + 2 * kHalo, kImgH = kTileH + 2 * kHalo;  // 42 x 18
constexpr int kScW = kTileW + 2, kScH = kTileH + 2;                    // 34 x 10

struct DetectLevels {
  const uint8_t* img[SVO_B200_MAX_LEVELS];
  int w[SVO_B200_MAX_LEVELS], h[SVO_B200_MAX_LEVELS];
  int tiles_x[SVO_B200_MAX_LEVELS];
  int tile_base[SVO_B200_MAX_LEVELS + 1];  // first CTA of each level
  unsigned order_base[SVO_B200_MAX_LEVELS];  // scan-order offset of each level
  int n_levels;
};

__device__ __forceinline__ bool has_arc10(unsigned m16) {  // >= 10 contiguous set bits on the 16-ring
  unsigned m = m16 | (m16 << 16);
  m &= m >> 1;  // runs of 2
  m &= m >> 2;  // runs of 4
  m &= m >> 4;  // runs of 8
  m &= m >> 2;  // runs of 10
  return (m & 0xffffu) != 0u;
}

__global__ void __launch_bounds__(256) fast_detect_kernel(DetectLevels lv, int b, int ties_suppress, int cell_size, int grid_n_cols,
                                                          const uint8_t* __restrict__ occupancy, unsigned long long* __restrict__ cells) {
  __shared__ uint8_t img[kImgH][kImgW + 2];
  __shared__ int16_t sc[kScH][kScW];
  int L = 0;
  while (L + 1 < lv.n_levels && (int)blockIdx.x >= lv.tile_base[L + 1]) ++L;
  const int t = blockIdx.x - lv.tile_base[L];
  const int x0 = (t % lv.tiles_x[L]) * kTileW, y0 = (t / lv.tiles_x[L]) * kTileH;
  const int W = lv.w[L], H = lv.h[L];
  const uint8_t* __restrict__ src = lv.img[L];
  for (int i = threadIdx.x; i < kImgH * kImgW; i += blockDim.x) {
    const int ly = i / kImgW, lx = i - ly * kImgW;
    const int gx = x0 - kHalo + lx, gy = y0 - kHalo + ly;
    img[ly][lx] = (gx >= 0 && gx < W && gy >= 0 && gy < H) ? __ldg(src + (size_t)gy * W + gx) : 0;
  }
  __syncthreads();
  // ring offsets in the order of the `fast` library (clockwise from 12 o'clock)
  constexpr int RX[16] = {0, 1, 2, 3, 3, 3, 2, 1, 0, -1, -2, -3, -3, -3, -2, -1};
  constexpr int RY[16] = {-3, -3, -2, -1, 0, 1, 2, 3, 3, 3, 2, 1, 0, -1, -2, -3};
  for (int i = threadIdx.x; i < kScH * kScW; i += blockDim.x) {
    const int sy = i / kScW, sx = i - sy * kScW;
    const int gx = x0 - 1 + sx, gy = y0 - 1 + sy;
    int score = -1;  // not a corner; corner scores lie in [b, 254], and b may be 0
    if (gx >= 3 && gx < W - 3 && gy >= 3 && gy < H - 3) {  // fast_corner_detect_10: 3-pixel border
      const int lx = sx + kHalo - 1, ly = sy + kHalo - 1;
      const int c = img[ly][lx];
      int d[16];
      unsigned mb = 0, md = 0;
#pragma unroll
      for (int k = 0; k < 16; ++k) {
        d[k] = (int)img[ly + RY[k]][lx + RX[k]] - c;
        mb |= (d[k] > b ? 1u : 0u) << k;
        md |= (-d[k] > b ? 1u : 0u) << k;
      }
      const bool cb = has_arc10(mb), cd = has_arc10(md);
      if (cb || cd) {
        // fast_corner_score_10: the largest threshold that still passes = (max over arcs of min contrast) - 1.
        // Sliding minimum over 10 ring positions by doubling (2, 4, 8, 8+2), both polarities.
        int best = -256;
#pragma unroll
        for (int pol = 0; pol < 2; ++pol) {
          int e[16], m2[16], m4[16], m8[16];
#pragma unroll
          for (int k = 0; k < 16; ++k) e[k] = pol ? -d[k] : d[k];
#pragma unroll
          for (int k = 0; k < 16; ++k) m2[k] = min(e[k], e[(k + 1) & 15]);
#pragma unroll
          for (int k = 0; k < 16; ++k) m4[k] = min(m2[k], m2[(k + 2) & 15]);
#pragma unroll
          for (int k = 0; k < 16; ++k) m8[k] = min(m4[k], m4[(k + 4) & 15]);
#pragma unroll
          for (int k = 0; k < 16; ++k) best = max(best, min(m8[k], m2[(k + 8) & 15]));
        }
        score = min(max(best - 1, b), 254);
      }
    }
    sc[sy][sx] = (int16_t)score;
  }
  __syncthreads();
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int gx = x0 + tx, gy = y0 + ty;
  const int s = sc[ty + 1][tx + 1];
  if (s < 0 || gx >= W || gy >= H) return;
  // fast_nonmax_3x3: suppressed by a detected neighbour whose score compares >= (ties suppress) or >
  bool bad = false;
#pragma unroll
  for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
    for (int dx = -1; dx <= 1; ++dx) {
      if (dx == 0 && dy == 0) continue;
      const int n = sc[ty + 1 + dy][tx + 1 + dx];
      if (n >= 0 && (ties_suppress ? n >= s : n > s)) bad = true;
    }
  if (bad) return;
  const int scale = 1 << L;
  const int k = ((gy * scale) / cell_size) * grid_n_cols + (gx * scale) / cell_size;  // :98-99
  if (occupancy && occupancy[k]) return;
  // vk::shiTomasiScore [EXT]: 8x8 box of central differences, smaller eigenvalue
  if (gx - 4 < 1 || gx + 4 >= W - 1 || gy - 4 < 1 || gy + 4 >= H - 1) return;  // returns 0.0: can never beat the threshold
  const int lx = tx + kHalo, ly = ty + kHalo;
  int iXX = 0, iYY = 0, iXY = 0;
#pragma unroll
  for (int yy = -4; yy < 4; ++yy)
#pragma unroll
    for (int xx = -4; xx < 4; ++xx) {
      const int dxv = (int)img[ly + yy][lx + xx + 1] - (int)img[ly + yy][lx + xx - 1];
      const int dyv = (int)img[ly + yy + 1][lx + xx] - (int)img[ly + yy - 1][lx + xx];
      iXX += dxv * dxv; iYY += dyv * dyv; iXY += dxv * dyv;
    }
  const float fXX = (float)((double)(float)iXX / 128.0), fYY = (float)((double)(float)iYY / 128.0),
              fXY = (float)((double)(float)iXY / 128.0);
  const float a = __fadd_rn(fXX, fYY);
  const float r = __fsub_rn(__fmul_rn(a, a), __fmul_rn(4.0f, __fsub_rn(__fmul_rn(fXX, fYY), __fmul_rn(fXY, fXY))));
  const float score = (float)(0.5 * ((double)a - sqrt((double)r)));
  if (!(score > 0.0f)) return;  // NaN / non-positive never beats a non-negative threshold
  const unsigned order = lv.order_base[L] + (unsigned)gy * (unsigned)W + (unsigned)gx;
  const unsigned long long key = ((unsigned long long)__float_as_uint(score) << 32) | (unsigned long long)(0xffffffffu - order);
  atomicMax(cells + k, key);
}

}  // namespace svo

using namespace svo;

extern "C" int svo_b200_fast_detect(svo_b200_ctx* ctx, const svo_b200_frame* frame, const svo_b200_detect_options* opt,
                                    const uint8_t* grid_occupancy, int cap, int* x_out, int* y_out, int* level_out,
                                    float* score_out, int* n_out) {
  if (!ctx || !frame || !opt || !n_out || cap < 0 || (cap > 0 && (!x_out || !y_out || !level_out)))
    return set_err(ctx, SVO_B200_EINVAL, "fast_detect: bad arguments");
  if (opt->cell_size <= 0 || opt->n_pyr_levels <= 0 || opt->n_pyr_levels > frame->n_levels || opt->fast_threshold < 0 ||
      opt->fast_threshold > 254 || !(opt->detection_threshold >= 0.0))
    return set_err(ctx, SVO_B200_EINVAL, "fast_detect: bad options (cell_size %d, n_pyr_levels %d of %d, b %d, threshold %g)",
                   opt->cell_size, opt->n_pyr_levels, frame->n_levels, opt->fast_threshold, opt->detection_threshold);
  const FrameDesc fd = make_desc(frame);
  const int W0 = fd.w[0], H0 = fd.h[0];
  const int grid_n_cols = (int)std::ceil((double)W0 / opt->cell_size), grid_n_rows = (int)std::ceil((double)H0 / opt->cell_size);
  const int n_cells = grid_n_cols * grid_n_rows;
  DetectLevels lv;
  std::memset(&lv, 0, sizeof(lv));
  lv.n_levels = opt->n_pyr_levels;
  unsigned order = 0;
  for (int L = 0; L < lv.n_levels; ++L) {
    lv.img[L] = fd.lvl[L]; lv.w[L] = fd.w[L]; lv.h[L] = fd.h[L];
    lv.tiles_x[L] = (fd.w[L] + kTileW - 1) / kTileW;
    lv.tile_base[L + 1] = lv.tile_base[L] + lv.tiles_x[L] * ((fd.h[L] + kTileH - 1) / kTileH);
    lv.order_base[L] = order;
    order += (unsigned)fd.w[L] * (unsigned)fd.h[L];
  }
  cudaSetDevice(ctx->device);
  Carver c;
  const size_t o_cells = c.take(sizeof(unsigned long long) * n_cells), o_occ = c.take(grid_occupancy ? n_cells : 0);
  int rc;
  if ((rc = ensure_host(ctx, ctx->h_in, c.off))) return rc;
  if ((rc = ensure_dev(ctx, ctx->d_in, c.off))) return rc;
  SVO_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
  uint8_t* h = static_cast<uint8_t*>(ctx->h_in.p);
  uint8_t* d = static_cast<uint8_t*>(ctx->d_in.p);
  float thr_f = (float)opt->detection_threshold;  // Corner(0,0,detection_threshold,0,0.0f): stored as float (:72)
  // -0.0 compares like +0.0, but its sign bit would make the initial key larger than every positive score's key
  if (thr_f == 0.0f) thr_f = 0.0f;
  unsigned thr_bits;
  std::memcpy(&thr_bits, &thr_f, 4);
  const unsigned long long init = ((unsigned long long)thr_bits << 32) | 0xffffffffull;
  for (int k = 0; k < n_cells; ++k) reinterpret_cast<unsigned long long*>(h + o_cells)[k] = init;
  if (grid_occupancy) std::memcpy(h + o_occ, grid_occupancy, n_cells);
  SVO_CUDA_CHECK(ctx, cudaMemcpyAsync(d, h, c.off, cudaMemcpyHostToDevice, ctx->stream));
  kt_begin(ctx);
  fast_detect_kernel<<<lv.tile_base[lv.n_levels], 256, 0, ctx->stream>>>(
      lv, opt->fast_threshold, opt->nonmax_ties_suppress, opt->cell_size, grid_n_cols, grid_occupancy ? d + o_occ : nullptr,
      reinterpret_cast<unsigned long long*>(d + o_cells));
  ctx->launches++;
  kt_end(ctx);
  SVO_CUDA_CHECK(ctx, cudaGetLastError());
  SVO_CUDA_CHECK(ctx, cudaMemcpyAsync(h + o_cells, d + o_cells, sizeof(unsigned long long) * n_cells, cudaMemcpyDeviceToHost, ctx->stream));
  SVO_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
  // corners with a high enough score, in cell order (:106-110).  A cell no corner beat still holds the initial
  // Corner(0, 0, detection_threshold, 0): it decodes to (0, 0), level 0, and passes the check whenever the float32
  // threshold rounded above the double one -- the reference then emits it too.
  int n = 0;
  for (int k = 0; k < n_cells; ++k) {
    const unsigned long long key = reinterpret_cast<const unsigned long long*>(h + o_cells)[k];
    const unsigned bits = (unsigned)(key >> 32);
    float score;
    std::memcpy(&score, &bits, 4);
    if (!((double)score > opt->detection_threshold)) continue;
    unsigned ord = 0xffffffffu - (unsigned)(key & 0xffffffffull);
    int L = 0;
    while (L + 1 < lv.n_levels && ord >= lv.order_base[L + 1]) ++L;
    ord -= lv.order_base[L];
    if (n < cap) {
      x_out[n] = (int)(ord % (unsigned)lv.w[L]) << L;
      y_out[n] = (int)(ord / (unsigned)lv.w[L]) << L;
      level_out[n] = L;
      if (score_out) score_out[n] = score;
    }
    ++n;
  }
  *n_out = n;
  return 0;
}
