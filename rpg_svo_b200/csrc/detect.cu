// rpg_svo_b200/csrc/detect.cu -- C ABI entry points
//   svo_b200_fast_detect          <- feature_detection::FastDetector::detect (svo/src/feature_detection.cpp:66-115)
//   svo_b200_fast_detect_streams  <- the same for S streams' keyframes in one launch (DepthFilter::initializeSeeds of
//                                    S filters, depth_filter.cpp:116-132); the single call is S = 1 of it
//
// "Next" row f4 of SURVEY.md 8f: the seed-initialisation detector that runs after DepthFilter::updateSeeds on keyframes
// (depth_filter.cpp:114-132).  The reference runs, per pyramid level, the `fast` library's segment test (FAST-10, b=20),
// its score bisection and 3x3 non-maximum suppression [EXT], then vk::shiTomasiScore [EXT] per surviving corner and keeps
// the best corner per 30-px grid cell across levels.  Here ONE launch covers all levels of all streams: a CTA owns a 32x8
// pixel tile of one level of one stream (+5 px halo in shared memory), evaluates the segment test with two 16-bit ring
// masks, scores the few corners in closed form (score = max over the 16 arcs of the minimum ring contrast, minus one =
// what the bisection converges to), suppresses non-maxima inside the tile (+1 halo of scores), computes the Shi-Tomasi
// score from the same tile and competes for its stream's grid cell with one 64-bit atomicMax on (score bits, reverse scan
// order) -- which reproduces the reference's "first strictly greater score in (level, row, column) order wins".  Integer
// work throughout; the only floating-point step (the eigenvalue formula) uses the oracle's operation order, so results
// are bit-identical.
#include <climits>
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
  int tile_base[SVO_B200_MAX_LEVELS + 1];  // first CTA of each level, then the CTA count, then INT_MAX
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

// One stream's detect call: its levels, options, occupancy grid (NULL = all cells free) and cell keys, in device memory.
struct DetectStream {
  DetectLevels lv;
  const uint8_t* occupancy;
  unsigned long long* cells;
  int b, ties_suppress, cell_size, grid_n_cols;
};

// CTA i of the launch is tile i - cta_offset[s] of stream s = stream_of(cta_offset, n_streams, i) (numbered across that
// stream's levels by lv.tile_base).
__global__ void __launch_bounds__(256) fast_detect_kernel(const DetectStream* __restrict__ streams,
                                                          const int* __restrict__ cta_offset, int n_streams) {
  __shared__ uint8_t img[kImgH][kImgW + 2];
  __shared__ int16_t sc[kScH][kScW];
  const int s_id = stream_of(cta_offset, n_streams, (int)blockIdx.x);
  const DetectStream& st = streams[s_id];
  const DetectLevels& lv = st.lv;
  const int b = st.b, ties_suppress = st.ties_suppress;
  const int tile = (int)blockIdx.x - __ldg(cta_offset + s_id);
  // the last level whose first tile is <= tile (tile_base is INT_MAX past the stream's levels): every tile base is read
  // at once, so that finding the level costs one round trip to the table rather than one per level
  int L = 0;
#pragma unroll
  for (int l = 1; l < SVO_B200_MAX_LEVELS; ++l) L += tile >= lv.tile_base[l] ? 1 : 0;
  const int t = tile - lv.tile_base[L];
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
  const int scale = 1 << L, cell_size = st.cell_size;
  const int k = ((gy * scale) / cell_size) * st.grid_n_cols + (gx * scale) / cell_size;  // :98-99
  const uint8_t* __restrict__ occupancy = st.occupancy;
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
  atomicMax(st.cells + k, key);
}

}  // namespace svo

using namespace svo;

namespace {

// The single call's argument checks (every stream's, for the streams call); nothing is written.
int detect_check(svo_b200_ctx* ctx, const svo_b200_detect_stream& a) {
  const svo_b200_detect_options* opt = a.opt;
  if (!ctx || !a.frame || !opt || !a.n_out || a.cap < 0 || (a.cap > 0 && (!a.x_out || !a.y_out || !a.level_out)))
    return set_err(ctx, SVO_B200_EINVAL, "fast_detect: bad arguments");
  if (opt->cell_size <= 0 || opt->n_pyr_levels <= 0 || opt->n_pyr_levels > a.frame->n_levels || opt->fast_threshold < 0 ||
      opt->fast_threshold > 254 || !(opt->detection_threshold >= 0.0))
    return set_err(ctx, SVO_B200_EINVAL, "fast_detect: bad options (cell_size %d, n_pyr_levels %d of %d, b %d, threshold %g)",
                   opt->cell_size, opt->n_pyr_levels, a.frame->n_levels, opt->fast_threshold, opt->detection_threshold);
  return 0;
}

// One checked call: its table entry (device pointers set at staging), its grid and its CTA count.
struct DetectCall {
  DetectStream t;
  int n_cells = 0, n_ctas = 0;
};

void detect_setup(const svo_b200_detect_stream& a, DetectCall& r) {
  const svo_b200_detect_options* opt = a.opt;
  const FrameDesc fd = make_desc(a.frame);
  const int grid_n_cols = (int)std::ceil((double)fd.w[0] / opt->cell_size), grid_n_rows = (int)std::ceil((double)fd.h[0] / opt->cell_size);
  r.n_cells = grid_n_cols * grid_n_rows;
  std::memset(&r.t, 0, sizeof(r.t));
  DetectLevels& lv = r.t.lv;
  lv.n_levels = opt->n_pyr_levels;
  unsigned order = 0;
  for (int L = 0; L < lv.n_levels; ++L) {
    lv.img[L] = fd.lvl[L]; lv.w[L] = fd.w[L]; lv.h[L] = fd.h[L];
    lv.tiles_x[L] = (fd.w[L] + kTileW - 1) / kTileW;
    lv.tile_base[L + 1] = lv.tile_base[L] + lv.tiles_x[L] * ((fd.h[L] + kTileH - 1) / kTileH);
    lv.order_base[L] = order;
    order += (unsigned)fd.w[L] * (unsigned)fd.h[L];
  }
  r.n_ctas = lv.tile_base[lv.n_levels];
  for (int L = lv.n_levels + 1; L <= SVO_B200_MAX_LEVELS; ++L) lv.tile_base[L] = INT_MAX;
  r.t.b = opt->fast_threshold;
  r.t.ties_suppress = opt->nonmax_ties_suppress;
  r.t.cell_size = opt->cell_size;
  r.t.grid_n_cols = grid_n_cols;
}

// A cell's initial key: Corner(0, 0, detection_threshold, 0) of the reference, the threshold stored as float (:72).
unsigned long long detect_init_key(double detection_threshold) {
  float thr_f = (float)detection_threshold;
  // -0.0 compares like +0.0, but its sign bit would make the initial key larger than every positive score's key
  if (thr_f == 0.0f) thr_f = 0.0f;
  unsigned thr_bits;
  std::memcpy(&thr_bits, &thr_f, 4);
  return ((unsigned long long)thr_bits << 32) | 0xffffffffull;
}

// Corners with a high enough score, in cell order (:106-110).  A cell no corner beat still holds the initial
// Corner(0, 0, detection_threshold, 0): it decodes to (0, 0), level 0, and passes the check whenever the float32
// threshold rounded above the double one -- the reference then emits it too.
void detect_decode(const unsigned long long* keys, const DetectCall& r, const svo_b200_detect_stream& a) {
  const DetectLevels& lv = r.t.lv;
  int n = 0;
  for (int k = 0; k < r.n_cells; ++k) {
    const unsigned long long key = keys[k];
    const unsigned bits = (unsigned)(key >> 32);
    float score;
    std::memcpy(&score, &bits, 4);
    if (!((double)score > a.opt->detection_threshold)) continue;
    unsigned ord = 0xffffffffu - (unsigned)(key & 0xffffffffull);
    int L = 0;
    while (L + 1 < lv.n_levels && ord >= lv.order_base[L + 1]) ++L;
    ord -= lv.order_base[L];
    if (n < a.cap) {
      a.x_out[n] = (int)(ord % (unsigned)lv.w[L]) << L;
      a.y_out[n] = (int)(ord / (unsigned)lv.w[L]) << L;
      a.level_out[n] = L;
      if (a.score_out) a.score_out[n] = score;
    }
    ++n;
  }
  *a.n_out = n;
}

// Every stream checked before anything is written; then one host-to-device copy (table, CTA offsets, initial cell keys,
// occupancy grids), one launch, one copy back of all cells, and each stream's decode into its own outputs.
int detect_run(svo_b200_ctx* ctx, int S, const svo_b200_detect_stream* streams, const char* name) {
  std::vector<DetectCall> calls((size_t)S);
  LaunchTable<DetectStream> tab;
  for (int s = 0; s < S; ++s) {
    if (const int rc = detect_check(ctx, streams[s])) return entry_err(ctx, rc, name, "stream", s);
    detect_setup(streams[s], calls[s]);
    tab.add(calls[s].t, calls[s].n_ctas, 1);
  }
  if (tab.over) return set_err(ctx, SVO_B200_ELIMIT, "fast_detect: %lld CTAs exceed one launch's grid", tab.ctas);
  if (S == 0) return 0;
  cudaSetDevice(ctx->device);
  Staging st(ctx);
  for (int s = 0; s < S; ++s) {
    if (streams[s].grid_occupancy) st.in(streams[s].grid_occupancy, calls[s].n_cells, &tab.jobs[s].occupancy, 1);
    st.inout<unsigned long long>(nullptr, calls[s].n_cells, &tab.jobs[s].cells, alignof(unsigned long long));  // initial keys in
  }
  tab.stage(st);
  int rc;
  if ((rc = st.open())) return rc;
  for (int s = 0; s < S; ++s) {
    const unsigned long long init = detect_init_key(streams[s].opt->detection_threshold);
    unsigned long long* keys = st.host(tab.jobs[s].cells);
    for (int k = 0; k < calls[s].n_cells; ++k) keys[k] = init;
  }
  if ((rc = st.send())) return rc;
  if (tab.ctas > 0 && (rc = launch_kernels(ctx, 1, [&] {
        fast_detect_kernel<<<(unsigned)tab.ctas, 256, 0, ctx->stream>>>(tab.jobs_at, tab.off_at, S);
      })))
    return rc;
  if ((rc = st.receive())) return rc;
  for (int s = 0; s < S; ++s) detect_decode(st.host(tab.jobs[s].cells), calls[s], streams[s]);
  return 0;
}

}  // namespace

extern "C" int svo_b200_fast_detect(svo_b200_ctx* ctx, const svo_b200_frame* frame, const svo_b200_detect_options* opt,
                                    const uint8_t* grid_occupancy, int cap, int* x_out, int* y_out, int* level_out,
                                    float* score_out, int* n_out) {
  const svo_b200_detect_stream a = {frame, opt, grid_occupancy, cap, x_out, y_out, level_out, score_out, n_out};
  return detect_run(ctx, 1, &a, nullptr);
}

extern "C" int svo_b200_fast_detect_streams(svo_b200_ctx* ctx, int S, const svo_b200_detect_stream* streams) {
  if (!ctx || S < 0 || (S > 0 && !streams))
    return set_err(ctx, SVO_B200_EINVAL, "fast_detect_streams: bad arguments (S %d)", S);
  return detect_run(ctx, S, streams, "fast_detect_streams");
}
