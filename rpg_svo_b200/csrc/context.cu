// rpg_svo_b200/csrc/context.cu -- context lifetime, frame (image pyramid) residency in HBM and the
// on-device pyramid build.  Replaces the image side of svo::Frame (svo/include/svo/frame.h:40-84,
// svo/src/frame.cpp:48-59,156-165).  The pyramid kernels' bodies are device functions shared by by-value launches (a single
// frame, a pool window) and table-driven launches over many frames of any sizes (svo_b200_frame_upload_streams; DESIGN.md
// section 4.5b), where a CTA finds its frame with stream_of.
#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <utility>
#include <vector>

#include "ctx.h"
#include "warp_align.cuh"

namespace svo {

int set_err(svo_b200_ctx* ctx, int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  if (ctx) ctx->err = buf;
  return code;
}

int ensure_dev(svo_b200_ctx* ctx, DevBuf& b, size_t bytes) {
  if (bytes <= b.cap) return 0;
  if (b.p) {
    SVO_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    cudaFree(b.p);
    b.p = nullptr;
    b.cap = 0;
  }
  size_t cap = bytes + bytes / 4 + 4096;
  SVO_CUDA_CHECK(ctx, cudaMalloc(&b.p, cap));
  b.cap = cap;
  return 0;
}

// [EXT] the constants vk::PinholeCamera / vk::ATANCamera derive in their constructors
int cam_to_dev(svo_b200_ctx* ctx, const svo_b200_camera* cam, CamDev& o) {
  memset(&o, 0, sizeof(o));
  if (!cam || cam->width <= 0 || cam->height <= 0 || cam->fx == 0.0 || cam->fy == 0.0)
    return set_err(ctx, SVO_B200_EINVAL, "camera: bad parameters");
  if (cam->model != SVO_B200_CAM_PINHOLE && cam->model != SVO_B200_CAM_ATAN)
    return set_err(ctx, SVO_B200_EINVAL, "camera: unknown model %d", cam->model);
  o.fx = cam->fx; o.fy = cam->fy; o.cx = cam->cx; o.cy = cam->cy;
  o.fx_inv = 1.0 / cam->fx; o.fy_inv = 1.0 / cam->fy;
  o.width = cam->width; o.height = cam->height;
  o.model = cam->model;
  for (int k = 0; k < 5; ++k) o.d[k] = cam->d[k];
  if (cam->model == SVO_B200_CAM_PINHOLE) {
    o.distorted = fabs(cam->d[0]) > 0.0000001;  // vk::PinholeCamera: distortion_(fabs(d0) > 0.0000001)
  } else {
    const double sv = cam->d[0];
    if (sv != 0.0) {  // vk::ATANCamera ctor
      o.tans = 2.0 * tan(sv / 2.0);
      o.tans_inv = 1.0 / o.tans;
      o.s_inv = 1.0 / sv;
      o.distorted = 1;
    }
  }
  return 0;
}

// svo::Frame refuses an image whose size is not its camera's (svo/src/frame.cpp:51), and the kernels bound their image reads
// by the camera's size: a camera whose size is not the level-0 size of each of the n frames is refused (NULL entries are the
// caller's to check).
int cam_check_frames(svo_b200_ctx* ctx, const char* who, const svo_b200_camera* cam, const svo_b200_frame* const* frames, int n) {
  for (int i = 0; i < n; ++i)
    if (frames[i] && (frames[i]->width != cam->width || frames[i]->height != cam->height))
      return set_err(ctx, SVO_B200_EINVAL, "%s: camera %dx%d, frame %dx%d", who, cam->width, cam->height, frames[i]->width,
                     frames[i]->height);
  return 0;
}

static int ensure_host(svo_b200_ctx* ctx, HostBuf& b, size_t bytes) {
  if (bytes <= b.cap) return 0;
  if (b.p) {
    SVO_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    cudaFreeHost(b.p);
    b.p = nullptr;
    b.cap = 0;
  }
  size_t cap = bytes + bytes / 4 + 4096;
  SVO_CUDA_CHECK(ctx, cudaMallocHost(&b.p, cap));
  b.cap = cap;
  return 0;
}

int Staging::open() {
  if (!hbuf_)
    for (const Region& r : regions_)
      if (r.back) return set_err(ctx_, SVO_B200_EINVAL, "Staging: a pageable staging copies nothing back");
  Carver c;
  const auto lay = [&](bool in, bool back) {
    for (Region& r : regions_)
      if (r.in == in && r.back == back) r.off = c.take(r.bytes, r.align);
  };
  lay(true, false);
  front_ = c.off;
  back_ = c.take(0);
  lay(true, true);
  if (c.off > back_) front_ = c.off;
  lay(false, true);
  end_ = c.off;
  int rc;
  if (hbuf_ && (rc = ensure_host(ctx_, *hbuf_, end_))) return rc;
  if ((rc = ensure_dev(ctx_, *dbuf_, end_))) return rc;
  if (hbuf_) {
    SVO_CUDA_CHECK(ctx_, cudaStreamSynchronize(ctx_->stream));
    h_ = static_cast<uint8_t*>(hbuf_->p);
  } else {
    page_.resize(end_);
    h_ = page_.data();
  }
  d_ = static_cast<uint8_t*>(dbuf_->p);
  for (const Region& r : regions_) r.bind(r.at, d_ + r.off);
  for (const Region& r : regions_)
    if (r.in && r.src && r.bytes) memcpy(h_ + r.off, r.src, r.bytes);
  return 0;
}

int Staging::send() {
  SVO_CUDA_CHECK(ctx_, cudaMemcpyAsync(d_, h_, front_, cudaMemcpyHostToDevice, ctx_->stream));
  return 0;
}

int Staging::receive() {
  SVO_CUDA_CHECK(ctx_, cudaMemcpyAsync(h_ + back_, d_ + back_, end_ - back_, cudaMemcpyDeviceToHost, ctx_->stream));
  SVO_CUDA_CHECK(ctx_, cudaStreamSynchronize(ctx_->stream));
  for (const Region& r : regions_)
    if (r.back && r.dst && r.bytes) memcpy(r.dst, h_ + r.off, r.bytes);
  return 0;
}

int entry_err(svo_b200_ctx* ctx, int rc, const char* name, const char* what, int i) {
  if (!ctx || !name) return rc;
  const std::string why = ctx->err;
  return set_err(ctx, rc, "%s: %s %d: %s", name, what, i, why.c_str());
}

int check_ref_levels(svo_b200_ctx* ctx, const char* who, const char* level_name, const svo_b200_frame* const* ref_frames,
                     int n_ref, int M, const int* ref_index, const int* level) {
  for (int m = 0; m < M; ++m) {
    if (ref_index[m] < 0 || ref_index[m] >= n_ref) return set_err(ctx, SVO_B200_EINVAL, "%s: ref_index[%d] out of range", who, m);
    if (level[m] < 0 || level[m] >= ref_frames[ref_index[m]]->n_levels)
      return set_err(ctx, SVO_B200_EINVAL, "%s: %s[%d] outside the pyramid", who, level_name, m);
  }
  return 0;
}

int check_ref_table(svo_b200_ctx* ctx, const char* who, const char* level_name, const svo_b200_frame* const* ref_frames,
                    int n_ref, int M, const int* ref_index, const int* level, const svo_b200_frame* cur,
                    const svo_b200_camera* cam, int max_search_level) {
  if (const int rc = check_ref_levels(ctx, who, level_name, ref_frames, n_ref, M, ref_index, level)) return rc;
  if (max_search_level >= cur->n_levels)
    return set_err(ctx, SVO_B200_EINVAL, "%s: max_search_level %d >= %d pyramid levels", who, max_search_level, cur->n_levels);
  if (const int rc = cam_check_frames(ctx, who, cam, &cur, 1)) return rc;
  return cam_check_frames(ctx, who, cam, ref_frames, n_ref);
}

// [EXT] vk::halfSample (svo/src/frame.cpp:156-165), both branches of rpg_vikit's vision.cpp:
//   scalar: out = (a + b + c + d) / 4, integer division;
//   SSE2 (what an x86 build runs when in_w % 16 == 0): vertical _mm_avg_epu8, then _mm_avg_epu16 of adjacent columns,
//          i.e. avg(avg(a, c), avg(b, d)) with round-half-up at both steps.
// Packed forms on 32-bit words holding four consecutive pixels of the top / bottom row: the two results come back in
// bytes 0 and 2.
__device__ __forceinline__ uint32_t half2_scalar(uint32_t top, uint32_t bot) {
  const uint32_t s = (top & 0x00ff00ffu) + ((top >> 8) & 0x00ff00ffu) + (bot & 0x00ff00ffu) + ((bot >> 8) & 0x00ff00ffu);
  return (s >> 2) & 0x00ff00ffu;
}
__device__ __forceinline__ uint32_t half2_avg(uint32_t top, uint32_t bot) {
  const uint32_t v = __vavgu4(top, bot);          // per byte (a + c + 1) >> 1
  return __vavgu4(v, v >> 8) & 0x00ff00ffu;       // bytes 0, 2: (v0 + v1 + 1) >> 1, (v2 + v3 + 1) >> 1
}
__device__ __forceinline__ uint32_t half2(uint32_t top, uint32_t bot, bool avg) {
  return avg ? half2_avg(top, bot) : half2_scalar(top, bot);
}
__device__ __forceinline__ uint32_t half1(uint32_t a, uint32_t b, uint32_t c, uint32_t d, bool avg) {  // one output pixel
  return avg ? ((((a + c + 1u) >> 1) + ((b + d + 1u) >> 1) + 1u) >> 1) : ((a + b + c + d) >> 2);
}

// Fused pyramid build for a batch of frames laid out with a constant stride: one CTA turns a
// 128x16 tile of level 0 into the matching 64x8 / 32x4 / 16x2 / 8x1 tiles of levels 1..4 (as many as
// the frame has), reading level 0 from HBM exactly once.  Every level is the halfSample of the one
// above it, so a deeper pyramid is built by further passes starting from the last level built.
// The kernel also writes the block-tiled copies (ctx.h) of the levels it reads or produces: whole 4x4 blocks from the
// level-0 .. level-2 tiles, and the rows of level 3 / 4 blocks that fall into this tile.
struct PyrGeom {
  int w[SVO_B200_MAX_LEVELS], h[SVO_B200_MAX_LEVELS];
  uint8_t* slab[SVO_B200_MAX_LEVELS];            // level l of frame i at slab[l] + i*stride[l]
  unsigned long long stride[SVO_B200_MAX_LEVELS];
  uint8_t* tslab[SVO_B200_MAX_LEVELS];           // tiled copy of level l of frame i at tslab[l] + i*tstride[l]
  unsigned long long tstride[SVO_B200_MAX_LEVELS];
  int n_levels;
  int tiles_x;
  unsigned avg_mask;  // bit l: level l is produced with the SSE2 rounding (avg of avg) instead of (a+b+c+d)/4
};
// Row word `w` of a block whose first column is x, of row y of a W x H level: pixels outside the level zeroed.
__device__ __forceinline__ uint32_t tile_word(uint32_t w, int x, int y, int W, int H) {
  if (y >= H || x >= W) return 0u;
  return W - x >= 4 ? w : w & ((1u << (8 * (W - x))) - 1u);
}
// Rows r0..r0+n-1 (n = 1, 2 or 4) of block (bx, by) of the tiled copy of a W x H level from a shared tile `t` (pitch P, the
// block's first column at c0 of tile row tr0): the words of rows r0.. are stored at word r0 of the block.  Blocks outside
// the copy are skipped.
template <int N>
__device__ __forceinline__ void put_block_rows(uint8_t* tiled, int W, int H, int bx, int by, int r0, const uint8_t* t, int P,
                                               int tr0, int c0) {
  if (bx >= (W + 3) / 4 || by >= (H + 3) / 4) return;
  uint32_t w[N];
#pragma unroll
  for (int r = 0; r < N; ++r)
    w[r] = tile_word(*reinterpret_cast<const uint32_t*>(t + (tr0 + r) * P + c0), 4 * bx, 4 * by + r0 + r, W, H);
  uint8_t* dst = tiled + ((size_t)by * ((W + 3) / 4) + bx) * 16 + 4 * r0;
  if constexpr (N == 4) *reinterpret_cast<uint4*>(dst) = make_uint4(w[0], w[1], w[2], w[3]);
  else if constexpr (N == 2) *reinterpret_cast<uint2*>(dst) = make_uint2(w[0], w[1]);
  else *reinterpret_cast<uint32_t*>(dst) = w[0];
}
// Tile (tx, ty) of frame fi of g, by one CTA of 128 threads.
__device__ __forceinline__ void pyramid_fused_tile(const PyrGeom& g, size_t fi, int tx, int ty) {
  __shared__ __align__(16) uint8_t t0[16][128];
  __shared__ __align__(16) uint8_t t1[8][64];
  __shared__ __align__(16) uint8_t t2[4][32];
  __shared__ __align__(16) uint8_t t3[2][16];
  __shared__ __align__(16) uint8_t t4[1][8];
  const int t = threadIdx.x;
  const int W0 = g.w[0], H0 = g.h[0];
  auto tiled = [&](int l) { return g.tslab[l] + fi * g.tstride[l]; };
  {  // level-0 tile -> shared (16 B per thread)
    const int r = t >> 3, c = (t & 7) * 16;
    const int y = ty * 16 + r, x = tx * 128 + c;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (y < H0) {
      const uint8_t* src = g.slab[0] + fi * g.stride[0] + (size_t)y * W0 + x;
      if (x + 16 <= W0 && ((W0 & 15) == 0)) {
        v = *reinterpret_cast<const uint4*>(src);
      } else {
        uint8_t tmp[16];
#pragma unroll
        for (int k = 0; k < 16; ++k) tmp[k] = (x + k < W0) ? src[k] : 0;
        v = *reinterpret_cast<uint4*>(tmp);
      }
    }
    *reinterpret_cast<uint4*>(&t0[r][c]) = v;
  }
  __syncthreads();
  // level 0 tiled: 4 x 32 blocks, one per thread
  put_block_rows<4>(tiled(0), W0, H0, tx * 32 + (t & 31), ty * 4 + (t >> 5), 0, &t0[0][0], 128, 4 * (t >> 5), 4 * (t & 31));
  if (g.n_levels > 1) {  // level 1: 8 x 64, four pixels per thread
    const int r = t >> 4, c = (t & 15) * 4;
    const uint2 a = *reinterpret_cast<const uint2*>(&t0[2 * r][2 * c]);
    const uint2 b = *reinterpret_cast<const uint2*>(&t0[2 * r + 1][2 * c]);
    const bool avg = (g.avg_mask >> 1) & 1u;
    const uint32_t q0 = half2(a.x, b.x, avg), q1 = half2(a.y, b.y, avg);
    const uint32_t o = (q0 & 0xffu) | ((q0 >> 8) & 0xff00u) | ((q1 & 0xffu) << 16) | ((q1 << 8) & 0xff000000u);
    *reinterpret_cast<uint32_t*>(&t1[r][c]) = o;
    const int y = ty * 8 + r, x = tx * 64 + c, W1 = g.w[1];
    if (y < g.h[1]) {
      uint8_t* dst = g.slab[1] + fi * g.stride[1] + (size_t)y * W1 + x;
      if (x + 4 <= W1 && ((W1 & 3) == 0)) *reinterpret_cast<uint32_t*>(dst) = o;
      else
        for (int k = 0; k < 4; ++k)
          if (x + k < W1) dst[k] = (uint8_t)(o >> (8 * k));
    }
  }
  __syncthreads();
  if (g.n_levels > 1 && t < 32)  // level 1 tiled: 2 x 16 blocks
    put_block_rows<4>(tiled(1), g.w[1], g.h[1], tx * 16 + (t & 15), ty * 2 + (t >> 4), 0, &t1[0][0], 64, 4 * (t >> 4), 4 * (t & 15));
  if (g.n_levels > 2) {  // level 2: 4 x 32
    const int r = t >> 5, c = t & 31;
    const uint8_t o = (uint8_t)half1(t1[2 * r][2 * c], t1[2 * r][2 * c + 1], t1[2 * r + 1][2 * c], t1[2 * r + 1][2 * c + 1],
                                     (g.avg_mask >> 2) & 1u);
    t2[r][c] = o;
    const int y = ty * 4 + r, x = tx * 32 + c;
    if (y < g.h[2] && x < g.w[2]) g.slab[2][fi * g.stride[2] + (size_t)y * g.w[2] + x] = o;
  }
  __syncthreads();
  if (g.n_levels > 2 && t < 8)  // level 2 tiled: 1 x 8 blocks
    put_block_rows<4>(tiled(2), g.w[2], g.h[2], tx * 8 + t, ty, 0, &t2[0][0], 32, 0, 4 * t);
  if (g.n_levels > 3 && t < 32) {  // level 3: 2 x 16
    const int r = t >> 4, c = t & 15;
    const uint8_t o = (uint8_t)half1(t2[2 * r][2 * c], t2[2 * r][2 * c + 1], t2[2 * r + 1][2 * c], t2[2 * r + 1][2 * c + 1],
                                     (g.avg_mask >> 3) & 1u);
    t3[r][c] = o;
    const int y = ty * 2 + r, x = tx * 16 + c;
    if (y < g.h[3] && x < g.w[3]) g.slab[3][fi * g.stride[3] + (size_t)y * g.w[3] + x] = o;
  }
  __syncthreads();
  if (g.n_levels > 3 && t < 4)  // level 3 tiled: rows 2ty, 2ty+1 of 4 blocks
    put_block_rows<2>(tiled(3), g.w[3], g.h[3], tx * 4 + t, ty >> 1, 2 * (ty & 1), &t3[0][0], 16, 0, 4 * t);
  if (g.n_levels > 4 && t < 8) {  // level 4: 1 x 8
    const int y = ty, x = tx * 8 + t;
    const uint8_t o = (uint8_t)half1(t3[0][2 * t], t3[0][2 * t + 1], t3[1][2 * t], t3[1][2 * t + 1], (g.avg_mask >> 4) & 1u);
    t4[0][t] = o;
    if (y < g.h[4] && x < g.w[4]) g.slab[4][fi * g.stride[4] + (size_t)y * g.w[4] + x] = o;
  }
  __syncthreads();
  if (g.n_levels > 4 && t < 2)  // level 4 tiled: row ty of 2 blocks
    put_block_rows<1>(tiled(4), g.w[4], g.h[4], tx * 2 + t, ty >> 2, ty & 3, &t4[0][0], 8, 0, 4 * t);
}
// Frames [first, first + gridDim.y) of one pool window, g by value.
__global__ void __launch_bounds__(128) pyramid_fused_kernel(int first, PyrGeom g) {
  pyramid_fused_tile(g, (size_t)(first + blockIdx.y), blockIdx.x % g.tiles_x, blockIdx.x / g.tiles_x);
}
// One frame per entry of `geoms` (level pointers of the frame itself, strides unused): CTA i is tile i - cta_offset[e] of
// entry e = stream_of(cta_offset, n, i).
__global__ void __launch_bounds__(128) pyramid_fused_table_kernel(const PyrGeom* __restrict__ geoms, const int* __restrict__ cta_offset,
                                                                  int n) {
  const int e = stream_of(cta_offset, n, (int)blockIdx.x);
  const PyrGeom& g = geoms[e];
  const int t = (int)blockIdx.x - __ldg(cta_offset + e);
  pyramid_fused_tile(g, 0, t % g.tiles_x, t / g.tiles_x);
}


// Level 0 -> level 1 for a batch of frames as a pure streaming kernel: 94 % of the pyramid's bytes move
// here, so it is written against the HBM roofline -- a persistent grid (a few CTAs per SM), each work
// item = 16 level-0 pixels of two consecutive rows (2 x 128-bit loads) -> 8 level-1 pixels (one 64-bit
// store), plus those two rows of the four level-0 blocks they cover in the tiled copy t0 (four 64-bit stores).
// The 2x2 reductions are formed SIMD-in-register (scalar rule: two 16-bit lanes per word; SSE2 rule: two __vavgu4).  An
// odd last level-0 row is tiled alone.  Requires W0 % 16 == 0.
// Item (y, ix) of one frame: l0, l1 and t0 point at the frame's level 0, level 1 and tiled level 0.
__device__ __forceinline__ void pyramid_l0_l1_item(const uint8_t* __restrict__ l0, uint8_t* __restrict__ l1, uint8_t* __restrict__ t0,
                                                   int W0, int H0, int y, int ix, int avg) {
  const int W1 = W0 >> 1, H1 = H0 >> 1, BW0 = W0 >> 2;
  const uint8_t* src = l0 + (size_t)(2 * y) * W0 + 16 * ix;
  const uint4 a = __ldg(reinterpret_cast<const uint4*>(src));
  const uint4 b = y < H1 ? __ldg(reinterpret_cast<const uint4*>(src + W0)) : make_uint4(0u, 0u, 0u, 0u);
  const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, bw[4] = {b.x, b.y, b.z, b.w};
  uint2* tl = reinterpret_cast<uint2*>(t0 + ((size_t)(y >> 1) * BW0 + 4 * ix) * 16 + 8 * (y & 1));
#pragma unroll
  for (int k = 0; k < 4; ++k) tl[2 * k] = make_uint2(aw[k], bw[k]);
  if (y >= H1) return;
  uint32_t o[2] = {0u, 0u};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const uint32_t q = half2(aw[k], bw[k], avg != 0);        // two results, bytes 0 and 2
    const uint32_t two = (q & 0xffu) | ((q >> 8) & 0xff00u);  // packed into the low 16 bits
    o[k >> 1] |= two << (16 * (k & 1));
  }
  *reinterpret_cast<uint2*>(l1 + (size_t)y * W1 + 8 * ix) = make_uint2(o[0], o[1]);
}
__global__ void __launch_bounds__(256) pyramid_l0_l1_stream_kernel(const uint8_t* __restrict__ l0, size_t stride0,
                                                                   uint8_t* __restrict__ l1, size_t stride1,
                                                                   uint8_t* __restrict__ t0, size_t tstride0, int first,
                                                                   int count, int W0, int H0, int avg) {
  const int items_x = W0 >> 4;
  const long long per_frame = (long long)items_x * ((H0 + 1) >> 1), total = per_frame * count;
  for (long long it = (long long)blockIdx.x * blockDim.x + threadIdx.x; it < total; it += (long long)gridDim.x * blockDim.x) {
    const int fr = (int)(it / per_frame);
    const int rem = (int)(it - (long long)fr * per_frame);
    const int y = rem / items_x, ix = rem - y * items_x;
    const size_t f = (size_t)(first + fr);
    pyramid_l0_l1_item(l0 + f * stride0, l1 + f * stride1, t0 + f * tstride0, W0, H0, y, ix, avg);
  }
}

// One frame's level (src, w x h) and its tiled copy, or (the streaming kernel) its level 0 (src), level 1 (dst) and tiled
// level 0, with the rounding of level 1 (avg): an entry of the table-driven streaming and tiling launches.
struct PyrJob {
  const uint8_t* src;
  uint8_t* dst;
  uint8_t* tiled;
  int w, h, avg;
};
// the streaming kernel over one frame per job: CTA i holds items (i - cta_offset[j]) * 256 ... of job j = stream_of(..., i)
__global__ void __launch_bounds__(256) pyramid_l0_l1_table_kernel(const PyrJob* __restrict__ jobs, const int* __restrict__ cta_offset,
                                                                  int n) {
  const int j = stream_of(cta_offset, n, (int)blockIdx.x);
  const PyrJob& jb = jobs[j];
  const int items_x = jb.w >> 4;
  const int i = ((int)blockIdx.x - __ldg(cta_offset + j)) * 256 + (int)threadIdx.x;
  if (i >= items_x * ((jb.h + 1) >> 1)) return;
  const int y = i / items_x, ix = i - y * items_x;
  pyramid_l0_l1_item(jb.src, jb.dst, jb.tiled, jb.w, jb.h, y, ix, jb.avg);
}

// Block-tiled copy of levels [first_level, first_level + gridDim.y) of `count` frames, level l of frame i at lvl[l] +
// i * stride[l], its copy at tl[l] + i * tstride[l]: one thread per 4x4 block, zero outside the level.  Tiles the levels no
// pyramid kernel tiles: levels uploaded from the host below the first fused pass, and the streaming kernel's level 1 of a
// two-level pyramid.
struct TileGeom {
  uint8_t* lvl[SVO_B200_MAX_LEVELS];
  unsigned long long stride[SVO_B200_MAX_LEVELS];
  uint8_t* tl[SVO_B200_MAX_LEVELS];
  unsigned long long tstride[SVO_B200_MAX_LEVELS];
  int w[SVO_B200_MAX_LEVELS], h[SVO_B200_MAX_LEVELS];
};
// Block b of the W x H level at src into its tiled copy at tiled.
__device__ __forceinline__ void tile_block(const uint8_t* src, int W, int H, uint8_t* tiled, int b) {
  const int BW = (W + 3) >> 2;
  const int by = b / BW, bx = b - by * BW;
  uint32_t w[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int y = 4 * by + r, x = 4 * bx;
    w[r] = 0u;
    if (y < H) {
      const uint8_t* p = src + (size_t)y * W + x;
      if ((W & 3) == 0) {
        w[r] = *reinterpret_cast<const uint32_t*>(p);
      } else {
        for (int k = 0; k < 4 && x + k < W; ++k) w[r] |= (uint32_t)p[k] << (8 * k);
      }
    }
  }
  reinterpret_cast<uint4*>(tiled)[b] = make_uint4(w[0], w[1], w[2], w[3]);
}
__global__ void __launch_bounds__(256) tile_levels_kernel(TileGeom g, int first_level, int count) {
  const int l = first_level + (int)blockIdx.y;
  const int W = g.w[l], H = g.h[l], BW = (W + 3) >> 2;
  const long long per_frame = (long long)BW * ((H + 3) >> 2), total = per_frame * count;
  for (long long it = (long long)blockIdx.x * blockDim.x + threadIdx.x; it < total; it += (long long)gridDim.x * blockDim.x) {
    const int fr = (int)(it / per_frame);
    const int b = (int)(it - (long long)fr * per_frame);
    tile_block(g.lvl[l] + (size_t)fr * g.stride[l], W, H, g.tl[l] + (size_t)fr * g.tstride[l], b);
  }
}
// one level of one frame per job: CTA i holds blocks (i - cta_offset[j]) * 256 ... of job j = stream_of(..., i)
__global__ void __launch_bounds__(256) tile_levels_table_kernel(const PyrJob* __restrict__ jobs, const int* __restrict__ cta_offset,
                                                                int n) {
  const int j = stream_of(cta_offset, n, (int)blockIdx.x);
  const PyrJob& jb = jobs[j];
  const int b = ((int)blockIdx.x - __ldg(cta_offset + j)) * 256 + (int)threadIdx.x;
  if (b >= ((jb.w + 3) >> 2) * ((jb.h + 3) >> 2)) return;
  tile_block(jb.src, jb.w, jb.h, jb.tiled, b);
}

// The tile_levels_kernel launch over levels [from, to) of frames [first, first + count) of `pool`
static void tile_levels(svo_b200_ctx* ctx, const svo_b200_frame_pool* pool, int first, int count, int from, int to) {
  const svo_b200_frame& f = pool->frames[first];
  TileGeom g;
  memset(&g, 0, sizeof(g));
  for (int l = from; l < to; ++l) {
    g.lvl[l] = f.lv[l]; g.stride[l] = pool->stride[l]; g.tl[l] = f.tv[l]; g.tstride[l] = pool->tstride[l];
    g.w[l] = f.w[l]; g.h[l] = f.h[l];
  }
  const long long n = (long long)((f.w[from] + 3) / 4) * ((f.h[from] + 3) / 4) * count;  // blocks of the largest level
  long long blocks = (n + 255) / 256;
  if (blocks > ctx->sm_count * 8LL) blocks = ctx->sm_count * 8LL;
  tile_levels_kernel<<<dim3((unsigned)blocks, (unsigned)(to - from)), 256, 0, ctx->stream>>>(g, from, count);
}

// does producing a level from a source level of width `src_w` use vikit's SSE2 rounding?  (x86 rule: width % 16 == 0;
// cv::Mat buffers are always 16-byte aligned)
static inline int pyr_avg(const svo_b200_ctx* ctx, int src_w) {
  return ctx->pyramid_rule == SVO_B200_PYR_X86 && (src_w % 16) == 0;
}

// The fused pass of frame f (and, with strides, of the frames that follow it in its pool) whose level 0 is level `top`.
static PyrGeom pass_geom(const svo_b200_ctx* ctx, const svo_b200_frame& f, int top, const size_t* stride, const size_t* tstride) {
  PyrGeom g;
  memset(&g, 0, sizeof(g));
  g.n_levels = f.n_levels - top < 5 ? f.n_levels - top : 5;
  for (int l = 0; l < g.n_levels; ++l) {
    g.w[l] = f.w[top + l]; g.h[l] = f.h[top + l]; g.slab[l] = f.lv[top + l]; g.tslab[l] = f.tv[top + l];
    if (stride) { g.stride[l] = stride[top + l]; g.tstride[l] = tstride[top + l]; }
    if (l && pyr_avg(ctx, g.w[l - 1])) g.avg_mask |= 1u << l;
  }
  g.tiles_x = (g.w[0] + 127) / 128;
  return g;
}

// The stages of a level-0 upload of frame f: whether the streaming kernel builds level 1, the levels [tile_from, tile_to)
// that only the tiling kernel copies, and the level 0 of the first fused pass (passes follow every 4 levels while
// top + 1 < n_levels).
struct UploadPlan {
  bool l0_l1;
  int tile_from, tile_to, top;
};
static UploadPlan upload_plan(const svo_b200_frame& f, int n_given) {
  UploadPlan p;
  p.l0_l1 = n_given == 1 && f.n_levels > 1 && f.w[0] % 16 == 0;
  p.top = p.l0_l1 ? 1 : n_given - 1;  // the highest level built; levels [tile_from, ..) lack a pyramid kernel's copy
  p.tile_from = p.l0_l1 ? 1 : 0;
  p.tile_to = p.top + 1 < f.n_levels ? p.top : f.n_levels;
  return p;
}

// The missing levels and the tiled copies of every level of frames [first, first + count) of `pool`, whose levels
// [0, n_given) are on the device.  Level 0 -> 1 with the streaming kernel when only level 0 is given and the width allows
// 128-bit rows, then passes of the fused kernel over the whole window, each from the highest level built so far to up to
// four levels further.
static int build_pyramid(svo_b200_ctx* ctx, const svo_b200_frame_pool* pool, int first, int count, int n_given) {
  const svo_b200_frame& f0 = pool->frames[0];
  const int n_levels = f0.n_levels;
  const UploadPlan p = upload_plan(f0, n_given);
  const int passes = (n_levels + 2 - p.top) / 4;  // top = p.top, p.top + 4, ... while top + 1 < n_levels
  const int chunks = (count + 32767) / 32768;     // gridDim.y limit 65535
  return launch_kernels(ctx, p.l0_l1 + (p.tile_from < p.tile_to) + passes * chunks, [&] {
    if (p.l0_l1)
      pyramid_l0_l1_stream_kernel<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(pool->slab[0], pool->stride[0], pool->slab[1],
                                                                              pool->stride[1], pool->tslab[0], pool->tstride[0],
                                                                              first, count, f0.w[0], f0.h[0], pyr_avg(ctx, f0.w[0]));
    if (p.tile_from < p.tile_to) tile_levels(ctx, pool, first, count, p.tile_from, p.tile_to);
    for (int top = p.top; top + 1 < n_levels; top += 4) {  // the fused kernel's level 0 = our level `top`
      const PyrGeom g = pass_geom(ctx, f0, top, pool->stride, pool->tstride);
      const int tiles_y = (g.h[0] + 15) / 16;
      for (int done = 0; done < count; done += 32768) {
        const int n = count - done < 32768 ? count - done : 32768;
        pyramid_fused_kernel<<<dim3(g.tiles_x * tiles_y, n), 128, 0, ctx->stream>>>(first + done, g);
      }
    }
  });
}

// svo_b200_frame_upload(ctx, entries[s].frame, &entries[s].level0, 1) of every entry, with one launch per stage: every
// entry is checked before anything is copied or launched; then each level 0 is copied into its frame, the tables of every
// launch go to the device in one copy, and one streaming launch, one tiling launch and one fused launch per pass serve
// all entries that have the stage.
static int upload_streams(svo_b200_ctx* ctx, int S, const svo_b200_frame_upload_entry* entries) {
  static const char* who = "frame_upload_streams";
  std::vector<std::pair<const svo_b200_frame*, int>> seen((size_t)S);
  for (int s = 0; s < S; ++s) {
    if (!entries[s].frame || !entries[s].level0) return set_err(ctx, SVO_B200_EINVAL, "%s: entry %d: NULL frame or image", who, s);
    seen[s] = {entries[s].frame, s};
  }
  std::sort(seen.begin(), seen.end());
  for (size_t k = 1; k < seen.size(); ++k)
    if (seen[k].first == seen[k - 1].first)
      return set_err(ctx, SVO_B200_EINVAL, "%s: entries %d and %d name one frame", who, std::min(seen[k - 1].second, seen[k].second),
                     std::max(seen[k - 1].second, seen[k].second));
  LaunchTable<PyrJob> l0_l1, tile;
  std::vector<LaunchTable<PyrGeom>> passes;
  for (int s = 0; s < S; ++s) {
    const svo_b200_frame& f = *entries[s].frame;
    const UploadPlan p = upload_plan(f, 1);
    if (p.l0_l1)
      l0_l1.add(PyrJob{f.lv[0], f.lv[1], f.tv[0], f.w[0], f.h[0], pyr_avg(ctx, f.w[0])}, (long long)(f.w[0] >> 4) * ((f.h[0] + 1) >> 1),
                256);
    for (int l = p.tile_from; l < p.tile_to; ++l)
      tile.add(PyrJob{f.lv[l], nullptr, f.tv[l], f.w[l], f.h[l], 0}, (long long)((f.w[l] + 3) >> 2) * ((f.h[l] + 3) >> 2), 256);
    size_t k = 0;
    for (int top = p.top; top + 1 < f.n_levels; top += 4, ++k) {
      if (k == passes.size()) passes.emplace_back();
      const PyrGeom g = pass_geom(ctx, f, top, nullptr, nullptr);
      passes[k].add(g, (long long)g.tiles_x * ((g.h[0] + 15) / 16), 1);
    }
  }
  bool over = l0_l1.over || tile.over;
  for (const auto& t : passes) over = over || t.over;
  if (over) return set_err(ctx, SVO_B200_ELIMIT, "%s: a launch's work exceeds one grid", who);
  if (S == 0) return 0;
  Staging st(ctx, Staging::Pageable{});
  l0_l1.stage(st);
  tile.stage(st);
  for (auto& t : passes) t.stage(st);
  cudaSetDevice(ctx->device);
  int rc;
  if ((rc = st.open())) return rc;
  for (int s = 0; s < S; ++s) {
    const svo_b200_frame& f = *entries[s].frame;
    SVO_CUDA_CHECK(ctx, cudaMemcpyAsync(f.lv[0], entries[s].level0, (size_t)f.w[0] * f.h[0], cudaMemcpyHostToDevice, ctx->stream));
  }
  if ((rc = st.send())) return rc;
  return launch_kernels(ctx, (l0_l1.n() > 0) + (tile.n() > 0) + (int)passes.size(), [&] {
    if (l0_l1.n()) pyramid_l0_l1_table_kernel<<<(unsigned)l0_l1.ctas, 256, 0, ctx->stream>>>(l0_l1.jobs_at, l0_l1.off_at, l0_l1.n());
    if (tile.n()) tile_levels_table_kernel<<<(unsigned)tile.ctas, 256, 0, ctx->stream>>>(tile.jobs_at, tile.off_at, tile.n());
    for (const auto& t : passes) pyramid_fused_table_kernel<<<(unsigned)t.ctas, 128, 0, ctx->stream>>>(t.jobs_at, t.off_at, t.n());
  });
}

// A zeroed pool of `count` frames of one geometry (arguments checked by the caller); `who` prefixes the error messages.
static int pool_create(svo_b200_ctx* ctx, const char* who, int width, int height, int n_levels, int count,
                       svo_b200_frame_pool** pool_out) {
  cudaSetDevice(ctx->device);
  svo_b200_frame proto;
  proto.width = width; proto.height = height; proto.n_levels = n_levels;
  svo_b200_frame_pool* pool = new svo_b200_frame_pool();
  pool->count = count;
  pool->n_levels = n_levels;
  size_t total = 0, slab_off[SVO_B200_MAX_LEVELS];
  for (int l = 0; l < n_levels; ++l) {
    proto.w[l] = l ? proto.w[l - 1] / 2 : width;
    proto.h[l] = l ? proto.h[l - 1] / 2 : height;
    if (proto.w[l] <= 0 || proto.h[l] <= 0) {
      delete pool;
      return set_err(ctx, SVO_B200_EINVAL, "%s: level %d is empty", who, l);
    }
    pool->stride[l] = ((size_t)proto.w[l] * proto.h[l] + 255) / 256 * 256;
    slab_off[l] = total;
    total += pool->stride[l] * (size_t)count + 256;  // slack: kernels fetch aligned words around footprints
  }
  size_t tslab_off[SVO_B200_MAX_LEVELS];
  for (int l = 0; l < n_levels; ++l) {
    pool->tstride[l] = (tiled_bytes(proto.w[l], proto.h[l]) + 255) / 256 * 256;
    tslab_off[l] = total;
    total += pool->tstride[l] * (size_t)count;
  }
  cudaError_t e = cudaMalloc((void**)&pool->mem, total);
  if (e != cudaSuccess) {
    delete pool;
    return set_err(ctx, SVO_B200_ENOMEM, "%s: cudaMalloc(%zu): %s", who, total, cudaGetErrorString(e));
  }
  ctx->sia_chain = false;
  cudaMemsetAsync(pool->mem, 0, total, ctx->stream);
  for (int l = 0; l < n_levels; ++l) {
    pool->slab[l] = pool->mem + slab_off[l];
    pool->tslab[l] = pool->mem + tslab_off[l];
  }
  proto.pool = pool;
  pool->frames.assign(count, proto);
  for (int i = 0; i < count; ++i) {
    pool->frames[i].index = i;
    for (int l = 0; l < n_levels; ++l) {
      pool->frames[i].lv[l] = pool->slab[l] + (size_t)i * pool->stride[l];
      pool->frames[i].tv[l] = pool->tslab[l] + (size_t)i * pool->tstride[l];
    }
  }
  *pool_out = pool;
  return 0;
}

}  // namespace svo

using namespace svo;

extern "C" {

int svo_b200_last_kernel_ms(svo_b200_ctx* ctx, float* ms_out) {
  if (!ctx || !ms_out) return SVO_B200_EINVAL;
  cudaSetDevice(ctx->device);
  SVO_CUDA_CHECK(ctx, cudaEventSynchronize(ctx->ev_k1));
  SVO_CUDA_CHECK(ctx, cudaEventElapsedTime(ms_out, ctx->ev_k0, ctx->ev_k1));
  return 0;
}

int svo_b200_set_pyramid_rule(svo_b200_ctx* ctx, int rule) {
  if (!ctx) return SVO_B200_EINVAL;
  if (rule != SVO_B200_PYR_X86 && rule != SVO_B200_PYR_SCALAR) return set_err(ctx, SVO_B200_EINVAL, "set_pyramid_rule: unknown rule %d", rule);
  ctx->pyramid_rule = rule;
  return 0;
}

const char* svo_b200_version(void) { return "svo_b200 0.1 (sm_90a)"; }

int svo_b200_create(svo_b200_ctx** ctx_out, int device) {
  if (!ctx_out) return SVO_B200_EINVAL;
  *ctx_out = nullptr;
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n <= 0 || device < 0 || device >= n) {
    fprintf(stderr, "svo_b200_create: no usable CUDA device %d (%s); there is no CPU fallback\n", device,
            e != cudaSuccess ? cudaGetErrorString(e) : "device index out of range");
    return SVO_B200_ECUDA;
  }
  svo_b200_ctx* ctx = new svo_b200_ctx();
  ctx->device = device;
  if (cudaSetDevice(device) != cudaSuccess ||
      cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess) {
    fprintf(stderr, "svo_b200_create: cannot initialise device %d: %s\n", device,
            cudaGetErrorString(cudaGetLastError()));
    delete ctx;
    return SVO_B200_ECUDA;
  }
  cudaEventCreate(&ctx->ev_k0);
  cudaEventCreate(&ctx->ev_k1);
  cudaDeviceGetAttribute(&ctx->sm_count, cudaDevAttrMultiProcessorCount, device);
  cudaDeviceGetAttribute(&ctx->max_smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
  *ctx_out = ctx;
  return SVO_B200_OK;
}

void svo_b200_destroy(svo_b200_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  sia_batch_free(ctx);
  sia_split_free(ctx);
  if (ctx->d_in.p) cudaFree(ctx->d_in.p);
  if (ctx->h_in.p) cudaFreeHost(ctx->h_in.p);
  if (ctx->ev_k0) cudaEventDestroy(ctx->ev_k0);
  if (ctx->ev_k1) cudaEventDestroy(ctx->ev_k1);
  cudaStreamDestroy(ctx->stream);
  delete ctx;
}

const char* svo_b200_last_error(const svo_b200_ctx* ctx) { return ctx ? ctx->err.c_str() : "null context"; }
void* svo_b200_stream(svo_b200_ctx* ctx) { return ctx ? (void*)ctx->stream : nullptr; }
uint64_t svo_b200_launch_count(const svo_b200_ctx* ctx) { return ctx ? ctx->launches : 0; }

int svo_b200_synchronize(svo_b200_ctx* ctx) {
  if (!ctx) return SVO_B200_EINVAL;
  SVO_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
  return 0;
}

int svo_b200_frame_create(svo_b200_ctx* ctx, int width, int height, int n_levels,
                          svo_b200_frame** frame_out) {
  if (!ctx || !frame_out || width <= 0 || height <= 0 || n_levels < 1 || n_levels > SVO_B200_MAX_LEVELS)
    return set_err(ctx, SVO_B200_EINVAL, "frame_create: bad size %dx%d levels %d", width, height, n_levels);
  svo_b200_frame_pool* pool = nullptr;
  if (int rc = pool_create(ctx, "frame_create", width, height, n_levels, 1, &pool)) return rc;
  pool->frames[0].owns_pool = true;
  *frame_out = &pool->frames[0];
  return 0;
}

int svo_b200_frame_upload(svo_b200_ctx* ctx, svo_b200_frame* fr, const uint8_t* const* levels, int n_given) {
  if (!ctx || !fr || !levels || n_given < 1 || n_given > fr->n_levels)
    return set_err(ctx, SVO_B200_EINVAL, "frame_upload: bad arguments");
  cudaSetDevice(ctx->device);
  for (int l = 0; l < n_given; ++l) {
    if (!levels[l]) return set_err(ctx, SVO_B200_EINVAL, "frame_upload: level %d is NULL", l);
    SVO_CUDA_CHECK(ctx, cudaMemcpyAsync(fr->lvl(l), levels[l], (size_t)fr->w[l] * fr->h[l],
                                        cudaMemcpyHostToDevice, ctx->stream));
  }
  return build_pyramid(ctx, fr->pool, fr->index, 1, n_given);
}

int svo_b200_frame_upload_streams(svo_b200_ctx* ctx, int S, const svo_b200_frame_upload_entry* entries) {
  if (!ctx || S < 0 || (S > 0 && !entries)) return set_err(ctx, SVO_B200_EINVAL, "frame_upload_streams: bad arguments (S %d)", S);
  return upload_streams(ctx, S, entries);
}

int svo_b200_frame_upload_device(svo_b200_ctx* ctx, svo_b200_frame* fr, const void* level0_dev) {
  if (!ctx || !fr || !level0_dev) return set_err(ctx, SVO_B200_EINVAL, "frame_upload_device: bad arguments");
  cudaSetDevice(ctx->device);
  SVO_CUDA_CHECK(ctx, cudaMemcpyAsync(fr->lvl(0), level0_dev, (size_t)fr->w[0] * fr->h[0],
                                      cudaMemcpyDeviceToDevice, ctx->stream));
  return build_pyramid(ctx, fr->pool, fr->index, 1, 1);
}

int svo_b200_frame_download_level_tiled(svo_b200_ctx* ctx, const svo_b200_frame* fr, int level, uint8_t* out) {
  if (!ctx || !fr || !out || level < 0 || level >= fr->n_levels)
    return set_err(ctx, SVO_B200_EINVAL, "frame_download_level_tiled: bad arguments");
  cudaSetDevice(ctx->device);
  ctx->sia_chain = false;
  SVO_CUDA_CHECK(ctx, cudaMemcpyAsync(out, fr->tv[level],
                                      tiled_bytes(fr->w[level], fr->h[level]), cudaMemcpyDeviceToHost, ctx->stream));
  SVO_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
  return 0;
}

int svo_b200_frame_download_level(svo_b200_ctx* ctx, const svo_b200_frame* fr, int level, uint8_t* out) {
  if (!ctx || !fr || !out || level < 0 || level >= fr->n_levels)
    return set_err(ctx, SVO_B200_EINVAL, "frame_download_level: bad arguments");
  cudaSetDevice(ctx->device);
  ctx->sia_chain = false;
  SVO_CUDA_CHECK(ctx, cudaMemcpyAsync(out, fr->lvl(level), (size_t)fr->w[level] * fr->h[level],
                                      cudaMemcpyDeviceToHost, ctx->stream));
  SVO_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
  return 0;
}

void svo_b200_frame_destroy(svo_b200_ctx* ctx, svo_b200_frame* fr) {
  if (fr && fr->owns_pool) svo_b200_frame_pool_destroy(ctx, fr->pool);  // else a borrowed handle of a pool
}


int svo_b200_frame_pool_create(svo_b200_ctx* ctx, int width, int height, int n_levels, int count,
                               svo_b200_frame_pool** pool_out) {
  if (!ctx || !pool_out || width <= 0 || height <= 0 || n_levels < 1 || n_levels > SVO_B200_MAX_LEVELS || count <= 0)
    return set_err(ctx, SVO_B200_EINVAL, "frame_pool_create: bad arguments");
  return pool_create(ctx, "frame_pool_create", width, height, n_levels, count, pool_out);
}

svo_b200_frame* svo_b200_frame_pool_get(svo_b200_frame_pool* pool, int index) {
  if (!pool || index < 0 || index >= pool->count) return nullptr;
  return &pool->frames[index];
}

int svo_b200_frame_pool_upload(svo_b200_ctx* ctx, svo_b200_frame_pool* pool, int first, int count,
                               const uint8_t* level0_host, size_t host_stride_bytes) {
  if (!ctx || !pool || !level0_host || first < 0 || count <= 0 || first + count > pool->count)
    return set_err(ctx, SVO_B200_EINVAL, "frame_pool_upload: bad arguments");
  cudaSetDevice(ctx->device);
  const svo_b200_frame& f0 = pool->frames[0];
  const size_t img = (size_t)f0.w[0] * f0.h[0];
  if (host_stride_bytes < img) return set_err(ctx, SVO_B200_EINVAL, "frame_pool_upload: host stride < image size");
  uint8_t* dst = pool->slab[0] + (size_t)first * pool->stride[0];
  if (host_stride_bytes == img && pool->stride[0] == img) {  // fully contiguous on both sides: one flat copy
    SVO_CUDA_CHECK(ctx, cudaMemcpyAsync(dst, level0_host, img * (size_t)count, cudaMemcpyHostToDevice, ctx->stream));
  } else {  // ONE strided copy: row i = level 0 of frame first+i
    SVO_CUDA_CHECK(ctx, cudaMemcpy2DAsync(dst, pool->stride[0], level0_host, host_stride_bytes, img, (size_t)count,
                                          cudaMemcpyHostToDevice, ctx->stream));
  }
  return build_pyramid(ctx, pool, first, count, 1);
}

void svo_b200_frame_pool_destroy(svo_b200_ctx* ctx, svo_b200_frame_pool* pool) {
  if (!pool) return;
  if (ctx) {
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
  }
  if (pool->mem) cudaFree(pool->mem);
  delete pool;
}

}  // extern "C"
