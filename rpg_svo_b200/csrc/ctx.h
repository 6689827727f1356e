// rpg_svo_b200/csrc/ctx.h -- internal: context, frame and helper declarations shared by the .cu files.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/svo_b200.h"

namespace svo {
// Every pyramid level is stored twice: row-major (pitch == width, what the reference indexes), and as a block-tiled copy.
// Block (bx, by) of the copy is 16 B: rows 4by..4by+3 of columns 4bx..4bx+3, one 32-bit word per row; block-rows are
// ceil(W/4) blocks long and pixels outside the level are zero.  Any 5x5 footprint then lies in 2x2 blocks and any 7x7
// footprint in at most 3x3: the alignment kernel gathers them with a few 16-byte loads instead of one or two loads per row
// (its gathers are priced by the number of L1 requests, not by bytes).  Every frame lives in a frame pool (a single frame is
// a pool of one), which keeps the tiled copies in slabs of their own, so that the pool's row-major level-0 images stay
// contiguous and a window of them uploads as one flat copy.
inline size_t tiled_bytes(int W, int H) { return (size_t)((W + 3) / 4) * ((H + 3) / 4) * 16; }
}  // namespace svo

struct svo_b200_frame_pool;

struct svo_b200_frame {
  int width = 0, height = 0, n_levels = 0;
  int w[SVO_B200_MAX_LEVELS] = {0}, h[SVO_B200_MAX_LEVELS] = {0};
  svo_b200_frame_pool* pool = nullptr;  // the pool holding the frame's memory, frame `index` of it
  int index = 0;
  bool owns_pool = false;  // made by svo_b200_frame_create: destroying the frame destroys its pool of one
  uint8_t* lv[SVO_B200_MAX_LEVELS] = {nullptr};  // level pointers, into the pool's per-level slabs
  uint8_t* tv[SVO_B200_MAX_LEVELS] = {nullptr};  // block-tiled copies of the levels
  uint8_t* lvl(int l) const { return lv[l]; }
};

struct svo_b200_frame_pool {
  int count = 0;
  int n_levels = 0;
  // one slab per pyramid level: level l of frame i at slab[l] + i*stride[l], each slab followed by 256 B of read slack
  // (kernels fetch aligned words around unaligned footprints).  Level 0 of consecutive frames is contiguous up to the
  // 256-byte rounding, so a window uploads as ONE copy (flat when the rounding adds nothing) whose rows are whole images.
  // The tiled copies live in slabs of their own: level l of frame i at tslab[l] + i*tstride[l].
  uint8_t* slab[SVO_B200_MAX_LEVELS] = {nullptr};
  size_t stride[SVO_B200_MAX_LEVELS] = {0};
  uint8_t* tslab[SVO_B200_MAX_LEVELS] = {nullptr};
  size_t tstride[SVO_B200_MAX_LEVELS] = {0};
  uint8_t* mem = nullptr;  // the single allocation behind all slabs
  std::vector<svo_b200_frame> frames;
};

// Grow-only device / pinned-host buffers owned by the context.
struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
};
struct HostBuf {
  void* p = nullptr;
  size_t cap = 0;
};

namespace svo {
struct SiaBatchState;  // defined in sparse_align.cu
}

struct svo_b200_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  std::string err;
  uint64_t launches = 0;
  int sm_count = 0;
  int max_smem_optin = 0;
  // generic scratch: h_in / d_in hold an entry point's Staging (the alignment batch has a pair of its own, SiaBatchState)
  DevBuf d_in;
  HostBuf h_in;
  svo::SiaBatchState* sia = nullptr;
  cudaEvent_t ev_k0 = nullptr, ev_k1 = nullptr;  // around the kernel(s) of the last entry point (svo_b200_last_kernel_ms)
  int pyramid_rule = SVO_B200_PYR_X86;  // svo_b200_set_pyramid_rule
  // feature split of single pairs over GPUs (svo_b200_sia_split_*): exchange buffers in peer memory
  int xg_rank = 0, xg_world = 1, xg_pairs = 0;
  bool xg_connected = false;
  void* xg_buf = nullptr;      // our exchange buffer
  void* xg_peer[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};  // rank r's buffer as mapped here
  bool xg_peer_ipc[8] = {false, false, false, false, false, false, false, false};
  int sia_cluster = -1;  // svo_b200_sia_config: CTAs per pair (-1 = by batch size)
  int sia_fpt = 0;       //                      features per thread (0 = automatic)
  int sia_upfront = -1;  // svo_b200_sia_upfront: all levels prepared before the first iteration (-1 = automatic, 0 = off)
  // cudaOccupancyMaxActiveClusters of the 4-CTA cluster kernel ([0] upfront, [1] per level) at the shared memory it was asked for
  size_t sia_occ_smem[2] = {0, 0};
  int sia_occ_clusters[2] = {0, 0};
  svo_b200_sia_launch sia_last = {};  // svo_b200_sia_last_launch
  bool sia_last_valid = false;
  // svo_b200_sia_robust: robust cost of svo_b200_sparse_img_align / svo_b200_sia_batch_stage (UNIT scale = off)
  int sia_scale_est = SVO_B200_SCALE_UNIT, sia_weight_fn = SVO_B200_WEIGHT_UNIT;
  bool sia_last_robust = false;   // the last alignment launch ran the robust kernel
  std::vector<float> sia_scales;  // its per-pair, per-level scales (svo_b200_sia_last_scales), fetched with its outputs
  // The last work enqueued on `stream` is a run of the staged batch (svo_b200_sia_batch_run): the next run of that batch
  // may then overlap it on the device.  Every other enqueue clears it (kt_begin for kernels; the copy-only entry points).
  bool sia_chain = false;
  // svo_b200_set_epipolar_options: Matcher::Options of the depth filter / epipolar matcher launches
  svo_b200_epipolar_options epi = {0, 1, 1, 0.7};
  // per candidate of the last svo_b200_find_epipolar_match_direct call: Matcher::h_inv_ and whether align1D set it
  // (svo_b200_epipolar_last_h_inv)
  std::vector<double> epi_h_inv;
  std::vector<uint8_t> epi_ran_1d;
  bool epi_last_valid = false;
};

namespace svo {

int set_err(svo_b200_ctx* ctx, int code, const char* fmt, ...);
int ensure_dev(svo_b200_ctx* ctx, DevBuf& b, size_t bytes);

#define SVO_CUDA_CHECK(ctx, call)                                                                   \
  do {                                                                                              \
    cudaError_t _e = (call);                                                                        \
    if (_e != cudaSuccess)                                                                          \
      return svo::set_err((ctx), SVO_B200_ECUDA, "%s failed: %s (%s:%d)", #call,                    \
                          cudaGetErrorString(_e), __FILE__, __LINE__);                              \
  } while (0)

// Bump allocator over a byte buffer (host staging mirrored 1:1 on the device).
struct Carver {
  size_t off = 0;
  size_t take(size_t bytes, size_t align = 256) {
    off = (off + align - 1) / align * align;
    size_t o = off;
    off += bytes;
    return o;
  }
};

void sia_batch_free(svo_b200_ctx* ctx);
void sia_split_free(svo_b200_ctx* ctx);
// CUDA events on the context's stream bracketing the kernel launch(es) of an entry point (no copies): the live
// per-kernel device time bench.py's roofline figures divide by.  Every entry point that launches a kernel calls kt_begin,
// which also ends a chain of batch runs (svo_b200_ctx::sia_chain).
inline void kt_begin(svo_b200_ctx* ctx) {
  ctx->sia_chain = false;
  if (ctx->ev_k0) cudaEventRecord(ctx->ev_k0, ctx->stream);
}
inline void kt_end(svo_b200_ctx* ctx) { if (ctx->ev_k1) cudaEventRecord(ctx->ev_k1, ctx->stream); }

// The kernel launches of an entry point: `launch` enqueues n of them between kt_begin and kt_end; they are counted for
// svo_b200_launch_count and their launch error is returned.
template <class F>
int launch_kernels(svo_b200_ctx* ctx, int n, F&& launch) {
  kt_begin(ctx);
  launch();
  ctx->launches += n;
  kt_end(ctx);
  SVO_CUDA_CHECK(ctx, cudaGetLastError());
  return 0;
}

// An entry point's arrays staged through a pinned buffer and its device mirror: the context's h_in / d_in, or a pair of the
// caller's own (the alignment batch's).  Each region is declared once, by kind, element count and the pointer `at` that
// open() sets to its device address:
//   in     copied in from src; a NULL src is filled by the caller through host() between open() and send();
//   inout  copied in from io and back to it; a NULL io is filled and read by the caller;
//   out    copied back to dst; a NULL dst is read by the caller through host(), or by nobody.
// open() lays out the copied-in regions as one front range and the copied-back ones as one tail range (in-only, then
// in-out, then out-only regions), grows the buffers, waits for the stream (an earlier copy may still read the pinned
// buffer), sets every `at` and then copies the sources in, so that a table whose entries hold region addresses can itself
// be a source.  send() copies the front range to the device; receive() copies the tail range back, waits for it and
// copies every region with a destination out.
// The pageable form (Staging(ctx, Staging::Pageable{})) stages in-only regions into d_in through a host buffer of its own,
// made per call.  The runtime stages a copy from pageable memory before the copy returns, so open() does not wait for the
// stream (only growing d_in does), and a call that only copies in does not wait on earlier work.  open() refuses in-out and
// out regions.
class Staging {
  template <class T>
  struct same { using type = T; };
  template <class T>
  using same_t = typename same<T>::type;  // element types come from `at` alone

 public:
  struct Pageable {};
  explicit Staging(svo_b200_ctx* ctx) : Staging(ctx, ctx->h_in, ctx->d_in) {}
  Staging(svo_b200_ctx* ctx, HostBuf& h, DevBuf& d) : ctx_(ctx), hbuf_(&h), dbuf_(&d) {}
  Staging(svo_b200_ctx* ctx, Pageable) : ctx_(ctx), hbuf_(nullptr), dbuf_(&ctx->d_in) {}
  template <class T>
  void in(const same_t<T>* src, size_t n, T** at, size_t align = 256) { add(src, nullptr, sizeof(T) * n, align, true, false, at); }
  template <class T>
  void inout(same_t<T>* io, size_t n, T** at, size_t align = 256) { add(io, io, sizeof(T) * n, align, true, true, at); }
  template <class T>
  void out(same_t<T>* dst, size_t n, T** at) { add(nullptr, dst, sizeof(T) * n, 256, false, true, at); }
  int open();
  int send();
  int receive();
  template <class T>
  typename std::remove_const<T>::type* host(T* dev) const {  // the pinned mirror of a region's device address
    return reinterpret_cast<typename std::remove_const<T>::type*>(h_ + (reinterpret_cast<const uint8_t*>(dev) - d_));
  }
  uint8_t* tail() const { return d_ + back_; }  // the device tail range, tail_bytes() long
  size_t tail_bytes() const { return end_ - back_; }

 private:
  struct Region {
    const void* src;
    void* dst;
    size_t bytes, align, off;
    bool in, back;
    void* at;
    void (*bind)(void* at, uint8_t* p);
  };
  template <class T>
  void add(const void* src, void* dst, size_t bytes, size_t align, bool in, bool back, T** at) {
    regions_.push_back({src, dst, bytes, align, 0, in, back, at, [](void* a, uint8_t* p) { *static_cast<T**>(a) = reinterpret_cast<T*>(p); }});
  }
  svo_b200_ctx* ctx_;
  HostBuf* hbuf_;  // NULL: pageable, through page_
  DevBuf* dbuf_;
  std::vector<uint8_t> page_;
  std::vector<Region> regions_;
  uint8_t *h_ = nullptr, *d_ = nullptr;
  size_t front_ = 0, back_ = 0, end_ = 0;
};

// The entries of one table-driven launch, where a CTA finds its entry with stream_of over the CTA offsets: entry j holds
// `items` work items, `per_cta` to a CTA, and CTAs cta_offset[j] .. cta_offset[j + 1] - 1.  stage() declares the entries
// and the offsets as two in-regions of `st`, whose device addresses open() sets in `jobs_at` / `off_at`.  An entry that
// holds region addresses is added before any region binding into it is declared, so that `jobs` never reallocates under a
// bound pointer.
template <class Job>
struct LaunchTable {
  std::vector<Job> jobs;
  std::vector<int> cta_offset = {0};
  long long ctas = 0;
  bool over = false;  // more CTAs than one grid holds, or an entry whose thread index leaves int
  const Job* jobs_at = nullptr;
  const int* off_at = nullptr;
  void add(const Job& j, long long items, int per_cta) {
    ctas += (items + per_cta - 1) / per_cta;
    over = over || ctas > INT32_MAX || items > INT32_MAX - per_cta;
    jobs.push_back(j);
    cta_offset.push_back((int)std::min<long long>(ctas, INT32_MAX));
  }
  int n() const { return (int)jobs.size(); }
  void stage(Staging& st) {
    st.in(jobs.data(), jobs.size(), &jobs_at);
    st.in(cta_offset.data(), cta_offset.size(), &off_at);
  }
};

// Re-prefixes the error that the check of entry i of a many-entry call left: "<name>: <what> <i>: <message>".  A single
// call (name NULL) keeps the message.
int entry_err(svo_b200_ctx* ctx, int rc, const char* name, const char* what, int i);

// The candidates' reference features of the matcher entry points (`who`): every ref_index inside the n_ref keyframes and
// every level (the array `level_name`) inside its keyframe's pyramid.
int check_ref_levels(svo_b200_ctx* ctx, const char* who, const char* level_name, const svo_b200_frame* const* ref_frames,
                     int n_ref, int M, const int* ref_index, const int* level);
// check_ref_levels, then max_search_level below the current frame's levels and the camera's size that of cur and of
// every keyframe.
int check_ref_table(svo_b200_ctx* ctx, const char* who, const char* level_name, const svo_b200_frame* const* ref_frames,
                    int n_ref, int M, const int* ref_index, const int* level, const svo_b200_frame* cur,
                    const svo_b200_camera* cam, int max_search_level);

// Device-side camera ([EXT] vk::PinholeCamera / vk::ATANCamera): the C-ABI parameters plus the derived constants
// the vikit constructors precompute.  Passed by value inside kernel parameter structs.
struct CamDev {
  double fx, fy, cx, cy;
  double fx_inv, fy_inv;
  double d[5];       // pinhole: k1 k2 p1 p2 k3;  ATAN: d[0] = s
  double s_inv, tans, tans_inv;  // ATAN: 1/s, 2 tan(s/2), 1/tans
  int model, distorted;
  int width, height;
};
int cam_to_dev(svo_b200_ctx* ctx, const svo_b200_camera* cam, CamDev& out);
int cam_check_frames(svo_b200_ctx* ctx, const char* who, const svo_b200_camera* cam, const svo_b200_frame* const* frames, int n);

}  // namespace svo
