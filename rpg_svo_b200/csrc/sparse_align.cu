// rpg_svo_b200/csrc/sparse_align.cu -- svo::SparseImgAlign on sm_90a.
//
// Replaces svo/src/sparse_img_align.cpp:43-258 (run / precomputeReferencePatches /
// computeResiduals / solve / update) together with the Gauss-Newton driver of
// vk::NLLSSolver<6,SE3>::optimizeGaussNewton [EXT] that the class derives from.
//
// Design (GPU-first, not a translation):
//   * one CTA per frame pair -- or, for small batches, one thread-block CLUSTER per pair with the
//     features split over its CTAs -- runs the WHOLE coarse-to-fine loop on the device: no host
//     round trip per Gauss-Newton iteration, batches of pairs fill the SMs.
//   * one thread owns one feature (FPT features when N > blockDim): the 4x4 reference patch, and its two
//     gradient images, live in shared memory in pixel-major (SoA) order so a warp's accesses are conflict
//     free; the feature's bearing/depth state lives in registers, or -- throughput geometry -- in shared memory.
//   * inverse-compositional structure is exploited: the per-pixel Jacobian is
//     J_p = dx_p * a + dy_p * b with a, b per-FEATURE 6-vectors, hence
//        sum_p J_p J_p^T = Sxx aa^T + Sxy (ab^T + ba^T) + Syy bb^T     (pose independent)
//        sum_p J_p r_p   = (sum dx_p r_p) a + (sum dy_p r_p) b
//     so the 6x6 normal matrix is reduced and factorised ONCE per level (and re-formed only in the
//     iterations where some patch leaves the current image), and an iteration costs 3 f32 FMAs per
//     pixel plus ~15 f64 FMAs per feature instead of the reference's 27 f64 MACs per pixel.
//   * the current image is staged in shared memory where the instantiation has room: whole coarse levels with
//     one TMA bulk copy (cp.async.bulk + mbarrier), at the fine levels a 16x8-byte window around each
//     feature's projection with cp.async (once per level; a footprint that drifts out of its window
//     falls back to global loads).  The packed feature records of the pair arrive by TMA as well.
//   * ONE block barrier pair per iteration: each warp folds its partial sums (6 Jres + chi2 + counts)
//     with a transposed shuffle reduction and parks them in a double-buffered shared array; after
//     the barrier warp 0 adds the per-warp partials and runs the 6x6 substitution, SE3 exp and the
//     accept / rollback decision in registers (all lanes redundantly), and publishes the pose in shared memory.
//     Cluster geometry: every warp of every CTA receives all partials and runs that tail redundantly
//     (bit-identical everywhere); its "upfront" variant prepares the reference patches, H and LDL^T of ALL
//     levels before the first iteration and exchanges the per-iteration sums with st.async + complete_tx on
//     the receivers' mbarriers instead of DSMEM stores + barrier.cluster.
//   * the throughput instantiation is kept SMALL: staging modes and features it cannot use are compiled out
//     and its loops over a thread's features are loops, not unrolled copies -- three CTAs in different phases
//     share one instruction cache, and instruction-fetch stalls were a leading stall reason of the unrolled form.
// Precision follows the reference per quantity: f32 interpolation/residual/chi2, f64 geometry and
// normal equations (SURVEY.md 8a).
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <type_traits>
#include <vector>

#include "ctx.h"
#include "sia_patch_layout.h"
#include "svo_math.cuh"

namespace svo {

#ifndef SVO_SIA_DEBUG
#define SVO_SIA_DEBUG 0  // 1: thread 0 accumulates clock64 section timings and a few CTAs print them
#endif
#if SVO_SIA_DEBUG
#define SIA_DBG(...) __VA_ARGS__
#else
#define SIA_DBG(...)
#endif
constexpr int kPatchArea = 16;
constexpr int kPartK = 24;     // widest block reduction: 21 unique H entries + 1 count, padded to 16 + 8
constexpr int kWinRows = 8;    // per-feature window of the current image: 8 rows x 16 bytes
constexpr int kWinBytes = kWinRows * 16;  // 128 B per feature slot

struct SiaJob {  // one frame pair; array lives in device memory
  const uint8_t* ref_lvl[SVO_B200_MAX_LEVELS];
  const uint8_t* cur_lvl[SVO_B200_MAX_LEVELS];
  // block-tiled copies of the levels (ctx.h).  Pointers of their own, not an offset from the row-major level: a frame pool
  // keeps its copies apart so that its level-0 images stay contiguous (one flat upload per window).
  const uint8_t* ref_tl[SVO_B200_MAX_LEVELS];
  const uint8_t* cur_tl[SVO_B200_MAX_LEVELS];
  const uint8_t* blob;  // packed features: px[np*2] f[np*3] pos[np*3] (f64) then has_point[np] (u8)
  int n_feat, n_pad;
  int feat_off;  // offset of this pair in visible_out
  int pad_;
  double T[12];
  double ref_pos[3];
};

// ---- single-stream feature split over GPUs (SURVEY.md 8e): the per-iteration sums of one pair are exchanged between the
// ranks' kernels through peer memory (NVLink P2P stores into every rank's exchange buffer, system-scope flags), so the
// whole coarse-to-fine loop still runs inside ONE kernel per GPU -- no host round trip, no collective library call.
constexpr int kMaxSplit = 8;
struct XgSlot {  // what one rank publishes for one exchange
  double v[kPartK];
  int cnt[2];
  unsigned seq;  // sequence number of the exchange this slot holds (written last, release)
  unsigned pad_;
};
struct XgPair {  // per frame pair, in every rank's exchange buffer
  XgSlot slot[2][kMaxSplit];  // [parity of the exchange][publishing rank]
  unsigned xseq;              // exchanges completed so far (persists across launches; identical on all ranks)
  unsigned err;               // sticky: a peer did not arrive within the timeout
  unsigned pad_[2];
};
struct XgParams {
  int rank, world;
  XgPair* peer[kMaxSplit];  // rank r's exchange buffer as mapped in this process (peer[rank] = our own)
};

struct SiaParams {
  const SiaJob* jobs;
  XgParams xg;
  int w[SVO_B200_MAX_LEVELS], h[SVO_B200_MAX_LEVELS];
  CamDev cam;
  int max_level, min_level, n_iter;
  double eps;
  int stage_cap;  // bytes of the staging region in shared memory (TMA image / cp.async windows)
  double* T_out;
  double* H_out;
  uint8_t* visible_out;
  svo_b200_sia_stats* stats;
  svo_b200_sia_iter* trace;
  int trace_cap;
  int* n_trace;
  int debug;  // env SVO_B200_SIA_DEBUG=1: thread 0 of a few CTAs prints clock64 section timings
  // EVAL mode (svo_b200_sparse_residuals)
  int eval_level;
  const uint8_t* visible_in;
  float* ref_patch_out;
  float* residuals_out;
  uint8_t* in_image_out;
  double* Jres_out;
  double* chi2_out;
  long long* n_meas_out;
};

struct SiaState {  // model_ / old_model of NLLSSolver::optimizeGaussNewton [EXT]
  Pose model, old_model;
};

// Shared-memory control block of one CTA.  NWC = warps of this CTA, CS = CTAs of the pair (cluster size).
template <int NWC, int CS>
struct SiaSharedT {
  static constexpr int kPairWarps = NWC * CS;
  uint64_t mbar;
  uint64_t xbar[2];  // cluster geometry, asynchronous exchange: one mbarrier per parity of the running iteration counter
  // per-warp partial sums of one residual pass (6 Jres + chi2, slot 7 unused) for every warp of the
  // pair (all CTAs of the cluster), double-buffered by the parity of the running iteration counter
  double part[2][kPairWarps][8];
  int cnt[2][kPairWarps][2];
  double hpart[NWC * kPartK];                   // per-warp partials of the 24-value H reduction
  double hsum_cta[CS > 1 ? CS : 1][kPartK];     // per-CTA H sums (cluster variant: written remotely)
  double sums[kPartK];                          // H totals of the pair
  double Hs[36];                                // H_ of the current pass (scaled), full symmetric
  double Htot[36];                              // sum over the level's visible set (scaled)
  Solver6 sol_cur;                              // factorisation used for the current solve (slow path)
  Solver6 sol_tot;                              // factorisation of Htot
  SiaState st[2];                               // double-buffered like `part`
  int h_is_tot, n_iters, sum_vis, sum_in, n_in_last, n_trace;  // thread 0 of CTA rank 0 only
  unsigned xg_seq;     // feature split over GPUs: exchanges completed (warp 0) ...
  unsigned xg_failed;  // ... and "an exchange timed out" (must directly follow xg_seq)
  alignas(16) double pub[12];  // CS == 1: the pose (R row-major, t) warp 0 publishes after its Gauss-Newton tail
  const uint4* cur_tl;         // tiled copy of the current image of the running level (throughput geometry)
  int pub_done, pub_slow;
#if SVO_SIA_DEBUG
  long long tkx[4];
  long long tk[8];  // debug: cycles in [level setup, pass, reduce, tail, total]
#endif
};

// "Upfront" variant (small batches: a thread-block cluster per pair, every CTA with an SM of its own): the reference patches,
// H sums and factorisations of ALL pyramid levels -- none of which depends on the pose -- are computed before the first
// Gauss-Newton iteration, with one cluster exchange for all levels, so a level starts with nothing but the staging of its
// current image.  Per-level results live here (behind the control block) and in per-level patch arrays.
template <int NWC, int CS>
struct SiaUpT {
  double hpart[SVO_B200_MAX_LEVELS][NWC * kPartK];      // per-warp partials of every level
  double hsum_cta[SVO_B200_MAX_LEVELS][CS][kPartK];     // per-CTA sums of every level (written remotely)
  double sums[SVO_B200_MAX_LEVELS][kPartK];
  double Htot[SVO_B200_MAX_LEVELS][36];
  Solver6 sol[SVO_B200_MAX_LEVELS];
};

// ---------------------------------------------------------------------------------------------
// Unaligned byte-row fetch: consecutive bytes starting at byte offset `off` from a 4-byte aligned
// base, as two (or three) aligned 32-bit loads + funnel shifts.
// ---------------------------------------------------------------------------------------------
template <bool SMEM>
__device__ __forceinline__ uint32_t ld_word(const uint8_t* base, int word_off) {
  if (SMEM) return *reinterpret_cast<const uint32_t*>(base + word_off);
  return __ldg(reinterpret_cast<const uint32_t*>(base + word_off));
}
template <bool SMEM>
__device__ __forceinline__ void fetch8(const uint8_t* base, int off, uint32_t& lo, uint32_t& hi) {
  const int a = off & ~3;
  const unsigned sh = (unsigned)(off & 3) * 8u;
  const uint32_t w0 = ld_word<SMEM>(base, a), w1 = ld_word<SMEM>(base, a + 4);
  lo = __funnelshift_r(w0, w1, sh);
  hi = w1 >> sh;  // byte 4 of the row in its low byte
}
// 7 consecutive bytes at byte offset `off` from an 8-byte aligned global base: one aligned 64-bit load, plus the next
// one only when the span crosses it -- 1.75 memory requests per row on average instead of 3 (the residual loops are
// bound by the number of uncoalesced requests the L1 can take, not by bytes)
__device__ __forceinline__ void fetch7_g64(const uint8_t* base, int off, uint32_t& lo, uint32_t& hi) {
  const int a = off & ~7, p = off & 7;
  const uint2 A = __ldg(reinterpret_cast<const uint2*>(base + a));
  uint2 B = make_uint2(0u, 0u);
  if (p > 1) B = __ldg(reinterpret_cast<const uint2*>(base + a + 8));
  const bool k = p >= 4;
  const uint32_t x0 = k ? A.y : A.x, x1 = k ? B.x : A.y, x2 = k ? B.y : B.x;
  const unsigned sh = (unsigned)(p & 3) * 8u;
  lo = __funnelshift_r(x0, x1, sh);
  hi = __funnelshift_r(x1, x2, sh);
}
template <bool SMEM>
__device__ __forceinline__ void fetch12(const uint8_t* base, int off, uint32_t& lo, uint32_t& hi) {
  const int a = off & ~3;
  const unsigned sh = (unsigned)(off & 3) * 8u;
  const uint32_t w0 = ld_word<SMEM>(base, a), w1 = ld_word<SMEM>(base, a + 4),
                 w2 = ld_word<SMEM>(base, a + 8);
  lo = __funnelshift_r(w0, w1, sh);
  hi = __funnelshift_r(w1, w2, sh);
}

// Footprint gathers from the block-tiled copy of a level (ctx.h: 16-byte blocks of 4x4 pixels, one 32-bit
// word per row, `bw` blocks per block-row).  A column of blocks yields a sequence of row words q = 0, 1, ... from the block-row
// of the footprint's first row y0; row r of the footprint is word q = r + (y0 & 3), picked by two select stages (rotate by
// 2, then by 1).  The same funnel shifts as the row-major fetches then give the same bytes, so the pixel values and everything
// computed from them are unchanged.
template <int N>
__device__ __forceinline__ void rotate_rows(const uint32_t (&q)[N + 3], int s, uint32_t (&out)[N]) {
  uint32_t v[N + 1];
#pragma unroll
  for (int i = 0; i <= N; ++i) v[i] = (s & 2) ? q[i + 2] : q[i];
#pragma unroll
  for (int r = 0; r < N; ++r) out[r] = (s & 1) ? v[r + 1] : v[r];
}
// 5x5: rows y0..y0+4, columns x0..x0+4 lie in exactly 2x2 blocks -- four loads.  lo[r] = columns x0..x0+3 of row y0+r, the
// low byte of hi[r] = column x0+4 (as fetch8).  Of the 8 row words of a block column the footprint needs words s..s+4
// (s = y0 & 3), so words (s & 2) .. (s & 2) + 5 are loaded -- one whole block and the adjacent half of the other, 6 registers
// instead of 8 (the residual pass runs at the register limit) -- and the first select stage of rotate_rows is done by the
// addresses.
__device__ __forceinline__ void fetch5x5_tiled(const uint4* tl, int bw, int x0, int y0, uint32_t (&lo)[5], uint32_t (&hi)[5]) {
  const uint4* b = tl + (y0 >> 2) * bw + (x0 >> 2);
  const bool s2 = (y0 & 2) != 0, s1 = (y0 & 1) != 0;
  // s2: the bottom block whole, words 2, 3 of the top one; else the top block whole, words 0, 1 of the bottom one
  const uint4* pw = s2 ? b + bw : b;
  const uint2* ph = reinterpret_cast<const uint2*>(s2 ? b : b + bw) + (s2 ? 1 : 0);
  const uint4 l4 = __ldg(pw), r4 = __ldg(pw + 1);
  const uint2 l2 = __ldg(ph), r2 = __ldg(ph + 2);
  const uint32_t vl[6] = {s2 ? l2.x : l4.x, s2 ? l2.y : l4.y, s2 ? l4.x : l4.z, s2 ? l4.y : l4.w, s2 ? l4.z : l2.x, s2 ? l4.w : l2.y};
  const uint32_t vr[6] = {s2 ? r2.x : r4.x, s2 ? r2.y : r4.y, s2 ? r4.x : r4.z, s2 ? r4.y : r4.w, s2 ? r4.z : r2.x, s2 ? r4.w : r2.y};
  uint32_t wl[5], wr[5];
#pragma unroll
  for (int r = 0; r < 5; ++r) {
    wl[r] = s1 ? vl[r + 1] : vl[r];
    wr[r] = s1 ? vr[r + 1] : vr[r];
  }
  const unsigned sh = (unsigned)(x0 & 3) * 8u;
#pragma unroll
  for (int r = 0; r < 5; ++r) {
    lo[r] = __funnelshift_r(wl[r], wr[r], sh);
    hi[r] = wr[r] >> sh;
  }
}
// 7x7: rows y0..y0+6, columns x0..x0+6 lie in 2 or 3 blocks per axis (6.25 loads on average).  Walked one block-row at a time,
// each block-row's words funnel-shifted into two words per row at once, so that the raw words of a block-row need not stay live.  lo[r] = columns
// x0..x0+3 of row y0+r, bytes 0..2 of hi[r] = columns x0+4..x0+6 (as fetch7_g64).  The third block column / block-row is
// loaded only when the footprint reaches into it (always inside the level when the footprint is).
__device__ __forceinline__ void fetch7x7_tiled(const uint4* tl, int bw, int x0, int y0, uint32_t (&lo)[7], uint32_t (&hi)[7]) {
  const uint4* b = tl + (y0 >> 2) * bw + (x0 >> 2);
  const int s = y0 & 3;
  const bool col3 = (x0 & 3) >= 2;
  const unsigned sh = (unsigned)(x0 & 3) * 8u;
  uint32_t ql[10], qh[10];  // funnel-shifted words of rows q = 0..9 from block-row y0 >> 2 (rows s..s+6 are the footprint's)
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const bool load = j < 2 || s >= 2;
    const uint4 zero = make_uint4(0u, 0u, 0u, 0u);
    const uint4 x = load ? __ldg(b + j * bw) : zero, y = load ? __ldg(b + j * bw + 1) : zero;
    const uint4 z = load && col3 ? __ldg(b + j * bw + 2) : zero;
    const uint32_t xw[4] = {x.x, x.y, x.z, x.w}, yw[4] = {y.x, y.y, y.z, y.w}, zw[4] = {z.x, z.y, z.z, z.w};
#pragma unroll
    for (int w = 0; w < 4; ++w) {
      if (4 * j + w >= 10) break;
      ql[4 * j + w] = __funnelshift_r(xw[w], yw[w], sh);
      qh[4 * j + w] = __funnelshift_r(yw[w], zw[w], sh);
    }
  }
  rotate_rows<7>(ql, s, lo);
  rotate_rows<7>(qh, s, hi);
}

// Element k of a per-feature register array, read with compile-time indices only: in a loop over the thread's features that
// is not unrolled, a[k] would put the whole array in local memory.
template <class T, int FPT>
__device__ __forceinline__ T sel_k(const T (&a)[FPT], int k) {
  T v = a[0];
#pragma unroll
  for (int j = 1; j < FPT; ++j) v = k == j ? a[j] : v;
  return v;
}

// precomputeReferencePatches' arithmetic (:115-136) for one feature: the 4x4 reference patch and its two gradient images
// from the 7x7 footprint (rows vi-3..vi+3, columns ui-3..ui+3; row r = bytes 0..3 of lo[r], 0..2 of hi[r]) at the sub-pixel
// offset (su, sv).  The footprint is streamed row by row to keep the register footprint small: Bq row r (bilinear blends
// with top-left tap P[r][c]) needs footprint rows r, r+1; patch row y needs Bq rows y, y+1, y+2.  emit(p, val, dx, dy) takes
// pixel p = 4 y + x.  The same operations in the same order as level_patches in sia_kernel, which keeps them inline: called
// from there, this function changes the local-memory slot assignment of ten of its instantiations.
template <class Emit>
__device__ __forceinline__ void ref_patch_7x7(const uint32_t (&rlo)[7], const uint32_t (&rhi)[7], float su, float sv, Emit emit) {
  float wtl, wtr, wbl, wbr;
  bilin_weights(su, sv, wtl, wtr, wbl, wbr);
  float pr0[7], pr1[7], b0[6], b1[6], b2[6];
  auto load_row = [&](int r, float (&dst)[7]) {
    const uint32_t lo = rlo[r], hi = rhi[r];
    dst[0] = byte_to_float<0>(lo); dst[1] = byte_to_float<1>(lo); dst[2] = byte_to_float<2>(lo);
    dst[3] = byte_to_float<3>(lo); dst[4] = byte_to_float<0>(hi); dst[5] = byte_to_float<1>(hi);
    dst[6] = byte_to_float<2>(hi);
  };
  load_row(0, pr0);
#pragma unroll
  for (int r = 0; r < 6; ++r) {
    load_row(r + 1, pr1);
#pragma unroll
    for (int c = 0; c < 6; ++c) b2[c] = bilin(wtl, wtr, wbl, wbr, pr0[c], pr0[c + 1], pr1[c], pr1[c + 1]);
    if (r >= 2) {  // rows b0 (= Bq[y]), b1 (= Bq[y+1]), b2 (= Bq[y+2]) with y = r-2 are complete
      const int y = r - 2;
#pragma unroll
      for (int x = 0; x < 4; ++x) {
        const int p = y * 4 + x;
        const float val = b1[x + 1];
        const float dx = __fmul_rn(0.5f, __fsub_rn(b1[x + 2], b1[x]));
        const float dy = __fmul_rn(0.5f, __fsub_rn(b2[x + 1], b0[x + 1]));
        emit(p, val, dx, dy);
      }
    }
#pragma unroll
    for (int c = 0; c < 6; ++c) { b0[c] = b1[c]; b1[c] = b2[c]; }
#pragma unroll
    for (int c = 0; c < 7; ++c) pr0[c] = pr1[c];
  }
}

// per-feature unscaled Jacobian rows: a = row0 of jacobian_xyz2uv, b = row1 (frame.h:116-138)
__device__ __forceinline__ void jac_rows(double x, double y, double zi, double (&a)[6], double (&b)[6]) {
  const double X = x * zi, Y = y * zi;
  a[0] = -zi; a[1] = 0.0; a[2] = X * zi; a[3] = X * Y; a[4] = -(1.0 + X * X); a[5] = Y;
  b[0] = 0.0; b[1] = -zi; b[2] = Y * zi; b[3] = 1.0 + Y * Y; b[4] = -(X * Y); b[5] = -X;
}
// Entry `idx` (0..20, upper triangle row-major) of Sxx aa^T + Sxy (ab^T + ba^T) + Syy bb^T.
template <int IDX>
__device__ __forceinline__ double h_entry(const double (&a)[6], const double (&b)[6], double sxx, double sxy, double syy) {
  constexpr int R = IDX < 6 ? 0 : IDX < 11 ? 1 : IDX < 15 ? 2 : IDX < 18 ? 3 : IDX < 20 ? 4 : 5;
  constexpr int BASE = R == 0 ? 0 : R == 1 ? 6 : R == 2 ? 11 : R == 3 ? 15 : R == 4 ? 18 : 20;
  constexpr int C = R + (IDX - BASE);
  return fma(sxx, a[R] * a[C], fma(sxy, fma(a[R], b[C], b[R] * a[C]), syy * (b[R] * b[C])));
}
template <int CHUNK, int J>
__device__ __forceinline__ double h_chunk_value(const double (&a)[6], const double (&b)[6], double sxx, double sxy,
                                                double syy, double cnt) {
  constexpr int IDX = CHUNK * 8 + J;
  if constexpr (IDX < 21) return h_entry<IDX>(a, b, sxx, sxy, syy);
  else if constexpr (IDX == 21) return cnt;
  else return 0.0;
}
// one feature's contribution to the 8 values of chunk CH
template <int CH>
__device__ __forceinline__ void h_chunk_add(double (&v)[8], const double (&a)[6], const double (&b)[6], double sxx, double sxy,
                                            double syy, double cnt) {
  v[0] += h_chunk_value<CH, 0>(a, b, sxx, sxy, syy, cnt);
  v[1] += h_chunk_value<CH, 1>(a, b, sxx, sxy, syy, cnt);
  v[2] += h_chunk_value<CH, 2>(a, b, sxx, sxy, syy, cnt);
  v[3] += h_chunk_value<CH, 3>(a, b, sxx, sxy, syy, cnt);
  v[4] += h_chunk_value<CH, 4>(a, b, sxx, sxy, syy, cnt);
  v[5] += h_chunk_value<CH, 5>(a, b, sxx, sxy, syy, cnt);
  v[6] += h_chunk_value<CH, 6>(a, b, sxx, sxy, syy, cnt);
  v[7] += h_chunk_value<CH, 7>(a, b, sxx, sxy, syy, cnt);
}

// ---- cluster helpers (CS == 1: plain CTA, everything below folds to local shared memory) ------------
__device__ __forceinline__ unsigned cluster_rank() {
  unsigned r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
template <int CS>
__device__ __forceinline__ void pair_sync() {  // all threads of the pair: the CTA, or every CTA of its cluster
  if constexpr (CS == 1) {
    __syncthreads();
  } else {
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
  }
}
// store a double into the same shared-memory variable of CTA `rank` of the cluster (DSMEM)
__device__ __forceinline__ void st_cluster_f64(double* local_ptr, unsigned rank, double v) {
  uint32_t remote;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(smem_u32(local_ptr)), "r"(rank));
  asm volatile("st.shared::cluster.f64 [%0], %1;" ::"r"(remote), "d"(v) : "memory");
}
__device__ __forceinline__ void st_cluster_v2s32(int* local_ptr, unsigned rank, int a, int b) {
  uint32_t remote;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(smem_u32(local_ptr)), "r"(rank));
  asm volatile("st.shared::cluster.v2.s32 [%0], {%1, %2};" ::"r"(remote), "r"(a), "r"(b) : "memory");
}

// asynchronous remote store that also counts its bytes on an mbarrier of the SAME remote CTA (st.async + complete_tx): data
// and "it has arrived" travel together, one DSMEM hop, and the receiver sleeps on its own mbarrier instead of a cluster barrier
__device__ __forceinline__ uint32_t cluster_addr(const void* local_ptr, unsigned rank) {
  uint32_t remote;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(smem_u32(local_ptr)), "r"(rank));
  return remote;
}
__device__ __forceinline__ void st_async_f64(uint32_t remote_addr, double v, uint32_t remote_mbar) {
  asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.f64 [%0], %1, [%2];" ::"r"(remote_addr), "d"(v), "r"(remote_mbar)
               : "memory");
}
__device__ __forceinline__ void st_async_v2s32(uint32_t remote_addr, int a, int b, uint32_t remote_mbar) {
  asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v2.s32 [%0], {%1, %2}, [%3];" ::"r"(remote_addr), "r"(a), "r"(b),
               "r"(remote_mbar)
               : "memory");
}

// ---- system-scope accesses to (peer) global memory
__device__ __forceinline__ void st_sys_f64(double* p, double v) { asm volatile("st.relaxed.sys.global.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory"); }
__device__ __forceinline__ void st_sys_s32(int* p, int v) { asm volatile("st.relaxed.sys.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ void st_release_sys_u32(unsigned* p, unsigned v) { asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ unsigned ld_acquire_sys_u32(const unsigned* p) { unsigned v; asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ double ld_sys_f64(const double* p) { double v; asm volatile("ld.relaxed.sys.global.f64 %0, [%1];" : "=d"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ int ld_sys_s32(const int* p) { int v; asm volatile("ld.relaxed.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }

// All-reduce (sum) of K <= 24 doubles + two counts of one pair over the ranks of a feature split, executed by ONE warp of
// the pair's CTA on every rank: lane k holds value k.  Every rank stores its values into slot [parity][rank] of EVERY
// rank's exchange buffer (peer memory), then its sequence number (release); it then waits until all slots of its own
// buffer carry that number (acquire) and adds them in rank order, so all ranks obtain bit-identical sums.  A slot is
// rewritten two exchanges later, by which time every peer has consumed it (a rank cannot run more than one exchange
// ahead).  A peer that never arrives trips a ~2 s timeout: the sticky error flag is set and the kernel finishes with
// meaningless numbers instead of hanging the GPU.
template <int K>
__device__ __forceinline__ void xg_allreduce(const XgParams& X, int pair, unsigned* seq_smem, double& val, int& c0, int& c1) {
  const int lane = threadIdx.x & 31;
  const unsigned failed = seq_smem[1];  // a previous exchange of this launch already timed out: do not wait again
  const unsigned xseq = *seq_smem;
  const unsigned par = xseq & 1u, want = xseq + 1u;
  for (int r = 0; r < X.world; ++r) {
    XgSlot* dst = &X.peer[r][pair].slot[par][X.rank];
    if (lane < K) st_sys_f64(&dst->v[lane], val);
    if (lane == 0) { st_sys_s32(&dst->cnt[0], c0); st_sys_s32(&dst->cnt[1], c1); }
  }
  __threadfence_system();
  __syncwarp();
  if (lane == 0)
    for (int r = 0; r < X.world; ++r) st_release_sys_u32(&X.peer[r][pair].slot[par][X.rank].seq, want);
  XgPair* own = &X.peer[X.rank][pair];
  bool ok = true;
  if (lane < X.world && !failed) {
    const long long t0 = clock64();
    while (ld_acquire_sys_u32(&own->slot[par][lane].seq) != want) {
      if (clock64() - t0 > 4000000000LL) { ok = false; break; }
    }
  }
  ok = __all_sync(0xffffffffu, ok);
  __threadfence_system();
  double acc = 0.0;
  int a0 = 0, a1 = 0;
  for (int r = 0; r < X.world; ++r) {
    if (lane < K) acc += ld_sys_f64(&own->slot[par][r].v[lane]);
    a0 += ld_sys_s32(&own->slot[par][r].cnt[0]);
    a1 += ld_sys_s32(&own->slot[par][r].cnt[1]);
  }
  val = acc; c0 = a0; c1 = a1;
  if (lane == 0) {
    *seq_smem = want;
    if (!ok) { own->err = 1u; seq_smem[1] = 1u; }
  }
  __syncwarp();
}

// Per-warp part of the H reduction: the 24 values (21 unique entries of sum_f Sxx aa^T + Sxy (ab^T + ba^T) + Syy bb^T, the
// feature count, two pads) of this warp's features, into dst[0..23] (shared memory): three transposed 8-value warp
// reductions.  `get(k, x, y, zi, sxx, sxy, syy, cnt)` yields feature k's data.
// ROLL (throughput geometry): ONE loop over the thread's features (a loop, not FPT copies: instruction-cache footprint), each
// feature's data and Jacobian rows formed once and added to all 24 accumulators.  Otherwise the sums are computed chunk by
// chunk, the loop unrolled, so that only ~8 accumulators are live at a time.  Every accumulator sees the same operands in
// the same order (feature 0, 1, ...) either way, so the partials are bit-identical.
template <int FPT, bool ROLL, class Get>
__device__ __forceinline__ void warp_h_partials(Get get, double* dst) {
  const int lane = threadIdx.x & 31;
  if constexpr (ROLL) {
    double v0[8], v1[8], v2[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) v0[j] = v1[j] = v2[j] = 0.0;
#pragma unroll 1
    for (int k = 0; k < FPT; ++k) {
      double x, y, zi, sxx, sxy, syy, cnt;
      get(k, x, y, zi, sxx, sxy, syy, cnt);
      double a[6], b[6];
      jac_rows(x, y, zi, a, b);
      h_chunk_add<0>(v0, a, b, sxx, sxy, syy, cnt);
      h_chunk_add<1>(v1, a, b, sxx, sxy, syy, cnt);
      h_chunk_add<2>(v2, a, b, sxx, sxy, syy, cnt);
    }
    warp_reduce_t<8>(v0);
    if ((lane & 3) == 0) dst[lane >> 2] = v0[0];
    warp_reduce_t<8>(v1);
    if ((lane & 3) == 0) dst[8 + (lane >> 2)] = v1[0];
    warp_reduce_t<8>(v2);
    if ((lane & 3) == 0) dst[16 + (lane >> 2)] = v2[0];
  } else {
    auto do_chunk = [&](auto chunk_tag) {
      constexpr int CH = decltype(chunk_tag)::value;
      double v[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = 0.0;
#pragma unroll(FPT)
      for (int k = 0; k < FPT; ++k) {
        double x, y, zi, sxx, sxy, syy, cnt;
        get(k, x, y, zi, sxx, sxy, syy, cnt);
        double a[6], b[6];
        jac_rows(x, y, zi, a, b);
        h_chunk_add<CH>(v, a, b, sxx, sxy, syy, cnt);
      }
      warp_reduce_t<8>(v);
      if ((lane & 3) == 0) dst[CH * 8 + (lane >> 2)] = v[0];
    };
    do_chunk(std::integral_constant<int, 0>{});
    do_chunk(std::integral_constant<int, 1>{});
    do_chunk(std::integral_constant<int, 2>{});
  }
}

// Named barrier `id` (not 0, which __syncthreads uses) of `n` threads: bar.arrive releases this thread's prior shared-memory
// writes to the threads that bar.sync on it and does not wait; bar.sync waits until all n have arrived.
__device__ __forceinline__ void named_bar_arrive(int id, int n) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ void named_bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
constexpr int kHsumBarrier = 1;  // the level's H partials (one CTA per pair)

// Programmatic dependent launch.  launch_dependents: once every CTA of this grid has executed it, a grid launched after it
// with cudaLaunchAttributeProgrammaticStreamSerialization may start its CTAs in the slots this grid's CTAs free.  wait: returns
// once the grid this one depends on has completed and its memory writes are visible (at once when launched without the attribute).
__device__ __forceinline__ void griddep_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// Sum of the 21 unique H entries + one count over the per-feature moments of the whole pair, once per level
// (and in the rare "slow path"): per-warp partials, one shared-memory hop, warp 0 adds the per-warp partials (and, in the
// cluster variant, the per-CTA sums every CTA received through DSMEM, after a cluster barrier).  On return the totals are in
// s.sums[0..23] of EVERY CTA of the pair, visible to warp 0 only (callers that need them elsewhere synchronise).
// (`sum_warp`: the warp that adds the per-warp partials and afterwards sees s.sums -- warp 0, or, one CTA per pair, another
// warp of the caller's choice.)
// ARRIVE (one CTA per pair): the other warps do not wait for the sum -- they arrive on a named barrier after writing their
// partials and return at once; only `sum_warp` waits on it.  The caller must keep s.hpart from being rewritten, and the
// barrier from being arrived on again, until `sum_warp` has summed (a block barrier that `sum_warp` reaches after it).
template <int FPT, int CS, bool XG, bool ROLL, class SH, bool ARRIVE = false, class Get>
__device__ __forceinline__ void pair_sum_h_to_warp0(Get get, SH& s, int nwarps, const XgParams& xg, int xg_pair, int sum_warp = 0) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  warp_h_partials<FPT, ROLL>(get, &s.hpart[warp * kPartK]);
  if constexpr (CS == 1 && ARRIVE) {
    if (warp != sum_warp) {
      named_bar_arrive(kHsumBarrier, nwarps * 32);
      return;
    }
    named_bar_sync(kHsumBarrier, nwarps * 32);
  } else {
    __syncthreads();
  }
  if constexpr (CS == 1) {
    if (warp == sum_warp) {
      double acc = 0.0;
      if (lane < kPartK)
        for (int wv = 0; wv < nwarps; ++wv) acc += s.hpart[wv * kPartK + lane];
      if (XG && xg.world > 1) {  // feature split over GPUs: the other ranks' partial sums arrive through peer memory
        int z0 = 0, z1 = 0;
        xg_allreduce<kPartK>(xg, xg_pair, &s.xg_seq, acc, z0, z1);
      }
      if (lane < kPartK) s.sums[lane] = acc;
      __syncwarp();
    }
  } else {
    const unsigned rank = cluster_rank();
    if (warp == 0 && lane < kPartK) {
      double acc = 0.0;
      for (int wv = 0; wv < nwarps; ++wv) acc += s.hpart[wv * kPartK + lane];
#pragma unroll
      for (int r = 0; r < CS; ++r) st_cluster_f64(&s.hsum_cta[rank][lane], (unsigned)r, acc);
    }
    pair_sync<CS>();
    if (warp == 0) {
      if (lane < kPartK) {
        double acc = 0.0;
#pragma unroll
        for (int r = 0; r < CS; ++r) acc += s.hsum_cta[r][lane];
        s.sums[lane] = acc;
      }
      __syncwarp();
    }
  }
}

// Warp 0: scale the 21 summed H entries into the full symmetric 6x6 `Hdst` and factorise it into `S`.
// Every lane runs the register-resident unpivoted LDL^T redundantly (same cost as one lane), lane 0 stores
// the factors; the pivoted Eigen-like fallback handles a degenerate H.
__device__ __forceinline__ void warp_scale_and_factor(const double* sums, double s2, double* Hdst, Solver6& S) {
  const int lane = threadIdx.x & 31;
  double h[21];
#pragma unroll
  for (int k = 0; k < 21; ++k) h[k] = sums[k] * s2;
  if (lane == 0) {
#pragma unroll
    for (int r = 0; r < 6; ++r)
#pragma unroll
      for (int c = r; c < 6; ++c) { Hdst[r * 6 + c] = h[upper_idx(r, c)]; Hdst[c * 6 + r] = h[upper_idx(r, c)]; }
  }
  Fact6 F;
  const bool ok = fact6_compute_upper(h, F);
  if (lane == 0) {
    if (ok) {
      S.F = F;
      S.pivoted = 0;
    } else {
      for (int k = 0; k < 36; ++k) S.ldl[k] = Hdst[k];
      ldlt6_factor(S.ldl, S.tr);
      S.pivoted = 1;
    }
  }
  __syncwarp();
}

// Tail of one NLLSSolver::optimizeGaussNewton iteration [EXT] -- solve, accept/rollback, update -- executed
// redundantly by EVERY thread of the pair on bit-identical inputs (tot[], n_in, the shared factorisation and the
// double-buffered state), so that all threads leave with the same new pose in registers and the same `done`.
// Thread 0 of every CTA (`cta_leader`) writes that CTA's state buffer of the next iteration; thread 0 of CTA rank 0
// (`leader`) also keeps the counters and the trace.
template <class SH>
__device__ __forceinline__ void gn_tail(SH& s, unsigned g, const Solver6* S, const double (&tot)[7], double jscale,
                                        int n_in, int iter, int level, double eps, bool cta_leader, bool leader, svo_b200_sia_iter* trace,
                                        int trace_cap, double& chi2_prev, int& stop, int& done, double (&R)[9],
                                        double (&t)[3]) {
#if SVO_SIA_DEBUG
  long long tg0 = clock64();
#endif
  const int n_meas = n_in * kPatchArea;
  const float chi2f = (float)tot[6];
  const double new_chi2 = (double)(chi2f / (float)n_meas);  // sparse_img_align.cpp:242 (NaN if 0)
  double x[6];
  if (S == nullptr) {  // Eigen's LDLT of an all-zero matrix solves to x = 0
#pragma unroll
    for (int k = 0; k < 6; ++k) x[k] = 0.0;
  } else if (!S->pivoted) {
    const Fact6 F = S->F;
    double b[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) b[k] = -(tot[k] * jscale);  // Jres_ = -sum J r
    fact6_solve(F, b, x);
  } else {
    double b[6];
    for (int k = 0; k < 6; ++k) b[k] = -(tot[k] * jscale);
    ldlt6_solve(S->ldl, S->tr, b);
    for (int k = 0; k < 6; ++k) x[k] = b[k];
  }
#if SVO_SIA_DEBUG
  long long tg1 = clock64() + (long long)(x[0] != x[0]) + (long long)(x[3] != x[3]);
#endif
  const SiaState& cur = s.st[g & 1u];
  const Pose model = cur.model;
  if (isnan(x[0])) stop = 1;  // solve() == 0 (:248-250); stop_ latches
  int accepted;
  Pose out;
  done = 0;
  if ((iter > 0 && new_chi2 > chi2_prev) || stop) {
    out = cur.old_model;  // rollback
    done = 1;
    accepted = 0;
    if (cta_leader) { s.st[(g + 1u) & 1u].model = out; s.st[(g + 1u) & 1u].old_model = out; }
  } else {
    double mx[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) mx[k] = -x[k];
    out = pose_mul_fast(model, se3_exp_fast(mx));  // T_new = T_old * exp(-x)  (:257)
    chi2_prev = new_chi2;
    accepted = 1;
    const double m = fmax(fmax(fmax(fabs(x[0]), fabs(x[1])), fmax(fabs(x[2]), fabs(x[3]))), fmax(fabs(x[4]), fabs(x[5])));
    if (m <= eps) done = 1;
    if (cta_leader) { s.st[(g + 1u) & 1u].model = out; s.st[(g + 1u) & 1u].old_model = model; }
  }
  qmatrix(out.q, R);
  t[0] = out.t[0]; t[1] = out.t[1]; t[2] = out.t[2];
#if SVO_SIA_DEBUG
  long long tg2 = clock64() + (long long)(R[0] != R[0]) + (long long)(t[0] != t[0]);
  if (leader) { s.tk[5] += tg1 - tg0; s.tk[6] += tg2 - tg1; }
#endif
  if (leader) {
    s.n_in_last = n_in;
    s.n_iters++;
    s.sum_in += n_in;
    if (trace) {
      if (s.n_trace < trace_cap) {
        svo_b200_sia_iter& r = trace[s.n_trace];
        r.level = level; r.iter = iter; r.accepted = accepted; r.n_meas = n_meas; r.chi2 = new_chi2;
        for (int k = 0; k < 6; ++k) r.x[k] = x[k];
        pose_to_rt12(out, r.T);
      }
      s.n_trace++;
    }
  }
}

// 4-byte asynchronous global->shared copy (LDGSTS): no register staging, completion per thread
__device__ __forceinline__ void cp_async4(void* dst_smem, const void* src_gmem) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(dst_smem)), "l"(src_gmem) : "memory");
}
__device__ __forceinline__ void cp_async8(void* dst_smem, const void* src_gmem) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_u32(dst_smem)), "l"(src_gmem) : "memory");
}
__device__ __forceinline__ void cp_async16(void* dst_smem, const void* src_gmem) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst_smem)), "l"(src_gmem) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
__device__ __forceinline__ void prefetch_l2_bulk(const void* p, uint32_t bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p), "r"(bytes) : "memory");
}

enum { kModeGlobal = 0, kModeImage = 1, kModeWindow = 2 };
static_assert(kModeGlobal == SVO_B200_SIA_STAGE_GLOBAL && kModeImage == SVO_B200_SIA_STAGE_IMAGE && kModeWindow == SVO_B200_SIA_STAGE_WINDOW,
              "the staging modes are reported through the ABI");

// How the current image of a W x Hh level reaches the residual loop: whole by one TMA copy when it fits the staging region
// (with 16 bytes to spare: the aligned-word fetches read past the last pixel), else -- in instantiations that have windows
// (`win`) -- one window per feature slot when the rows are 8-byte aligned and `slots` windows fit, else gathers from global
// memory.  The kernel and svo_b200_sia_last_launch both decide with this function.
__host__ __device__ __forceinline__ uint32_t sia_image_bytes(int W, int Hh) { return ((uint32_t)(W * Hh) + 15u) & ~15u; }
__host__ __device__ __forceinline__ int sia_stage_mode(uint32_t img_bytes, int W, int stage_cap, bool win, int slots) {
  int mode = kModeGlobal;
  if (img_bytes + 16u <= (uint32_t)stage_cap) mode = kModeImage;
  else if (win && (W & 7) == 0 && kWinBytes * slots <= stage_cap) mode = kModeWindow;
  return mode;
}

// xyz_cur = T_cur_from_ref * xyz_ref.  One CTA per pair (CS == 1): the pose is read from shared memory (s.pub, published by
// warp 0's Gauss-Newton tail) at the point of use -- six 128-bit shared loads per feature instead of 24 registers that stay
// live across the residual loops (at 128 registers per thread those were spilled to local memory, which misses the small L1
// left beside 3 x 75 KB of shared memory).  Cluster per pair: every
// warp runs the tail itself and keeps the pose in registers.
template <int CS>
__device__ __forceinline__ void sia_transform(const double* pub, const double (&R)[9], const double (&t)[3], double x, double y,
                                              double z, double& xc, double& yc, double& zc) {
  if constexpr (CS == 1) {
    double r[12];
    const uint32_t a = smem_u32(pub);
#pragma unroll
    for (int k = 0; k < 6; ++k)
      asm volatile("ld.shared.v2.f64 {%0, %1}, [%2];" : "=d"(r[2 * k]), "=d"(r[2 * k + 1]) : "r"(a + 16u * k));
    xc = fma(r[0], x, fma(r[1], y, fma(r[2], z, r[9])));
    yc = fma(r[3], x, fma(r[4], y, fma(r[5], z, r[10])));
    zc = fma(r[6], x, fma(r[7], y, fma(r[8], z, r[11])));
  } else {
    xc = fma(R[0], x, fma(R[1], y, fma(R[2], z, t[0])));
    yc = fma(R[3], x, fma(R[4], y, fma(R[5], z, t[1])));
    zc = fma(R[6], x, fma(R[7], y, fma(R[8], z, t[2])));
  }
}

template <bool CG>
__device__ __forceinline__ void sia_world2cam(const CamDev& c, double x, double y, double& u, double& v) {
  if constexpr (CG) {
    cam_world2cam(c, x, y, u, v);
  } else {  // undistorted pinhole (the host dispatches on svo_b200_camera: model == PINHOLE, no distortion)
    u = fma(c.fx, x, c.cx);
    v = fma(c.fy, y, c.cy);
  }
}

// Feature slots of the throughput geometry's shared arrays (the host selects it for at most this many features per pair).
constexpr int kSiaThroughputSlots = 304;

// One instantiation of sia_kernel (EVAL aside): its template arguments and the shared-memory layout that follows from them.
// The kernel finds its regions with it and the host (kSiaEntries) sizes and reports launches with it.
template <int FPT_, int MAXT_, int MINB_, int CS_, bool CG_, bool UP_>
struct SiaInst {
  static constexpr int FPT = FPT_, MAXT = MAXT_, MINB = MINB_, CS = CS_;
  static constexpr bool CG = CG_, UP = UP_;
  static constexpr int NWC = MAXT / 32;  // warps of one CTA; the host launches exactly MAXT threads
  // Throughput geometry (160 threads x 2 features, three CTAs per SM): the shared arrays are allocated for
  // kSiaThroughputSlots slots, which leaves room for the per-feature state xyz_ref in shared memory next to the two coarsest
  // current images.  Kept in registers that state was spilled at 128 registers per thread, and local memory misses the small
  // L1 left beside 3 x 75 KB of shared memory (each miss at the head of a feature's projection chain).
  static constexpr bool SS = FPT == 2 && MAXT == 160 && CS == 1;
  static constexpr int SA = SS ? kSiaThroughputSlots : MAXT * FPT;  // stride of the per-slot shared arrays
  // The throughput geometry has no room for windows (its staging region holds the two coarsest current images) and is never
  // used for the multi-GPU feature split: both code paths are compiled out of it, and its residual pass loops over the
  // thread's features instead of being unrolled -- the instruction stream of one Gauss-Newton iteration shrinks from ~27 KB to
  // ~20 KB, which matters with three CTAs in different phases sharing one instruction cache.
  static constexpr bool WIN = !SS;  // per-feature cp.async windows of the current image exist in this instantiation
  static constexpr bool XG = CS == 1 && !SS;  // multi-GPU feature split (svo_b200_sia_split_*) compiled in
  // The throughput geometry gathers from global memory -- the reference footprints of every level, the current footprints of
  // the levels not staged whole -- from the block-tiled copy of the level (two 16-byte and two 8-byte loads per 5x5 footprint
  // instead of ten 32-bit loads, 6.25 16-byte loads instead of ~12 8-byte ones per 7x7 one).  The other geometries stage windows or whole images and keep the
  // row-major gathers.
  static constexpr bool TL = SS;
  using SH = SiaSharedT<NWC, CS>;
  using UPT = SiaUpT<NWC, CS>;
  // dynamic shared memory: control block (SH, then UPT when UP), patch array sets, xyz_ref (SS), staging region
  static constexpr size_t kShBytes = (sizeof(SH) + 15) & ~size_t(15);
  static constexpr size_t kCtlBytes = kShBytes + (UP ? ((sizeof(UPT) + 15) & ~size_t(15)) : 0);
  static constexpr size_t kSetFloats = (size_t)3 * kPatchArea * SA;  // one set: SA slots of patch and gradients (sia_patch_chunk)
  static constexpr size_t kXyzDoubles = SS ? (size_t)3 * SA : 0;     // [3][SA] f64 xyz_ref
  // bytes in front of the staging region with n_sets patch array sets (1, or one per level when UP)
  static constexpr size_t fixed_bytes(int n_sets) {
    return kCtlBytes + (size_t)n_sets * kSetFloats * sizeof(float) + kXyzDoubles * sizeof(double);
  }
};

// One CTA (CS == 1) or one cluster of CS CTAs per frame pair; the pair's features are dealt to the CTAs in
// contiguous blocks of S = MAXT*FPT slots.
// (__launch_bounds__(160, 3) yields 128 registers although 3 x 160 x 136 <= 64 K: the register file is split over the
// four SM sub-partitions, 15 warps put 4 on one of them, and 4 warps x 32 lanes x 136 > 16 K.  Forcing 136 with
// __maxnreg__ drops the kernel to two CTAs per SM.  Issuing both features' reference-footprint loads before computing
// either patch makes the extra live registers spill.)
//
// CG = false compiles the projection for the undistorted pinhole only (px = fx * uv + cx): the general vk::AbstractCamera
// dispatch (radial-tangential pinhole, ATAN with its atan() slow path) stays out of the instruction stream of the
// residual loop, which is what BASELINE's synthetic camera and any rectified stream run.
//
// UP = true (cluster geometry, every CTA alone on its SM): patches / H / factorisations of all levels are computed before
// the first iteration (SiaUpT); shared memory then holds one patch array set per level.
template <int FPT, bool EVAL, int MAXT, int MINB, int CS, bool CG, bool UP>
__global__ void __launch_bounds__(MAXT, MINB) sia_kernel(const SiaParams P) {
  static_assert(!UP || (CS > 1 && FPT == 1 && !EVAL), "the upfront variant exists for the cluster geometry only");
  extern __shared__ __align__(16) unsigned char smem_raw[];
  using G = SiaInst<FPT, MAXT, MINB, CS, CG, UP>;
  using SH = typename G::SH;
  using UPT = typename G::UPT;
  SH& s = *reinterpret_cast<SH*>(smem_raw);
  constexpr int S = MAXT * FPT;  // feature slots of this CTA
  constexpr bool SS = G::SS;
  constexpr int SA = G::SA;
  constexpr bool WIN = G::WIN;
  constexpr bool XG = G::XG;
  constexpr bool TL = G::TL;
  UPT& up = *reinterpret_cast<UPT*>(smem_raw + G::kShBytes);  // only touched when UP
  const int n_lvl_bufs = UP ? (P.max_level - P.min_level + 1) : 1;  // patch array sets (one per level when UP)
  // the regions in the order of SiaInst::fixed_bytes (pointer steps in the regions' element types: stepping in bytes
  // instead changes the generated address arithmetic)
  float* const pat_base = reinterpret_cast<float*>(smem_raw + G::kCtlBytes);
  // set li (0 = coarsest level): each slot's reference patch and gradients as 16-byte chunks, addressed by sia_patch_chunk
  auto pat_of = [&](int li) -> uint8_t* { return reinterpret_cast<uint8_t*>(pat_base + (size_t)li * G::kSetFloats); };
  auto pchunk = [&](uint8_t* set, int slot, int c) -> float4* { return reinterpret_cast<float4*>(set + sia_patch_chunk(SA, slot, c)); };
  uint8_t* pat = pat_of(0);
  double* const st_xyz = reinterpret_cast<double*>(pat_base + (size_t)n_lvl_bufs * G::kSetFloats);  // SS: [3][SA] xyz_ref
  uint8_t* stage = reinterpret_cast<uint8_t*>(st_xyz + G::kXyzDoubles);  // 16-byte aligned
  uint4* win = reinterpret_cast<uint4*>(stage);                                                      // [kWinRows][SA] 16-byte window rows

  const unsigned crank = CS == 1 ? 0u : cluster_rank();
  const int pair = CS == 1 ? (int)blockIdx.x : (int)(blockIdx.x / CS);
  const SiaJob& job = P.jobs[pair];
  const int tid = threadIdx.x, T = blockDim.x, nwarps = (T + 31) >> 5;
  const int lane = tid & 31, warp = tid >> 5;
  const int fbase = (int)crank * S;  // first feature of this CTA
  const int N = job.n_feat;          // features of the pair
  const int np = job.n_pad;
  const bool cta_leader = tid == 0, leader = tid == 0 && crank == 0;
  // features of this CTA: [fbase, min(N, fbase + S)); their records are np_loc padded entries of the pair's blob
  const int n_loc = max(0, min(N - fbase, S));
  const int np_loc = (n_loc + 15) & ~15;

  // Throughput geometry: the next run of the same staged batch (svo_b200_sia_batch_run) may start its CTAs while this
  // launch's last wave drains; it reads nothing this launch writes, and orders its output stores after this launch (below).
  if constexpr (SS && !EVAL) griddep_launch_dependents();

  if (tid == 0) {
    mbar_init(&s.mbar, 1);
    mbar_init(&s.xbar[0], 1);
    mbar_init(&s.xbar[1], 1);
    fence_mbar_init();
    // ---- TMA: the packed feature records of this CTA's features, four bulk copies (px, f, pos, has_point
    //      sections of the pair's blob) into the (idle) patch arrays -- issued first, everything else this thread
    //      initialises runs in the shadow of that copy
    fence_proxy_async();
    if (np_loc > 0) {
      const uint32_t bytes = (uint32_t)np_loc * 65u;
      mbar_expect_tx(&s.mbar, bytes);
      uint8_t* dst = pat;
      const uint8_t* src = job.blob;
      tma_bulk_g2s(dst, src + (size_t)fbase * 16, (uint32_t)np_loc * 16u, &s.mbar);                                   // px
      tma_bulk_g2s(dst + (size_t)np_loc * 16, src + (size_t)np * 16 + (size_t)fbase * 24, (uint32_t)np_loc * 24u, &s.mbar);  // f
      tma_bulk_g2s(dst + (size_t)np_loc * 40, src + (size_t)np * 40 + (size_t)fbase * 24, (uint32_t)np_loc * 24u, &s.mbar);  // pos
      tma_bulk_g2s(dst + (size_t)np_loc * 64, src + (size_t)np * 64 + (size_t)fbase, (uint32_t)np_loc, &s.mbar);             // has_point
    } else {
      mbar_arrive(&s.mbar);  // a CTA without features still completes use 0 of the barrier: the phase parities of the image copies stay in step
    }
    s.st[0].model = pose_from_rt12(job.T);
    s.st[0].old_model = s.st[0].model;
    s.h_is_tot = 0; s.n_in_last = 0;
    s.n_iters = 0; s.sum_vis = 0; s.sum_in = 0; s.n_trace = 0;
    s.xg_seq = (CS == 1 && P.xg.world > 1) ? P.xg.peer[P.xg.rank][pair].xseq : 0u;
    s.xg_failed = 0u;
#if SVO_SIA_DEBUG
    for (int k = 0; k < 8; ++k) s.tk[k] = 0;
    for (int k = 0; k < 4; ++k) s.tkx[k] = 0;
    s.tk[4] = clock64();
#endif
    for (int k = 0; k < 36; ++k) s.Hs[k] = 0.0;
    // tiled copy of the running level's current image, read by the residual passes: the first level's here, every further
    // one at the end of the level before it
    if (TL) s.cur_tl = reinterpret_cast<const uint4*>(job.cur_tl[EVAL ? P.eval_level : P.max_level]);
  }
  __syncthreads();
  mbar_wait(&s.mbar, 0);
  const uint8_t* blob = pat;
  const double* b_f = reinterpret_cast<const double*>(blob) + 2 * np_loc;
  const double* b_pos = b_f + 3 * np_loc;
  const uint8_t* b_hp = reinterpret_cast<const uint8_t*>(b_pos + 3 * np_loc);

  // per-feature register state
  double fx_[FPT], fy_[FPT], fz_[FPT], fzi_[FPT];
  double fxs[FPT], fys[FPT], fzs[FPT];  // SS: copies that go to shared memory once the staged blob has been consumed
  int wx_[FPT], wy_[FPT];  // origin of the feature's current-image window (kModeWindow)
  unsigned hp_mask = 0, vis_mask = 0, in_mask = 0;
#pragma unroll
  for (int k = 0; k < FPT; ++k) {
    const int i = tid + k * T;
    fx_[k] = fy_[k] = 0.0; fz_[k] = fzi_[k] = 1.0;
    wx_[k] = wy_[k] = -(1 << 20);
    if (i < n_loc) {
      const double dxp = b_pos[3 * i] - job.ref_pos[0], dyp = b_pos[3 * i + 1] - job.ref_pos[1],
                   dzp = b_pos[3 * i + 2] - job.ref_pos[2];
      const double depth = sqrt(dxp * dxp + dyp * dyp + dzp * dzp);  // :107  |pos - ref_pos|
      fx_[k] = b_f[3 * i] * depth;                                    // :108  xyz_ref = f * depth
      fy_[k] = b_f[3 * i + 1] * depth;
      fz_[k] = b_f[3 * i + 2] * depth;
      fzi_[k] = 1.0 / fz_[k];
      if constexpr (SS) { fxs[k] = fx_[k]; fys[k] = fy_[k]; fzs[k] = fz_[k]; }
      if (b_hp[i]) hp_mask |= 1u << k;
      if (EVAL && P.visible_in[fbase + i]) vis_mask |= 1u << k;
    }
  }
  // solver state every thread carries (uniform over the pair): chi2_ and stop_ of NLLSSolver (reset(): 1e10 / false
  // [EXT]), the running iteration counter that selects the state / partial-sum buffers, and the current pose
  double chi2_prev = 1e10;
  int stop = 0;
  unsigned g = 0;
  double R[9], t[3];
  {
    const Pose m0 = pose_from_rt12(job.T);  // same arithmetic as thread 0's s.st[0].model
    qmatrix(m0.q, R);
    t[0] = m0.t[0]; t[1] = m0.t[1]; t[2] = m0.t[2];
    if (CS == 1 && tid == 0) {
#pragma unroll
      for (int k = 0; k < 9; ++k) s.pub[k] = R[k];
      s.pub[9] = t[0]; s.pub[10] = t[1]; s.pub[11] = t[2];
      s.pub_done = 0; s.pub_slow = 0;
    }
  }
  if constexpr (UP) {
    // Latency of a live pair is a chain of first-touch DRAM reads (reference footprints and current-image windows of every
    // level): all of them are known now -- the footprints exactly, the windows at the initial pose, which the
    // iterations move by a few pixels at most -- so every thread pulls its feature's rows of every level into L2 at once.
    // (Only here: with the CTA alone on its SM the extra L1 requests cost nothing; in the batched geometries they do.)
    const int i = tid;
    if (i < n_loc) {
      const double2 pxy = *reinterpret_cast<const double2*>(blob + (size_t)i * 16);
      double xc, yc, zc;
      sia_transform<CS>(s.pub, R, t, fx_[0], fy_[0], fz_[0], xc, yc, zc);
      const double rz = fast_rcp(zc);
      double ud, vd;
      sia_world2cam<CG>(P.cam, div_rn(xc, zc, rz), div_rn(yc, zc, rz), ud, vd);
      for (int level = P.max_level; level >= P.min_level; --level) {
        const int W = P.w[level], Hh = P.h[level];
        const double sc = 1.0 / (double)(1 << level);
        const int ur = (int)(pxy.x * sc), vr = (int)(pxy.y * sc);
        if (ur - 3 >= 0 && vr - 3 >= 0 && ur + 4 < W && vr + 4 < Hh) {
          const uint8_t* p0 = job.ref_lvl[level] + (size_t)(vr - 3) * W + (ur - 3);
#pragma unroll
          for (int r = 0; r < 7; ++r) prefetch_l2(p0 + (size_t)r * W);
        }
        const int uc = (int)(ud * sc), vc = (int)(vd * sc);
        if ((uint32_t)(W * Hh) + 32u > (uint32_t)P.stage_cap && uc - 4 >= 0 && vc - 4 >= 0 && uc + 4 < W && vc + 4 < Hh && ud >= 0.0 && vd >= 0.0) {
          const uint8_t* p0 = job.cur_lvl[level] + (size_t)(vc - 4) * W + (uc - 4);
#pragma unroll
          for (int r = 0; r < kWinRows; ++r) prefetch_l2(p0 + (size_t)r * W);
        }
      }
    }
    if (tid == 0 && crank == 0) {  // the coarse current images that are staged whole
      for (int level = P.max_level; level >= P.min_level; --level) {
        const uint32_t nb = ((uint32_t)(P.w[level] * P.h[level]) + 15u) & ~15u;
        if (nb + 16u <= (uint32_t)P.stage_cap) prefetch_l2_bulk(job.cur_lvl[level], nb);
      }
    }
  }
  pair_sync<CS>();  // everyone is done with the staged blob (the patch arrays may be written) and, in the cluster
                    // variant, every CTA's shared memory is initialised before remote stores arrive
    SIA_DBG(if ((SVO_SIA_DEBUG && P.debug) && tid == 0) s.tkx[3] = clock64() - s.tk[4];)
  if constexpr (SS) {
#pragma unroll
    for (int k = 0; k < FPT; ++k) {
      const int slot = tid + k * T;
      if (slot < n_loc) { st_xyz[slot] = fxs[k]; st_xyz[SA + slot] = fys[k]; st_xyz[2 * SA + slot] = fzs[k]; }
    }
  }
  // xyz_ref of feature k of this thread, and 1/z (SS: re-read from shared memory / recomputed, correctly rounded like the division)
  auto feat_xyz = [&](const int k, const int slot, double& x, double& y, double& z) {
    if constexpr (SS) {
      // slots without a feature (and the slots >= SA the last half-warp maps to) yield the neutral (0, 0, 1) the register
      // variant initialises: the H reduction multiplies their Jacobian rows by zero moments, which must stay finite
      x = 0.0; y = 0.0; z = 1.0;
      if (slot < n_loc) { x = st_xyz[slot]; y = st_xyz[SA + slot]; z = st_xyz[2 * SA + slot]; }
    } else { x = fx_[k]; y = fy_[k]; z = fz_[k]; }
  };
  auto feat_zi = [&](const int k, const double z) -> double {
    if constexpr (SS) return rcp_rn(z);
    else return fzi_[k];
  };

  // ---- one feature's window of the current image at this level (kModeWindow): 16 columns x 8 rows around the projection
  //      with the pose the level starts from, requested with cp.async (completion: cp_async_wait_all by the same thread)
  auto stage_window = [&](const int k, const int slot, const int W, const int Hh, const float scale, const uint8_t* cur_img) {
    double x, y, z;
    feat_xyz(k, slot, x, y, z);
    double xc, yc, zc;
    sia_transform<CS>(s.pub, R, t, x, y, z, xc, yc, zc);
    const double rz = fast_rcp(zc);
    double ud, vd;
    sia_world2cam<CG>(P.cam, div_rn(xc, zc, rz), div_rn(yc, zc, rz), ud, vd);
    const float u0 = __fmul_rn((float)ud, scale), v0 = __fmul_rn((float)vd, scale);
    if (u0 >= 0.f && v0 >= 0.f && u0 < 1e6f && v0 < 1e6f) {
      float tmp;
      const int cu = floor_pos(__fadd_rn(u0, 0.5f), tmp), cv = floor_pos(__fadd_rn(v0, 0.5f), tmp);
      {
        // 16 columns x 8 rows around (round(u), round(v)): the 5x5 footprint stays inside for at least +-1.5 px of
        // drift.  One 16-byte cp.async per row when columns round(u)-4 .. round(u)+3 fall into one 16-byte aligned
        // block (and the pitch keeps every row 16-byte aligned), else two 8-byte copies from the 8-byte aligned column.
        const int c4 = cu - 4, wy = cv - 4;
        const bool one = ((c4 & 15) <= 8) && (W & 15) == 0;
        const int wx = one ? (c4 & ~15) : (c4 & ~7);
        if (wx >= 0 && wy >= 0 && wx + 16 <= W && wy + kWinRows <= Hh) {
          wx_[k] = wx; wy_[k] = wy;
          const uint8_t* src = cur_img + (size_t)wy * W + wx;
          if (one) {
#pragma unroll
            for (int r = 0; r < kWinRows; ++r) cp_async16(win + r * SA + slot, src + (size_t)r * W);
          } else {
#pragma unroll
            for (int r = 0; r < kWinRows; ++r) {
              cp_async8(reinterpret_cast<uint8_t*>(win + r * SA + slot), src + (size_t)r * W);
              cp_async8(reinterpret_cast<uint8_t*>(win + r * SA + slot) + 8, src + (size_t)r * W + 8);
            }
          }
        }
      }
    }
  };
  // ---- gradient moments Sxx, Sxy, Syy of feature k of this thread if it is in `mask` (else zero), summed pixel by pixel
  //      from the gradients of patch array set `set` in shared memory; patch_moments: of all its features
  auto feat_moments = [&](uint8_t* set, const unsigned mask, const int k, double& sxx, double& sxy, double& syy) {
    sxx = sxy = syy = 0.0;
    if (!((mask >> k) & 1u)) return;
    const int slot = tid + k * T;
#pragma unroll
    for (int j = 0; j < 8; ++j) {  // gradient chunk j: pixels 2j, 2j + 1
      const float4 gr = *pchunk(set, slot, 4 + j);
      const double dx0 = (double)gr.x, dy0 = (double)gr.y, dx1 = (double)gr.z, dy1 = (double)gr.w;
      sxx = fma(dx0, dx0, sxx);
      sxy = fma(dx0, dy0, sxy);
      syy = fma(dy0, dy0, syy);
      sxx = fma(dx1, dx1, sxx);
      sxy = fma(dx1, dy1, sxy);
      syy = fma(dy1, dy1, syy);
    }
  };
  auto patch_moments = [&](uint8_t* set, const unsigned mask, double (&sxx)[FPT], double (&sxy)[FPT], double (&syy)[FPT]) {
#pragma unroll
    for (int k = 0; k < FPT; ++k) feat_moments(set, mask, k, sxx[k], sxy[k], syy[k]);
  };
  // ---- precomputeReferencePatches (:84-145) of one level into the patch array set `set`: visibility bits, the f32 patch and
  //      its gradients, and the per-feature gradient moments m_* the H reduction needs.  `with_windows`: also request the
  //      current-image windows (between the footprint loads and the arithmetic, so that both latencies overlap).
  //      Throughput geometry: the loop over the thread's features is not unrolled, so moments stored here would be indexed by
  //      the feature and live in local memory, which misses the small L1 left beside 3 x 75 KB of shared memory; it leaves
  //      m_* alone and the H sum takes them from the set with feat_moments(set, vis_mask) -- a visible patch has its
  //      gradients there (zero for a stale one), summed in the same order.  The other geometries unroll the loop and keep the moments of
  //      the patch arithmetic (a second pass over the gradients would lengthen the latency path of the cluster geometries).
  auto level_patches = [&](const int level, uint8_t* set, uint8_t* set_stale, const int mode, const bool with_windows,
                           double (&m_sxx)[FPT], double (&m_sxy)[FPT], double (&m_syy)[FPT]) {
    const int W = P.w[level], Hh = P.h[level];
    const float scale = 1.0f / (float)(1 << level);
    const uint8_t* ref_img = job.ref_lvl[level];
    const uint8_t* cur_img = job.cur_lvl[level];
    const uint4* ref_tl = reinterpret_cast<const uint4*>(job.ref_tl[level]);
#pragma unroll(SS ? 1 : FPT)
    for (int k = 0; k < FPT; ++k) {
      if constexpr (!SS) m_sxx[k] = m_sxy[k] = m_syy[k] = 0.0;
      const int slot = tid + k * T;
      // px is re-read from the pair's blob in global memory (L2) once per level instead of living in registers
      const double2 pxy = slot < n_loc ? __ldg(reinterpret_cast<const double2*>(job.blob) + fbase + slot) : make_double2(-1e6, -1e6);
      const float u_ref = (float)(pxy.x * (double)scale);
      const float v_ref = (float)(pxy.y * (double)scale);
      const bool rng = u_ref >= 0.f && v_ref >= 0.f && u_ref < 1e6f && v_ref < 1e6f;  // else: outside, floor not needed
      float ufl = 0.f, vfl = 0.f;
      const int ui = rng ? floor_pos(u_ref, ufl) : -1, vi = rng ? floor_pos(v_ref, vfl) : -1;
      const bool ok = ((hp_mask >> k) & 1u) && ui - 3 >= 0 && vi - 3 >= 0 && ui + 3 < W && vi + 3 < Hh;
      // all seven footprint rows are requested before anything else: one exposed L2/HBM latency per level
      uint32_t rlo[7], rhi[7];
      if (ok) {
        vis_mask |= 1u << k;
        if constexpr (TL) {
          fetch7x7_tiled(ref_tl, (W + 3) >> 2, ui - 3, vi - 3, rlo, rhi);
        } else {
#pragma unroll
          for (int r = 0; r < 7; ++r) fetch7_g64(ref_img, (vi - 3 + r) * W + (ui - 3), rlo[r], rhi[r]);
        }
      }
      // ---- current-image window of this feature (fine levels): projected with the pose the level starts from
      if constexpr (WIN) {
        if (with_windows) {
          wx_[k] = wy_[k] = -(1 << 20);
          if (((vis_mask >> k) & 1u) && mode == kModeWindow) stage_window(k, slot, W, Hh, scale, cur_img);
        }
      }
      if (ok) {
        float wtl, wtr, wbl, wbr;
        bilin_weights(__fsub_rn(u_ref, ufl), __fsub_rn(v_ref, vfl), wtl, wtr, wbl, wbr);
        // 7x7 footprint rows vi-3..vi+3, cols ui-3..ui+3, streamed row by row to keep the register
        // footprint small: Bq row r (bilinear blends with top-left tap P[r][c]) needs footprint rows
        // r, r+1; patch row y needs Bq rows y, y+1, y+2.
        float pr0[7], pr1[7], b0[6], b1[6], b2[6];
        double sxx = 0, sxy = 0, syy = 0;
        auto load_row = [&](int r, float (&dst)[7]) {
          const uint32_t lo = rlo[r], hi = rhi[r];
          dst[0] = byte_to_float<0>(lo); dst[1] = byte_to_float<1>(lo); dst[2] = byte_to_float<2>(lo);
          dst[3] = byte_to_float<3>(lo); dst[4] = byte_to_float<0>(hi); dst[5] = byte_to_float<1>(hi);
          dst[6] = byte_to_float<2>(hi);
        };
        load_row(0, pr0);
#pragma unroll
        for (int r = 0; r < 6; ++r) {
          load_row(r + 1, pr1);
#pragma unroll
          for (int c = 0; c < 6; ++c) b2[c] = bilin(wtl, wtr, wbl, wbr, pr0[c], pr0[c + 1], pr1[c], pr1[c + 1]);
          if (r >= 2) {  // rows b0 (= Bq[y]), b1 (= Bq[y+1]), b2 (= Bq[y+2]) with y = r-2 are complete
            const int y = r - 2;
            float dx[4], dy[4];
#pragma unroll
            for (int x = 0; x < 4; ++x) {
              dx[x] = __fmul_rn(0.5f, __fsub_rn(b1[x + 2], b1[x]));
              dy[x] = __fmul_rn(0.5f, __fsub_rn(b2[x + 1], b0[x + 1]));
              sxx = fma((double)dx[x], (double)dx[x], sxx);
              sxy = fma((double)dx[x], (double)dy[x], sxy);
              syy = fma((double)dy[x], (double)dy[x], syy);
            }
            *pchunk(set, slot, y) = make_float4(b1[1], b1[2], b1[3], b1[4]);
            *pchunk(set, slot, 4 + 2 * y) = make_float4(dx[0], dy[0], dx[1], dy[1]);
            *pchunk(set, slot, 5 + 2 * y) = make_float4(dx[2], dy[2], dx[3], dy[3]);
          }
#pragma unroll
          for (int c = 0; c < 6; ++c) { b0[c] = b1[c]; b1[c] = b2[c]; }
#pragma unroll
          for (int c = 0; c < 7; ++c) pr0[c] = pr1[c];
        }
        if constexpr (!SS) { m_sxx[k] = sxx; m_sxy[k] = sxy; m_syy[k] = syy; }
      } else if ((vis_mask >> k) & 1u) {
        // visible from a coarser level but failing here: the reference would keep the stale patch
        // and a zeroed Jacobian (jacobian_cache_.setZero() per level, :64).  Unreachable for
        // dyadic pyramids (SURVEY.md quirk 1) but kept bit-faithful.
#pragma unroll
        for (int j = 0; j < 8; ++j) *pchunk(set, slot, 4 + j) = make_float4(0.f, 0.f, 0.f, 0.f);
        if (set_stale)  // per-level arrays (upfront variant): the stale patch is the previous level's
          for (int y = 0; y < 4; ++y) *pchunk(set, slot, y) = *pchunk(set_stale, slot, y);
      }
    }
  };

  const int lvl_hi = EVAL ? P.eval_level : P.max_level;
  const int lvl_lo = EVAL ? P.eval_level : P.min_level;
  unsigned vis_levels = 0;  // UP: bit li = this thread's feature is visible at level lvl_hi - li (set-only across levels)
  unsigned img_phase = 0;   // parity of the most recent use of s.mbar (the blob copy of the prologue was use 0)
  if constexpr (UP) {
    SIA_DBG(long long tu0 = 0;)
      SIA_DBG(if ((SVO_SIA_DEBUG && P.debug) && tid == 0) tu0 = clock64();)
    // ---- all levels' reference patches and per-warp H partials, coarse to fine (the visibility mask accumulates in that order)
    for (int level = lvl_hi; level >= lvl_lo; --level) {
      const int li = lvl_hi - level;
      double m_sxx[FPT], m_sxy[FPT], m_syy[FPT];
      level_patches(level, pat_of(li), li > 0 ? pat_of(li - 1) : (uint8_t*)nullptr, kModeGlobal, false,
                    m_sxx, m_sxy, m_syy);
      vis_levels |= (vis_mask & 1u) << li;
      warp_h_partials<FPT, false>(
          [&](int k, double& x, double& y, double& zi, double& sxx, double& sxy, double& syy, double& cnt) {
            { double z_; feat_xyz(k, (int)threadIdx.x + k * (int)blockDim.x, x, y, z_); zi = feat_zi(k, z_); } sxx = sel_k(m_sxx, k); sxy = sel_k(m_sxy, k); syy = sel_k(m_syy, k); cnt = ((vis_mask >> k) & 1u) ? 1.0 : 0.0;
          },
          &up.hpart[li][warp * kPartK]);
    }
    __syncthreads();
    // ---- one exchange for all levels: every CTA receives every CTA's per-level sums (DSMEM), one cluster barrier
    const int nlv = lvl_hi - lvl_lo + 1;
    for (int e = tid; e < nlv * kPartK; e += T) {
      const int li = e / kPartK, j = e - li * kPartK;
      double acc = 0.0;
      for (int wv = 0; wv < nwarps; ++wv) acc += up.hpart[li][wv * kPartK + j];
#pragma unroll
      for (int r = 0; r < CS; ++r) st_cluster_f64(&up.hsum_cta[li][crank][j], (unsigned)r, acc);
    }
    pair_sync<CS>();
    // ---- every CTA scales and factorises its own copy, the levels dealt to its warps
    for (int li = warp; li < nlv; li += nwarps) {
      if (lane < kPartK) {
        double acc = 0.0;
#pragma unroll
        for (int r = 0; r < CS; ++r) acc += up.hsum_cta[li][r][lane];
        up.sums[li][lane] = acc;
      }
      __syncwarp();
      const double js = P.cam.fx / (double)(1 << (lvl_hi - li));
      warp_scale_and_factor(up.sums[li], js * js, up.Htot[li], up.sol[li]);
    }
    __syncthreads();
      SIA_DBG(if ((SVO_SIA_DEBUG && P.debug) && tid == 0) s.tkx[2] += clock64() - tu0;)
  }
  for (int level = lvl_hi; level >= lvl_lo; --level) {
    const int W = P.w[level], Hh = P.h[level];
    const float scale = 1.0f / (float)(1 << level);
    const double jscale = P.cam.fx / (double)(1 << level);  // focal_length / (1<<level_)  (:140)
    const uint8_t* cur_img = job.cur_lvl[level];

    // ---- how the current image of this level reaches the residual loop --------------------------
    const uint32_t img_bytes = sia_image_bytes(W, Hh);
    int mode = sia_stage_mode(img_bytes, W, P.stage_cap, WIN, SA);
    // Phase parity of this use of s.mbar, kept by every thread in a register (use k completes parity k & 1; the blob copy was
    // use 0).  NOT read from shared memory: in the upfront variant no barrier separates thread 0's update from the other
    // warps' wait, and a stale parity lets them through before the image has landed (found by running the tests under
    // compute-sanitizer, whose timing exposed it; `mode` is the same in all threads).
    if (mode == kModeImage) img_phase ^= 1u;
    if (mode == kModeImage && tid == 0) {
      fence_proxy_async();
      mbar_expect_tx(&s.mbar, img_bytes);
      tma_bulk_g2s(stage, cur_img, img_bytes, &s.mbar);
    }
    if (cta_leader) s.st[g & 1u].old_model = s.st[g & 1u].model;  // optimizeGaussNewton: ModelType old_model(model) [EXT]
    // next level: pull its current image (coarse levels, staged whole) into L2 while this level iterates
    if (tid == 0 && crank == 0 && level > lvl_lo) {
      const uint32_t nb = ((uint32_t)(P.w[level - 1] * P.h[level - 1]) + 15u) & ~15u;
      if (nb + 16u <= (uint32_t)P.stage_cap) prefetch_l2_bulk(job.cur_lvl[level - 1], nb);
    }

    SIA_DBG(long long tq0 = 0;)
      SIA_DBG(if ((SVO_SIA_DEBUG && P.debug) && tid == 0) tq0 = clock64();)
    SIA_DBG(long long tq1 = 0;)
    SIA_DBG(long long tq2 = 0;)
    const Solver6* sol_level = &s.sol_tot;  // factorisation of this level's H over its visible set
    const int fwarp = SS ? nwarps - 1 : 0;  // the warp that sums and factorises this level's H
    if constexpr (!UP) {
      // ---- precomputeReferencePatches (:84-145), one feature per thread; the windows of the current image are requested
      //      between the footprint loads and the patch arithmetic
      double m_sxx[FPT], m_sxy[FPT], m_syy[FPT];
      level_patches(level, pat, (uint8_t*)nullptr, mode, true, m_sxx, m_sxy, m_syy);
      SIA_DBG(if ((SVO_SIA_DEBUG && P.debug) && tid == 0) { tq1 = clock64(); s.tk[7] += tq1 - tq0; })
      // Only fwarp waits for the other warps' H partials (!EVAL: a named barrier the others arrive on and pass).  fwarp
      // reads s.hpart before it reaches barrier A of iteration 0, and nothing rewrites s.hpart -- the slow path's sum, the
      // next level's partials -- or arrives on the named barrier again before every warp has passed that barrier A
      // (n_iter == 0: the barrier at the end of the level).  sum_vis is fwarp's alone until the outputs.  EVAL keeps the block
      // barrier: it runs one pass of one level.
      pair_sum_h_to_warp0<FPT, CS, XG, SS, SH, !EVAL>(
          [&](int k, double& x, double& y, double& zi, double& sxx, double& sxy, double& syy, double& cnt) {
            { double z_; feat_xyz(k, (int)threadIdx.x + k * (int)blockDim.x, x, y, z_); zi = feat_zi(k, z_); }
            if constexpr (SS) feat_moments(pat, vis_mask, k, sxx, sxy, syy);
            else { sxx = sel_k(m_sxx, k); sxy = sel_k(m_sxy, k); syy = sel_k(m_syy, k); }
            cnt = ((vis_mask >> k) & 1u) ? 1.0 : 0.0;
            // opaque to the optimiser: otherwise the level-invariant Jacobian rows are hoisted out of the level loop and
            // parked in local memory (17 doubles per thread, written once and re-read every level)
            asm volatile("" : "+d"(x), "+d"(y), "+d"(zi));
          },
          s, nwarps, P.xg, pair, fwarp);
      // The scaling and LDL^T factorisation of this level's H is serial work nobody needs before the first solve: one warp
      // does it while the others already run the first residual pass; its results (s.sol_tot, s.Htot) become visible to
      // everybody through the barrier of that pass.  Throughput geometry: the LAST warp, which owns fewer features than the
      // others (44 of 300 against 64) and would reach that barrier early -- not warp 0, which runs the Gauss-Newton tail.
      SIA_DBG(if ((SVO_SIA_DEBUG && P.debug) && tid == 0) { tq2 = clock64(); s.tkx[0] += tq2 - tq1; })
      if (warp == fwarp) {
        if (lane == 0) s.sum_vis += (int)s.sums[21];
        warp_scale_and_factor(s.sums, jscale * jscale, s.Htot, s.sol_tot);
      }
    } else {
      // everything pose independent was prepared before the first level: select this level's arrays, request the windows
      const int li = lvl_hi - level;
      pat = pat_of(li);
      sol_level = &up.sol[li];
      vis_mask = (vis_levels >> li) & 1u;
#pragma unroll
      for (int k = 0; k < FPT; ++k) {
        wx_[k] = wy_[k] = -(1 << 20);
        if (((vis_mask >> k) & 1u) && mode == kModeWindow) stage_window(k, tid + k * T, W, Hh, scale, cur_img);
      }
      if (leader) s.sum_vis += (int)up.sums[li][21];
      SIA_DBG(if ((SVO_SIA_DEBUG && P.debug) && tid == 0) { tq1 = tq2 = clock64(); s.tk[7] += tq1 - tq0; })
    }
    if (mode == kModeImage) mbar_wait(&s.mbar, img_phase);
    if (mode == kModeWindow) cp_async_wait_all();  // each thread reads only the window it copied itself
      SIA_DBG(if ((SVO_SIA_DEBUG && P.debug) && tid == 0) { s.tk[0] += clock64() - tq0; s.tkx[1] += clock64() - tq2; })

    // ---- Gauss-Newton iterations at this level ---------------------------------------------
    const int n_iter = EVAL ? 1 : P.n_iter;
    for (int iter = 0; iter < n_iter; ++iter) {
      SIA_DBG(long long ti0 = 0;)
      SIA_DBG(if ((SVO_SIA_DEBUG && P.debug) && tid == 0) ti0 = clock64();)
      double acc[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) acc[k] = 0.0;
      int n_in_t = 0, n_out_t = 0;
      in_mask = 0;
#pragma unroll(SS ? 1 : FPT)
      for (int k = 0; k < FPT; ++k) {
        if (!((vis_mask >> k) & 1u)) continue;
        const int slot = tid + k * T;
        double x, y, z;
        feat_xyz(k, slot, x, y, z);
        double xc, yc, zc;
        sia_transform<CS>(s.pub, R, t, x, y, z, xc, yc, zc);
        const double rz = fast_rcp(zc);
        double ud, vd;
        sia_world2cam<CG>(P.cam, div_rn(xc, zc, rz), div_rn(yc, zc, rz), ud, vd);  // [EXT] world2cam(project2d(xyz))
        const float u_cur = __fmul_rn((float)ud, scale);  // .cast<float>() * scale (:183)
        const float v_cur = __fmul_rn((float)vd, scale);
        // negative / non-finite / huge coordinates can never pass the border test (:190)
        const bool rng = u_cur >= 0.f && v_cur >= 0.f && u_cur < 1e6f && v_cur < 1e6f;
        float ufl = 0.f, vfl = 0.f;
        const int ui = rng ? floor_pos(u_cur, ufl) : -1, vi = rng ? floor_pos(v_cur, vfl) : -1;
        const bool in = ui >= 0 && vi >= 0 && ui - 3 >= 0 && vi - 3 >= 0 && ui + 3 < W && vi + 3 < Hh;  // :190
        if (!in) {
          ++n_out_t;
          if (EVAL) {
            for (int p = 0; p < kPatchArea; ++p)
              P.residuals_out[(size_t)(fbase + slot) * kPatchArea + p] = __int_as_float(0x7fc00000);
          }
          continue;
        }
        in_mask |= 1u << k;
        ++n_in_t;
        float wtl, wtr, wbl, wbr;
        bilin_weights(__fsub_rn(u_cur, ufl), __fsub_rn(v_cur, vfl), wtl, wtr, wbl, wbr);
        uint32_t lo[5], hi[5];
        if (mode == kModeImage) {
#pragma unroll
          for (int r = 0; r < 5; ++r) fetch8<true>(stage, (vi - 2 + r) * W + (ui - 2), lo[r], hi[r]);
        } else {
          const int c0 = WIN ? (ui - 2) - wx_[SS ? 0 : k] : -1, r0 = WIN ? (vi - 2) - wy_[SS ? 0 : k] : -1;
          if (WIN && mode == kModeWindow && (unsigned)c0 <= 11u && (unsigned)r0 <= (unsigned)(kWinRows - 5)) {
            const uint4* wp = win + r0 * SA + slot;
            const int kw = c0 >> 2;  // 0..2: the footprint row starts in word kw of the 16-byte window row
            const unsigned sh = (unsigned)(c0 & 3) * 8u;
#pragma unroll
            for (int r = 0; r < 5; ++r) {
              const uint4 q = wp[r * SA];
              const uint32_t w0 = kw == 0 ? q.x : kw == 1 ? q.y : q.z, w1 = kw == 0 ? q.y : kw == 1 ? q.z : q.w;
              lo[r] = __funnelshift_r(w0, w1, sh);
              hi[r] = w1 >> sh;
            }
          } else if constexpr (TL) {
            // the copy's address is read from shared memory here, not kept in registers across the level
            fetch5x5_tiled(s.cur_tl, (W + 3) >> 2, ui - 2, vi - 2, lo, hi);
          } else {
#pragma unroll
            for (int r = 0; r < 5; ++r) fetch8<false>(cur_img, (vi - 2 + r) * W + (ui - 2), lo[r], hi[r]);
          }
        }
        float c2 = 0.f, gx = 0.f, gy = 0.f;
        float q0[5], q1[5];
        q0[0] = byte_to_float<0>(lo[0]); q0[1] = byte_to_float<1>(lo[0]); q0[2] = byte_to_float<2>(lo[0]);
        q0[3] = byte_to_float<3>(lo[0]); q0[4] = byte_to_float<0>(hi[0]);
#pragma unroll
        for (int yy = 0; yy < 4; ++yy) {
          q1[0] = byte_to_float<0>(lo[yy + 1]); q1[1] = byte_to_float<1>(lo[yy + 1]); q1[2] = byte_to_float<2>(lo[yy + 1]);
          q1[3] = byte_to_float<3>(lo[yy + 1]); q1[4] = byte_to_float<0>(hi[yy + 1]);
          // patch row yy: its values and gradients, three 128-bit loads (one row at a time: at most 12 more live floats)
          const float4 pv = *pchunk(pat, slot, yy), pg0 = *pchunk(pat, slot, 4 + 2 * yy), pg1 = *pchunk(pat, slot, 5 + 2 * yy);
          const float val_r[4] = {pv.x, pv.y, pv.z, pv.w};
          const float gx_r[4] = {pg0.x, pg0.z, pg1.x, pg1.z}, gy_r[4] = {pg0.y, pg0.w, pg1.y, pg1.w};
#pragma unroll
          for (int xx = 0; xx < 4; ++xx) {
            const int p = yy * 4 + xx;
            const float I = bilin(wtl, wtr, wbl, wbr, q0[xx], q0[xx + 1], q1[xx], q1[xx + 1]);
            const float res = __fsub_rn(I, val_r[xx]);
            c2 = fmaf(res, res, c2);  // chi2 += res*res*weight, weight == 1 (:222); order differs from the serial sum anyway
            gx = fmaf(gx_r[xx], res, gx);
            gy = fmaf(gy_r[xx], res, gy);
            if (EVAL) P.residuals_out[(size_t)(fbase + slot) * kPatchArea + p] = res;
          }
#pragma unroll
          for (int c = 0; c < 5; ++c) q0[c] = q1[c];
        }
        const double zi = feat_zi(k, z), X = x * zi, Y = y * zi, dgx = (double)gx, dgy = (double)gy;
        acc[0] = fma(-zi, dgx, acc[0]);
        acc[1] = fma(-zi, dgy, acc[1]);
        acc[2] = fma(zi, fma(X, dgx, Y * dgy), acc[2]);
        acc[3] = fma(X * Y, dgx, fma(fma(Y, Y, 1.0), dgy, acc[3]));
        acc[4] = fma(-fma(X, X, 1.0), dgx, fma(-(X * Y), dgy, acc[4]));
        acc[5] = fma(Y, dgx, fma(-X, dgy, acc[5]));
        acc[6] += (double)c2;
      }
      SIA_DBG(long long ti1 = 0;)
      SIA_DBG(if ((SVO_SIA_DEBUG && P.debug) && tid == 0) ti1 = clock64();)

      // ---- pair-wide sums: per-warp transposed reduction, one shared-memory hop, ONE barrier; then every warp adds
      //      the per-warp partials in the same order (bit-identical totals everywhere)
      const unsigned buf = g & 1u;
      warp_reduce_t<8>(acc);
      const int w_in = __reduce_add_sync(0xffffffffu, n_in_t), w_out = __reduce_add_sync(0xffffffffu, n_out_t);
      const int gw = (int)crank * nwarps + warp;  // warp index within the pair
      if constexpr (CS == 1) {
        if ((lane & 3) == 0) s.part[buf][gw][lane >> 2] = acc[0];
        if (lane == 0) { s.cnt[buf][gw][0] = w_in; s.cnt[buf][gw][1] = w_out; }
      } else if constexpr (UP) {
        // every CTA of the cluster receives every warp's partials by st.async: each store completes its 8 bytes on the
        // receiver's mbarrier of this parity, which one local thread arms with the byte count of all warps of the pair; the
        // receiver wakes when the last byte has landed -- one DSMEM hop, no cluster barrier.  (Two barriers: traffic of
        // iteration g+1 goes to the other one, and nobody can send g+2 before everybody has consumed g.)
        uint64_t* xb = &s.xbar[buf];
        if (tid == 0) mbar_expect_tx(xb, 72u * (uint32_t)(nwarps * CS));
        if ((lane & 3) == 0) {
#pragma unroll
          for (int r = 0; r < CS; ++r) st_async_f64(cluster_addr(&s.part[buf][gw][lane >> 2], (unsigned)r), acc[0], cluster_addr(xb, (unsigned)r));
        }
        if (lane == 0) {
#pragma unroll
          for (int r = 0; r < CS; ++r) st_async_v2s32(cluster_addr(&s.cnt[buf][gw][0], (unsigned)r), w_in, w_out, cluster_addr(xb, (unsigned)r));
        }
        mbar_wait(xb, (g >> 1) & 1u);
      } else {
        // per-level cluster flow: every CTA of the cluster receives every warp's partials (distributed shared memory stores)
        if ((lane & 3) == 0) {
#pragma unroll
          for (int r = 0; r < CS; ++r) st_cluster_f64(&s.part[buf][gw][lane >> 2], (unsigned)r, acc[0]);
        }
        if (lane == 0) {
#pragma unroll
          for (int r = 0; r < CS; ++r) st_cluster_v2s32(&s.cnt[buf][gw][0], (unsigned)r, w_in, w_out);
        }
      }
      if constexpr (!UP) pair_sync<CS>();  // barrier A: every warp's partial sums are in place
      // warps of the pair as a constant (the host launches exactly MAXT threads): the totals' loops below run one or two
      // steps per lane, and unrolled from a constant they leave the serial path without their loop control and remainders
      constexpr int nw_pair = G::NWC * CS;
      double tot[7];
      int n_in = 0, n_out = 0, done = 0;
      auto compute_totals = [&]() {
        const int kk = lane & 7;
        double a = 0.0;
        for (int wv = lane >> 3; wv < nw_pair; wv += 4) a += s.part[buf][wv][kk];
        a += __shfl_xor_sync(0xffffffffu, a, 8);
        a += __shfl_xor_sync(0xffffffffu, a, 16);
#pragma unroll
        for (int e = 0; e < 7; ++e) tot[e] = __shfl_sync(0xffffffffu, a, e);
        int ci = 0, co = 0;
        for (int wv = lane; wv < nw_pair; wv += 32) { ci += s.cnt[buf][wv][0]; co += s.cnt[buf][wv][1]; }
        n_in = __reduce_add_sync(0xffffffffu, ci);
        n_out = __reduce_add_sync(0xffffffffu, co);
      };
      // some visible patches fell outside the current image (or EVAL wants H): H_ = sum over the patches that
      // contributed in this pass ("slow path"; all threads, one block barrier inside)
      auto slow_sum_h = [&]() {
        double q_sxx[FPT], q_sxy[FPT], q_syy[FPT];
        if constexpr (!SS) patch_moments(pat, in_mask, q_sxx, q_sxy, q_syy);
        pair_sum_h_to_warp0<FPT, CS, XG, SS, SH>(
            [&](int k, double& x, double& y, double& zi, double& sxx, double& sxy, double& syy, double& cnt) {
              // a feature outside the image contributes nothing, also where its Jacobian rows are not finite (a point at
              // zero depth, or with f_z == 0): 1/z is selected away, the rows are then finite and the moments zero
              { double z_; feat_xyz(k, (int)threadIdx.x + k * (int)blockDim.x, x, y, z_); zi = feat_zi(k, z_); }
              if constexpr (SS) feat_moments(pat, in_mask, k, sxx, sxy, syy);
              else { sxx = sel_k(q_sxx, k); sxy = sel_k(q_sxy, k); syy = sel_k(q_syy, k); }
              cnt = 0.0;
              asm volatile("" : "+d"(x), "+d"(y), "+d"(zi));  // see the per-level call: no hoisting into local memory
              if (!((in_mask >> k) & 1u)) zi = 0.0;
            },
            s, nwarps, P.xg, pair);
      };
      auto eval_outputs = [&]() {  // EVAL, leader: computeResiduals' scalar outputs
        for (int k = 0; k < 6; ++k) P.Jres_out[k] = -(tot[k] * jscale);
        const float chi2f = (float)tot[6];
        *P.chi2_out = (double)(chi2f / (float)(n_in * kPatchArea));
        *P.n_meas_out = (long long)n_in * kPatchArea;
        s.n_in_last = n_in;
      };
      auto fast_path_solver = [&]() -> const Solver6* {  // every visible patch contributed: H_ is the level's H
        if (n_in == 0) {  // H_ == 0 exactly: Eigen's LDLT yields x = 0
          if (leader) {
            for (int k = 0; k < 36; ++k) s.Hs[k] = 0.0;
            s.h_is_tot = 0;
          }
          return nullptr;
        }
        if (leader) s.h_is_tot = 1;
        return sol_level;
      };
      SIA_DBG(long long ti2 = 0;)
      if constexpr (CS == 1) {
        // One CTA per pair: warp 0 alone adds the per-warp partials and runs the Gauss-Newton tail, then publishes the
        // new pose through shared memory (barrier B); the other warps would only replicate that work on the same SM.
        bool slow = false;
        if (warp == 0) {
          compute_totals();
          if (XG && P.xg.world > 1) {  // feature split over GPUs: sum the 7 doubles + 2 counts of this pass over the ranks
            double v = 0.0;
#pragma unroll
            for (int e = 0; e < 7; ++e) v = lane == e ? tot[e] : v;
            xg_allreduce<8>(P.xg, pair, &s.xg_seq, v, n_in, n_out);
#pragma unroll
            for (int e = 0; e < 7; ++e) tot[e] = __shfl_sync(0xffffffffu, v, e);
          }
      SIA_DBG(if ((SVO_SIA_DEBUG && P.debug) && tid == 0) { ti2 = clock64(); s.tk[1] += ti1 - ti0; s.tk[2] += ti2 - ti1; })
          slow = EVAL || (n_out > 0 && n_in > 0);
          if (!slow) {
            const Solver6* S6 = fast_path_solver();
            gn_tail(s, g, S6, tot, jscale, n_in, iter, level, P.eps, cta_leader, leader, P.trace, P.trace_cap, chi2_prev, stop,
                    done, R, t);
            if (lane == 0) {
#pragma unroll
              for (int k = 0; k < 9; ++k) s.pub[k] = R[k];
              s.pub[9] = t[0]; s.pub[10] = t[1]; s.pub[11] = t[2];
              s.pub_done = done;
            }
          }
          if (lane == 0) s.pub_slow = slow ? 1 : 0;
        }
        __syncthreads();  // barrier B
        if (s.pub_slow) {
          slow_sum_h();
          if (warp == 0) {
            warp_scale_and_factor(s.sums, jscale * jscale, s.Hs, s.sol_cur);
            if (leader) s.h_is_tot = 0;
            if (EVAL) {
              if (leader) eval_outputs();
            } else {
              gn_tail(s, g, &s.sol_cur, tot, jscale, n_in, iter, level, P.eps, cta_leader, leader, P.trace, P.trace_cap,
                      chi2_prev, stop, done, R, t);
              if (lane == 0) {
#pragma unroll
                for (int k = 0; k < 9; ++k) s.pub[k] = R[k];
                s.pub[9] = t[0]; s.pub[10] = t[1]; s.pub[11] = t[2];
                s.pub_done = done;
              }
            }
          }
          __syncthreads();  // barrier C
        }
        if (!EVAL) done = s.pub_done;  // the new pose stays in s.pub: sia_transform reads it there
      } else {
        // Cluster per pair: every warp of every CTA adds the partials in the same order and runs the tail redundantly in
        // registers (bit-identical everywhere), which saves a second cluster barrier + DSMEM broadcast per iteration.
        compute_totals();
      SIA_DBG(if ((SVO_SIA_DEBUG && P.debug) && tid == 0) { ti2 = clock64(); s.tk[1] += ti1 - ti0; s.tk[2] += ti2 - ti1; })
        const Solver6* S6;
        const bool slow = EVAL || (n_out > 0 && n_in > 0);
        if (!slow) {
          S6 = fast_path_solver();
        } else {
          slow_sum_h();
          if (warp == 0) {
            warp_scale_and_factor(s.sums, jscale * jscale, s.Hs, s.sol_cur);
            if (leader) s.h_is_tot = 0;
          }
          if (EVAL && leader) eval_outputs();
          __syncthreads();  // s.sol_cur is visible to every warp of this CTA (each CTA factorised its own copy)
          S6 = &s.sol_cur;
        }
        if (!EVAL)
          gn_tail(s, g, S6, tot, jscale, n_in, iter, level, P.eps, cta_leader, leader, P.trace, P.trace_cap, chi2_prev, stop,
                  done, R, t);
      }
      if (EVAL) {
#pragma unroll
        for (int k = 0; k < FPT; ++k) {
          const int i = tid + k * T;
          if (i < n_loc) {
            P.in_image_out[fbase + i] = (in_mask >> k) & 1u;
            if (!((vis_mask >> k) & 1u))
              for (int p = 0; p < kPatchArea; ++p)
                P.residuals_out[(size_t)(fbase + i) * kPatchArea + p] = __int_as_float(0x7fc00000);
            for (int y = 0; y < 4; ++y) {
              const float4 v = *pchunk(pat, i, y);
              float* o = P.ref_patch_out + (size_t)(fbase + i) * kPatchArea + 4 * y;
              o[0] = v.x; o[1] = v.y; o[2] = v.z; o[3] = v.w;
            }
          }
        }
        break;
      }
      ++g;
      SIA_DBG(if ((SVO_SIA_DEBUG && P.debug) && tid == 0) s.tk[3] += clock64() - ti2;)
      if (done) break;
    }
    // stage region / patches are rewritten by the next level; the leader's state writes are visible.  Upfront variant: only
    // CTA-local buffers are reused between levels (every level has its own patch arrays, the exchange buffers alternate by
    // the parity of the running iteration counter), so the CTAs of the pair need not meet here.
    // One CTA per pair: the barrier publishes the next level's s.cur_tl -- the warps that do not sum the level's H reach its
    // first residual pass without another barrier -- and, when n_iter == 0, orders the H sum against the next level's.
    if constexpr (UP) {
      __syncthreads();
    } else {
      if (TL && cta_leader && level > lvl_lo) s.cur_tl = reinterpret_cast<const uint4*>(job.cur_tl[level - 1]);
      pair_sync<CS>();
    }
  }
  if constexpr (UP) pair_sync<CS>();  // no CTA of the cluster exits while another may still write into its shared memory

  // ---- outputs ---------------------------------------------------------------------------------
  // Launched as a dependent of the previous run of its batch, this launch writes the same outputs: wait for that run to
  // complete.  These are the first global stores of the instantiation (the iteration trace is written only by the
  // single-pair svo_b200_sparse_img_align, whose launch is never a dependent).
  if constexpr (SS && !EVAL) griddep_wait();
#pragma unroll
  for (int k = 0; k < FPT; ++k) {
    const int i = tid + k * T;
    if (i < n_loc && P.visible_out) P.visible_out[job.feat_off + fbase + i] = (vis_mask >> k) & 1u;
  }
  if (leader) {
    if (P.T_out) pose_to_rt12(s.st[g & 1u].model, P.T_out + 12 * (size_t)pair);
    if (P.H_out)
      for (int k = 0; k < 36; ++k)  // H_ of the last residual pass: the level's H (of the finest level run) or the slow path's
        P.H_out[36 * (size_t)pair + k] = s.h_is_tot ? (UP ? up.Htot[lvl_hi - lvl_lo][k] : s.Htot[k]) : s.Hs[k];
    if (P.stats) {
      svo_b200_sia_stats st;
      st.n_iters = s.n_iters; st.sum_visible = s.sum_vis; st.sum_in_image = s.sum_in;
      st.n_tracked = s.n_in_last;  // n_meas_/patch_area_ of the last pass (:74)
      P.stats[pair] = st;
    }
    if (P.n_trace) *P.n_trace = s.n_trace;
    if (CS == 1 && P.xg.world > 1) P.xg.peer[P.xg.rank][pair].xseq = s.xg_seq;
#if SVO_SIA_DEBUG
    if (SVO_SIA_DEBUG && P.debug && (pair == 0 || pair == (int)(gridDim.x / CS) / 2 || pair == (int)(gridDim.x / CS) - 1))
      printf("[sia dbg] pair %d iters %d cycles: setup %lld pass %lld reduce %lld tail %lld (solve %lld update %lld) total %lld | setup parts: loads+patches %lld hsum %lld factor+wait %lld upfront %lld prologue %lld\n", pair, s.n_iters,
             s.tk[0], s.tk[1], s.tk[2], s.tk[3], s.tk[5], s.tk[6], (long long)clock64() - s.tk[4], s.tk[7], s.tkx[0], s.tkx[1], s.tkx[2], s.tkx[3]);
#endif
  }
}

// =============================================================================================
// Robust cost (NLLSSolver::setRobustCostFunction with MADScale; DESIGN.md 4.1c)
// =============================================================================================
// With a per-pixel weight H is no longer pose independent, so the factorisation of sia_kernel (H summed and factorised once
// per level) does not apply: this kernel re-sums the weighted H from per-feature weighted moments and factorises it in every
// iteration.  One CTA per pair, kSiaRobustThreads threads, features dealt round robin (feature i to thread i % T); the
// reference patches, gradients and xyz_ref of all the pair's features live in shared memory, the current image is read from
// global memory.  It is a kernel of its own so that the instantiations of sia_kernel keep their code.
constexpr int kSiaRobustThreads = 256;
constexpr int kSiaRobustWarps = kSiaRobustThreads / 32;
constexpr int kSiaRobustMaxFeat = 1024;

struct SiaRobustParams {
  SiaParams P;        // jobs, pyramid, camera, levels, iterations and the outputs of sia_kernel (EVAL fields unused)
  int weight;         // SVO_B200_WEIGHT_UNIT / _TUKEY / _HUBER
  int slots;          // stride of the per-feature shared arrays (>= the largest feature count of the batch)
  float* scales_out;  // [B][SVO_B200_MAX_LEVELS]: scale_ the iterations of each level used, NaN outside [min, max]
};

struct SiaRobustShared {
  SiaState st[2];                       // double-buffered by the running iteration counter, as in sia_kernel
  double part[kSiaRobustWarps][32];     // per-warp sums: 21 H entries, 6 Jres, chi2 (slots 28..31 unused)
  double sums[kPartK];                  // pair totals of the 21 H entries (warp_scale_and_factor reads them)
  double Hs[36];                        // H_ of the last pass (scaled, full symmetric)
  Solver6 sol;
  alignas(16) double pub[12];           // the pose warp 0 publishes after its Gauss-Newton tail
  unsigned hist[256];                   // radix-select histogram
  int cnt[kSiaRobustWarps];
  int n_in_last, n_iters, sum_vis, sum_in, n_trace;  // gn_tail's counters (thread 0)
  int pub_done, sel_bin, sel_k, n_pre;
#if SVO_SIA_DEBUG
  long long tk[8];
#endif
};
__host__ __device__ constexpr size_t sia_robust_ctl_bytes() { return (sizeof(SiaRobustShared) + 15) & ~size_t(15); }
// dynamic shared memory: control block, [16][SA] f32 reference patch, [16][SA] float2 gradients, [3][SA] f64 xyz_ref
__host__ __device__ constexpr size_t sia_robust_smem_bytes(int slots) {
  return sia_robust_ctl_bytes() + (size_t)slots * (kPatchArea * (sizeof(float) + sizeof(float2)) + 3 * sizeof(double));
}

// [EXT] vk::robust_cost weight functions restated in f32 (oracle/svo_oracle_robust.cpp): x = res / scale_.
__device__ __forceinline__ float robust_weight(int wf, float res, float scale) {
  const float x = __fdiv_rn(res, scale);
  if (wf == SVO_B200_WEIGHT_TUKEY) {  // b = 4.6851
    constexpr float b2 = 4.6851f * 4.6851f;
    const float x2 = __fmul_rn(x, x);
    if (x2 <= b2) {
      const float tmp = __fsub_rn(1.0f, __fdiv_rn(x2, b2));
      return __fmul_rn(tmp, tmp);
    }
    return 0.0f;  // also for x = +-inf and NaN
  }
  if (wf == SVO_B200_WEIGHT_HUBER) {  // k = 1.345: NaN for x = NaN (0 / 0)
    const float t = fabsf(x);
    return t < 1.345f ? 1.0f : __fdiv_rn(1.345f, t);
  }
  return 1.0f;
}

__global__ void __launch_bounds__(kSiaRobustThreads, 1) sia_robust_kernel(const SiaRobustParams RP) {
  const SiaParams& P = RP.P;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  SiaRobustShared& s = *reinterpret_cast<SiaRobustShared*>(smem_raw);
  const int SA = RP.slots;
  float* const pat_ref = reinterpret_cast<float*>(smem_raw + sia_robust_ctl_bytes());  // [16][SA]
  float2* const pat_dxy = reinterpret_cast<float2*>(pat_ref + kPatchArea * SA);        // [16][SA]
  double* const xyz = reinterpret_cast<double*>(pat_dxy + kPatchArea * SA);            // [3][SA]
  constexpr int T = kSiaRobustThreads, FPT = kSiaRobustMaxFeat / kSiaRobustThreads;
  const int pair = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const SiaJob& job = P.jobs[pair];
  const int N = job.n_feat, np = job.n_pad;
  const bool leader = tid == 0;
  const double* b_px = reinterpret_cast<const double*>(job.blob);
  const double* b_f = b_px + 2 * np;
  const double* b_pos = b_f + 3 * np;
  const uint8_t* b_hp = reinterpret_cast<const uint8_t*>(b_pos + 3 * np);

  // No features: run() returns before it touches anything (:47-51), as svo_b200_sparse_img_align does without a launch --
  // the pose exactly as given (no quaternion round trip), H and the stats 0, no level run (scales NaN).  N is the same in
  // every thread of the CTA, so the whole CTA leaves before its first barrier.
  if (N == 0) {
    if (leader) {
      if (P.T_out)
        for (int k = 0; k < 12; ++k) P.T_out[12 * (size_t)pair + k] = job.T[k];
      if (P.H_out)
        for (int k = 0; k < 36; ++k) P.H_out[36 * (size_t)pair + k] = 0.0;
      if (P.stats) P.stats[pair] = svo_b200_sia_stats{};
      if (RP.scales_out)
        for (int l = 0; l < SVO_B200_MAX_LEVELS; ++l) RP.scales_out[(size_t)pair * SVO_B200_MAX_LEVELS + l] = __int_as_float(0x7fc00000);
      if (P.n_trace) *P.n_trace = 0;
    }
    return;
  }

  // xyz_ref = f * |pos - ref_pos| (:107-108), as sia_kernel forms it
  for (int i = tid; i < N; i += T) {
    const double dxp = b_pos[3 * i] - job.ref_pos[0], dyp = b_pos[3 * i + 1] - job.ref_pos[1], dzp = b_pos[3 * i + 2] - job.ref_pos[2];
    const double depth = sqrt(dxp * dxp + dyp * dyp + dzp * dzp);
    xyz[i] = b_f[3 * i] * depth;
    xyz[SA + i] = b_f[3 * i + 1] * depth;
    xyz[2 * SA + i] = b_f[3 * i + 2] * depth;
  }
  double R[9], t[3];
  if (leader) {
    s.st[0].model = pose_from_rt12(job.T);
    s.st[0].old_model = s.st[0].model;
    s.n_in_last = 0; s.n_iters = 0; s.sum_vis = 0; s.sum_in = 0; s.n_trace = 0;
    for (int k = 0; k < 36; ++k) s.Hs[k] = 0.0;
    qmatrix(s.st[0].model.q, R);
    for (int k = 0; k < 9; ++k) s.pub[k] = R[k];
    for (int k = 0; k < 3; ++k) s.pub[9 + k] = s.st[0].model.t[k];
    if (RP.scales_out)
      for (int l = 0; l < SVO_B200_MAX_LEVELS; ++l) RP.scales_out[(size_t)pair * SVO_B200_MAX_LEVELS + l] = __int_as_float(0x7fc00000);
  }
  __syncthreads();
  auto load_pose = [&]() {
#pragma unroll
    for (int k = 0; k < 9; ++k) R[k] = s.pub[k];
    t[0] = s.pub[9]; t[1] = s.pub[10]; t[2] = s.pub[11];
  };
  load_pose();

  // The feature's 16 residuals at the current pose (computeResiduals :179-210): false if the patch is outside the current
  // image (:190).  emit(p, res, gradient) per pixel.
  auto residuals = [&](int i, int W, int Hh, float scale, const uint8_t* cur_img, auto emit) -> bool {
    const double x = xyz[i], y = xyz[SA + i], z = xyz[2 * SA + i];
    const double xc = fma(R[0], x, fma(R[1], y, fma(R[2], z, t[0])));
    const double yc = fma(R[3], x, fma(R[4], y, fma(R[5], z, t[1])));
    const double zc = fma(R[6], x, fma(R[7], y, fma(R[8], z, t[2])));
    const double rz = fast_rcp(zc);
    double ud, vd;
    cam_world2cam(P.cam, div_rn(xc, zc, rz), div_rn(yc, zc, rz), ud, vd);
    const float u_cur = __fmul_rn((float)ud, scale), v_cur = __fmul_rn((float)vd, scale);
    const bool rng = u_cur >= 0.f && v_cur >= 0.f && u_cur < 1e6f && v_cur < 1e6f;
    float ufl = 0.f, vfl = 0.f;
    const int ui = rng ? floor_pos(u_cur, ufl) : -1, vi = rng ? floor_pos(v_cur, vfl) : -1;
    if (!(ui - 3 >= 0 && vi - 3 >= 0 && ui + 3 < W && vi + 3 < Hh)) return false;
    float wtl, wtr, wbl, wbr;
    bilin_weights(__fsub_rn(u_cur, ufl), __fsub_rn(v_cur, vfl), wtl, wtr, wbl, wbr);
    uint32_t lo[5], hi[5];
#pragma unroll
    for (int r = 0; r < 5; ++r) fetch8<false>(cur_img, (vi - 2 + r) * W + (ui - 2), lo[r], hi[r]);
    float q0[5], q1[5];
    q0[0] = byte_to_float<0>(lo[0]); q0[1] = byte_to_float<1>(lo[0]); q0[2] = byte_to_float<2>(lo[0]);
    q0[3] = byte_to_float<3>(lo[0]); q0[4] = byte_to_float<0>(hi[0]);
#pragma unroll
    for (int yy = 0; yy < 4; ++yy) {
      q1[0] = byte_to_float<0>(lo[yy + 1]); q1[1] = byte_to_float<1>(lo[yy + 1]); q1[2] = byte_to_float<2>(lo[yy + 1]);
      q1[3] = byte_to_float<3>(lo[yy + 1]); q1[4] = byte_to_float<0>(hi[yy + 1]);
#pragma unroll
      for (int xx = 0; xx < 4; ++xx) {
        const int p = yy * 4 + xx;
        const float I = bilin(wtl, wtr, wbl, wbr, q0[xx], q0[xx + 1], q1[xx], q1[xx + 1]);
        emit(p, __fsub_rn(I, pat_ref[p * SA + i]), pat_dxy[p * SA + i]);
      }
#pragma unroll
      for (int c = 0; c < 5; ++c) q0[c] = q1[c];
    }
    return true;
  };

  double chi2_prev = 1e10;  // chi2_ of NLLSSolver::reset() [EXT]
  int stop = 0;
  unsigned g = 0;
  float wscale = 0.0f;   // scale_ (NLLSSolver() initialises it to 0 [EXT])
  int iter_end = 0;      // iter_ as the previous level's loop left it (reset(): 0)
  long long n_meas_pre = 0;  // n_meas_ counted by the pre-calls (reset only by the loop)
  unsigned vis_mask = 0;     // bit k: feature tid + k T is visible (set-only across levels, :57)
  for (int level = P.max_level; level >= P.min_level; --level) {
    const int W = P.w[level], Hh = P.h[level];
    const float scale = 1.0f / (float)(1 << level);
    const double jscale = P.cam.fx / (double)(1 << level);
    const uint8_t* ref_img = job.ref_lvl[level];
    const uint8_t* cur_img = job.cur_lvl[level];
    // ---- precomputeReferencePatches (:84-145)
    int n_vis_t = 0;
#pragma unroll 1
    for (int k = 0; k < FPT; ++k) {
      const int i = tid + k * T;
      if (i >= N) break;
      const float u_ref = (float)(b_px[2 * i] * (double)scale), v_ref = (float)(b_px[2 * i + 1] * (double)scale);
      const bool rng = u_ref >= 0.f && v_ref >= 0.f && u_ref < 1e6f && v_ref < 1e6f;
      float ufl = 0.f, vfl = 0.f;
      const int ui = rng ? floor_pos(u_ref, ufl) : -1, vi = rng ? floor_pos(v_ref, vfl) : -1;
      if (b_hp[i] && ui - 3 >= 0 && vi - 3 >= 0 && ui + 3 < W && vi + 3 < Hh) {
        vis_mask |= 1u << k;
        uint32_t rlo[7], rhi[7];
#pragma unroll
        for (int r = 0; r < 7; ++r) fetch7_g64(ref_img, (vi - 3 + r) * W + (ui - 3), rlo[r], rhi[r]);
        ref_patch_7x7(rlo, rhi, __fsub_rn(u_ref, ufl), __fsub_rn(v_ref, vfl), [&](int p, float val, float dx, float dy) {
          pat_ref[p * SA + i] = val;
          pat_dxy[p * SA + i] = make_float2(dx, dy);
        });
      } else if ((vis_mask >> k) & 1u) {  // visible at a coarser level only: stale patch, zero Jacobian (as sia_kernel)
        for (int p = 0; p < kPatchArea; ++p) pat_dxy[p * SA + i] = make_float2(0.f, 0.f);
      }
      n_vis_t += (vis_mask >> k) & 1u;
    }
    n_vis_t = __reduce_add_sync(0xffffffffu, n_vis_t);
    if (lane == 0) s.cnt[warp] = n_vis_t;
    if (leader) s.st[g & 1u].old_model = s.st[g & 1u].model;
    __syncthreads();
    if (leader) for (int w = 0; w < kSiaRobustWarps; ++w) s.sum_vis += s.cnt[w];

    // ---- the pre-call computeResiduals(model, false, true) of optimizeGaussNewton [EXT]: counts n_meas_ and, when iter_ is
    //      0 (:239), sets scale_ = 1.48 * the upper median of |res| (MAD) -- an exact MSB-first radix select on the bit
    //      patterns of the non-negative f32 |res| (ordered like the values), 8 bits per sweep; every sweep recomputes the
    //      residuals instead of storing 16 N of them.
    {
      const bool want_scale = iter_end == 0;
      unsigned prefix = 0, pmask = 0;
      int kth = 0;
      for (int sweep = 0; sweep < (want_scale ? 4 : 1); ++sweep) {
        const int shift = 24 - 8 * sweep;
        for (int b = tid; b < 256; b += T) s.hist[b] = 0u;
        __syncthreads();
        int n_in_t = 0;
#pragma unroll 1
        for (int k = 0; k < FPT; ++k) {
          const int i = tid + k * T;
          if (i >= N) break;
          if (!((vis_mask >> k) & 1u)) continue;
          n_in_t += residuals(i, W, Hh, scale, cur_img, [&](int, float res, float2) {
            const unsigned key = __float_as_uint(fabsf(res));
            if (want_scale && (key & pmask) == prefix) atomicAdd(&s.hist[(key >> shift) & 255u], 1u);
          });
        }
        if (sweep == 0) {
          n_in_t = __reduce_add_sync(0xffffffffu, n_in_t);
          if (lane == 0) s.cnt[warp] = n_in_t;
        }
        __syncthreads();
        if (sweep == 0) {
          int n = 0;
          for (int w = 0; w < kSiaRobustWarps; ++w) n += s.cnt[w];
          if (leader) s.n_pre = n;
          n_meas_pre += (long long)n * kPatchArea;
          // getMedian of no errors is undefined in the reference: scale_ stays (not pinned).  n is the same in every thread;
          // the barrier keeps s.cnt from being rewritten (the first pass below, or the next level's precompute when n_iter
          // is 0) before every warp has read it here
          if (n == 0 || !want_scale) { __syncthreads(); break; }
          kth = n * kPatchArea / 2;  // vk::getMedian: nth_element at floor(n / 2)
        }
        if (warp == 0) {  // lane l scans bins [8 l, 8 l + 8)
          unsigned loc[8], sum = 0;
#pragma unroll
          for (int j = 0; j < 8; ++j) { loc[j] = s.hist[8 * lane + j]; sum += loc[j]; }
          unsigned inc = sum;
#pragma unroll
          for (int o = 1; o < 32; o <<= 1) {
            const unsigned v = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += v;
          }
          const unsigned hit = __ballot_sync(0xffffffffu, inc > (unsigned)kth);
          if (lane == __ffs(hit) - 1) {
            unsigned cum = inc - sum;
            int bin = 8 * lane;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              if (cum + loc[j] > (unsigned)kth) { bin = 8 * lane + j; break; }
              cum += loc[j];
            }
            s.sel_bin = bin;
            s.sel_k = kth - (int)cum;
          }
        }
        __syncthreads();
        prefix |= (unsigned)s.sel_bin << shift;
        pmask |= 255u << shift;
        kth = s.sel_k;
        if (sweep == 3) wscale = __fmul_rn(1.48f, __uint_as_float(prefix));  // MADScaleEstimator [EXT]
        __syncthreads();  // s.sel_* and s.hist are rewritten by the next sweep
      }
    }
    if (leader && RP.scales_out) RP.scales_out[(size_t)pair * SVO_B200_MAX_LEVELS + level] = wscale;

    // ---- Gauss-Newton iterations: every pass re-sums the weighted H and factorises it
    iter_end = P.n_iter;
    for (int iter = 0; iter < P.n_iter; ++iter) {
      double acc[32];
#pragma unroll
      for (int e = 0; e < 32; ++e) acc[e] = 0.0;
      int n_in_t = 0;
#pragma unroll 1
      for (int k = 0; k < FPT; ++k) {
        const int i = tid + k * T;
        if (i >= N) break;
        if (!((vis_mask >> k) & 1u)) continue;
        // weighted moments of the patch: sum w dx^2, w dx dy, w dy^2, w dx r, w dy r (f64) and chi2 += res^2 w (f32, :222)
        double sxx = 0.0, sxy = 0.0, syy = 0.0, sxr = 0.0, syr = 0.0;
        float c2 = 0.f;
        const bool in = residuals(i, W, Hh, scale, cur_img, [&](int, float res, float2 gr) {
          const float w = robust_weight(RP.weight, res, wscale);
          c2 = fmaf(__fmul_rn(res, res), w, c2);
          const double wd = (double)w, dx = (double)gr.x, dy = (double)gr.y, r = (double)res;
          sxx = fma(wd * dx, dx, sxx);
          sxy = fma(wd * dx, dy, sxy);
          syy = fma(wd * dy, dy, syy);
          sxr = fma(wd * dx, r, sxr);
          syr = fma(wd * dy, r, syr);
        });
        if (!in) continue;
        ++n_in_t;
        const double z = xyz[2 * SA + i];
        double a[6], b[6];
        jac_rows(xyz[i], xyz[SA + i], rcp_rn(z), a, b);
#define SIA_ROBUST_H(IDX) acc[IDX] += h_entry<IDX>(a, b, sxx, sxy, syy);
        SIA_ROBUST_H(0) SIA_ROBUST_H(1) SIA_ROBUST_H(2) SIA_ROBUST_H(3) SIA_ROBUST_H(4) SIA_ROBUST_H(5) SIA_ROBUST_H(6)
        SIA_ROBUST_H(7) SIA_ROBUST_H(8) SIA_ROBUST_H(9) SIA_ROBUST_H(10) SIA_ROBUST_H(11) SIA_ROBUST_H(12) SIA_ROBUST_H(13)
        SIA_ROBUST_H(14) SIA_ROBUST_H(15) SIA_ROBUST_H(16) SIA_ROBUST_H(17) SIA_ROBUST_H(18) SIA_ROBUST_H(19) SIA_ROBUST_H(20)
#undef SIA_ROBUST_H
#pragma unroll
        for (int e = 0; e < 6; ++e) acc[21 + e] = fma(a[e], sxr, fma(b[e], syr, acc[21 + e]));
        acc[27] += (double)c2;
      }
      // ---- pair sums: four transposed 8-value warp reductions, one shared-memory hop, warp 0 adds the warps' partials
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        double v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = acc[8 * c + j];
        warp_reduce_t<8>(v);
        if ((lane & 3) == 0) s.part[warp][8 * c + (lane >> 2)] = v[0];
      }
      n_in_t = __reduce_add_sync(0xffffffffu, n_in_t);
      if (lane == 0) s.cnt[warp] = n_in_t;
      __syncthreads();
      if (warp == 0) {
        double tot_l = 0.0;
        int n_in = 0;
        for (int w = 0; w < kSiaRobustWarps; ++w) { tot_l += s.part[w][lane]; n_in += s.cnt[w]; }
        if (lane < 21) s.sums[lane] = tot_l;
        double tot[7];
#pragma unroll
        for (int e = 0; e < 7; ++e) tot[e] = __shfl_sync(0xffffffffu, tot_l, 21 + e);
        __syncwarp();
        warp_scale_and_factor(s.sums, jscale * jscale, s.Hs, s.sol);
        int done = 0;
        gn_tail(s, g, &s.sol, tot, jscale, n_in, iter, level, P.eps, leader, leader, P.trace, P.trace_cap, chi2_prev, stop, done,
                R, t);
        if (lane == 0) {
#pragma unroll
          for (int k = 0; k < 9; ++k) s.pub[k] = R[k];
          s.pub[9] = t[0]; s.pub[10] = t[1]; s.pub[11] = t[2];
          s.pub_done = done;
        }
      }
      __syncthreads();
      load_pose();
      const int done = s.pub_done;  // (chi2_ and stop_ live in warp 0, which alone runs the tail)
      ++g;
      __syncthreads();  // s.pub_done / s.part are rewritten by the next pass
      if (done) { iter_end = iter; break; }
    }
  }

  // ---- outputs
#pragma unroll 1
  for (int k = 0; k < FPT; ++k) {
    const int i = tid + k * T;
    if (i < N && P.visible_out) P.visible_out[job.feat_off + i] = (vis_mask >> k) & 1u;
  }
  if (leader) {
    if (P.T_out) pose_to_rt12(s.st[g & 1u].model, P.T_out + 12 * (size_t)pair);
    if (P.H_out)
      for (int k = 0; k < 36; ++k) P.H_out[36 * (size_t)pair + k] = s.Hs[k];
    if (P.stats) {
      svo_b200_sia_stats st;
      st.n_iters = s.n_iters; st.sum_visible = s.sum_vis; st.sum_in_image = s.sum_in;
      // run() returns n_meas_ / patch_area_ (:74): the last pass's count, or -- no iteration ran at all -- what the pre-calls
      // of every level added up (only the loop resets n_meas_)
      st.n_tracked = P.n_iter > 0 ? s.n_in_last : (int)(n_meas_pre / kPatchArea);
      P.stats[pair] = st;
    }
    if (P.n_trace) *P.n_trace = s.n_trace;
  }
}

// =============================================================================================
// Host side
// =============================================================================================
using SiaKernel = void (*)(SiaParams);

// What the host needs of one alignment instantiation (SiaInst), and its kernels.
struct SiaEntry {
  int fpt, threads, min_blocks, cluster;              // FPT, MAXT (the block size), MINB (resident CTAs per SM), CS
  bool general_camera, upfront, throughput, windows;  // CG, UP, SS, WIN
  int slots;                                          // SA
  size_t (*fixed_bytes)(int n_sets);
  SiaKernel kern[2];  // EVAL = false / true (no residual pass: nullptr)
};

template <int FPT, int MAXT, int MINB, int CS, bool CG, bool UP>
static SiaEntry sia_entry() {
  using G = SiaInst<FPT, MAXT, MINB, CS, CG, UP>;
  SiaKernel eval = nullptr;
  if constexpr (CG && !UP) eval = sia_kernel<FPT, true, MAXT, MINB, CS, CG, UP>;
  return {FPT, MAXT, MINB, CS, CG, UP, G::SS, G::WIN, G::SA, G::fixed_bytes, {sia_kernel<FPT, false, MAXT, MINB, CS, CG, UP>, eval}};
}

// Every alignment instantiation.  pick_launch takes the first general-camera, per-level entry that fits, so the one-CTA
// entries are in the order it tries them.  The undistorted pinhole has its own instantiation of the geometries that carry the
// throughput / latency figures; the residual pass and the rarely used geometries run the general-camera code only.
static const SiaEntry kSiaEntries[] = {
    sia_entry<1, 96, 2, 2, true, false>(),
    sia_entry<1, 96, 2, 4, true, false>(),  sia_entry<1, 96, 2, 4, false, false>(),
    sia_entry<1, 96, 1, 4, true, true>(),   sia_entry<1, 96, 1, 4, false, true>(),
    sia_entry<1, 96, 2, 8, true, false>(),
    sia_entry<2, 160, 3, 1, true, false>(), sia_entry<2, 160, 3, 1, false, false>(),
    sia_entry<1, 320, 2, 1, true, false>(), sia_entry<1, 320, 2, 1, false, false>(),
    sia_entry<1, 384, 2, 1, true, false>(),
    sia_entry<1, 512, 1, 1, true, false>(),
    sia_entry<2, 512, 1, 1, true, false>(),
};

// The entry of e's geometry (CTAs per pair, threads, features per thread) with the given camera and upfront flags.
static const SiaEntry* sia_variant(const SiaEntry& e, bool general_camera, bool upfront) {
  for (const SiaEntry& v : kSiaEntries)
    if (v.cluster == e.cluster && v.threads == e.threads && v.fpt == e.fpt && v.general_camera == general_camera &&
        v.upfront == upfront)
      return &v;
  return nullptr;
}

struct SiaBatchState {
  int B = 0;
  int total_feat = 0;
  int max_feat = 0;
  SiaParams P;
  // The batch API owns its staging buffers: stage / run / fetch may be interleaved with any other entry point of the
  // context (align, pose optimizer, depth filter ... stage through the context's h_in / d_in) without clobbering a staged
  // batch.  `io` is the Staging of the last stage, over this pair; it bound the addresses in P and `scales`.
  HostBuf h;
  DevBuf d;
  Staging io;
  const SiaEntry* geo = nullptr;  // the launch geometry pick_launch chose (nullptr: the robust kernel)
  size_t smem = 0;
  bool staged = false;
  // robust cost (svo_b200_sia_robust) the batch was staged with: weight function, or -1 = unweighted (sia_kernel)
  int robust_weight = -1;
  int robust_slots = 0;
  float* scales = nullptr;  // the robust kernel's per-pair, per-level scales (device)
  // features whose xyz_ref is not finite (sia_kernel only): staged without their point, visibility as the reference has it
  struct Nonfinite { int feat, pair, vis_levels; };  // vis_levels: the levels the set-only mask holds it at
  std::vector<Nonfinite> nonfinite;
  explicit SiaBatchState(svo_b200_ctx* ctx) : io(ctx, h, d) {}
};

void sia_batch_free(svo_b200_ctx* ctx) {
  if (ctx->sia) {
    if (ctx->sia->d.p) cudaFree(ctx->sia->d.p);
    if (ctx->sia->h.p) cudaFreeHost(ctx->sia->h.p);
  }
  delete ctx->sia;
  ctx->sia = nullptr;
}

void sia_split_free(svo_b200_ctx* ctx) {
  for (int r = 0; r < 8; ++r) {
    if (ctx->xg_peer_ipc[r] && ctx->xg_peer[r]) cudaIpcCloseMemHandle(ctx->xg_peer[r]);
    ctx->xg_peer[r] = nullptr;
    ctx->xg_peer_ipc[r] = false;
  }
  if (ctx->xg_buf) cudaFree(ctx->xg_buf);
  ctx->xg_buf = nullptr;
  ctx->xg_world = 1; ctx->xg_rank = 0; ctx->xg_pairs = 0; ctx->xg_connected = false;
}

// Minimum staging region: holds the current image of level >= 2 of 640x480 (TMA).  The next coarse, TMA-staged current
// image is bulk-prefetched into L2 while a level iterates; there are no per-feature L2 prefetches of the next level's
// footprints: the extra uncoalesced requests cost more L1 time than the DRAM latency they hide.
constexpr size_t kSiaMinStageBytes = 20 * 1024;

// How many clusters of the (upfront or per-level) 4-CTA geometry `e` the device holds at once with `smem` bytes of dynamic
// shared memory per CTA.  The general-camera instantiation stands for both: the plain-pinhole one has the same shared memory,
// and at 96 threads per CTA registers do not limit residency.
static int max_active_clusters(svo_b200_ctx* ctx, const SiaEntry& e, size_t smem, int& n) {
  const int k = e.upfront ? 0 : 1;
  if (ctx->sia_occ_smem[k] != smem) {
    SVO_CUDA_CHECK(ctx, cudaFuncSetAttribute(e.kern[0], cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    SVO_CUDA_CHECK(ctx, cudaFuncSetAttribute(e.kern[0], cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared));
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)e.cluster);
    cfg.blockDim = dim3((unsigned)e.threads);
    cfg.dynamicSmemBytes = smem;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = (unsigned)e.cluster;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    int c = 0;
    SVO_CUDA_CHECK(ctx, cudaOccupancyMaxActiveClusters(&c, (const void*)e.kern[0], &cfg));
    ctx->sia_occ_smem[k] = smem;
    ctx->sia_occ_clusters[k] = c;
  }
  n = ctx->sia_occ_clusters[k];
  return 0;
}

// Launch geometry (an entry of kSiaEntries) for a batch of B pairs with at most max_feat features each: one CTA per pair,
// or (small batches) the pair's features split over the CTAs of a thread-block cluster.
// `fallback` (internal): 1 = the upfront clusters of this batch are not all resident at once, 2 = no cluster geometry is.
static int pick_launch(svo_b200_ctx* ctx, int B, int max_feat, int n_lvl, const SiaEntry*& geo, int& stage_cap, size_t& smem,
                       int fallback = 0) {
  if (max_feat > 1024)
    return set_err(ctx, SVO_B200_ELIMIT, "sparse_img_align: %d features per pair > 1024 (shared-memory patch cache)", max_feat);
  int want = ctx->sia_cluster;
  const bool auto_cluster = want < 0 && !ctx->xg_connected;
  if (ctx->xg_connected) {
    // feature split over GPUs: the ranks' CTAs of a pair wait for each other, so every CTA must be resident at once
    if (B > ctx->xg_pairs || B > 2 * ctx->sm_count)
      return set_err(ctx, SVO_B200_ELIMIT, "sia split: %d pairs per launch exceed the split's capacity (%d) or the resident CTAs (%d)",
                     B, ctx->xg_pairs, 2 * ctx->sm_count);
    want = 1;
  }
  // small batch (live streams, BASELINE configs[4]'s 32 pairs per GPU): spread each pair over 4 SMs while every CTA
  // still has an SM of its own (two cluster CTAs sharing an SM lose to one 320-thread CTA per pair)
  if (want < 0) want = (fallback < 2 && B * 4 <= ctx->sm_count) ? 4 : 1;
  // full batches (more pairs than 2 per SM): the throughput geometry, 160 threads x 2 features, three CTAs per SM; in
  // between, 320 x 1 with windows (with its state in shared memory and its loops rolled the throughput geometry also serves
  // batches below two CTAs per SM, so the one-feature geometries are left for pairs beyond its slots, the multi-GPU split and
  // explicit requests); otherwise the smallest one-CTA geometry whose slots hold the pair's features
  const bool fpt2 = ctx->sia_fpt != 1 && !ctx->xg_connected;
  auto first = [&](auto accept) -> const SiaEntry* {  // the first general-camera, per-level entry that holds max_feat
    for (const SiaEntry& c : kSiaEntries)
      if (c.general_camera && !c.upfront && max_feat <= c.cluster * c.slots && accept(c)) return &c;
    return nullptr;
  };
  const SiaEntry* e = want > 1 ? first([&](const SiaEntry& c) { return c.cluster == want; }) : nullptr;
  if (!e) e = first([&](const SiaEntry& c) { return c.cluster == 1 && (fpt2 || !c.throughput); });
  // cluster geometry with every CTA alone on its SM: one patch array set per level, everything pose independent prepared
  // before the first iteration (only the 4-CTA geometry has an upfront instantiation; 2 and 8 keep the per-level flow)
  const SiaEntry* up = sia_variant(*e, true, true);
  if (up && ctx->sia_upfront != 0 && fallback == 0 && B * e->cluster <= ctx->sm_count && n_lvl >= 1 &&
      n_lvl <= SVO_B200_MAX_LEVELS && up->fixed_bytes(n_lvl) + kSiaMinStageBytes + 1024 <= (size_t)ctx->max_smem_optin)
    e = up;
  const size_t base = e->fixed_bytes(e->upfront ? n_lvl : 1);
  // shared memory one CTA may use so that the MINB CTAs the instantiation is compiled for stay resident per SM (228 KB per
  // SM, 1 KB reserved per CTA)
  size_t budget = (size_t)ctx->max_smem_optin;
  const size_t per_cta = (size_t)(228 * 1024) / e->min_blocks - 1024;
  if (per_cta < budget) budget = per_cta;
  if (base + 1024 > budget)
    return set_err(ctx, SVO_B200_ELIMIT, "sparse_img_align: %d features need %zu B of shared memory", max_feat, base);
  // staging region: the coarse current-level images (TMA) or, at the fine levels, one 128-byte window per feature slot
  size_t cap = kSiaMinStageBytes;
  const size_t win = (size_t)kWinBytes * e->slots;
  if (win > cap && base + win <= budget) cap = win;
  if (base + cap > budget) cap = (budget - base) & ~size_t(15);
  geo = e;
  stage_cap = (int)cap;
  smem = base + cap;
  // The CTAs of a cluster run within one GPC, so whether all B clusters are resident at once depends on the GPC layout and
  // the shared memory per CTA; B * 4 <= #SMs does not imply it (an H100's 132 SMs sit in GPCs of different sizes).  A second
  // wave of clusters would double a small batch's latency: fall back to the per-level cluster flow (less shared memory per
  // CTA), and from there to one CTA per pair.  Explicit requests (svo_b200_sia_config / svo_b200_sia_upfront(1)) are kept.
  if (auto_cluster && e->cluster == 4 && !(e->upfront && ctx->sia_upfront == 1)) {
    int n = 0;
    if (int rc = max_active_clusters(ctx, *e, smem, n)) return rc;
    if (B > n) return pick_launch(ctx, B, max_feat, n_lvl, geo, stage_cap, smem, e->upfront ? 1 : 2);
  }
  return 0;
}

// Launches geometry `geo` (from pick_launch) and records the launch for svo_b200_sia_last_launch.  The undistorted pinhole
// runs the geometry's plain-pinhole instantiation where it has one; the residual pass (eval) runs its general-camera,
// per-level instantiation.
// `chain`: the last work on the stream is a run of the same staged batch.  The throughput geometry then launches as its
// programmatic dependent -- its CTAs fill the slots the previous run's last wave frees, and wait for that run before they
// store the outputs -- without the kernel-time events, whose records between the two kernels would serialise them again.
// The other geometries run few CTAs per SM or small batches, where an overlap would shorten the time per launch and not a
// pair's latency: they are never chained.
static int launch_sia(svo_b200_ctx* ctx, const SiaParams& P, int B, const SiaEntry& geo, size_t smem, bool eval, bool chain) {
  const bool plain = !eval && !P.cam.distorted && P.cam.model == SVO_B200_CAM_PINHOLE;
  const SiaEntry* e = sia_variant(geo, !plain, geo.upfront && !eval);
  if (!e) e = &geo;
  const SiaKernel kern = e->kern[eval];
  SVO_CUDA_CHECK(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  // ask for the full shared-memory carveout so that two CTAs of ~95 KB fit one SM
  SVO_CUDA_CHECK(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout,
                                           (int)cudaSharedmemCarveoutMaxShared));
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)(B * e->cluster));
  cfg.blockDim = dim3((unsigned)e->threads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = ctx->stream;
  const bool dependent = chain && !eval && e->throughput;
  cudaLaunchAttribute attr[2];
  cfg.attrs = attr;
  if (e->cluster > 1) {
    attr[cfg.numAttrs].id = cudaLaunchAttributeClusterDimension;
    attr[cfg.numAttrs].val.clusterDim.x = (unsigned)e->cluster;
    attr[cfg.numAttrs].val.clusterDim.y = 1;
    attr[cfg.numAttrs].val.clusterDim.z = 1;
    cfg.numAttrs++;
  }
  if (dependent) {
    attr[cfg.numAttrs].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[cfg.numAttrs].val.programmaticStreamSerializationAllowed = 1;
    cfg.numAttrs++;
  }
  if (!dependent) kt_begin(ctx);
  SVO_CUDA_CHECK(ctx, cudaLaunchKernelEx(&cfg, kern, P));
  if (!dependent) kt_end(ctx);
  ctx->launches++;
  SVO_CUDA_CHECK(ctx, cudaGetLastError());
  svo_b200_sia_launch& L = ctx->sia_last;  // what ran, for svo_b200_sia_last_launch
  L = svo_b200_sia_launch{};
  L.n_pairs = B; L.ctas_per_pair = e->cluster; L.threads = e->threads; L.features_per_thread = e->fpt; L.min_blocks = e->min_blocks;
  L.upfront = e->upfront; L.general_camera = e->general_camera;
  L.residuals_only = eval; L.stage_cap = P.stage_cap; L.smem_bytes = (int)smem; L.resident_clusters = ctx->sia_occ_clusters[0];
  L.sm_count = ctx->sm_count;
  L.min_level = eval ? P.eval_level : P.min_level;
  L.max_level = eval ? P.eval_level : P.max_level;
  for (int l = 0; l < SVO_B200_MAX_LEVELS; ++l)
    L.level_stage[l] = l >= L.min_level && l <= L.max_level ? sia_stage_mode(sia_image_bytes(P.w[l], P.h[l]), P.w[l], P.stage_cap, e->windows, e->slots) : -1;
  ctx->sia_last_valid = true;
  ctx->sia_last_robust = false;
  return 0;
}

// Launches the robust kernel for a staged batch and records it for svo_b200_sia_last_launch / svo_b200_sia_last_scales.
static int launch_sia_robust(svo_b200_ctx* ctx, const SiaBatchState& st) {
  SiaRobustParams RP;
  RP.P = st.P;
  RP.weight = st.robust_weight;
  RP.slots = st.robust_slots;
  RP.scales_out = st.scales;
  SVO_CUDA_CHECK(ctx, cudaFuncSetAttribute(sia_robust_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)st.smem));
  if (int rc = launch_kernels(ctx, 1, [&] { sia_robust_kernel<<<st.B, kSiaRobustThreads, st.smem, ctx->stream>>>(RP); })) return rc;
  svo_b200_sia_launch& L = ctx->sia_last;
  L = svo_b200_sia_launch{};
  L.n_pairs = st.B; L.ctas_per_pair = 1; L.threads = kSiaRobustThreads;
  L.features_per_thread = (st.max_feat + kSiaRobustThreads - 1) / kSiaRobustThreads;
  L.min_blocks = 1; L.upfront = 0; L.general_camera = 1; L.residuals_only = 0; L.stage_cap = 0; L.smem_bytes = (int)st.smem;
  L.resident_clusters = ctx->sia_occ_clusters[0];
  L.sm_count = ctx->sm_count;
  L.min_level = st.P.min_level; L.max_level = st.P.max_level;
  for (int l = 0; l < SVO_B200_MAX_LEVELS; ++l) L.level_stage[l] = l >= L.min_level && l <= L.max_level ? SVO_B200_SIA_STAGE_GLOBAL : -1;
  ctx->sia_last_valid = true;
  ctx->sia_last_robust = true;
  ctx->sia_scales.assign((size_t)st.B * SVO_B200_MAX_LEVELS, __builtin_nanf(""));  // filled by svo_b200_sia_batch_fetch
  return 0;
}

static inline int pad16(int n) { return (n + 15) / 16 * 16; }

// A point whose xyz_ref = f * |pos - ref_pos| is not finite projects to NaN at every pose: the reference keeps it visible
// where its reference patch fits, and it never enters a residual pass.  sia_kernel, which sums every visible feature's
// Jacobian rows times its moments (zero where the feature is not in the image), would turn 0 * NaN into a NaN normal matrix:
// such features are staged as a slot without a point at a finite position, and their visibility is the reference's border
// test (precomputeReferencePatches, sparse_img_align.cpp:84-99), counted in the pair's sum_visible as the kernel counts.
static bool finite_xyz_ref(const double* f, const double* pos, const double* ref_pos) {
  // every input finite (the common case): 0 * (a sum of them) is 0, where any is inf or NaN it is NaN
  if (std::isfinite(0.0 * (f[0] + f[1] + f[2] + pos[0] + pos[1] + pos[2] + ref_pos[0] + ref_pos[1] + ref_pos[2]))) {
    const double m = fmax(fmax(fabs(pos[0] - ref_pos[0]), fabs(pos[1] - ref_pos[1])), fabs(pos[2] - ref_pos[2]));
    if (m < 1e150) return true;  // no overflow in the depth either
  }
  const double dx = pos[0] - ref_pos[0], dy = pos[1] - ref_pos[1], dz = pos[2] - ref_pos[2];
  const double depth = sqrt(dx * dx + dy * dy + dz * dz);
  return std::isfinite(f[0] * depth) && std::isfinite(f[1] * depth) && std::isfinite(f[2] * depth);
}
// The number of levels (max..min) at which the set-only visibility mask holds a feature: from the first level its reference
// patch fits on.  0: never visible.
static int ref_patch_levels(const double* px, const SiaParams& P, const svo_b200_frame* ref) {
  int n = 0;
  bool vis = false;
  for (int l = P.max_level; l >= P.min_level; --l) {
    const float scale = 1.0f / (float)(1 << l);
    const float u = (float)(px[0] * scale), v = (float)(px[1] * scale);
    if (u >= 0.f && v >= 0.f && u < 1e6f && v < 1e6f) {
      const int ui = (int)floorf(u), vi = (int)floorf(v);
      vis = vis || (ui - 3 >= 0 && vi - 3 >= 0 && ui + 3 < ref->w[l] && vi + 3 < ref->h[l]);
    }
    n += vis ? 1 : 0;
  }
  return n;
}

// Pack one pair's features into the blob layout the kernel stages with TMA.
static void pack_blob(uint8_t* dst, int n, int np, const double* px, const double* f, const double* pos,
                      const uint8_t* hp) {
  double* d = reinterpret_cast<double*>(dst);
  memset(dst, 0, (size_t)np * 65);
  memcpy(d, px, sizeof(double) * 2 * n);
  memcpy(d + 2 * np, f, sizeof(double) * 3 * n);
  memcpy(d + 5 * np, pos, sizeof(double) * 3 * n);
  memcpy(dst + (size_t)np * 64, hp, n);
}

constexpr int kSiaUnboundedIters = 1000;  // iterations per level for a negative n_iter

static int fill_common(svo_b200_ctx* ctx, SiaParams& P, const svo_b200_frame* fr, const svo_b200_camera* cam,
                       const svo_b200_sia_options* opt) {
  memset(&P, 0, sizeof(P));
  if (opt->max_level < opt->min_level || opt->min_level < 0 || opt->max_level >= fr->n_levels)
    return set_err(ctx, SVO_B200_EINVAL, "sparse_img_align: levels [%d,%d] outside the pyramid (%d levels)",
                   opt->min_level, opt->max_level, fr->n_levels);
  for (int l = 0; l < fr->n_levels; ++l) { P.w[l] = fr->w[l]; P.h[l] = fr->h[l]; }
  int rc = cam_to_dev(ctx, cam, P.cam);
  if (rc) return rc;
  P.max_level = opt->max_level; P.min_level = opt->min_level; P.eps = opt->eps;
  // The reference's n_iter_ is a size_t: a negative n_iter wraps around to no limit.  Here it is kSiaUnboundedIters per level,
  // which no converging level reaches, while a level that never stops (no measurement or a zero residual, with a NaN or
  // negative eps) ends within milliseconds instead of running for hours.  The robust kernel takes the same bound.
  P.n_iter = opt->n_iter < 0 ? kSiaUnboundedIters : opt->n_iter;
  P.debug = getenv("SVO_B200_SIA_DEBUG") ? 1 : 0;
  P.xg.rank = 0; P.xg.world = 1;
  if (ctx->xg_connected) {
    P.xg.rank = ctx->xg_rank; P.xg.world = ctx->xg_world;
    for (int r = 0; r < ctx->xg_world; ++r) P.xg.peer[r] = static_cast<XgPair*>(ctx->xg_peer[r]);
  }
  return 0;
}

}  // namespace svo

using namespace svo;

extern "C" {

int svo_b200_sia_split_create(svo_b200_ctx* ctx, int rank, int world, int max_pairs, void* ipc_handle_out, void** local_ptr_out) {
  if (!ctx || world < 1 || world > kMaxSplit || rank < 0 || rank >= world || max_pairs < 1)
    return set_err(ctx, SVO_B200_EINVAL, "sia_split_create: need 1 <= world <= %d, 0 <= rank < world, max_pairs >= 1", kMaxSplit);
  cudaSetDevice(ctx->device);
  sia_split_free(ctx);
  const size_t bytes = sizeof(XgPair) * (size_t)max_pairs;
  SVO_CUDA_CHECK(ctx, cudaMalloc(&ctx->xg_buf, bytes));
  SVO_CUDA_CHECK(ctx, cudaMemset(ctx->xg_buf, 0, bytes));
  ctx->xg_rank = rank; ctx->xg_world = world; ctx->xg_pairs = max_pairs;
  if (ipc_handle_out) {
    static_assert(sizeof(cudaIpcMemHandle_t) == SVO_B200_IPC_HANDLE_BYTES, "IPC handle size");
    cudaIpcMemHandle_t h;
    SVO_CUDA_CHECK(ctx, cudaIpcGetMemHandle(&h, ctx->xg_buf));
    memcpy(ipc_handle_out, &h, sizeof(h));
  }
  if (local_ptr_out) *local_ptr_out = ctx->xg_buf;
  return 0;
}

int svo_b200_sia_split_connect(svo_b200_ctx* ctx, const void* ipc_handles, void* const* in_process_ptrs) {
  if (!ctx || !ctx->xg_buf || (!ipc_handles && !in_process_ptrs))
    return set_err(ctx, SVO_B200_EINVAL, "sia_split_connect: call sia_split_create first and pass the peers' handles or pointers");
  cudaSetDevice(ctx->device);
  for (int r = 0; r < ctx->xg_world; ++r) {
    if (r == ctx->xg_rank) { ctx->xg_peer[r] = ctx->xg_buf; continue; }
    if (in_process_ptrs) {
      if (!in_process_ptrs[r]) return set_err(ctx, SVO_B200_EINVAL, "sia_split_connect: NULL pointer for rank %d", r);
      ctx->xg_peer[r] = in_process_ptrs[r];
    } else {
      cudaIpcMemHandle_t h;
      memcpy(&h, static_cast<const uint8_t*>(ipc_handles) + (size_t)r * sizeof(h), sizeof(h));
      SVO_CUDA_CHECK(ctx, cudaIpcOpenMemHandle(&ctx->xg_peer[r], h, cudaIpcMemLazyEnablePeerAccess));
      ctx->xg_peer_ipc[r] = true;
    }
  }
  // the buffers start from a known state on every rank (sequence counters 0): the caller connects all ranks before any
  // of them launches (a barrier of the launcher's own, e.g. torch.distributed.barrier)
  SVO_CUDA_CHECK(ctx, cudaMemset(ctx->xg_buf, 0, sizeof(XgPair) * (size_t)ctx->xg_pairs));
  SVO_CUDA_CHECK(ctx, cudaDeviceSynchronize());
  ctx->xg_connected = ctx->xg_world > 1;
  return 0;
}

int svo_b200_sia_split_destroy(svo_b200_ctx* ctx) {
  if (!ctx) return SVO_B200_EINVAL;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  sia_split_free(ctx);
  return 0;
}

int svo_b200_sia_config(svo_b200_ctx* ctx, int ctas_per_pair, int features_per_thread) {
  if (!ctx) return SVO_B200_EINVAL;
  if (!(ctas_per_pair == -1 || ctas_per_pair == 1 || ctas_per_pair == 2 || ctas_per_pair == 4 || ctas_per_pair == 8) ||
      features_per_thread < 0 || features_per_thread > 2)
    return set_err(ctx, SVO_B200_EINVAL, "sia_config: ctas_per_pair must be -1, 1, 2, 4 or 8 and features_per_thread 0, 1 or 2");
  ctx->sia_cluster = ctas_per_pair;
  ctx->sia_fpt = features_per_thread;
  return 0;
}

int svo_b200_sia_upfront(svo_b200_ctx* ctx, int mode) {
  if (!ctx) return SVO_B200_EINVAL;
  if (mode < -1 || mode > 1) return set_err(ctx, SVO_B200_EINVAL, "sia_upfront: mode must be -1, 0 or 1");
  ctx->sia_upfront = mode;
  return 0;
}

int svo_b200_sia_robust(svo_b200_ctx* ctx, int scale_estimator, int weight_function) {
  if (!ctx) return SVO_B200_EINVAL;
  if (scale_estimator < SVO_B200_SCALE_UNIT || scale_estimator > SVO_B200_SCALE_NORMAL || weight_function < SVO_B200_WEIGHT_UNIT ||
      weight_function > SVO_B200_WEIGHT_HUBER)
    return set_err(ctx, SVO_B200_EINVAL, "sia_robust: scale estimator %d / weight function %d is not an SVO_B200_SCALE_* / SVO_B200_WEIGHT_* value",
                   scale_estimator, weight_function);
  if (scale_estimator == SVO_B200_SCALE_UNIT) {  // use_weights_ = false: plain Gauss-Newton whatever the weight function
    ctx->sia_scale_est = SVO_B200_SCALE_UNIT;
    ctx->sia_weight_fn = SVO_B200_WEIGHT_UNIT;
    return 0;
  }
  if (scale_estimator != SVO_B200_SCALE_MAD)
    return set_err(ctx, SVO_B200_EINVAL, "sia_robust: only the MAD scale estimator is supported (T-distribution and normal scales are not)");
  if (weight_function == SVO_B200_WEIGHT_TDIST)
    return set_err(ctx, SVO_B200_EINVAL, "sia_robust: the T-distribution weight function is not supported (unit, Tukey or Huber)");
  if (ctx->xg_connected)
    return set_err(ctx, SVO_B200_EINVAL, "sia_robust: the robust cost does not run with a multi-GPU feature split");
  ctx->sia_scale_est = scale_estimator;
  ctx->sia_weight_fn = weight_function;
  return 0;
}

int svo_b200_sia_last_scales(const svo_b200_ctx* ctx, int B, float* out) {
  if (!ctx || !out || B < 1) return SVO_B200_EINVAL;
  if (!ctx->sia_last_valid || !ctx->sia_last_robust)
    return set_err(const_cast<svo_b200_ctx*>(ctx), SVO_B200_EINVAL, "sia_last_scales: the last alignment launch was not weighted");
  if ((size_t)B * SVO_B200_MAX_LEVELS > ctx->sia_scales.size())
    return set_err(const_cast<svo_b200_ctx*>(ctx), SVO_B200_EINVAL, "sia_last_scales: the last launch had %d pairs",
                   (int)(ctx->sia_scales.size() / SVO_B200_MAX_LEVELS));
  memcpy(out, ctx->sia_scales.data(), sizeof(float) * SVO_B200_MAX_LEVELS * (size_t)B);
  return 0;
}

int svo_b200_sia_last_launch(const svo_b200_ctx* ctx, svo_b200_sia_launch* out) {
  if (!ctx || !out) return SVO_B200_EINVAL;
  if (!ctx->sia_last_valid) return set_err(const_cast<svo_b200_ctx*>(ctx), SVO_B200_EINVAL, "sia_last_launch: no alignment kernel launched yet");
  *out = ctx->sia_last;
  return 0;
}

}  // extern "C"

namespace svo {
// svo_b200_sia_batch_stage with the robust cost of the context (`robust`) or without it (svo_b200_sparse_residuals).
// `more(st)` declares the extra regions of a single-pair call in st.io, after every check and before it opens.
template <class More>
static int sia_stage(svo_b200_ctx* ctx, int B, const svo_b200_frame* const* ref, const svo_b200_frame* const* cur,
                     const svo_b200_camera* cam, const svo_b200_sia_options* opt, const double* T, const int* feat_offset,
                     const double* px, const double* f, const double* point_pos, const uint8_t* has_point, const double* ref_pos,
                     bool robust, More&& more) {
  if (!ctx || B <= 0 || !ref || !cur || !cam || !opt || !T || !feat_offset || !ref_pos)
    return set_err(ctx, SVO_B200_EINVAL, "sia_batch_stage: bad arguments");
  cudaSetDevice(ctx->device);
  if (!ctx->sia) ctx->sia = new SiaBatchState(ctx);
  SiaBatchState& st = *ctx->sia;
  st.staged = false;
  ctx->sia_chain = false;
  st.B = B;
  st.total_feat = feat_offset[B] - feat_offset[0];
  st.max_feat = 0;
  st.nonfinite.clear();
  for (int b = 0; b < B; ++b) {
    const int n = feat_offset[b + 1] - feat_offset[b];
    if (n < 0) return set_err(ctx, SVO_B200_EINVAL, "sia_batch_stage: feat_offset not monotone");
    if (n > st.max_feat) st.max_feat = n;
    if (!ref[b] || !cur[b] || ref[b]->n_levels != ref[0]->n_levels || ref[b]->width != ref[0]->width ||
        ref[b]->height != ref[0]->height || cur[b]->width != ref[0]->width ||
        cur[b]->height != ref[0]->height || cur[b]->n_levels != ref[0]->n_levels)
      return set_err(ctx, SVO_B200_EINVAL, "sia_batch_stage: all frames of a batch must share one geometry");
  }
  if (int rc_sz = cam_check_frames(ctx, "sia_batch_stage", cam, ref, 1)) return rc_sz;  // ref[0]: the batch's one geometry
  if (st.total_feat > 0 && (!px || !f || !point_pos || !has_point))
    return set_err(ctx, SVO_B200_EINVAL, "sia_batch_stage: NULL feature arrays");
  int rc = fill_common(ctx, st.P, ref[0], cam, opt);
  if (rc) return rc;
  // weights on: the robust kernel, chosen before pick_launch (svo_b200_sia_config / _upfront do not apply to it)
  const bool weighted = robust && ctx->sia_scale_est == SVO_B200_SCALE_MAD;
  st.robust_weight = -1;
  if (weighted) {
    if (ctx->xg_connected)
      return set_err(ctx, SVO_B200_EINVAL, "sparse_img_align: the robust cost does not run with a multi-GPU feature split");
    if (st.max_feat > kSiaRobustMaxFeat)
      return set_err(ctx, SVO_B200_ELIMIT, "sparse_img_align: %d features per pair > %d (robust cost)", st.max_feat, kSiaRobustMaxFeat);
    st.robust_slots = ((st.max_feat > 1 ? st.max_feat : 1) + 31) & ~31;
    st.smem = sia_robust_smem_bytes(st.robust_slots);
    if (st.smem > (size_t)ctx->max_smem_optin)
      return set_err(ctx, SVO_B200_ELIMIT, "sparse_img_align: %d features need %zu B of shared memory (robust cost)", st.max_feat, st.smem);
    st.geo = nullptr;
    st.robust_weight = ctx->sia_weight_fn;
  } else {
    rc = pick_launch(ctx, B, st.max_feat, opt->max_level - opt->min_level + 1, st.geo, st.P.stage_cap, st.smem);
    if (rc) return rc;
  }

  // in: the jobs, then the pairs' feature blobs, each on a 128-byte boundary (the jobs hold the blobs' addresses: both are
  // filled after open()); out: read back by svo_b200_sia_batch_fetch
  const auto blob_span = [](int n) { return ((size_t)pad16(n) * 65 + 16 + 127) / 128 * 128; };
  size_t blob_bytes = 0;
  for (int b = 0; b < B; ++b) blob_bytes += blob_span(feat_offset[b + 1] - feat_offset[b]);
  st.io = Staging(ctx, st.h, st.d);
  st.io.in(nullptr, B, &st.P.jobs);
  const uint8_t* blobs = nullptr;
  st.io.in(nullptr, blob_bytes, &blobs, 128);
  st.io.out(nullptr, 12 * (size_t)B, &st.P.T_out);
  st.io.out(nullptr, 36 * (size_t)B, &st.P.H_out);
  st.io.out(nullptr, B, &st.P.stats);
  st.io.out(nullptr, (size_t)st.total_feat + 16, &st.P.visible_out);
  if (weighted) st.io.out(nullptr, SVO_B200_MAX_LEVELS * (size_t)B, &st.scales);
  more(st);
  if ((rc = st.io.open())) return rc;
  SiaJob* jobs = st.io.host(st.P.jobs);
  const uint8_t* blob = blobs;
  for (int b = 0; b < B; ++b) {
    SiaJob& j = jobs[b];
    memset(&j, 0, sizeof(j));
    for (int l = 0; l < ref[b]->n_levels; ++l) {
      j.ref_lvl[l] = ref[b]->lvl(l); j.cur_lvl[l] = cur[b]->lvl(l);
      j.ref_tl[l] = ref[b]->tv[l]; j.cur_tl[l] = cur[b]->tv[l];
    }
    const int o = feat_offset[b], n = feat_offset[b + 1] - o;
    j.n_feat = n;
    j.n_pad = pad16(n);
    j.feat_off = o - feat_offset[0];
    j.blob = blob;
    blob += blob_span(n);
    memcpy(j.T, T + 12 * (size_t)b, sizeof(double) * 12);
    memcpy(j.ref_pos, ref_pos + 3 * (size_t)b, sizeof(double) * 3);
    uint8_t* hb = st.io.host(j.blob);
    if (n > 0) pack_blob(hb, n, j.n_pad, px + 2 * (size_t)o, f + 3 * (size_t)o, point_pos + 3 * (size_t)o, has_point + o);
    if (!weighted)
      for (int i = 0; i < n; ++i)
        if (has_point[o + i] && !finite_xyz_ref(f + 3 * (size_t)(o + i), point_pos + 3 * (size_t)(o + i), ref_pos + 3 * (size_t)b)) {
          double* d = reinterpret_cast<double*>(hb);
          const double* rp = ref_pos + 3 * (size_t)b;
          for (int c = 0; c < 3; ++c) {  // the neutral xyz_ref (0, 0, ~1) of a slot without a feature
            d[2 * (size_t)j.n_pad + 3 * i + c] = c == 2 ? 1.0 : 0.0;
            d[5 * (size_t)j.n_pad + 3 * i + c] = c == 2 ? rp[c] + 1.0 : rp[c];
          }
          hb[(size_t)j.n_pad * 64 + i] = 0;
          st.nonfinite.push_back({j.feat_off + i, b, ref_patch_levels(px + 2 * (size_t)(o + i), st.P, ref[b])});
        }
  }
  if ((rc = st.io.send())) return rc;
  st.staged = true;
  return 0;
}
}  // namespace svo

extern "C" {

int svo_b200_sia_batch_stage(svo_b200_ctx* ctx, int B, const svo_b200_frame* const* ref,
                             const svo_b200_frame* const* cur, const svo_b200_camera* cam,
                             const svo_b200_sia_options* opt, const double* T, const int* feat_offset,
                             const double* px, const double* f, const double* point_pos,
                             const uint8_t* has_point, const double* ref_pos) {
  return sia_stage(ctx, B, ref, cur, cam, opt, T, feat_offset, px, f, point_pos, has_point, ref_pos, true, [](SiaBatchState&) {});
}

int svo_b200_sia_batch_run(svo_b200_ctx* ctx) {
  if (!ctx || !ctx->sia || !ctx->sia->staged) return set_err(ctx, SVO_B200_EINVAL, "sia_batch_run: nothing staged");
  cudaSetDevice(ctx->device);
  SiaBatchState& st = *ctx->sia;
  const int rc = st.robust_weight >= 0 ? launch_sia_robust(ctx, st) : launch_sia(ctx, st.P, st.B, *st.geo, st.smem, false, ctx->sia_chain);
  ctx->sia_chain = rc == 0;
  return rc;
}

int svo_b200_sia_batch_fetch(svo_b200_ctx* ctx, double* T_out, uint8_t* visible_out, double* H_out,
                             svo_b200_sia_stats* stats_out) {
  if (!ctx || !ctx->sia || !ctx->sia->staged) return set_err(ctx, SVO_B200_EINVAL, "sia_batch_fetch: nothing staged");
  cudaSetDevice(ctx->device);
  SiaBatchState& st = *ctx->sia;
  ctx->sia_chain = false;
  if (int rc = st.io.receive()) return rc;
  if (ctx->xg_connected) {  // did every peer take part in every exchange?  (if not, no caller array is written)
    std::vector<unsigned> err((size_t)st.B, 0u);
    SVO_CUDA_CHECK(ctx, cudaMemcpy2D(err.data(), sizeof(unsigned), static_cast<const uint8_t*>(ctx->xg_buf) + offsetof(XgPair, err),
                                     sizeof(XgPair), sizeof(unsigned), (size_t)st.B, cudaMemcpyDeviceToHost));
    for (int b = 0; b < st.B; ++b)
      if (err[b]) return set_err(ctx, SVO_B200_ECUDA, "sia split: a peer rank did not arrive at an exchange of pair %d (timeout); reconnect the split", b);
  }
  if (T_out) memcpy(T_out, st.io.host(st.P.T_out), sizeof(double) * 12 * (size_t)st.B);
  if (H_out) memcpy(H_out, st.io.host(st.P.H_out), sizeof(double) * 36 * (size_t)st.B);
  if (stats_out) memcpy(stats_out, st.io.host(st.P.stats), sizeof(svo_b200_sia_stats) * (size_t)st.B);
  if (visible_out) memcpy(visible_out, st.io.host(st.P.visible_out), (size_t)st.total_feat);
  if (st.P.n_iter == 0 && st.robust_weight < 0) {
    // no iteration: SparseImgAlign computes the reference patches, and so the visibility, only inside the first residual
    // pass (the robust cost's scale pass at the start pose computes them there): no feature is visible at any level
    if (visible_out) memset(visible_out, 0, (size_t)st.total_feat);
    if (stats_out)
      for (int b = 0; b < st.B; ++b) stats_out[b].sum_visible = 0;
  } else {
    for (const auto& q : st.nonfinite) {  // the points staged without their position (finite_xyz_ref)
      if (visible_out) visible_out[q.feat] = q.vis_levels > 0;
      if (stats_out) stats_out[q.pair].sum_visible += q.vis_levels;
    }
  }
  if (st.robust_weight >= 0 && ctx->sia_last_robust && ctx->sia_scales.size() == (size_t)st.B * SVO_B200_MAX_LEVELS)
    memcpy(ctx->sia_scales.data(), st.io.host(st.scales), sizeof(float) * SVO_B200_MAX_LEVELS * (size_t)st.B);
  return 0;
}

int svo_b200_sparse_img_align(svo_b200_ctx* ctx, const svo_b200_frame* ref, const svo_b200_frame* cur,
                              const svo_b200_camera* cam, const svo_b200_sia_options* opt,
                              double* T_io, const double* px, const double* f, const double* point_pos,
                              const uint8_t* has_point, const double* ref_pos, int N,
                              uint8_t* visible_out, double* H_out, svo_b200_sia_stats* stats_out,
                              svo_b200_sia_iter* trace_out, int trace_cap, int* n_trace_out) {
  if (!ctx || !ref || !cur || !cam || !opt || !T_io || !ref_pos || N < 0)
    return set_err(ctx, SVO_B200_EINVAL, "sparse_img_align: bad arguments");
  if (N == 0) {  // "SparseImgAlign: no features to track!" -> return 0 (sparse_img_align.cpp:47-51)
    if (stats_out) memset(stats_out, 0, sizeof(*stats_out));
    if (H_out) memset(H_out, 0, sizeof(double) * 36);
    if (n_trace_out) *n_trace_out = 0;
    return 0;
  }
  const bool tracing = trace_out && trace_cap > 0;
  const int off[2] = {0, N};
  int rc = sia_stage(ctx, 1, &ref, &cur, cam, opt, T_io, off, px, f, point_pos, has_point, ref_pos, true, [&](SiaBatchState& st) {
    if (!tracing) return;
    st.io.out(nullptr, (size_t)trace_cap, &st.P.trace);
    st.io.out(nullptr, 1, &st.P.n_trace);
    st.P.trace_cap = trace_cap;
  });
  if (rc) return rc;
  SiaBatchState& st = *ctx->sia;
  if ((rc = svo_b200_sia_batch_run(ctx))) return rc;
  if ((rc = svo_b200_sia_batch_fetch(ctx, T_io, visible_out, H_out, stats_out))) return rc;
  int ntr = 0;
  if (tracing) {
    ntr = *st.io.host(st.P.n_trace);
    const int ncopy = ntr < trace_cap ? ntr : trace_cap;
    if (ncopy > 0) memcpy(trace_out, st.io.host(st.P.trace), sizeof(svo_b200_sia_iter) * (size_t)ncopy);
  }
  if (n_trace_out) *n_trace_out = ntr;
  st.staged = false;  // the single-pair call leaves nothing staged behind
  return 0;
}

int svo_b200_sparse_residuals(svo_b200_ctx* ctx, const svo_b200_frame* ref, const svo_b200_frame* cur,
                              const svo_b200_camera* cam, int level, const double* T, const double* px,
                              const double* f, const double* point_pos, const uint8_t* has_point,
                              const double* ref_pos, int N, uint8_t* visible_io, float* ref_patch_out,
                              float* residuals_out, uint8_t* in_image_out, double* H_out, double* Jres_out,
                              double* chi2_out, int64_t* n_meas_out) {
  if (!ctx || !ref || !cur || !cam || !T || !ref_pos || N <= 0 || !visible_io)
    return set_err(ctx, SVO_B200_EINVAL, "sparse_residuals: bad arguments");
  svo_b200_sia_options opt = {level, level, 1, 1e-6};
  const int off[2] = {0, N};
  size_t nslots = 0;  // feature slots of the launch geometry: the kernel writes a patch row of each
  const auto regions = [&](SiaBatchState& st) {
    nslots = (size_t)st.geo->threads * st.geo->fpt * st.geo->cluster;
    st.io.in(visible_io, N, &st.P.visible_in);
    st.io.out(nullptr, 16 * nslots, &st.P.ref_patch_out);
    st.io.out(nullptr, 16 * nslots, &st.P.residuals_out);
    st.io.out(nullptr, N, &st.P.in_image_out);
    st.io.out(nullptr, 6, &st.P.Jres_out);
    st.io.out(nullptr, 1, &st.P.chi2_out);
    st.io.out(nullptr, 1, &st.P.n_meas_out);
  };
  int rc = sia_stage(ctx, 1, &ref, &cur, cam, &opt, T, off, px, f, point_pos, has_point, ref_pos, false, regions);  // never weighted
  if (rc) return rc;
  SiaBatchState& st = *ctx->sia;
  SVO_CUDA_CHECK(ctx, cudaMemsetAsync(st.P.residuals_out, 0xff, sizeof(float) * 16 * nslots, ctx->stream));
  st.P.eval_level = level;
  if ((rc = launch_sia(ctx, st.P, 1, *st.geo, st.smem, true, false))) return rc;
  double Tdummy[12];
  if ((rc = svo_b200_sia_batch_fetch(ctx, Tdummy, visible_io, H_out, nullptr))) return rc;
  if (ref_patch_out) memcpy(ref_patch_out, st.io.host(st.P.ref_patch_out), sizeof(float) * 16 * (size_t)N);
  if (residuals_out) memcpy(residuals_out, st.io.host(st.P.residuals_out), sizeof(float) * 16 * (size_t)N);
  if (in_image_out) memcpy(in_image_out, st.io.host(st.P.in_image_out), N);
  if (Jres_out) memcpy(Jres_out, st.io.host(st.P.Jres_out), sizeof(double) * 6);
  if (chi2_out) *chi2_out = *st.io.host(st.P.chi2_out);
  if (n_meas_out) *n_meas_out = *st.io.host(st.P.n_meas_out);
  st.staged = false;
  return 0;
}

}  // extern "C"
