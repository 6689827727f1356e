/* include/svo_b200.h -- C ABI of libsvo_b200.so, the H100 (sm_90a) implementation of the rpg_svo
 * direct-tracking hot path.  Plain pointers and sizes only; no torch / C++ types cross this line.
 *
 * Each entry point replaces one reference interface (paths relative to the rpg_svo tree):
 *   svo_b200_sparse_img_align*      <- svo::SparseImgAlign::run               svo/include/svo/sparse_img_align.h:43-57
 *                                      (+ getFisherInformation via H_out)     svo/src/sparse_img_align.cpp:43-82
 *   svo_b200_sparse_residuals       <- SparseImgAlign::computeResiduals       svo/src/sparse_img_align.cpp:147-243
 *   svo_b200_align2d_batch/_1d      <- feature_alignment::align2D / align1D   svo/include/svo/feature_alignment.h:29-44
 *   svo_b200_find_match_direct      <- Matcher::findMatchDirect               svo/include/svo/matcher.h:109-112
 *   svo_b200_reproject_map          <- Reprojector::reprojectMap              svo/include/svo/reprojector.h:58-62, svo/src/reprojector.cpp:64-217
 *   svo_b200_fast_detect            <- feature_detection::FastDetector::detect svo/include/svo/feature_detection.h:107-122, svo/src/feature_detection.cpp:66-115
 *   svo_b200_pose_optimize(_batch)  <- pose_optimizer::optimizeGaussNewton    svo/include/svo/pose_optimizer.h:37-45
 *   svo_b200_point_optimize_batch   <- Point::optimize                        svo/include/svo/point.h:86, svo/src/point.cpp:119-177
 *   svo_b200_find_epipolar_match_direct <- Matcher::findEpipolarMatchDirect   svo/include/svo/matcher.h:114-121
 *   svo_b200_depth_filter_update    <- DepthFilter::updateSeeds               svo/include/svo/depth_filter.h:155
 *                                      (Matcher::findEpipolarMatchDirect, updateSeed, computeTau inside)
 *   svo_b200_set_epipolar_options   <- Matcher::Options of both               svo/include/svo/matcher.h:74-91
 *   (_streams: S streams' calls of reprojectMap / updateSeeds / FastDetector::detect in one launch each)
 *   svo_b200_frame_*                <- svo::Frame image pyramid               svo/include/svo/frame.h:52, svo/src/frame.cpp:156-165
 *   svo_b200_klt_*                  <- initialization::trackKlt's             svo/src/initialization.cpp:127-169
 *                                      cv::calcOpticalFlowPyrLK
 *
 * Conventions
 *   - every function returns 0 on success, a negative SVO_B200_E* code on argument / CUDA errors;
 *     svo_b200_last_error(ctx) gives the text.  Algorithmic "failures" (no features, GN rollback,
 *     align not converged, seed without match) are reported in-band exactly like the reference and
 *     are NOT errors.  Nothing throws across this boundary.
 *   - SE3 = row-major 3x4 [R|t] doubles (12 values).  Images are 8-bit, row pitch == width.
 *   - host pointers are caller-owned and only read/written during the call; device memory is owned
 *     by the context.  One context = one GPU + one CUDA stream; use one context per calling host
 *     thread (tracking / mapping), as the reference's two threads do.
 *   - there is NO CPU fallback: if no CUDA device is usable, svo_b200_create fails.
 */
#ifndef SVO_B200_H_
#define SVO_B200_H_
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define SVO_B200_MAX_LEVELS 8

#define SVO_B200_OK 0
#define SVO_B200_EINVAL (-1)   /* bad argument */
#define SVO_B200_ECUDA (-2)    /* CUDA runtime error */
#define SVO_B200_ENOMEM (-3)   /* allocation failure */
#define SVO_B200_ELIMIT (-4)   /* size beyond what the kernels support */

typedef struct svo_b200_ctx svo_b200_ctx;
typedef struct svo_b200_frame svo_b200_frame;

/* [EXT] vk::AbstractCamera: the two models the reference ships parameter files for
 * (svo_ros/param/camera_pinhole.yaml, camera_atan.yaml; svo/include/svo/frame_handler_mono.h:64).
 *   SVO_B200_CAM_PINHOLE  vk::PinholeCamera(width, height, fx, fy, cx, cy, d0, d1, d2, d3, d4): d = radial-tangential
 *                         coefficients (k1, k2, p1, p2, k3); all zero = no distortion.
 *   SVO_B200_CAM_ATAN     vk::ATANCamera(width, height, fx, fy, cx, cy, s) (PTAM's FOV model): fx, fy, cx, cy are the
 *                         PIXEL values the vikit constructor derives (fx_ = width*fx, cx_ = width*cx - 0.5, ...),
 *                         d[0] = s (0 = no distortion).
 * Zero-initialising model and d gives the undistorted pinhole camera.
 * width x height must be the level-0 size of every frame a call hands with the camera (the current frame, the keyframes;
 * for the streams calls, each stream's current frame and the keyframes its seeds refer to), as svo::Frame requires
 * (svo/src/frame.cpp:51): every entry point that takes a camera returns SVO_B200_EINVAL otherwise, before any work. */
#define SVO_B200_CAM_PINHOLE 0
#define SVO_B200_CAM_ATAN 1
typedef struct {
  double fx, fy, cx, cy;
  int width, height;
  int model; /* SVO_B200_CAM_* */
  int reserved_;
  double d[5];
} svo_b200_camera;

/* ------------------------------------------------------------------ context ------------- */
int svo_b200_create(svo_b200_ctx** ctx_out, int device);
void svo_b200_destroy(svo_b200_ctx* ctx);
const char* svo_b200_last_error(const svo_b200_ctx* ctx);
/* cudaStream_t of the context (for CUDA-event timing by the caller) */
void* svo_b200_stream(svo_b200_ctx* ctx);
int svo_b200_synchronize(svo_b200_ctx* ctx);
/* device time (CUDA events on the context's stream) of the kernel launch(es) of the most recent entry point that
 * launched any, excluding its host<->device copies; synchronises on that launch.  Runs of a staged batch that overlap the
 * run before them (svo_b200_sia_batch_run) record no events: after back-to-back runs this is the time of the first one. */
int svo_b200_last_kernel_ms(svo_b200_ctx* ctx, float* ms_out);
/* number of kernels this context has launched since creation */
uint64_t svo_b200_launch_count(const svo_b200_ctx* ctx);
const char* svo_b200_version(void);

/* ------------------------------------------------------------------ frames -------------- */
/* A frame = an image pyramid resident in HBM (svo::Frame::img_pyr_).  Level l has size
 * (width >> l, height >> l) (integer division, svo/src/frame.cpp:162). */
int svo_b200_frame_create(svo_b200_ctx* ctx, int width, int height, int n_levels,
                          svo_b200_frame** frame_out);
/* Rounding of the device-side pyramid build (vk::halfSample [EXT], called by frame_utils::createImgPyramid,
 * svo/src/frame.cpp:156-165).  vikit has two branches that round differently:
 *   SVO_B200_PYR_X86 (default)  what the reference computes on its own platform (x86): the SSE2 branch
 *       avg(avg(top, bottom)) of adjacent columns, round-half-up twice (_mm_avg_epu8, _mm_avg_epu16), whenever the
 *       source level's width is a multiple of 16 (cv::Mat buffers are 16-byte aligned), else the scalar branch;
 *   SVO_B200_PYR_SCALAR         (a+b+c+d)/4 with integer division at every level (non-SIMD builds).
 * 640, 752 and 1920 are multiples of 16, so on x86 at least the first level always takes the SSE2 branch. */
#define SVO_B200_PYR_SCALAR 0
#define SVO_B200_PYR_X86 1
int svo_b200_set_pyramid_rule(svo_b200_ctx* ctx, int rule);

/* Upload n_given >= 1 levels from host memory (levels[l] has pitch == width>>l).  Levels
 * n_given..n_levels-1 are built on the device with vk::halfSample's rule (svo_b200_set_pyramid_rule).
 * The copy is asynchronous on the context stream when host memory is pinned. */
int svo_b200_frame_upload(svo_b200_ctx* ctx, svo_b200_frame* frame, const uint8_t* const* levels,
                          int n_given);
/* The arguments of one single-level svo_b200_frame_upload call, for svo_b200_frame_upload_streams. */
typedef struct svo_b200_frame_upload_entry {
  svo_b200_frame* frame;  /* a frame of this context's device; frame-pool frames allowed */
  const uint8_t* level0;  /* host image, pitch == frame width */
} svo_b200_frame_upload_entry;
/* S frames (e.g. the new frames of S camera streams) uploaded and their pyramids built together: each level 0 is copied
 * straight into its frame, then one launch builds level 1 of every entry whose width is a multiple of 16 and that has more
 * than one level, one launch makes the tiled copies no pyramid kernel makes, and one launch per fused pass (four levels
 * each) serves every entry that needs the pass -- the launch count depends on the deepest pyramid, not on S: at most four
 * for SVO_B200_MAX_LEVELS levels, two for 5-level frames whose widths are multiples of 16.  Entries may differ in size and
 * level count, and may name frames of one pool, in any order.  Every frame's levels and tiled copies equal those of
 * svo_b200_frame_upload(ctx, frame, &level0, 1), byte for byte, under either pyramid rule.  Every entry is checked before
 * anything is copied, launched or written (SVO_B200_EINVAL for S < 0, NULL `entries`, a NULL frame or image and a frame
 * listed twice), so a refused call leaves every frame as it was.  SVO_B200_ELIMIT when a launch's work exceeds one grid.
 * S == 0 returns 0 without a launch.  The copies are asynchronous on the context stream when the host memory is pinned. */
int svo_b200_frame_upload_streams(svo_b200_ctx* ctx, int S, const svo_b200_frame_upload_entry* entries);
/* Device-to-device variant: level 0 already on this GPU. */
int svo_b200_frame_upload_device(svo_b200_ctx* ctx, svo_b200_frame* frame, const void* level0_dev);
int svo_b200_frame_download_level(svo_b200_ctx* ctx, const svo_b200_frame* frame, int level,
                                  uint8_t* out);
/* Every upload also writes a block-tiled copy of each level, which the alignment kernel gathers its footprints from.
 * This copies it out, ceil(w/4) * ceil(h/4) * 16 bytes for a w x h level: block (bx, by) at byte 16 * (by * ceil(w/4) + bx)
 * holds rows 4by..4by+3 of columns 4bx..4bx+3, four bytes per row; pixels outside the level are zero. */
int svo_b200_frame_download_level_tiled(svo_b200_ctx* ctx, const svo_b200_frame* frame, int level, uint8_t* out);
void svo_b200_frame_destroy(svo_b200_ctx* ctx, svo_b200_frame* frame);

/* A pool = `count` frames of one geometry in ONE device slab (constant stride), so that a window of
 * a camera stream is uploaded with a single strided host->device copy and its pyramids are built by a
 * single fused kernel (levels 1..4 from one read of level 0).  Frames obtained from a pool are
 * borrowed handles: valid until the pool is destroyed, never passed to svo_b200_frame_destroy. */
typedef struct svo_b200_frame_pool svo_b200_frame_pool;
int svo_b200_frame_pool_create(svo_b200_ctx* ctx, int width, int height, int n_levels, int count,
                               svo_b200_frame_pool** pool_out);
svo_b200_frame* svo_b200_frame_pool_get(svo_b200_frame_pool* pool, int index);
/* Upload level 0 of frames [first, first+count) from host memory (image i at level0_host +
 * i*host_stride_bytes, row pitch == width) and build their pyramids.  Asynchronous on the context
 * stream when the host memory is pinned. */
int svo_b200_frame_pool_upload(svo_b200_ctx* ctx, svo_b200_frame_pool* pool, int first, int count,
                               const uint8_t* level0_host, size_t host_stride_bytes);
void svo_b200_frame_pool_destroy(svo_b200_ctx* ctx, svo_b200_frame_pool* pool);

/* ------------------------------------------------------------------ SparseImgAlign ------ */
typedef struct {
  int max_level, min_level; /* coarsest / finest pyramid level (ctor args) */
  int n_iter;               /* max GN iterations per level (< 0: 1000, the reference's unbounded size_t) */
  double eps;               /* convergence threshold on |x|_inf; reference: 1e-6 */
} svo_b200_sia_options;

/* Per-iteration record, same fields as the oracle's trace (tests only). */
typedef struct {
  int level, iter, accepted, n_meas;
  double chi2;
  double x[6];
  double T[12];
} svo_b200_sia_iter;

/* Per-pair counters used for the algorithmic-bytes model (SURVEY.md 8d). */
typedef struct {
  int32_t n_iters;      /* residual passes executed, all levels */
  int32_t sum_visible;  /* sum over levels of |visible set| at that level */
  int32_t sum_in_image; /* sum over passes of patches inside the current image */
  int32_t n_tracked;    /* return value of run(): patches in the last pass */
} svo_b200_sia_stats;

/* One frame pair.  T_cur_from_ref_io: in = cur.T_f_w * ref.T_f_w^-1, out = optimised value
 * (the caller forms cur.T_f_w_ = T_cur_from_ref * ref.T_f_w_, sparse_img_align.cpp:70).
 * px: N x 2 level-0 pixels; f: N x 3 unit bearings; point_pos: N x 3 world points;
 * has_point: N flags (point != NULL); ref_pos = ref_frame->pos().
 * Outputs (each may be NULL): visible_out N bytes; H_out 36 doubles (H_ of the last pass);
 * stats_out; trace_out/trace_cap/n_trace_out. */
int svo_b200_sparse_img_align(svo_b200_ctx* ctx, const svo_b200_frame* ref, const svo_b200_frame* cur,
                              const svo_b200_camera* cam, const svo_b200_sia_options* opt,
                              double* T_cur_from_ref_io, const double* px, const double* f,
                              const double* point_pos, const uint8_t* has_point,
                              const double* ref_pos, int N, uint8_t* visible_out, double* H_out,
                              svo_b200_sia_stats* stats_out, svo_b200_sia_iter* trace_out,
                              int trace_cap, int* n_trace_out);

/* Batch of B independent frame pairs (one CTA -- or, for small B, one thread-block cluster -- each).  Three-phase API so that the caller can
 * time the device part alone: stage (H2D of poses + features), run (kernels), fetch (D2H).
 * feat_offset has B+1 entries; pair b owns features [feat_offset[b], feat_offset[b+1]). */
int svo_b200_sia_batch_stage(svo_b200_ctx* ctx, int B, const svo_b200_frame* const* ref,
                             const svo_b200_frame* const* cur, const svo_b200_camera* cam,
                             const svo_b200_sia_options* opt, const double* T_cur_from_ref /*B*12*/,
                             const int* feat_offset, const double* px, const double* f,
                             const double* point_pos, const uint8_t* has_point,
                             const double* ref_pos /*B*3*/);
/* Consecutive runs of one staged batch may overlap on the device: when one CTA per pair runs (the throughput geometry of
 * full batches) and the last work the library enqueued on the context's stream is a run of the same batch, the next run's
 * CTAs start while the previous run's last wave drains.  Each run reads only what the stage and the frame uploads wrote, and
 * stores its outputs after the run before it has completed, so a fetch returns the outputs of the last run.  Any other call
 * that enqueues work (stage, fetch, uploads, the other kernels) ends the overlap.  Work of the caller's own enqueued on the
 * context's stream between two runs must not write the frames or anything else the batch reads. */
int svo_b200_sia_batch_run(svo_b200_ctx* ctx);
int svo_b200_sia_batch_fetch(svo_b200_ctx* ctx, double* T_out /*B*12*/, uint8_t* visible_out,
                             double* H_out /*B*36 or NULL*/, svo_b200_sia_stats* stats_out /*B or NULL*/);

/* Launch geometry of the alignment kernel (tuning / tests; results agree to rounding between geometries).
 *   ctas_per_pair: -1 = automatic (a 4-CTA thread-block cluster per pair while 4*B <= #SMs, i.e. live streams and
 *                  small batches; one CTA per pair otherwise), or 1, 2, 4, 8 (clusters need <= 96*ctas features per pair).
 *   features_per_thread: 0 = automatic (2 whenever one CTA per pair is used and every pair has <= 304 features), 1, or 2
 *                  (one CTA per pair only; pairs with more than 304 features run with 1). */
int svo_b200_sia_config(svo_b200_ctx* ctx, int ctas_per_pair, int features_per_thread);
/* Small batches in the 4-CTA cluster geometry (every CTA alone on an SM) prepare the reference patches, H and its
 * factorisation of ALL pyramid levels before the first Gauss-Newton iteration ("upfront"; none of it depends on the pose,
 * svo/src/sparse_img_align.cpp:84-145 runs it lazily per level).  mode: -1 = automatic (default), 0 = per level, 1 = as -1. */
int svo_b200_sia_upfront(svo_b200_ctx* ctx, int mode);

/* How the current image of one pyramid level reaches the alignment kernel's residual loop. */
#define SVO_B200_SIA_STAGE_GLOBAL 0 /* gathered from global memory */
#define SVO_B200_SIA_STAGE_IMAGE 1  /* the whole level copied into shared memory by one TMA bulk copy */
#define SVO_B200_SIA_STAGE_WINDOW 2 /* a 16x8-byte window per feature copied into shared memory with cp.async */
/* The launch of the most recent svo_b200_sparse_img_align, svo_b200_sparse_residuals or svo_b200_sia_batch_run:
 * which kernel instantiation ran and how it staged every level (tests and tuning). */
typedef struct {
  int n_pairs;             /* B */
  int ctas_per_pair;       /* 1, or the thread-block cluster size 2, 4, 8 */
  int threads;             /* per CTA */
  int features_per_thread; /* 1 or 2 */
  int min_blocks;          /* resident CTAs per SM the instantiation is compiled for (__launch_bounds__) */
  int upfront;             /* cluster geometry with all levels prepared before the first iteration; it exchanges the
                              per-iteration sums by st.async + mbarrier instead of DSMEM stores + barrier.cluster */
  int general_camera;      /* 1 = general camera models compiled in, 0 = the undistorted-pinhole instantiation */
  int residuals_only;      /* 1 = the svo_b200_sparse_residuals pass */
  int stage_cap;           /* bytes of the shared-memory staging region */
  int smem_bytes;          /* dynamic shared memory per CTA */
  int resident_clusters;   /* cudaOccupancyMaxActiveClusters of the 4-CTA upfront cluster kernel as the choice last consulted
                              it (0 = not consulted by this context yet) */
  int sm_count;            /* multiprocessors of the device */
  int min_level, max_level;
  int level_stage[SVO_B200_MAX_LEVELS]; /* SVO_B200_SIA_STAGE_* of levels min_level..max_level, -1 elsewhere */
} svo_b200_sia_launch;
/* Returns SVO_B200_EINVAL if the context has not launched the alignment kernel yet. */
int svo_b200_sia_last_launch(const svo_b200_ctx* ctx, svo_b200_sia_launch* out);

/* ---- robust cost of SparseImgAlign: vk::NLLSSolver::setRobustCostFunction(scale_estimator, weight_function) ----
 * Numbering as vikit's ScaleEstimatorType / WeightFunctionType. */
#define SVO_B200_SCALE_UNIT 0   /* weights off: plain Gauss-Newton, whatever the weight function (default) */
#define SVO_B200_SCALE_TDIST 1  /* not supported */
#define SVO_B200_SCALE_MAD 2    /* scale_ = 1.48 * upper median of |res| */
#define SVO_B200_SCALE_NORMAL 3 /* not supported */
#define SVO_B200_WEIGHT_UNIT 0
#define SVO_B200_WEIGHT_TDIST 1 /* not supported */
#define SVO_B200_WEIGHT_TUKEY 2 /* b = 4.6851 */
#define SVO_B200_WEIGHT_HUBER 3 /* k = 1.345 */
/* Context setting like svo_b200_sia_config.  It applies to svo_b200_sparse_img_align and svo_b200_sia_batch_stage (a staged
 * batch keeps the mode it was staged with); svo_b200_sparse_residuals ignores it.  With weights on (MAD scale) the robust
 * kernel runs: one CTA per pair, 0..1024 features (SVO_B200_ELIMIT above), every camera model; svo_b200_sia_config and
 * svo_b200_sia_upfront do not apply to it, and it does not run with a multi-GPU feature split (SVO_B200_EINVAL).
 * The scale is computed as the reference does it: by the pre-pass each level's Gauss-Newton loop starts with, and only when
 * iter_ is 0 there -- at the first level, and at a later level only if the previous level's loop ended at iteration 0;
 * otherwise the scale carries over.  SVO_B200_EINVAL for the T-distribution / normal scales, the T-distribution weight and
 * values outside the enums. */
int svo_b200_sia_robust(svo_b200_ctx* ctx, int scale_estimator, int weight_function);
/* The scale_ each of the B pairs of the last alignment launch used at each level, out[b * SVO_B200_MAX_LEVELS + level]; NaN
 * outside [min_level, max_level].  Available once the launch's outputs are fetched (svo_b200_sparse_img_align,
 * svo_b200_sia_batch_fetch).  SVO_B200_EINVAL if the last alignment launch was not weighted or had fewer than B pairs. */
int svo_b200_sia_last_scales(const svo_b200_ctx* ctx, int B, float* out);

/* ---- one stream's features split over several GPUs (SURVEY.md 8e; a demonstration mode: a pair fits one GPU) ----
 * Every rank (one process or thread per GPU) holds both pyramids and passes ITS contiguous slice of the pair's features
 * to svo_b200_sparse_img_align / svo_b200_sia_batch_*; the kernels of the ranks exchange the per-iteration sums
 * (6 Jres + chi2 + counts, and the 21 H entries once per level) directly through peer memory over NVLink -- no host
 * round trip, no collective-library call inside the Gauss-Newton loop -- and all ranks finish with the same pose, H and
 * n_tracked; the visibility mask covers the rank's slice.  All ranks must issue the same sequence of alignment calls.
 *   create   allocates this rank's exchange buffer (max_pairs pairs per launch) and returns its CUDA IPC handle
 *            (SVO_B200_IPC_HANDLE_BYTES bytes) and / or its device pointer;
 *   connect  maps the peers: `ipc_handles` = world handles in rank order (other processes; all-gather them with the
 *            launcher's own means), or `in_process_ptrs` = world device pointers (ranks that share the process).
 *            Every rank must have connected before any rank launches (launcher barrier);
 *   destroy  unmaps / frees.  An exchange a peer never joins times out after ~2 s: the next fetch returns SVO_B200_ECUDA. */
#define SVO_B200_IPC_HANDLE_BYTES 64
int svo_b200_sia_split_create(svo_b200_ctx* ctx, int rank, int world, int max_pairs, void* ipc_handle_out, void** local_ptr_out);
int svo_b200_sia_split_connect(svo_b200_ctx* ctx, const void* ipc_handles, void* const* in_process_ptrs);
int svo_b200_sia_split_destroy(svo_b200_ctx* ctx);

/* computeResiduals(model, linearize=true) at one level and pose, exposing the caches; visible_io
 * carries the set-only visibility flags in and out. */
int svo_b200_sparse_residuals(svo_b200_ctx* ctx, const svo_b200_frame* ref, const svo_b200_frame* cur,
                              const svo_b200_camera* cam, int level, const double* T_cur_from_ref,
                              const double* px, const double* f, const double* point_pos,
                              const uint8_t* has_point, const double* ref_pos, int N,
                              uint8_t* visible_io, float* ref_patch_out /*N*16*/,
                              float* residuals_out /*N*16, NaN where not evaluated*/,
                              uint8_t* in_image_out /*N*/, double* H_out /*36*/, double* Jres_out /*6*/,
                              double* chi2_out, int64_t* n_meas_out);

/* ------------------------------------------------------------------ feature alignment --- */
/* M independent align2D calls on levels of one frame: ref_patch_with_border M*100, ref_patch M*64,
 * level[M], px_io M*2 (level coordinates).  converged_out[M]: 1 / 0 as the reference's bool. */
int svo_b200_align2d_batch(svo_b200_ctx* ctx, const svo_b200_frame* cur, int M, const int* level,
                           const uint8_t* ref_patch_with_border, const uint8_t* ref_patch,
                           int n_iter, double* px_io, uint8_t* converged_out);
int svo_b200_align1d_batch(svo_b200_ctx* ctx, const svo_b200_frame* cur, int M, const int* level,
                           const float* dir /*M*2*/, const uint8_t* ref_patch_with_border,
                           const uint8_t* ref_patch, int n_iter, double* px_io,
                           uint8_t* converged_out, double* h_inv_out);

/* M Matcher::findMatchDirect calls (after Point::getCloseViewObs chose the reference feature):
 * warp the 10x10 reference patch (getWarpMatrixAffine, getBestSearchLevel, warpAffine) and align.
 * ref_index[M] selects one of n_ref reference frames / poses; every ref_frames entry must be non-NULL.
 * M == 0 returns 0 without reading the frames (n_ref may then be 0).  search_level_out, A_cur_ref_out
 * and h_inv_out may be NULL. */
typedef struct {
  int max_search_level; /* Config::nPyrLevels()-1 */
  int align_max_iter;   /* Matcher::Options::align_max_iter = 10 */
} svo_b200_match_options;
int svo_b200_find_match_direct(svo_b200_ctx* ctx, const svo_b200_frame* const* ref_frames,
                               const double* ref_T_f_w /*n_ref*12*/, int n_ref,
                               const svo_b200_frame* cur, const double* cur_T_f_w,
                               const svo_b200_camera* cam, const svo_b200_match_options* opt, int M,
                               const int* ref_index, const double* ref_px, const double* ref_f,
                               const int* ref_level, const int* ftr_type, const double* ref_grad,
                               const double* point_pos /*M*3*/, double* px_cur_io /*M*2*/,
                               uint8_t* success_out, int* search_level_out, double* A_cur_ref_out /*M*4*/,
                               double* h_inv_out);

/* ------------------------------------------------------------------ pose optimizer ------ */
typedef struct {
  double estimated_scale, error_init, error_final;
  int64_t num_obs;
  int n_iter_done;
  /* Which 6x6 solves ran, for tests and diagnostics (they sit in what was padding: size and offsets are unchanged).
   * n_pivoted_solves: Gauss-Newton iterations whose normal matrix failed the unpivoted LDL^T's pivot test
   * (a pivot <= 1e-13 * max diagonal) and took the pivoted LDL^T; cov_pivoted: 1 if the covariance took the
   * Gauss-Jordan inverse for the same reason. */
  int16_t n_pivoted_solves, cov_pivoted;
  double cov[36];
} svo_b200_pose_opt_result;
int svo_b200_pose_optimize(svo_b200_ctx* ctx, double reproj_thresh, int n_iter,
                           double fx /*cam->errorMultiplier2()*/, double* T_f_w_io, const double* f,
                           const double* point_pos, const int* level, uint8_t* has_point_io, int N,
                           svo_b200_pose_opt_result* out);

/* B frames in one launch (one CTA per frame): frame b owns observations [obs_offset[b], obs_offset[b+1]) of the
 * concatenated arrays; fx[b] = that frame's cam->errorMultiplier2().  Same results as B single calls.
 * Requires 0 <= obs_offset[0] <= obs_offset[1] <= ... <= obs_offset[B]; otherwise SVO_B200_EINVAL, nothing written
 * but out (zeroed). */
int svo_b200_pose_optimize_batch(svo_b200_ctx* ctx, int B, double reproj_thresh, int n_iter, const double* fx /*B*/,
                                 double* T_f_w_io /*B*12*/, const int* obs_offset /*B+1*/, const double* f,
                                 const double* point_pos, const int* level, uint8_t* has_point_io,
                                 svo_b200_pose_opt_result* out /*B*/);

/* Point::optimize (svo/src/point.cpp:119-177) for P independent points ("next" row f3: structure
 * refinement after the pose optimizer, frame_handler_base.cpp:178-196).  Point p owns observations
 * [obs_offset[p], obs_offset[p+1]); observation o is seen from frame obs_frame[o] (pose frame_T_f_w) with
 * unit bearing obs_f[o].  pos_io: P*3 world positions, updated in place.
 * Requires 0 <= obs_offset[0] <= obs_offset[1] <= ... <= obs_offset[P] and 0 <= obs_frame[o] < n_frames for the
 * observations in [obs_offset[0], obs_offset[P]) (entries before obs_offset[0] are not read); otherwise
 * SVO_B200_EINVAL before anything is launched or written. */
int svo_b200_point_optimize_batch(svo_b200_ctx* ctx, int P, int n_iter, const int* obs_offset,
                                  const int* obs_frame, const double* obs_f, const double* frame_T_f_w,
                                  int n_frames, double* pos_io);

/* ------------------------------------------------------------------ reprojector ("next" row f2) -------- */
/* Flat, read-only view of the map's pointer graph (Map::keyframes_, Frame::fts_, Feature, Point::obs_,
 * MapPointCandidates::candidates_), gathered by the host wrapper (rpg_svo_b200/host/svo_host.h: svo::Reprojector). */
typedef struct svo_b200_map_view {
  int n_kfs;                     /* Map::keyframes_ in list order (map.h:74) */
  const double* kf_T_f_w;        /* n_kfs*12 */
  const double* kf_keypt_pos;    /* n_kfs*5*3: key_pts_[i]->point->pos_ (frame.h:53) */
  const uint8_t* kf_keypt_valid; /* n_kfs*5: key_pts_[i] != NULL */
  const int* kf_fts_offset;      /* n_kfs+1: Frame::fts_ of keyframe k = kf_fts[offset[k] .. offset[k+1]);
                                    0 <= offset[0] <= offset[1] <= ... <= offset[n_kfs] */
  const int* kf_fts;             /* indices into the feature table, fts_ list order */
  int n_ftrs;                    /* feature table: every Feature a Frame::fts_ or Point::obs_ entry refers to */
  const int* ftr_kf;             /* Feature::frame as keyframe index */
  const double* ftr_px;          /* n_ftrs*2 */
  const double* ftr_f;           /* n_ftrs*3 */
  const int* ftr_level;
  const int* ftr_type;           /* 0 CORNER, 1 EDGELET (feature.h:29-32) */
  const double* ftr_grad;        /* n_ftrs*2 */
  const int* ftr_point;          /* Feature::point as point index, -1 = NULL */
  int n_points;
  const double* pt_pos;          /* n_points*3 */
  const int* pt_obs_offset;      /* n_points+1: Point::obs_ of point p = pt_obs[offset[p] .. offset[p+1]);
                                    0 <= offset[0] <= offset[1] <= ... <= offset[n_points] */
  const int* pt_obs;             /* Point::obs_ in list order, as feature-table indices */
  int n_candidates;
  const int* cand_point;         /* MapPointCandidates::candidates_ in list order, as point indices (map.h:44) */
} svo_b200_map_view;
typedef struct svo_b200_reproject_options {
  int grid_size;         /* Config::gridSize()  (config.cpp:32: 30) */
  int max_fts;           /* Config::maxFts()    (config.cpp:52: 120) */
  int max_n_kfs;         /* Reprojector::Options::max_n_kfs (reprojector.h:44: 10) */
  int find_match_direct; /* Reprojector::Options::find_match_direct (reprojector.h:45: true) */
  int max_search_level;  /* Config::nPyrLevels()-1 (matcher.cpp:153) */
  int align_max_iter;    /* Matcher::Options::align_max_iter (matcher.h:77: 10) */
} svo_b200_reproject_options;
typedef struct svo_b200_reproject_stats {
  int64_t n_matches, n_trials; /* Reprojector::n_matches_, n_trials_ (reprojector.h:51-52) */
  int n_new;                   /* features added to the frame */
  int n_overlap;               /* overlap_kfs.size() */
  int n_projected;             /* points that fell into a grid cell */
  int n_speculative;           /* matches computed on the device (>= n_trials: every in-frame point is aligned) */
} svo_b200_reproject_stats;
#define SVO_B200_PT_NONE 0
#define SVO_B200_PT_SAFE_DELETE 1      /* caller must run map_.safeDeletePoint(pt)               (reprojector.cpp:173-174) */
#define SVO_B200_PT_DELETE_CANDIDATE 2 /* caller must run point_candidates_.deleteCandidatePoint (reprojector.cpp:175-176) */
#define SVO_B200_PT_CANDIDATE_ERASED 3 /* candidate erased while projecting: deleteCandidate+erase (reprojector.cpp:117-122) */
/* Reprojector::reprojectMap.  The device projects every map point of the closest keyframes and every candidate into
 * `cur`, and aligns ALL in-frame points speculatively in one launch (getCloseViewObs + findMatchDirect per warp); the
 * host then replays the reference's one-match-per-cell policy over those results in `cell_order`
 * (Reprojector::Grid::cell_order, shuffled once by the caller as initializeGrid does), applying the reference's side
 * effects only to the candidates the sequential code would have reached.
 *   kf_frames: n_kfs uploaded keyframe pyramids.  Point types: 0 DELETED, 1 CANDIDATE, 2 UNKNOWN, 3 GOOD (point.h:40-45).
 *   pt_*_io: Point::type_, n_failed_reproj_, n_succeeded_reproj_ per point, updated in place; pt_action_out: SVO_B200_PT_*.
 *   overlap_kf_out / overlap_count_out: max_n_kfs entries (overlap_kfs of the reference, keyframe index + count).
 *   new_*: the Features the reference would add to the frame, in order (max_fts+1 entries): point index, px, level,
 *   type, grad. */
int svo_b200_reproject_map(svo_b200_ctx* ctx, const svo_b200_map_view* map, const svo_b200_frame* const* kf_frames,
                           const svo_b200_frame* cur, const double* cur_T_f_w, const svo_b200_camera* cam,
                           const svo_b200_reproject_options* opt, const int* cell_order, int* pt_type_io,
                           int* pt_n_failed_io, int* pt_n_succeeded_io, uint8_t* pt_action_out, int* overlap_kf_out,
                           int64_t* overlap_count_out, int* new_point_out, double* new_px_out, int* new_level_out,
                           int* new_type_out, double* new_grad_out, svo_b200_reproject_stats* stats);

/* The arguments of one svo_b200_reproject_map call, for svo_b200_reproject_map_streams. */
typedef struct svo_b200_reproject_stream {
  const svo_b200_map_view* map;
  const svo_b200_frame* const* kf_frames;
  const svo_b200_frame* cur;
  const double* cur_T_f_w;
  const svo_b200_camera* cam;
  const svo_b200_reproject_options* opt;
  const int* cell_order;
  int* pt_type_io;
  int* pt_n_failed_io;
  int* pt_n_succeeded_io;
  uint8_t* pt_action_out;
  int* overlap_kf_out;
  int64_t* overlap_count_out;
  int* new_point_out;
  double* new_px_out;
  int* new_level_out;
  int* new_type_out;
  double* new_grad_out;
  svo_b200_reproject_stats* stats;
} svo_b200_reproject_stream;
/* S streams' Reprojector::reprojectMap: one device launch over the enumerated points of every stream, then each
 * stream's one-match-per-cell replay into its own outputs.  Every output and the stats equal S calls of
 * svo_b200_reproject_map, bit for bit.  Streams may share frame handles and map views; the _io / _out arrays of
 * different streams must not overlap.  Every stream's arguments are checked before anything is launched or written
 * (SVO_B200_EINVAL for S < 0, a NULL frame, an index out of range in a map view, ...), so a refused call leaves every
 * output untouched.  S == 0 returns 0; streams that enumerate no point take no part in the launch. */
int svo_b200_reproject_map_streams(svo_b200_ctx* ctx, int S, const svo_b200_reproject_stream* streams);

/* ------------------------------------------------------------------ FAST detector ("next" row f4) -------- */
typedef struct svo_b200_detect_options {
  int cell_size;               /* Config::gridSize() (config.cpp:32: 30) */
  int n_pyr_levels;            /* Config::nPyrLevels() (config.cpp:30: 3): levels searched */
  int fast_threshold;          /* the literal 20 of feature_detection.cpp:78-92 */
  int nonmax_ties_suppress;    /* [EXT] fast_nonmax_3x3: 0 = only a larger neighbour suppresses (libCVD non-strict, default); 1 = ties too */
  double detection_threshold;  /* Config::triangMinCornerScore() (config.cpp:44: 20.0); must be >= 0 */
} svo_b200_detect_options;
/* FastDetector::detect: FAST-10 + score + 3x3 non-maximum suppression on levels 0..n_pyr_levels-1, Shi-Tomasi score of
 * every surviving corner, the best corner of every grid cell that is not flagged in grid_occupancy (ceil(w/cell) *
 * ceil(h/cell) bytes, NULL = all free; AbstractDetector::setExistingFeatures / setGridOccpuancy are the caller's).
 * Outputs in cell order, level-0 pixel coordinates (the reference then builds Feature(frame, Vector2d(x, y), level));
 * *n_out is the number found, at most `cap` of them are written; score_out may be NULL. */
int svo_b200_fast_detect(svo_b200_ctx* ctx, const svo_b200_frame* frame, const svo_b200_detect_options* opt,
                         const uint8_t* grid_occupancy, int cap, int* x_out, int* y_out, int* level_out, float* score_out,
                         int* n_out);

/* The arguments of one svo_b200_fast_detect call, for svo_b200_fast_detect_streams. */
typedef struct svo_b200_detect_stream {
  const svo_b200_frame* frame;
  const svo_b200_detect_options* opt;
  const uint8_t* grid_occupancy; /* NULL = all cells free */
  int cap;
  int *x_out, *y_out, *level_out;
  float* score_out; /* may be NULL */
  int* n_out;
} svo_b200_detect_stream;
/* S streams' FastDetector::detect (e.g. the keyframes of S depth filters' initializeSeeds) in one launch: one copy to the
 * device, one launch, one copy back.  Every stream's outputs and *n_out equal one svo_b200_fast_detect call with that
 * stream's arguments, bit for bit.  Streams may share frame handles (frame-pool frames included) with different options
 * and grids; the output arrays of different streams must not overlap.  Every stream's arguments are checked as
 * svo_b200_fast_detect checks them before anything is launched or written (SVO_B200_EINVAL, also for S < 0 or NULL
 * `streams`; SVO_B200_ELIMIT when the streams' tiles exceed one launch's grid), so a refused call leaves every output
 * untouched.  S == 0 returns 0 without a launch.  svo_b200_fast_detect is S = 1 of this call. */
int svo_b200_fast_detect_streams(svo_b200_ctx* ctx, int S, const svo_b200_detect_stream* streams);

/* ------------------------------------------------------------------ depth filter -------- */
#define SVO_B200_SEED_TOO_OLD 1
#define SVO_B200_SEED_BEHIND 2
#define SVO_B200_SEED_NOT_IN_FRAME 3
#define SVO_B200_SEED_NO_MATCH 4
#define SVO_B200_SEED_UPDATED 5
#define SVO_B200_SEED_CONVERGED 6
#define SVO_B200_SEED_NAN 7

typedef struct {
  int max_n_kfs;                         /* DepthFilter::Options::max_n_kfs = 3 */
  double seed_convergence_sigma2_thresh; /* 200 */
  int max_search_level;                  /* Config::nPyrLevels()-1 */
  int align_max_iter;                    /* 10 */
  int max_epi_search_steps;              /* 1000 */
} svo_b200_depth_options;

/* DepthFilter::updateSeeds over M seeds in SoA form.  Seeds are updated in place; status_out tells
 * the host which list operations / callbacks to replay in list order. */
int svo_b200_depth_filter_update(svo_b200_ctx* ctx, const svo_b200_frame* const* ref_frames,
                                 const double* ref_T_f_w, int n_ref, const svo_b200_frame* cur,
                                 const double* cur_T_f_w, const svo_b200_camera* cam,
                                 const svo_b200_depth_options* opt, int M, const int* ref_index,
                                 const double* ftr_px, const double* ftr_f, const int* ftr_level,
                                 const int* ftr_type, const double* ftr_grad, const int* batch_id,
                                 int batch_counter, float* a, float* b, float* mu, float* z_range,
                                 float* sigma2, uint8_t* status_out, double* px_cur_out,
                                 double* z_out, int* n_zmssd_out);

/* S streams' DepthFilter::updateSeeds in one launch; the result is bit-identical to S calls of
 * svo_b200_depth_filter_update.  Stream s has current frame cur[s], pose cur_T_f_w[12*s .. 12*s+11], camera cam[s]
 * (the models may differ between streams) and Seed::batch_counter batch_counter[s], and owns seeds
 * [seed_offset[s], seed_offset[s+1]) of the per-seed arrays, which are laid out as in svo_b200_depth_filter_update
 * (seed_offset has S+1 entries, seed_offset[0] == 0).  ref_index indexes ONE keyframe table (ref_frames, ref_T_f_w,
 * n_ref) shared by all streams; streams may share keyframe and current-frame handles.  One options struct for all.
 * SVO_B200_EINVAL for S < 0, a NULL frame, seed offsets that do not start at 0 or are not monotone, a ref_index or
 * ftr_level out of range, or a max_search_level beyond a current frame's pyramid -- all checked before anything is
 * launched or written, so a refused call leaves every output untouched.  S == 0, or no seeds at all, returns 0 without
 * a launch (the keyframe table is then not read). */
int svo_b200_depth_filter_update_streams(svo_b200_ctx* ctx, int S, const svo_b200_frame* const* cur /*S*/,
                                         const double* cur_T_f_w /*S*12*/, const svo_b200_camera* cam /*S*/,
                                         const int* batch_counter /*S*/, const int* seed_offset /*S+1*/,
                                         const svo_b200_frame* const* ref_frames, const double* ref_T_f_w, int n_ref,
                                         const svo_b200_depth_options* opt, const int* ref_index, const double* ftr_px,
                                         const double* ftr_f, const int* ftr_level, const int* ftr_type,
                                         const double* ftr_grad, const int* batch_id, float* a, float* b, float* mu,
                                         float* z_range, float* sigma2, uint8_t* status_out, double* px_cur_out,
                                         double* z_out, int* n_zmssd_out);

/* M independent Matcher::findEpipolarMatchDirect calls (svo/include/svo/matcher.h:114-121, svo/src/matcher.cpp:179-321):
 * candidate m is reference feature (ref_index, px, f, level, type, grad) searched in `cur` along the epipolar segment of
 * depths [d_min, d_max] around d_estimate.  Outputs = the return value, `depth`, and the Matcher's public scratch
 * members callers read afterwards (px_cur_, search_level_, epi_length_, reject_, A_cur_ref_); each may be NULL except
 * success_out.  n_zmssd_out: ZMSSD evaluations along the line (instrumentation). */
int svo_b200_find_epipolar_match_direct(svo_b200_ctx* ctx, const svo_b200_frame* const* ref_frames,
                                        const double* ref_T_f_w, int n_ref, const svo_b200_frame* cur,
                                        const double* cur_T_f_w, const svo_b200_camera* cam,
                                        const svo_b200_depth_options* opt, int M, const int* ref_index,
                                        const double* ftr_px, const double* ftr_f, const int* ftr_level,
                                        const int* ftr_type, const double* ftr_grad, const double* d_estimate,
                                        const double* d_min, const double* d_max, uint8_t* success_out,
                                        double* depth_out, double* px_cur_out /*M*2*/, int* search_level_out,
                                        double* epi_length_out, uint8_t* reject_out, double* A_cur_ref_out /*M*4*/,
                                        int* n_zmssd_out);

/* ---- Matcher::Options of the epipolar search (svo/include/svo/matcher.h:74-91, read by matcher.cpp:204-320) ----
 * align_max_iter and max_epi_search_steps are the fields of svo_b200_depth_options; max_epi_length_optim is never read by
 * the reference (matcher.cpp:226 uses the literal 2.0). */
typedef struct {
  int align_1d;                        /* Matcher::Options::align_1d (0): align1D along (px_A - px_B).cast<float>().normalized() */
  int subpix_refinement;               /* (1): 0 = the scan's best step is the match, triangulated without alignment */
  int epi_search_edgelet_filtering;    /* (1) */
  double epi_search_edgelet_max_angle; /* (0.7): an edgelet is rejected when cosangle < max_angle (NaN never rejects) */
} svo_b200_epipolar_options;
/* Context setting like svo_b200_sia_robust.  NULL = the reference's defaults.  Applies to svo_b200_find_epipolar_match_direct,
 * svo_b200_depth_filter_update and svo_b200_depth_filter_update_streams (all streams of a call).  At the defaults those
 * run the kernel they always ran; any other setting runs its general instantiation, which follows each option as
 * matcher.cpp does (the short-line branch, epi_length < 2, aligns whatever subpix_refinement says).  Any angle is
 * accepted.  SVO_B200_EINVAL for a flag other than 0 or 1, and the setting is left as it was. */
int svo_b200_set_epipolar_options(svo_b200_ctx* ctx, const svo_b200_epipolar_options* opt);
int svo_b200_get_epipolar_options(const svo_b200_ctx* ctx, svo_b200_epipolar_options* out);
/* Matcher::h_inv_ after each of the first M candidates of the last svo_b200_find_epipolar_match_direct call: ran_1d_out[m]
 * is 1 when align1D ran for candidate m (it sets h_inv_ on entry, whether or not it converges) and h_inv_out[m] is the
 * value it set; 0 and 0 when it did not run, and a Matcher's h_inv_ then keeps its previous value.  SVO_B200_EINVAL before
 * the first such call, or when the last one had fewer than M candidates.  A refused call changes nothing. */
int svo_b200_epipolar_last_h_inv(const svo_b200_ctx* ctx, int M, double* h_inv_out, uint8_t* ran_1d_out);

/* ------------------------------------------------------------------ KLT tracking of the two-view initialisation ------ */
/* initialization::trackKlt (svo/src/initialization.cpp:127-169) tracks every corner of the first keyframe into each new
 * frame with cv::calcOpticalFlowPyrLK(ref, cur, px_ref, px_cur, status, err, Size(30, 30), 4,
 * TermCriteria(COUNT + EPS, 30, 0.001), OPTFLOW_USE_INITIAL_FLOW).  These entry points run OpenCV's published algorithm
 * ([EXT] modules/video/src/lkpyramid.cpp) on the device; see DESIGN.md section 4.2d for the rules it follows.
 *
 * An LK pyramid is OpenCV's, not the frame's vk::halfSample pyramid: level l+1 = pyrDown(level l) ([1 4 6 4 1] filter,
 * reflect-101 borders, (sum + 128) >> 8, size ((w+1)/2, (h+1)/2)), and levels stop once the next one would be no larger
 * than the 30-pixel window (640 x 480 and 752 x 480 get 4 levels, 644 x 484 gets 5).  The pyramid of the previous image
 * also holds the Scharr derivatives of every level (interleaved int16 dx, dy; zero outside the level).  Build the
 * reference frame's pyramid once with derivatives and reuse it; each new frame needs its own pyramid without. */
typedef struct svo_b200_klt_pyramid svo_b200_klt_pyramid;
int svo_b200_klt_pyramid_create(svo_b200_ctx* ctx, svo_b200_klt_pyramid** pyr_out);
void svo_b200_klt_pyramid_destroy(svo_b200_ctx* ctx, svo_b200_klt_pyramid* pyr);
/* Builds the pyramid (at most max_level + 1 levels) from level 0 of `frame`, already on the device.  with_derivatives:
 * 1 = also the Scharr derivatives (the previous image of svo_b200_klt_track), 0 = images only.  A handle may be rebuilt
 * at any size; it keeps its allocation where the new pyramid fits.  Returns SVO_B200_EINVAL for max_level < 0, and where
 * OpenCV's cut would build more than SVO_B200_MAX_LEVELS levels (a side of 7681 pixels or more at max_level >= 8): such
 * a pyramid is refused, not cut short, before anything is allocated or launched, and the handle keeps its last build. */
int svo_b200_klt_pyramid_build(svo_b200_ctx* ctx, svo_b200_klt_pyramid* pyr, const svo_b200_frame* frame, int max_level,
                               int with_derivatives);
/* Number of levels the last build made (0 before the first).  A build that fails to allocate a larger block
 * (SVO_B200_ENOMEM) leaves the handle at 0 levels: svo_b200_klt_track refuses it until a build succeeds. */
int svo_b200_klt_pyramid_levels(const svo_b200_klt_pyramid* pyr);

/* The arguments of one svo_b200_klt_pyramid_build call, for svo_b200_klt_pyramid_build_streams. */
typedef struct svo_b200_klt_build {
  svo_b200_klt_pyramid* pyr;
  const svo_b200_frame* frame;
  int max_level;
  int with_derivatives;
} svo_b200_klt_build;
/* S pyramids (e.g. the new frames of S camera streams) built together: one launch for level 0 of every entry, one pyrDown
 * launch per level 1 .. L_max - 1 (L_max = the most levels any entry builds), and one Scharr launch over every level of
 * every entry with derivatives -- the launch count depends on the deepest pyramid, not on S.  Entries may differ in size,
 * max_level and with_derivatives; frame-pool frames are valid sources.  Every handle equals one svo_b200_klt_pyramid_build
 * with its entry's arguments, byte for byte, and svo_b200_klt_pyramid_build is one entry of this call.  Every entry is
 * checked as the single build checks it before anything is allocated, launched or written (SVO_B200_EINVAL, also for
 * S < 0, NULL `builds` and a handle listed twice), so a refused call leaves every handle as it was.  SVO_B200_ELIMIT when
 * a launch's tiles exceed one grid.  A failed allocation (SVO_B200_ENOMEM) returns before any launch; the handle it was
 * for, and any handle already given a new block in the same call, is left at 0 levels.  S == 0 returns 0 without a
 * launch. */
int svo_b200_klt_pyramid_build_streams(svo_b200_ctx* ctx, int S, const svo_b200_klt_build* builds);
/* Copies one level out: img_out w*h bytes, deriv_out w*h*2 int16 (interleaved dx, dy; needs a build with derivatives);
 * either may be NULL. */
int svo_b200_klt_pyramid_download(svo_b200_ctx* ctx, const svo_b200_klt_pyramid* pyr, int level, uint8_t* img_out,
                                  int16_t* deriv_out);

typedef struct {
  int win_size;  /* only the reference's 30 is supported */
  int max_level; /* coarsest level (initialization.cpp: 4); the levels used are min(max_level + 1, levels of both pyramids) */
  int max_iter;  /* iterations per level (30), clamped to [0, 100] as OpenCV does */
  double eps;    /* stop when |delta| <= eps (0.001), clamped to at most 10 as OpenCV does */
} svo_b200_klt_options;
/* Unlike OpenCV, which clamps them, max_level < 0 and a negative or NaN eps return SVO_B200_EINVAL. */
/* How a point's tracking ended at a level. */
#define SVO_B200_KLT_CONVERGED 0     /* delta . delta <= eps^2 */
#define SVO_B200_KLT_HALF_STEP 1     /* two consecutive steps nearly cancelled: stepped back half a step */
#define SVO_B200_KLT_MAX_ITER 2      /* max_iter steps taken */
#define SVO_B200_KLT_OUT_OF_BOUNDS 3 /* the window left the level (status 0 only at level 0) */
#define SVO_B200_KLT_SMALL_EIG 4     /* min eigenvalue of the window's gradient matrix / 900 < 1e-4, or its determinant
                                        < FLT_EPSILON (status 0 only at level 0) */
typedef struct {
  int32_t reason;                              /* SVO_B200_KLT_* at level 0 */
  int32_t level_reason[SVO_B200_MAX_LEVELS];   /* SVO_B200_KLT_* per level, -1 for levels not run */
  int32_t iters[SVO_B200_MAX_LEVELS];          /* steps taken per level */
} svo_b200_klt_exit;
/* calcOpticalFlowPyrLK with OPTFLOW_USE_INITIAL_FLOW for N points: prev_pts N*2 floats; next_pts_io N*2 floats, in = the
 * initial guess, out = the tracked points; status_out N bytes (1 tracked, 0 lost); exit_out (N entries) may be NULL.
 * OpenCV's `err` output is not produced.  `prev` must have been built with derivatives, `next` with or without; both from
 * frames of one size (one handle may be both).  N == 0 returns 0.  prev_pts and next_pts_io may be the same buffer.  A
 * point with a NaN, an infinite or a huge coordinate in prev_pts or in its guess is lost out of bounds at every level,
 * as OpenCV loses it; its next_pts entry keeps the guess. */
int svo_b200_klt_track(svo_b200_ctx* ctx, const svo_b200_klt_pyramid* prev, const svo_b200_klt_pyramid* next,
                       const svo_b200_klt_options* opt, int N, const float* prev_pts, float* next_pts_io, uint8_t* status_out,
                       svo_b200_klt_exit* exit_out);

/* The arguments of one svo_b200_klt_track call, for svo_b200_klt_track_streams. */
typedef struct svo_b200_klt_stream {
  const svo_b200_klt_pyramid* prev;
  const svo_b200_klt_pyramid* next;
  const svo_b200_klt_options* opt;
  int N;
  const float* prev_pts;
  float* next_pts_io;
  uint8_t* status_out;
  svo_b200_klt_exit* exit_out; /* may be NULL */
} svo_b200_klt_stream;
/* S streams' calcOpticalFlowPyrLK (e.g. the initialisation of S camera streams that start together) in one launch: one
 * copy to the device, one launch, one copy back, two stream synchronisations in all, as the single call makes.  Every
 * stream's next_pts, statuses and exit records equal one svo_b200_klt_track call with that stream's arguments, bit for
 * bit; svo_b200_klt_track is S = 1 of this call.  Streams may share pyramid handles (e.g. one first keyframe that several
 * streams track against) and differ in image size and options; the output arrays of different streams must not overlap,
 * while within one stream prev_pts and next_pts_io may be the same buffer.  Every stream's arguments are checked as
 * svo_b200_klt_track checks them before anything is launched or written (SVO_B200_EINVAL, also for S < 0 or NULL
 * `streams`), so a refused call leaves every output untouched.  SVO_B200_ELIMIT when the streams hold more than INT_MAX
 * points together.  S == 0, or no points at all, returns 0 without a launch. */
int svo_b200_klt_track_streams(svo_b200_ctx* ctx, int S, const svo_b200_klt_stream* streams);

#ifdef __cplusplus
}
#endif
#endif /* SVO_B200_H_ */
