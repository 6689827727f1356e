/* oracle/svo_oracle.h -- TEST INFRASTRUCTURE ONLY.
 *
 * C interface of the CPU oracle: a dependency-free, single-thread restatement of the
 * rpg_svo direct-tracking hot path (SURVEY.md section 8a).  Only tests/, __graft_entry__.smoke()
 * and bench.py's cpu_baseline / --impl reference legs may load this library.  The product
 * (rpg_svo_b200/, include/svo_b200.h) never links, imports or calls it.
 *
 * PINNING: everything that lives in the reference tree is pinned by executing it -- oracle/_ref is the
 * reference's own svo/src .cpp files of this path compiled where they lie (oracle/Makefile target `ref`,
 * oracle/ref_wrap.cpp) and tests/test_oracle_pins.py compares every function below with it.
 * PARITY UNPINNED at the third-party boundary: Eigen, OpenCV, Sophus, rpg_vikit, Boost are absent and
 * un-vendored, so oracle/_ref is built against stand-in headers (oracle/shim/) and the arithmetic inside
 * those libraries ([EXT] in the sources) is restated from their published algorithms, here and in the
 * stand-ins alike; the reference's own tests are print-only programs on an external dataset, so no
 * golden vector of the reference exists for those pieces.
 *
 * All SE3 arguments are row-major 3x4 [R|t] doubles; images are 8-bit, row pitch == cols
 * (the reference indexes with `cols` as stride: svo/src/sparse_img_align.cpp:88,165).
 */
#ifndef SVO_ORACLE_H_
#define SVO_ORACLE_H_
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define ORC_MAX_LEVELS 8

typedef struct {
  double fx, fy, cx, cy; /* [EXT] vk::PinholeCamera / vk::ATANCamera pixel parameters */
  int width, height;
  int model;             /* 0 = pinhole (d = k1 k2 p1 p2 k3, all 0 = undistorted), 1 = ATAN (d[0] = s) */
  int reserved_;
  double d[5];
} orc_camera;

/* One Gauss-Newton iteration of vk::NLLSSolver::optimizeGaussNewton as driven by
 * svo::SparseImgAlign::run (sparse_img_align.cpp:61-69). */
typedef struct {
  int level;
  int iter;
  int accepted; /* 1: update applied; 0: rollback (chi2 increase / solve failure) */
  int n_meas;   /* pixel residuals counted in this pass */
  double chi2;  /* value returned by computeResiduals */
  double x[6];
  double T[12]; /* model after the iteration */
} orc_sia_iter;

/* svo::SparseImgAlign::run restated on flat arrays.  Returns n_meas_/patch_area_. */
int64_t orc_sparse_img_align_run(
    const uint8_t* const* ref_levels, const uint8_t* const* cur_levels,
    const int* cols, const int* rows, int n_levels, const orc_camera* cam,
    double* T_cur_from_ref_io, const double* px /*N*2*/, const double* f /*N*3*/,
    const double* point_pos /*N*3*/, const uint8_t* has_point /*N*/, const double* ref_pos /*3*/,
    int N, int max_level, int min_level, int n_iter, double eps,
    uint8_t* visible_out /*N or NULL*/, double* H_out /*36 or NULL*/,
    float* residuals_out /*N*16 or NULL: last residual pass, NaN where not evaluated*/,
    orc_sia_iter* trace /*or NULL*/, int trace_cap, int* n_trace /*or NULL*/);

/* B independent runs of orc_sparse_img_align_run on n_threads host threads (std::thread, dynamic
 * work queue) -- the CPU arm of bench.py.  Level pointer arrays are [B * n_levels]; feat_offset has
 * B+1 entries; T_io is B*12; ref_pos B*3; n_tracked_out B (or NULL). */
void orc_sparse_img_align_batch(int B, const uint8_t* const* ref_levels,
                                const uint8_t* const* cur_levels, const int* cols, const int* rows,
                                int n_levels, const orc_camera* cam, double* T_io,
                                const int* feat_offset, const double* px, const double* f,
                                const double* point_pos, const uint8_t* has_point,
                                const double* ref_pos, int max_level, int min_level, int n_iter,
                                double eps, int64_t* n_tracked_out, int n_threads);

/* One computeResiduals(model, linearize=true) pass at a given level and pose, starting from
 * the visibility flags in visible_io (may be all zero).  Exposes every intermediate. */
int orc_sparse_residuals(
    const uint8_t* ref_img, const uint8_t* cur_img, int cols, int rows, int level,
    const orc_camera* cam, const double* T_cur_from_ref, const double* px, const double* f,
    const double* point_pos, const uint8_t* has_point, const double* ref_pos, int N,
    uint8_t* visible_io /*N*/, float* ref_patch_out /*N*16*/, double* jac_out /*N*16*6*/,
    float* residuals_out /*N*16*/, uint8_t* in_image_out /*N*/, double* H_out /*36*/,
    double* Jres_out /*6*/, double* chi2_out, int64_t* n_meas_out);

/* [EXT] vk::halfSample scalar path: out = (a+b+c+d)/4 (integer division). */
void orc_half_sample(const uint8_t* in, int in_cols, int in_rows, uint8_t* out);
/* [EXT] vk::AbstractCamera::world2cam(xyz) / cam2world(px) of the restated models, n points each. */
void orc_camera_world2cam(const orc_camera* cam, const double* xyz, int n, double* px_out);
void orc_camera_cam2world(const orc_camera* cam, const double* px, int n, double* f_out);
/* rule 0 = scalar, 1 = x86 (vikit's SSE2 avg(avg) branch when in_cols % 16 == 0, scalar otherwise). */
void orc_half_sample_rule(const uint8_t* in, int in_cols, int in_rows, uint8_t* out, int rule);

/* Sophus helpers exposed for the pinning tests. */
void orc_se3_exp(const double* x6, double* T12_out);
void orc_se3_mul(const double* A12, const double* B12, double* C12_out);
void orc_se3_inv(const double* A12, double* C12_out);
void orc_ldlt6_solve(const double* H36, const double* b6, double* x6_out);

/* ---- feature_alignment (svo/src/feature_alignment.cpp:30-277) ---- */
int orc_align2d(const uint8_t* cur_img, int cols, int rows, int step,
                const uint8_t* ref_patch_with_border /*100*/, const uint8_t* ref_patch /*64*/,
                int n_iter, double* px_io /*2*/);
int orc_align1d(const uint8_t* cur_img, int cols, int rows, int step, const float* dir /*2*/,
                const uint8_t* ref_patch_with_border, const uint8_t* ref_patch, int n_iter,
                double* px_io /*2*/, double* h_inv_out);
/* The same runs, also reporting how they ended (test instrumentation; the reference returns only the bool):
 * n_iter_done = loop iterations run, the converging one included and a rolled-back one not;
 * exit_reason = one of ORC_ALIGN_EXIT_*. */
enum {
  ORC_ALIGN_EXIT_BORDER_FIRST = 1, /* border test failed before the first step */
  ORC_ALIGN_EXIT_BORDER = 2,       /* border test failed after at least one step */
  ORC_ALIGN_EXIT_CONVERGED = 3,
  ORC_ALIGN_EXIT_MAX_ITER = 4,     /* n_iter steps (also n_iter <= 0) */
  ORC_ALIGN_EXIT_ROLLBACK = 5,     /* align1D only: chi2 rose, the last update was subtracted */
  ORC_ALIGN_EXIT_NAN = 6           /* NaN after the border test: unreachable */
};
int orc_align2d_ex(const uint8_t* cur_img, int cols, int rows, int step, const uint8_t* ref_patch_with_border,
                   const uint8_t* ref_patch, int n_iter, double* px_io, int* n_iter_done, int* exit_reason);
int orc_align1d_ex(const uint8_t* cur_img, int cols, int rows, int step, const float* dir,
                   const uint8_t* ref_patch_with_border, const uint8_t* ref_patch, int n_iter, double* px_io,
                   double* h_inv_out, int* n_iter_done, int* exit_reason);

/* ---- matcher warp (svo/src/matcher.cpp:33-133) ---- */
void orc_get_warp_matrix_affine(const orc_camera* cam_ref, const orc_camera* cam_cur,
                                const double* px_ref, const double* f_ref, double depth_ref,
                                const double* T_cur_ref, int level_ref, double* A_cur_ref_out /*4 row-major*/);
int orc_get_best_search_level(const double* A_cur_ref, int max_level);
int orc_warp_affine(const double* A_cur_ref, const uint8_t* img_ref, int cols, int rows,
                    const double* px_ref, int level_ref, int search_level, int halfpatch_size,
                    uint8_t* patch_io);
int orc_depth_from_triangulation(const double* T_search_ref, const double* f_ref,
                                 const double* f_cur, double* depth_out);

/* Matcher::findMatchDirect (matcher.cpp:135-177) with the reference feature already chosen
 * (Point::getCloseViewObs is host bookkeeping).  ftr_type: 0 corner, 1 edgelet. */
typedef struct {
  int success;
  int search_level;
  double px_cur[2];
  double A_cur_ref[4];
  double h_inv;
} orc_match_result;
void orc_find_match_direct(const uint8_t* const* ref_levels, const uint8_t* const* cur_levels,
                           const int* cols, const int* rows, int n_levels, const orc_camera* cam,
                           const double* T_cur_ref, const double* ref_px, const double* ref_f,
                           int ref_level, int ftr_type, const double* ref_grad, double depth_ref,
                           int max_search_level, int align_max_iter, const double* px_cur_in,
                           orc_match_result* out);

/* Matcher::findEpipolarMatchDirect (matcher.cpp:179-321). */
typedef struct {
  int success;
  int reject;
  int search_level;
  int n_zmssd_evals; /* ZMSSD scores actually computed (for the bytes model) */
  int n_align_iter;  /* not available from the reference; -1 */
  double epi_length;
  double px_cur[2];
  double depth;
  double h_inv;
  double A_cur_ref[4]; /* Matcher::A_cur_ref_, row-major */
} orc_epi_result;
void orc_find_epipolar_match_direct(const uint8_t* const* ref_levels,
                                    const uint8_t* const* cur_levels, const int* cols,
                                    const int* rows, int n_levels, const orc_camera* cam,
                                    const double* T_cur_ref, const double* ref_px,
                                    const double* ref_f, int ref_level, int ftr_type,
                                    const double* ref_grad, double d_estimate, double d_min,
                                    double d_max, int max_search_level, int align_max_iter,
                                    int max_epi_search_steps, int align_1d, orc_epi_result* out);

/* ---- depth filter (svo/src/depth_filter.cpp:197-350) ---- */
void orc_update_seed(float x, float tau2, float* a, float* b, float* mu, float* z_range,
                     float* sigma2);
double orc_compute_tau(const double* T_ref_cur, const double* f, double z, double px_error_angle);

/* status codes of one seed inside DepthFilter::updateSeeds */
enum {
  ORC_SEED_TOO_OLD = 1,      /* erased: older than max_n_kfs batches (:216-219) */
  ORC_SEED_BEHIND = 2,       /* behind the camera (:225-228) */
  ORC_SEED_NOT_IN_FRAME = 3, /* does not project into the image (:229-232) */
  ORC_SEED_NO_MATCH = 4,     /* findEpipolarMatchDirect failed: b++ (:237-244) */
  ORC_SEED_UPDATED = 5,      /* updateSeed applied (:247-252) */
  ORC_SEED_CONVERGED = 6,    /* updated and converged -> point created, erased (:261-282) */
  ORC_SEED_NAN = 7           /* updated, z_inv_min NaN -> erased (:283-287) */
};
/* DepthFilter::updateSeeds over SoA seeds.  All seeds share one reference keyframe per entry of
 * ref_index (index into ref_frames arrays). */
void orc_depth_filter_update(
    const uint8_t* const* ref_levels /*n_ref*n_levels*/, const double* ref_T_f_w /*n_ref*12*/,
    int n_ref, const uint8_t* const* cur_levels, const double* cur_T_f_w, const int* cols,
    const int* rows, int n_levels, const orc_camera* cam, int M, const int* ref_index,
    const double* ftr_px, const double* ftr_f, const int* ftr_level, const int* ftr_type,
    const double* ftr_grad, const int* batch_id, int batch_counter, int max_n_kfs,
    double seed_convergence_sigma2_thresh, int max_search_level, int align_max_iter,
    int max_epi_search_steps, float* a, float* b, float* mu, float* z_range, float* sigma2,
    uint8_t* status_out, double* px_cur_out /*M*2*/, double* z_out /*M*/,
    int* n_zmssd_out /*M or NULL*/);

/* ---- pose optimizer (svo/src/pose_optimizer.cpp:28-161) ---- */
typedef struct {
  double estimated_scale, error_init, error_final;
  int64_t num_obs;
  int n_iter_done;
  double cov[36];
} orc_pose_opt_result;
void orc_pose_optimize(double reproj_thresh, int n_iter, double fx /*errorMultiplier2*/,
                       double* T_f_w_io, const double* f /*N*3*/, const double* pos /*N*3*/,
                       const int* level /*N*/, uint8_t* has_point_io /*N*/, int N,
                       orc_pose_opt_result* out);

/* svo::Point::optimize (svo/src/point.cpp:119-177): one point, n_obs observing frames. */
void orc_point_optimize(int n_iter, double* pos_io /*3*/, int n_obs, const double* obs_T_f_w /*n_obs*12*/,
                        const double* obs_f /*n_obs*3*/);

/* ---- Reprojector::reprojectMap (svo/src/reprojector.cpp:64-217) on a flat view of the map ---- */
typedef struct {
  int n_kfs;                     /* Map::keyframes_, in list order */
  const double* kf_T_f_w;        /* n_kfs*12 */
  const double* kf_keypt_pos;    /* n_kfs*5*3: key_pts_[i]->point->pos_ (frame.h:48) */
  const uint8_t* kf_keypt_valid; /* n_kfs*5: key_pts_[i] != NULL */
  const int* kf_fts_offset;      /* n_kfs+1: Frame::fts_ of keyframe k = kf_fts[offset[k]..offset[k+1]) */
  const int* kf_fts;             /* indices into the feature table */
  int n_ftrs;                    /* feature table: every Feature some Point::obs_ or Frame::fts_ refers to */
  const int* ftr_kf;             /* Feature::frame as keyframe index */
  const double* ftr_px;          /* n_ftrs*2 */
  const double* ftr_f;           /* n_ftrs*3 */
  const int* ftr_level;
  const int* ftr_type;           /* 0 CORNER, 1 EDGELET */
  const double* ftr_grad;        /* n_ftrs*2 */
  const int* ftr_point;          /* Feature::point as point index, -1 = NULL */
  int n_points;
  const double* pt_pos;          /* n_points*3 */
  const int* pt_obs_offset;      /* n_points+1 */
  const int* pt_obs;             /* Point::obs_ in list order, as feature-table indices */
  int n_candidates;
  const int* cand_point;         /* MapPointCandidates::candidates_ in list order, as point indices */
} orc_map_view;
typedef struct {
  int grid_size;         /* Config::gridSize() (config.cpp:32: 30) */
  int max_fts;           /* Config::maxFts() (config.cpp:52: 120) */
  int max_n_kfs;         /* Reprojector::Options::max_n_kfs (reprojector.h:44: 10) */
  int find_match_direct; /* Reprojector::Options::find_match_direct (true) */
  int max_search_level;  /* Config::nPyrLevels()-1 (matcher.cpp:153) */
  int align_max_iter;    /* Matcher::Options::align_max_iter (10) */
} orc_reproject_options;
typedef struct {
  int64_t n_matches, n_trials; /* Reprojector::n_matches_, n_trials_ */
  int n_new;                   /* features added to the frame */
  int n_overlap;               /* keyframes reprojected from (overlap_kfs.size()) */
  int n_projected;             /* points that fell into a grid cell */
  int n_speculative;           /* unused by the oracle (it matches only what the cell policy reaches) */
} orc_reproject_stats;
enum {
  ORC_PT_NONE = 0,
  ORC_PT_SAFE_DELETE = 1,      /* map_.safeDeletePoint(pt)            (reprojector.cpp:173-174) */
  ORC_PT_DELETE_CANDIDATE = 2, /* point_candidates_.deleteCandidatePoint (reprojector.cpp:175-176) */
  ORC_PT_CANDIDATE_ERASED = 3  /* candidate erased while projecting   (reprojector.cpp:117-122) */
};
/* Point types: 0 DELETED, 1 CANDIDATE, 2 UNKNOWN, 3 GOOD (point.h:40-45).  new_* arrays hold max_fts+1 entries;
 * overlap_* hold max_n_kfs entries; cell_order has ceil(w/grid)*ceil(h/grid) entries. */
void orc_reproject_map(const orc_map_view* map, const uint8_t* const* kf_levels /*n_kfs*n_levels*/,
                       const uint8_t* const* cur_levels, const int* cols, const int* rows, int n_levels,
                       const orc_camera* cam, const double* cur_T_f_w, const orc_reproject_options* opt,
                       const int* cell_order, int* pt_type_io, int* pt_n_failed_io, int* pt_n_succeeded_io,
                       uint8_t* pt_action_out, int* overlap_kf_out, int64_t* overlap_count_out, int* new_point,
                       double* new_px, int* new_level, int* new_type, double* new_grad, orc_reproject_stats* stats);

/* ---- feature_detection::FastDetector::detect (svo/src/feature_detection.cpp:66-115) ----
 * FAST-10 (b = fast_threshold; the reference hard-codes 20) + score + 3x3 non-maximum suppression per pyramid level,
 * Shi-Tomasi score per surviving corner, best corner per grid cell over all levels, cells flagged in grid_occupancy
 * (NULL = none) skipped.  The `fast` library and vk::shiTomasiScore are [EXT] (oracle/fast_ext.h).  Output: corners in
 * cell order (level-0 pixel coordinates, level, score); returns their number (may exceed cap; only cap are written). */
int orc_fast_detect(const uint8_t* const* levels, const int* cols, const int* rows, int n_pyr_levels, int img_width,
                    int img_height, int cell_size, const uint8_t* grid_occupancy, double detection_threshold,
                    int fast_threshold, int nonmax_ties_suppress /*[EXT] 0 = libCVD non-strict (default)*/, int* out_x,
                    int* out_y, int* out_level, float* out_score, int cap);

#ifdef __cplusplus
}
#endif
#endif
