// rpg_svo_b200/csrc/reproject.cu -- C ABI entry point
//   svo_b200_reproject_map  <- Reprojector::reprojectMap (svo/src/reprojector.cpp:64-217)
//
// The reference walks the grid cell by cell and calls Matcher::findMatchDirect once per candidate until a cell has its
// match -- a data-dependent sequential loop.  Here the device projects every map point / candidate into the frame and
// aligns ALL in-frame points speculatively (one warp each: Point::getCloseViewObs over the observation list, then
// findMatchDirect), and the host replays the reference's policy -- cell order, quality sort, one match per cell, maxFts
// stop, point counters and deletions -- over those results, touching only what the sequential code would have reached
// (SURVEY.md 8f row 2).  Everything the replay needs is per-point and independent of the replay order, so the results
// equal the sequential ones.
#include <algorithm>
#include <climits>
#include <cstdint>
#include <cmath>
#include <cstring>
#include <vector>

#include "ctx.h"
#include "warp_align.cuh"

namespace svo {

constexpr int kRpWarps = 4;

struct ReprojIn {
  const int* e_pt;           // E: enumerated point indices (keyframe points in reference order, then candidates)
  const uint8_t* e_skip;     // E: input type == TYPE_DELETED -> projected but never matched
  const double* pt_pos;      // n_points*3
  const int* pt_obs_offset;  // n_points+1
  const int* pt_obs;
  const int* ftr_kf;
  const double* ftr_px;
  const double* ftr_f;
  const int* ftr_level;
  const int* ftr_type;
  const double* ftr_grad;
  const double* kf_T;        // n_kfs*12
  const FrameDesc* kf_frames;
};
struct ReprojOut {
  double* px;         // E*2  frame->w2c(pos)
  uint8_t* in_frame;  // E
  int* cell;          // E
  uint8_t* success;   // E    findMatchDirect
  double* px_match;   // E*2
  int* search_level;  // E
  double* A;          // E*4
  int* ref_ftr;       // E    feature picked by getCloseViewObs
};

__global__ void __launch_bounds__(kRpWarps * 32) reproject_match_kernel(
    FrameDesc cur, Cam cam, int E, ReprojIn in, ReprojOut out, const double* __restrict__ cur_T_f_w, int cell_size,
    int grid_n_cols, int find_match, int max_search_level, int align_max_iter) {
  __shared__ WarpAlignScratch scratch[kRpWarps];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int e = blockIdx.x * kRpWarps + warp;
  if (e >= E) return;
#include "reproject_match.inc"
}

// One stream of svo_b200_reproject_map_streams: the arguments reproject_match_kernel takes, in a per-launch device table.
struct ReprojStream {
  FrameDesc cur;
  Cam cam;
  ReprojIn in;
  ReprojOut out;
  const double* cur_T_f_w;
  int e_begin;  // the stream's first point in the launch's concatenated enumeration
  int cell_size, grid_n_cols, find_match, max_search_level, align_max_iter;
};

// The stream whose points include the launch's point g: the last s with e_begin <= g (every stream in the table has points).
__device__ __forceinline__ int reproject_stream_of(const ReprojStream* __restrict__ streams, int n_streams, int g) {
  int lo = 0, hi = n_streams - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (streams[mid].e_begin <= g) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__global__ void __launch_bounds__(kRpWarps * 32) reproject_match_streams_kernel(const ReprojStream* __restrict__ streams,
                                                                                int n_streams, int E_total) {
  __shared__ WarpAlignScratch scratch[kRpWarps];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = blockIdx.x * kRpWarps + warp;
  if (g >= E_total) return;
  const ReprojStream& rs = streams[reproject_stream_of(streams, n_streams, g)];
  const int e = g - rs.e_begin;
  const FrameDesc& cur = rs.cur;
  const Cam& cam = rs.cam;
  const ReprojIn& in = rs.in;
  const ReprojOut& out = rs.out;
  const double* __restrict__ cur_T_f_w = rs.cur_T_f_w;
  const int cell_size = rs.cell_size, grid_n_cols = rs.grid_n_cols, find_match = rs.find_match,
            max_search_level = rs.max_search_level, align_max_iter = rs.align_max_iter;
#include "reproject_match.inc"
}

}  // namespace svo

using namespace svo;

namespace {

// The argument checks of one reprojectMap call that precede any write (the single-stream call clears its stats and
// actions before the camera and cell-order checks; reproject_grid does those).
int reproject_check(svo_b200_ctx* ctx, const svo_b200_map_view* m, const svo_b200_frame* const* kf_frames,
                    const svo_b200_frame* cur, const double* cur_T_f_w, const svo_b200_camera* cam,
                    const svo_b200_reproject_options* opt, const int* cell_order, const int* pt_type_io,
                    const int* pt_n_failed_io, const int* pt_n_succeeded_io, const uint8_t* pt_action_out,
                    const int* overlap_kf_out, const int64_t* overlap_count_out, const int* new_point_out,
                    const double* new_px_out, const int* new_level_out, const int* new_type_out,
                    const double* new_grad_out, const svo_b200_reproject_stats* stats) {
  if (!ctx || !m || !cur || !cur_T_f_w || !cam || !opt || !cell_order || !pt_type_io || !pt_n_failed_io ||
      !pt_n_succeeded_io || !pt_action_out || !overlap_kf_out || !overlap_count_out || !new_point_out || !new_px_out ||
      !new_level_out || !new_type_out || !new_grad_out || !stats)
    return set_err(ctx, SVO_B200_EINVAL, "reproject_map: NULL argument");
  if (m->n_kfs < 0 || m->n_ftrs < 0 || m->n_points < 0 || m->n_candidates < 0 || (m->n_kfs > 0 && !kf_frames))
    return set_err(ctx, SVO_B200_EINVAL, "reproject_map: negative sizes / missing keyframe handles");
  if ((m->n_kfs > 0 && (!m->kf_T_f_w || !m->kf_keypt_pos || !m->kf_keypt_valid || !m->kf_fts_offset)) ||
      (m->n_ftrs > 0 && (!m->ftr_kf || !m->ftr_px || !m->ftr_f || !m->ftr_level || !m->ftr_type || !m->ftr_grad || !m->ftr_point)) ||
      (m->n_points > 0 && (!m->pt_pos || !m->pt_obs_offset)) || (m->n_candidates > 0 && !m->cand_point))
    return set_err(ctx, SVO_B200_EINVAL, "reproject_map: NULL array in the map view");
  for (int k = 0; k < m->n_kfs; ++k)
    if (!kf_frames[k]) return set_err(ctx, SVO_B200_EINVAL, "reproject_map: kf_frames[%d] is NULL", k);
  const int n_kf_fts = m->n_kfs ? m->kf_fts_offset[m->n_kfs] : 0, n_obs_total = m->n_points ? m->pt_obs_offset[m->n_points] : 0;
  if (n_kf_fts < 0 || n_obs_total < 0 || (n_kf_fts > 0 && !m->kf_fts) || (n_obs_total > 0 && !m->pt_obs))
    return set_err(ctx, SVO_B200_EINVAL, "reproject_map: inconsistent offsets in the map view");
  if (opt->grid_size <= 0 || opt->max_fts < 0 || opt->max_n_kfs < 0 || opt->max_search_level < 0 ||
      opt->max_search_level >= cur->n_levels)
    return set_err(ctx, SVO_B200_EINVAL, "reproject_map: bad options (grid_size %d, max_search_level %d of %d levels)",
                   opt->grid_size, opt->max_search_level, cur->n_levels);
  for (int i = 0; i < m->n_ftrs; ++i) {
    if (m->ftr_kf[i] < 0 || m->ftr_kf[i] >= m->n_kfs || m->ftr_point[i] >= m->n_points || m->ftr_point[i] < -1)
      return set_err(ctx, SVO_B200_EINVAL, "reproject_map: feature %d refers outside the map view", i);
    if (m->ftr_level[i] < 0 || m->ftr_level[i] >= kf_frames[m->ftr_kf[i]]->n_levels)
      return set_err(ctx, SVO_B200_EINVAL, "reproject_map: ftr_level[%d] outside the pyramid", i);
  }
  for (int j = 0; j < n_kf_fts; ++j)
    if (m->kf_fts[j] < 0 || m->kf_fts[j] >= m->n_ftrs) return set_err(ctx, SVO_B200_EINVAL, "reproject_map: kf_fts[%d] out of range", j);
  for (int j = 0; j < n_obs_total; ++j)
    if (m->pt_obs[j] < 0 || m->pt_obs[j] >= m->n_ftrs) return set_err(ctx, SVO_B200_EINVAL, "reproject_map: pt_obs[%d] out of range", j);
  for (int c = 0; c < m->n_candidates; ++c)
    if (m->cand_point[c] < 0 || m->cand_point[c] >= m->n_points) return set_err(ctx, SVO_B200_EINVAL, "reproject_map: cand_point[%d] out of range", c);
  return 0;
}

// initializeGrid (:47-58): the device camera, the grid and the check of the caller's cell order.
int reproject_grid(svo_b200_ctx* ctx, const svo_b200_camera* cam, const svo_b200_reproject_options* opt,
                   const int* cell_order, Cam& cm, int& grid_n_cols, size_t& n_cells) {
  { const int rc_cam = cam_to_dev(ctx, cam, cm); if (rc_cam) return rc_cam; }
  grid_n_cols = (int)std::ceil((double)cam->width / opt->grid_size);
  const int grid_n_rows = (int)std::ceil((double)cam->height / opt->grid_size);
  n_cells = (size_t)grid_n_cols * grid_n_rows;
  for (size_t i = 0; i < n_cells; ++i)
    if (cell_order[i] < 0 || (size_t)cell_order[i] >= n_cells) return set_err(ctx, SVO_B200_EINVAL, "reproject_map: cell_order[%zu] out of range", i);
  return 0;
}

// Map::getCloseKeyframes and the enumeration of the points to project, in the reference's order; writes the overlap
// keyframes and n_overlap.  src = overlap slot, or -1 for a candidate.
void reproject_enumerate(const svo_b200_map_view* m, const svo_b200_camera* cam, const Cam& cm, const double* cur_T_f_w,
                         const svo_b200_reproject_options* opt, int* overlap_kf_out, int64_t* overlap_count_out,
                         svo_b200_reproject_stats* stats, std::vector<int>& e_pt, std::vector<int>& e_src) {
  // Map::getCloseKeyframes (map.cpp:106-127) + sort by distance (:76-77); list::sort is stable
  const double* Tc = cur_T_f_w;
  std::vector<std::pair<int, double>> close_kfs;
  for (int k = 0; k < m->n_kfs; ++k)
    for (int i = 0; i < 5; ++i) {
      if (!m->kf_keypt_valid[5 * k + i]) continue;
      const double* kp = m->kf_keypt_pos + 3 * (5 * (size_t)k + i);
      const double x = Tc[0] * kp[0] + Tc[1] * kp[1] + Tc[2] * kp[2] + Tc[3];  // Frame::isVisible (frame.cpp:141-150)
      const double y = Tc[4] * kp[0] + Tc[5] * kp[1] + Tc[6] * kp[2] + Tc[7];
      const double z = Tc[8] * kp[0] + Tc[9] * kp[1] + Tc[10] * kp[2] + Tc[11];
      if (z < 0.0) continue;
      double u, v;
      cam_world2cam(cm, x / z, y / z, u, v);  // Frame::w2c
      if (u >= 0.0 && v >= 0.0 && u < cam->width && v < cam->height) {
        const double* Tk = m->kf_T_f_w + 12 * (size_t)k;
        const double dx = Tc[3] - Tk[3], dy = Tc[7] - Tk[7], dz = Tc[11] - Tk[11];
        close_kfs.emplace_back(k, std::sqrt(dx * dx + dy * dy + dz * dz));
        break;
      }
    }
  std::stable_sort(close_kfs.begin(), close_kfs.end(),
                   [](const std::pair<int, double>& a, const std::pair<int, double>& b) { return a.second < b.second; });

  // enumeration in the reference's order (:81-104, :108-127)
  std::vector<uint8_t> projected((size_t)m->n_points, 0);  // point->last_projected_kf_id_ == frame->id_
  size_t n_ov = 0;
  for (auto it = close_kfs.begin(); it != close_kfs.end() && n_ov < (size_t)opt->max_n_kfs; ++it, ++n_ov) {
    const int k = it->first;
    overlap_kf_out[n_ov] = k;
    overlap_count_out[n_ov] = 0;
    for (int j = m->kf_fts_offset[k]; j < m->kf_fts_offset[k + 1]; ++j) {
      const int p = m->ftr_point[m->kf_fts[j]];
      if (p < 0 || projected[p]) continue;
      projected[p] = 1;
      e_pt.push_back(p);
      e_src.push_back((int)n_ov);
    }
  }
  stats->n_overlap = (int)n_ov;
  for (int c = 0; c < m->n_candidates; ++c) { e_pt.push_back(m->cand_point[c]); e_src.push_back(-1); }
}

// Byte offsets of one call's device inputs and outputs in the context's staging buffer (mirrored host / device).
struct ReprojLayout {
  size_t o_ept, o_skip, o_pos, o_ooff, o_obs, o_fkf, o_fpx, o_ff, o_flv, o_fty, o_fgr, o_kT, o_kfr, o_cT;
  size_t o_px, o_in, o_cell, o_su, o_pm, o_sl, o_A, o_rf;
};

void reproject_carve_in(Carver& c, const svo_b200_map_view* m, int E, ReprojLayout& L) {
  const int n_obs = m->n_points ? m->pt_obs_offset[m->n_points] : 0;
  L.o_ept = c.take(sizeof(int) * E); L.o_skip = c.take(E); L.o_pos = c.take(sizeof(double) * 3 * m->n_points);
  L.o_ooff = c.take(sizeof(int) * (m->n_points + 1)); L.o_obs = c.take(sizeof(int) * n_obs);
  L.o_fkf = c.take(sizeof(int) * m->n_ftrs); L.o_fpx = c.take(sizeof(double) * 2 * m->n_ftrs);
  L.o_ff = c.take(sizeof(double) * 3 * m->n_ftrs); L.o_flv = c.take(sizeof(int) * m->n_ftrs);
  L.o_fty = c.take(sizeof(int) * m->n_ftrs); L.o_fgr = c.take(sizeof(double) * 2 * m->n_ftrs);
  L.o_kT = c.take(sizeof(double) * 12 * m->n_kfs); L.o_kfr = c.take(sizeof(FrameDesc) * m->n_kfs);
  L.o_cT = c.take(sizeof(double) * 12);
}

void reproject_carve_out(Carver& c, int E, ReprojLayout& L) {
  L.o_px = c.take(sizeof(double) * 2 * E); L.o_in = c.take(E); L.o_cell = c.take(sizeof(int) * E); L.o_su = c.take(E);
  L.o_pm = c.take(sizeof(double) * 2 * E); L.o_sl = c.take(sizeof(int) * E); L.o_A = c.take(sizeof(double) * 4 * E);
  L.o_rf = c.take(sizeof(int) * E);
}

void reproject_stage(uint8_t* h, const ReprojLayout& L, const svo_b200_map_view* m, const svo_b200_frame* const* kf_frames,
                     const double* cur_T_f_w, const std::vector<int>& e_pt, const int* pt_type_io) {
  const int E = (int)e_pt.size(), n_obs = m->n_points ? m->pt_obs_offset[m->n_points] : 0;
  auto cp = [&](size_t off, const void* src, size_t bytes) { if (bytes) memcpy(h + off, src, bytes); };  // empty tables may be NULL
  cp(L.o_ept, e_pt.data(), sizeof(int) * E);
  for (int e = 0; e < E; ++e) (h + L.o_skip)[e] = pt_type_io[e_pt[e]] == 0;
  cp(L.o_pos, m->pt_pos, sizeof(double) * 3 * m->n_points);
  cp(L.o_ooff, m->pt_obs_offset, sizeof(int) * (m->n_points + 1));
  cp(L.o_obs, m->pt_obs, sizeof(int) * n_obs);
  cp(L.o_fkf, m->ftr_kf, sizeof(int) * m->n_ftrs);
  cp(L.o_fpx, m->ftr_px, sizeof(double) * 2 * m->n_ftrs);
  cp(L.o_ff, m->ftr_f, sizeof(double) * 3 * m->n_ftrs);
  cp(L.o_flv, m->ftr_level, sizeof(int) * m->n_ftrs);
  cp(L.o_fty, m->ftr_type, sizeof(int) * m->n_ftrs);
  cp(L.o_fgr, m->ftr_grad, sizeof(double) * 2 * m->n_ftrs);
  cp(L.o_kT, m->kf_T_f_w, sizeof(double) * 12 * m->n_kfs);
  for (int k = 0; k < m->n_kfs; ++k) reinterpret_cast<FrameDesc*>(h + L.o_kfr)[k] = make_desc(kf_frames[k]);
  cp(L.o_cT, cur_T_f_w, sizeof(double) * 12);
}

ReprojIn reproject_in(uint8_t* d, const ReprojLayout& L) {
  return {reinterpret_cast<const int*>(d + L.o_ept), d + L.o_skip, reinterpret_cast<const double*>(d + L.o_pos),
          reinterpret_cast<const int*>(d + L.o_ooff), reinterpret_cast<const int*>(d + L.o_obs),
          reinterpret_cast<const int*>(d + L.o_fkf), reinterpret_cast<const double*>(d + L.o_fpx),
          reinterpret_cast<const double*>(d + L.o_ff), reinterpret_cast<const int*>(d + L.o_flv),
          reinterpret_cast<const int*>(d + L.o_fty), reinterpret_cast<const double*>(d + L.o_fgr),
          reinterpret_cast<const double*>(d + L.o_kT), reinterpret_cast<const FrameDesc*>(d + L.o_kfr)};
}

ReprojOut reproject_out(uint8_t* d, const ReprojLayout& L) {
  return {reinterpret_cast<double*>(d + L.o_px), d + L.o_in, reinterpret_cast<int*>(d + L.o_cell), d + L.o_su,
          reinterpret_cast<double*>(d + L.o_pm), reinterpret_cast<int*>(d + L.o_sl), reinterpret_cast<double*>(d + L.o_A),
          reinterpret_cast<int*>(d + L.o_rf)};
}

// The host replay of the sequential policy over the device results of one call (in the host staging buffer h).
void reproject_replay(const uint8_t* h, const ReprojLayout& L, const svo_b200_map_view* m,
                      const svo_b200_reproject_options* opt, size_t n_cells, const int* cell_order,
                      const std::vector<int>& e_pt, const std::vector<int>& e_src, int* pt_type_io, int* pt_n_failed_io,
                      int* pt_n_succeeded_io, uint8_t* pt_action_out, int64_t* overlap_count_out, int* new_point_out,
                      double* new_px_out, int* new_level_out, int* new_type_out, double* new_grad_out,
                      svo_b200_reproject_stats* stats) {
  const int E = (int)e_pt.size();
  const double* r_px = reinterpret_cast<const double*>(h + L.o_px);
  const uint8_t* r_in = h + L.o_in;
  const int* r_cell = reinterpret_cast<const int*>(h + L.o_cell);
  const uint8_t* r_su = h + L.o_su;
  const double* r_pm = reinterpret_cast<const double*>(h + L.o_pm);
  const int* r_sl = reinterpret_cast<const int*>(h + L.o_sl);
  const double* r_A = reinterpret_cast<const double*>(h + L.o_A);
  const int* r_rf = reinterpret_cast<const int*>(h + L.o_rf);
  std::vector<std::vector<int>> cells(n_cells);  // enumeration indices, push_back order
  for (int e = 0; e < E; ++e) {
    const int p = e_pt[e];
    if (r_in[e]) {
      cells[(size_t)r_cell[e]].push_back(e);
      ++stats->n_projected;
      if (e_src[e] >= 0) overlap_count_out[e_src[e]]++;
      if (opt->find_match_direct && pt_type_io[p] != 0) ++stats->n_speculative;
    } else if (e_src[e] < 0) {  // candidate that does not reproject (:113-122)
      pt_n_failed_io[p] += 3;
      if (pt_n_failed_io[p] > 30) {
        pt_type_io[p] = 0;
        pt_action_out[p] = SVO_B200_PT_CANDIDATE_ERASED;
      }
    }
  }
  for (size_t i = 0; i < n_cells; ++i) {
    std::vector<int>& cell = cells[(size_t)cell_order[i]];
    // cell.sort(pointQualityComparator): stable, better type first (:144-149,153)
    std::stable_sort(cell.begin(), cell.end(), [&](int l, int r) { return pt_type_io[e_pt[l]] > pt_type_io[e_pt[r]]; });
    bool matched = false;
    for (size_t ci = 0; ci < cell.size(); ++ci) {
      const int e = cell[ci], p = e_pt[e];
      ++stats->n_trials;
      if (pt_type_io[p] == 0) continue;  // TYPE_DELETED: erased from the cell
      const bool found_match = opt->find_match_direct ? r_su[e] != 0 : true;
      if (!found_match) {
        pt_n_failed_io[p]++;
        if (pt_type_io[p] == 2 && pt_n_failed_io[p] > 15) { pt_type_io[p] = 0; pt_action_out[p] = SVO_B200_PT_SAFE_DELETE; }
        if (pt_type_io[p] == 1 && pt_n_failed_io[p] > 30) { pt_type_io[p] = 0; pt_action_out[p] = SVO_B200_PT_DELETE_CANDIDATE; }
        continue;
      }
      pt_n_succeeded_io[p]++;
      if (pt_type_io[p] == 2 && pt_n_succeeded_io[p] > 10) pt_type_io[p] = 3;
      const int q = stats->n_new++;
      new_point_out[q] = p;
      new_px_out[2 * q] = opt->find_match_direct ? r_pm[2 * e] : r_px[2 * e];
      new_px_out[2 * q + 1] = opt->find_match_direct ? r_pm[2 * e + 1] : r_px[2 * e + 1];
      new_level_out[q] = r_sl[e];
      new_type_out[q] = 0;
      new_grad_out[2 * q] = 1.0;
      new_grad_out[2 * q + 1] = 0.0;
      const int ref = r_rf[e];
      if (ref >= 0 && m->ftr_type[ref] == 1) {  // EDGELET: grad = normalize(A_cur_ref * ref grad) (:190-195)
        const double gx = m->ftr_grad[2 * ref], gy = m->ftr_grad[2 * ref + 1];
        const double ax = r_A[4 * e] * gx + r_A[4 * e + 1] * gy, ay = r_A[4 * e + 2] * gx + r_A[4 * e + 3] * gy;
        const double nn = std::sqrt(ax * ax + ay * ay);
        new_type_out[q] = 1;
        new_grad_out[2 * q] = ax / nn;
        new_grad_out[2 * q + 1] = ay / nn;
      }
      matched = true;
      break;
    }
    if (matched) ++stats->n_matches;
    if (stats->n_matches > (int64_t)opt->max_fts) break;
  }
}

}  // namespace

extern "C" int svo_b200_reproject_map(svo_b200_ctx* ctx, const svo_b200_map_view* m, const svo_b200_frame* const* kf_frames,
                                      const svo_b200_frame* cur, const double* cur_T_f_w, const svo_b200_camera* cam,
                                      const svo_b200_reproject_options* opt, const int* cell_order, int* pt_type_io,
                                      int* pt_n_failed_io, int* pt_n_succeeded_io, uint8_t* pt_action_out,
                                      int* overlap_kf_out, int64_t* overlap_count_out, int* new_point_out,
                                      double* new_px_out, int* new_level_out, int* new_type_out, double* new_grad_out,
                                      svo_b200_reproject_stats* stats) {
  int rc = reproject_check(ctx, m, kf_frames, cur, cur_T_f_w, cam, opt, cell_order, pt_type_io, pt_n_failed_io,
                           pt_n_succeeded_io, pt_action_out, overlap_kf_out, overlap_count_out, new_point_out, new_px_out,
                           new_level_out, new_type_out, new_grad_out, stats);
  if (rc) return rc;
  std::memset(stats, 0, sizeof(*stats));
  for (int p = 0; p < m->n_points; ++p) pt_action_out[p] = SVO_B200_PT_NONE;
  Cam cm;
  int grid_n_cols;
  size_t n_cells;
  if ((rc = reproject_grid(ctx, cam, opt, cell_order, cm, grid_n_cols, n_cells))) return rc;
  std::vector<int> e_pt, e_src;
  reproject_enumerate(m, cam, cm, cur_T_f_w, opt, overlap_kf_out, overlap_count_out, stats, e_pt, e_src);
  const int E = (int)e_pt.size();
  if (E == 0) return 0;

  // ---- device: project + speculative getCloseViewObs / findMatchDirect for every enumerated point ----
  cudaSetDevice(ctx->device);
  Carver c;
  ReprojLayout L;
  reproject_carve_in(c, m, E, L);
  const size_t in_bytes = c.off;
  reproject_carve_out(c, E, L);
  if ((rc = ensure_host(ctx, ctx->h_in, c.off))) return rc;
  if ((rc = ensure_dev(ctx, ctx->d_in, c.off))) return rc;
  SVO_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
  uint8_t* h = static_cast<uint8_t*>(ctx->h_in.p);
  uint8_t* d = static_cast<uint8_t*>(ctx->d_in.p);
  reproject_stage(h, L, m, kf_frames, cur_T_f_w, e_pt, pt_type_io);
  SVO_CUDA_CHECK(ctx, cudaMemcpyAsync(d, h, in_bytes, cudaMemcpyHostToDevice, ctx->stream));
  const int blocks = (E + kRpWarps - 1) / kRpWarps;
  kt_begin(ctx);
  reproject_match_kernel<<<blocks, kRpWarps * 32, 0, ctx->stream>>>(
      make_desc(cur), cm, E, reproject_in(d, L), reproject_out(d, L), reinterpret_cast<const double*>(d + L.o_cT),
      opt->grid_size, grid_n_cols, opt->find_match_direct, opt->max_search_level, opt->align_max_iter);
  ctx->launches++;
  kt_end(ctx);
  SVO_CUDA_CHECK(ctx, cudaGetLastError());
  SVO_CUDA_CHECK(ctx, cudaMemcpyAsync(h + L.o_px, d + L.o_px, c.off - L.o_px, cudaMemcpyDeviceToHost, ctx->stream));
  SVO_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
  reproject_replay(h, L, m, opt, n_cells, cell_order, e_pt, e_src, pt_type_io, pt_n_failed_io, pt_n_succeeded_io,
                   pt_action_out, overlap_count_out, new_point_out, new_px_out, new_level_out, new_type_out, new_grad_out,
                   stats);
  return 0;
}

extern "C" int svo_b200_reproject_map_streams(svo_b200_ctx* ctx, int S, const svo_b200_reproject_stream* streams) {
  if (!ctx || S < 0 || (S > 0 && !streams))
    return set_err(ctx, SVO_B200_EINVAL, "reproject_map_streams: bad arguments (S %d)", S);
  // every stream is checked before anything is written
  std::vector<Cam> cm((size_t)S);
  std::vector<int> grid_n_cols((size_t)S);
  std::vector<size_t> n_cells((size_t)S);
  int64_t e_bound = 0;  // a stream enumerates at most its keyframe features and candidates
  for (int s = 0; s < S; ++s) {
    const svo_b200_reproject_stream& a = streams[s];
    int rc = reproject_check(ctx, a.map, a.kf_frames, a.cur, a.cur_T_f_w, a.cam, a.opt, a.cell_order, a.pt_type_io,
                             a.pt_n_failed_io, a.pt_n_succeeded_io, a.pt_action_out, a.overlap_kf_out, a.overlap_count_out,
                             a.new_point_out, a.new_px_out, a.new_level_out, a.new_type_out, a.new_grad_out, a.stats);
    if (!rc) rc = reproject_grid(ctx, a.cam, a.opt, a.cell_order, cm[s], grid_n_cols[s], n_cells[s]);
    if (rc) {
      const std::string why = ctx->err;
      return set_err(ctx, rc, "reproject_map_streams: stream %d: %s", s, why.c_str());
    }
    e_bound += (int64_t)(a.map->n_kfs ? a.map->kf_fts_offset[a.map->n_kfs] : 0) + a.map->n_candidates;
  }
  if (e_bound > INT32_MAX) return set_err(ctx, SVO_B200_ELIMIT, "reproject_map_streams: more than 2^31-1 points in one launch");
  std::vector<std::vector<int>> e_pt((size_t)S), e_src((size_t)S);
  std::vector<int> active;  // streams with points, in stream order
  int E_total = 0;
  for (int s = 0; s < S; ++s) {
    const svo_b200_reproject_stream& a = streams[s];
    std::memset(a.stats, 0, sizeof(*a.stats));
    for (int p = 0; p < a.map->n_points; ++p) a.pt_action_out[p] = SVO_B200_PT_NONE;
    reproject_enumerate(a.map, a.cam, cm[s], a.cur_T_f_w, a.opt, a.overlap_kf_out, a.overlap_count_out, a.stats, e_pt[s],
                        e_src[s]);
    if (e_pt[s].empty()) continue;
    active.push_back(s);
    E_total += (int)e_pt[s].size();
  }
  if (E_total == 0) return 0;

  // ---- device: one launch over the concatenated enumerations ----
  cudaSetDevice(ctx->device);
  const int A = (int)active.size();
  Carver c;
  std::vector<ReprojLayout> L((size_t)A);
  for (int j = 0; j < A; ++j) reproject_carve_in(c, streams[active[j]].map, (int)e_pt[active[j]].size(), L[j]);
  const size_t o_tab = c.take(sizeof(ReprojStream) * A);
  const size_t in_bytes = c.off;
  size_t o_out0 = 0;
  for (int j = 0; j < A; ++j) {
    reproject_carve_out(c, (int)e_pt[active[j]].size(), L[j]);
    if (j == 0) o_out0 = L[0].o_px;
  }
  int rc;
  if ((rc = ensure_host(ctx, ctx->h_in, c.off))) return rc;
  if ((rc = ensure_dev(ctx, ctx->d_in, c.off))) return rc;
  SVO_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
  uint8_t* h = static_cast<uint8_t*>(ctx->h_in.p);
  uint8_t* d = static_cast<uint8_t*>(ctx->d_in.p);
  ReprojStream* tab = reinterpret_cast<ReprojStream*>(h + o_tab);
  int e_begin = 0;
  for (int j = 0; j < A; ++j) {
    const svo_b200_reproject_stream& a = streams[active[j]];
    reproject_stage(h, L[j], a.map, a.kf_frames, a.cur_T_f_w, e_pt[active[j]], a.pt_type_io);
    ReprojStream t;
    std::memset(&t, 0, sizeof(t));
    t.cur = make_desc(a.cur);
    t.cam = cm[active[j]];
    t.in = reproject_in(d, L[j]);
    t.out = reproject_out(d, L[j]);
    t.cur_T_f_w = reinterpret_cast<const double*>(d + L[j].o_cT);
    t.e_begin = e_begin;
    t.cell_size = a.opt->grid_size;
    t.grid_n_cols = grid_n_cols[active[j]];
    t.find_match = a.opt->find_match_direct;
    t.max_search_level = a.opt->max_search_level;
    t.align_max_iter = a.opt->align_max_iter;
    tab[j] = t;
    e_begin += (int)e_pt[active[j]].size();
  }
  SVO_CUDA_CHECK(ctx, cudaMemcpyAsync(d, h, in_bytes, cudaMemcpyHostToDevice, ctx->stream));
  const int blocks = (E_total + kRpWarps - 1) / kRpWarps;
  kt_begin(ctx);
  reproject_match_streams_kernel<<<blocks, kRpWarps * 32, 0, ctx->stream>>>(reinterpret_cast<const ReprojStream*>(d + o_tab),
                                                                             A, E_total);
  ctx->launches++;
  kt_end(ctx);
  SVO_CUDA_CHECK(ctx, cudaGetLastError());
  SVO_CUDA_CHECK(ctx, cudaMemcpyAsync(h + o_out0, d + o_out0, c.off - o_out0, cudaMemcpyDeviceToHost, ctx->stream));
  SVO_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
  for (int j = 0; j < A; ++j) {
    const int s = active[j];
    const svo_b200_reproject_stream& a = streams[s];
    reproject_replay(h, L[j], a.map, a.opt, n_cells[s], a.cell_order, e_pt[s], e_src[s], a.pt_type_io, a.pt_n_failed_io,
                     a.pt_n_succeeded_io, a.pt_action_out, a.overlap_count_out, a.new_point_out, a.new_px_out,
                     a.new_level_out, a.new_type_out, a.new_grad_out, a.stats);
  }
  return 0;
}
