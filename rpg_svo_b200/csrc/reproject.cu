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

// One reprojectMap call of a launch, in a per-launch device table: its current frame, camera, map arrays, output arrays,
// grid and options.
struct ReprojStream {
  FrameDesc cur;
  Cam cam;
  ReprojIn in;
  ReprojOut out;
  double cur_T_f_w[12];
  int cell_size, grid_n_cols, find_match, max_search_level, align_max_iter;
};

// One warp per enumerated point of n_streams calls' concatenated enumerations: point g is point g - e_offset[s] of call
// s = stream_of(e_offset, n_streams, g).
__global__ void __launch_bounds__(kRpWarps * 32) reproject_match_kernel(const ReprojStream* __restrict__ streams,
                                                                        const int* __restrict__ e_offset, int n_streams,
                                                                        int E_total) {
  __shared__ WarpAlignScratch scratch[kRpWarps];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = blockIdx.x * kRpWarps + warp;
  if (g >= E_total) return;
  const int s = stream_of(e_offset, n_streams, g);
  const ReprojStream& rs = streams[s];
  const int e = g - __ldg(e_offset + s);
  const FrameDesc& cur = rs.cur;
  const Cam& cam = rs.cam;
  const ReprojIn& in = rs.in;
  const ReprojOut& out = rs.out;
  const int cell_size = rs.cell_size, grid_n_cols = rs.grid_n_cols, find_match = rs.find_match,
            max_search_level = rs.max_search_level, align_max_iter = rs.align_max_iter;
  const int p = in.e_pt[e];
  const double pos[3] = {in.pt_pos[3 * p], in.pt_pos[3 * p + 1], in.pt_pos[3 * p + 2]};
  const Pose T_cur_w = pose_from_rt12(rs.cur_T_f_w);
  // Reprojector::reprojectPoint (:206-217)
  double pc[3], u, v;
  pose_apply(T_cur_w, pos, pc);
  world2cam(cam, pc, u, v);
  const int ui = (int)u, vi = (int)v;
  const bool inside = ui >= 8 && ui < cam.width - 8 && vi >= 8 && vi < cam.height - 8;  // isInFrame(px.cast<int>(), 8)
  const int cell = inside ? (int)(v / cell_size) * grid_n_cols + (int)(u / cell_size) : -1;
  int success = 0, search_level = 0, ref = -1;
  double A[4] = {0, 0, 0, 0}, h_inv = 0.0, pu = u, pv = v;
  if (inside && find_match && !in.e_skip[e]) {
    // Point::getCloseViewObs (point.cpp:97-117): first observation with the largest cos(angle), must be > 60 deg
    const Pose T_cur_w_inv = pose_inv(T_cur_w);
    double ox = T_cur_w_inv.t[0] - pos[0], oy = T_cur_w_inv.t[1] - pos[1], oz = T_cur_w_inv.t[2] - pos[2];
    const double on = sqrt(ox * ox + oy * oy + oz * oz);
    ox /= on; oy /= on; oz /= on;
    const int b = in.pt_obs_offset[p], en = in.pt_obs_offset[p + 1];
    double best_c = 0.0;
    int best_j = b;
    for (int j = b + lane; j < en; j += 32) {
      // Frame::pos() = T_f_w_.inverse().translation() of the observing keyframe, computed by the lane that reads it:
      // nothing is staged per keyframe, so the number of keyframes in the map view has no limit
      const int k = in.ftr_kf[in.pt_obs[j]];
      const Pose Ti = pose_inv(pose_from_rt12(in.kf_T + 12 * (size_t)k));
      double dx = Ti.t[0] - pos[0], dy = Ti.t[1] - pos[1], dz = Ti.t[2] - pos[2];
      const double dn = sqrt(dx * dx + dy * dy + dz * dz);
      dx /= dn; dy /= dn; dz /= dn;
      const double c = ox * dx + oy * dy + oz * dz;
      if (c > best_c) { best_c = c; best_j = j; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double oc = __shfl_xor_sync(0xffffffffu, best_c, o);
      const int oj = __shfl_xor_sync(0xffffffffu, best_j, o);
      if (oc > best_c || (oc == best_c && oj < best_j)) { best_c = oc; best_j = oj; }
    }
    if (en > b) {
      ref = in.pt_obs[best_j];
      if (!(best_c < 0.5)) {
        const int k = in.ftr_kf[ref];
        const double ref_px[2] = {in.ftr_px[2 * ref], in.ftr_px[2 * ref + 1]};
        const double f_ref[3] = {in.ftr_f[3 * ref], in.ftr_f[3 * ref + 1], in.ftr_f[3 * ref + 2]};
        const double grad[2] = {in.ftr_grad[2 * ref], in.ftr_grad[2 * ref + 1]};
        success = warp_find_match_direct(cur, cam, in.kf_frames[k], pose_from_rt12(in.kf_T + 12 * (size_t)k), T_cur_w, ref_px,
                                         f_ref, in.ftr_level[ref], in.ftr_type[ref], grad, pos, max_search_level,
                                         align_max_iter, scratch[warp], pu, pv, search_level, A, h_inv)
                      ? 1 : 0;
      }
    }
  }
  if (lane == 0) {
    out.px[2 * e] = u; out.px[2 * e + 1] = v;
    out.in_frame[e] = inside ? 1 : 0;
    out.cell[e] = cell;
    out.success[e] = (uint8_t)success;
    out.px_match[2 * e] = pu; out.px_match[2 * e + 1] = pv;
    out.search_level[e] = search_level;
    for (int k = 0; k < 4; ++k) out.A[4 * e + k] = A[k];
    out.ref_ftr[e] = ref;
  }
}

}  // namespace svo

using namespace svo;

namespace {

// One reprojectMap call: its arguments, then its device camera and grid (reproject_grid) and its enumeration in the
// reference's order (reproject_enumerate; src = overlap slot, or -1 for a candidate).
struct ReprojCall {
  svo_b200_reproject_stream a;
  Cam cm;
  int grid_n_cols;
  size_t n_cells;
  std::vector<int> e_pt, e_src;
};

// The argument checks of one reprojectMap call that precede any write (the single-stream call clears its stats and
// actions before the camera and cell-order checks; reproject_grid does those).
int reproject_check(svo_b200_ctx* ctx, const svo_b200_reproject_stream& a) {
  const svo_b200_map_view* m = a.map;
  const svo_b200_frame* const* kf_frames = a.kf_frames;
  const svo_b200_reproject_options* opt = a.opt;
  if (!ctx || !m || !a.cur || !a.cur_T_f_w || !a.cam || !opt || !a.cell_order || !a.pt_type_io || !a.pt_n_failed_io ||
      !a.pt_n_succeeded_io || !a.pt_action_out || !a.overlap_kf_out || !a.overlap_count_out || !a.new_point_out ||
      !a.new_px_out || !a.new_level_out || !a.new_type_out || !a.new_grad_out || !a.stats)
    return set_err(ctx, SVO_B200_EINVAL, "reproject_map: NULL argument");
  if (m->n_kfs < 0 || m->n_ftrs < 0 || m->n_points < 0 || m->n_candidates < 0 || (m->n_kfs > 0 && !kf_frames))
    return set_err(ctx, SVO_B200_EINVAL, "reproject_map: negative sizes / missing keyframe handles");
  if ((m->n_kfs > 0 && (!m->kf_T_f_w || !m->kf_keypt_pos || !m->kf_keypt_valid || !m->kf_fts_offset)) ||
      (m->n_ftrs > 0 && (!m->ftr_kf || !m->ftr_px || !m->ftr_f || !m->ftr_level || !m->ftr_type || !m->ftr_grad || !m->ftr_point)) ||
      (m->n_points > 0 && (!m->pt_pos || !m->pt_obs_offset)) || (m->n_candidates > 0 && !m->cand_point))
    return set_err(ctx, SVO_B200_EINVAL, "reproject_map: NULL array in the map view");
  for (int k = 0; k < m->n_kfs; ++k)
    if (!kf_frames[k]) return set_err(ctx, SVO_B200_EINVAL, "reproject_map: kf_frames[%d] is NULL", k);
  if (const int rc = cam_check_frames(ctx, "reproject_map", a.cam, &a.cur, 1)) return rc;
  if (const int rc = cam_check_frames(ctx, "reproject_map", a.cam, kf_frames, m->n_kfs)) return rc;
  // the device and reproject_enumerate walk every [offset[i], offset[i+1]) range: each must lie inside the range
  // [0, offset[n]) whose entries are checked below
  for (int k = 0; k <= m->n_kfs && m->n_kfs > 0; ++k)
    if (m->kf_fts_offset[k] < (k ? m->kf_fts_offset[k - 1] : 0))
      return set_err(ctx, SVO_B200_EINVAL, "reproject_map: kf_fts_offset[%d] is negative or decreasing", k);
  for (int p = 0; p <= m->n_points && m->n_points > 0; ++p)
    if (m->pt_obs_offset[p] < (p ? m->pt_obs_offset[p - 1] : 0))
      return set_err(ctx, SVO_B200_EINVAL, "reproject_map: pt_obs_offset[%d] is negative or decreasing", p);
  const int n_kf_fts = m->n_kfs ? m->kf_fts_offset[m->n_kfs] : 0, n_obs_total = m->n_points ? m->pt_obs_offset[m->n_points] : 0;
  if (n_kf_fts < 0 || n_obs_total < 0 || (n_kf_fts > 0 && !m->kf_fts) || (n_obs_total > 0 && !m->pt_obs))
    return set_err(ctx, SVO_B200_EINVAL, "reproject_map: inconsistent offsets in the map view");
  if (opt->grid_size <= 0 || opt->max_fts < 0 || opt->max_n_kfs < 0 || opt->max_search_level < 0 ||
      opt->max_search_level >= a.cur->n_levels)
    return set_err(ctx, SVO_B200_EINVAL, "reproject_map: bad options (grid_size %d, max_search_level %d of %d levels)",
                   opt->grid_size, opt->max_search_level, a.cur->n_levels);
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
int reproject_grid(svo_b200_ctx* ctx, ReprojCall& r) {
  const svo_b200_camera* cam = r.a.cam;
  if (const int rc = cam_to_dev(ctx, cam, r.cm)) return rc;
  r.grid_n_cols = (int)std::ceil((double)cam->width / r.a.opt->grid_size);
  const int grid_n_rows = (int)std::ceil((double)cam->height / r.a.opt->grid_size);
  r.n_cells = (size_t)r.grid_n_cols * grid_n_rows;
  for (size_t i = 0; i < r.n_cells; ++i)
    if (r.a.cell_order[i] < 0 || (size_t)r.a.cell_order[i] >= r.n_cells)
      return set_err(ctx, SVO_B200_EINVAL, "reproject_map: cell_order[%zu] out of range", i);
  return 0;
}

// Map::getCloseKeyframes and the enumeration of the points to project, in the reference's order; writes the overlap
// keyframes and n_overlap.
void reproject_enumerate(ReprojCall& r) {
  const svo_b200_map_view* m = r.a.map;
  // Map::getCloseKeyframes (map.cpp:106-127) + sort by distance (:76-77); list::sort is stable
  const double* Tc = r.a.cur_T_f_w;
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
      cam_world2cam(r.cm, x / z, y / z, u, v);  // Frame::w2c
      if (u >= 0.0 && v >= 0.0 && u < r.a.cam->width && v < r.a.cam->height) {
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
  for (auto it = close_kfs.begin(); it != close_kfs.end() && n_ov < (size_t)r.a.opt->max_n_kfs; ++it, ++n_ov) {
    const int k = it->first;
    r.a.overlap_kf_out[n_ov] = k;
    r.a.overlap_count_out[n_ov] = 0;
    for (int j = m->kf_fts_offset[k]; j < m->kf_fts_offset[k + 1]; ++j) {
      const int p = m->ftr_point[m->kf_fts[j]];
      if (p < 0 || projected[p]) continue;
      projected[p] = 1;
      r.e_pt.push_back(p);
      r.e_src.push_back((int)n_ov);
    }
  }
  r.a.stats->n_overlap = (int)n_ov;
  for (int c = 0; c < m->n_candidates; ++c) { r.e_pt.push_back(m->cand_point[c]); r.e_src.push_back(-1); }
}

// Declares one call's regions, their device addresses going into its table entry t: the map arrays and the enumeration
// in (the skip flags and keyframe descriptors filled by reproject_run), the device results out.
void reproject_stage(Staging& st, const ReprojCall& r, ReprojStream& t) {
  const svo_b200_map_view* m = r.a.map;
  const size_t E = r.e_pt.size(), n_pts = m->n_points, n_ftrs = m->n_ftrs, n_kfs = m->n_kfs;
  memset(&t, 0, sizeof(t));
  ReprojIn& in = t.in;
  ReprojOut& out = t.out;
  st.in(r.e_pt.data(), E, &in.e_pt);
  st.in(nullptr, E, &in.e_skip);
  st.in(m->pt_pos, 3 * n_pts, &in.pt_pos);
  st.in(m->pt_obs_offset, n_pts + 1, &in.pt_obs_offset);
  st.in(m->pt_obs, n_pts ? m->pt_obs_offset[n_pts] : 0, &in.pt_obs);
  st.in(m->ftr_kf, n_ftrs, &in.ftr_kf);
  st.in(m->ftr_px, 2 * n_ftrs, &in.ftr_px);
  st.in(m->ftr_f, 3 * n_ftrs, &in.ftr_f);
  st.in(m->ftr_level, n_ftrs, &in.ftr_level);
  st.in(m->ftr_type, n_ftrs, &in.ftr_type);
  st.in(m->ftr_grad, 2 * n_ftrs, &in.ftr_grad);
  st.in(m->kf_T_f_w, 12 * n_kfs, &in.kf_T);
  st.in(nullptr, n_kfs, &in.kf_frames);
  st.out(nullptr, 2 * E, &out.px);
  st.out(nullptr, E, &out.in_frame);
  st.out(nullptr, E, &out.cell);
  st.out(nullptr, E, &out.success);
  st.out(nullptr, 2 * E, &out.px_match);
  st.out(nullptr, E, &out.search_level);
  st.out(nullptr, 4 * E, &out.A);
  st.out(nullptr, E, &out.ref_ftr);
  t.cur = make_desc(r.a.cur);
  t.cam = r.cm;
  memcpy(t.cur_T_f_w, r.a.cur_T_f_w, sizeof(double) * 12);
  t.cell_size = r.a.opt->grid_size;
  t.grid_n_cols = r.grid_n_cols;
  t.find_match = r.a.opt->find_match_direct;
  t.max_search_level = r.a.opt->max_search_level;
  t.align_max_iter = r.a.opt->align_max_iter;
}
// The host replay of the sequential policy over the device results `o` of one call, in st's pinned buffer.
void reproject_replay(const Staging& st, const ReprojOut& o, const ReprojCall& r) {
  const svo_b200_reproject_stream& a = r.a;
  const svo_b200_map_view* m = a.map;
  const svo_b200_reproject_options* opt = a.opt;
  const int E = (int)r.e_pt.size();
  const double *r_px = st.host(o.px), *r_pm = st.host(o.px_match), *r_A = st.host(o.A);
  const uint8_t *r_in = st.host(o.in_frame), *r_su = st.host(o.success);
  const int *r_cell = st.host(o.cell), *r_sl = st.host(o.search_level), *r_rf = st.host(o.ref_ftr);
  std::vector<std::vector<int>> cells(r.n_cells);  // enumeration indices, push_back order
  for (int e = 0; e < E; ++e) {
    const int p = r.e_pt[e];
    if (r_in[e]) {
      cells[(size_t)r_cell[e]].push_back(e);
      ++a.stats->n_projected;
      if (r.e_src[e] >= 0) a.overlap_count_out[r.e_src[e]]++;
      if (opt->find_match_direct && a.pt_type_io[p] != 0) ++a.stats->n_speculative;
    } else if (r.e_src[e] < 0) {  // candidate that does not reproject (:113-122)
      a.pt_n_failed_io[p] += 3;
      if (a.pt_n_failed_io[p] > 30) {
        a.pt_type_io[p] = 0;
        a.pt_action_out[p] = SVO_B200_PT_CANDIDATE_ERASED;
      }
    }
  }
  for (size_t i = 0; i < r.n_cells; ++i) {
    std::vector<int>& cell = cells[(size_t)a.cell_order[i]];
    // cell.sort(pointQualityComparator): stable, better type first (:144-149,153)
    std::stable_sort(cell.begin(), cell.end(), [&](int el, int er) { return a.pt_type_io[r.e_pt[el]] > a.pt_type_io[r.e_pt[er]]; });
    bool matched = false;
    for (size_t ci = 0; ci < cell.size(); ++ci) {
      const int e = cell[ci], p = r.e_pt[e];
      ++a.stats->n_trials;
      if (a.pt_type_io[p] == 0) continue;  // TYPE_DELETED: erased from the cell
      const bool found_match = opt->find_match_direct ? r_su[e] != 0 : true;
      if (!found_match) {
        a.pt_n_failed_io[p]++;
        if (a.pt_type_io[p] == 2 && a.pt_n_failed_io[p] > 15) { a.pt_type_io[p] = 0; a.pt_action_out[p] = SVO_B200_PT_SAFE_DELETE; }
        if (a.pt_type_io[p] == 1 && a.pt_n_failed_io[p] > 30) { a.pt_type_io[p] = 0; a.pt_action_out[p] = SVO_B200_PT_DELETE_CANDIDATE; }
        continue;
      }
      a.pt_n_succeeded_io[p]++;
      if (a.pt_type_io[p] == 2 && a.pt_n_succeeded_io[p] > 10) a.pt_type_io[p] = 3;
      const int q = a.stats->n_new++;
      a.new_point_out[q] = p;
      a.new_px_out[2 * q] = opt->find_match_direct ? r_pm[2 * e] : r_px[2 * e];
      a.new_px_out[2 * q + 1] = opt->find_match_direct ? r_pm[2 * e + 1] : r_px[2 * e + 1];
      a.new_level_out[q] = r_sl[e];
      a.new_type_out[q] = 0;
      a.new_grad_out[2 * q] = 1.0;
      a.new_grad_out[2 * q + 1] = 0.0;
      const int ref = r_rf[e];
      if (ref >= 0 && m->ftr_type[ref] == 1) {  // EDGELET: grad = normalize(A_cur_ref * ref grad) (:190-195)
        const double gx = m->ftr_grad[2 * ref], gy = m->ftr_grad[2 * ref + 1];
        const double ax = r_A[4 * e] * gx + r_A[4 * e + 1] * gy, ay = r_A[4 * e + 2] * gx + r_A[4 * e + 3] * gy;
        const double nn = std::sqrt(ax * ax + ay * ay);
        a.new_type_out[q] = 1;
        a.new_grad_out[2 * q] = ax / nn;
        a.new_grad_out[2 * q + 1] = ay / nn;
      }
      matched = true;
      break;
    }
    if (matched) ++a.stats->n_matches;
    if (a.stats->n_matches > (int64_t)opt->max_fts) break;
  }
}


// The device half of reprojectMap for checked and enumerated calls: one launch over the points of every call that has any
// (none when no call has), then each such call's replay into its own outputs.
int reproject_run(svo_b200_ctx* ctx, const std::vector<ReprojCall>& calls) {
  std::vector<const ReprojCall*> act;  // the calls with points, in order; act[j] owns points e_offset[j] .. e_offset[j+1]-1
  std::vector<int> e_offset(1, 0);
  for (const ReprojCall& r : calls)
    if (!r.e_pt.empty()) { act.push_back(&r); e_offset.push_back(e_offset.back() + (int)r.e_pt.size()); }
  const int A = (int)act.size(), E_total = e_offset.back();
  if (A == 0) return 0;
  cudaSetDevice(ctx->device);
  Staging st(ctx);
  std::vector<ReprojStream> tab((size_t)A);
  for (int j = 0; j < A; ++j) reproject_stage(st, *act[j], tab[j]);
  const ReprojStream* d_tab;
  const int* d_off;
  st.in(tab.data(), A, &d_tab);
  st.in(e_offset.data(), A + 1, &d_off);
  int rc;
  if ((rc = st.open())) return rc;
  for (int j = 0; j < A; ++j) {
    const ReprojCall& r = *act[j];
    uint8_t* skip = st.host(tab[j].in.e_skip);
    for (size_t e = 0; e < r.e_pt.size(); ++e) skip[e] = r.a.pt_type_io[r.e_pt[e]] == 0;
    FrameDesc* kfs = st.host(tab[j].in.kf_frames);
    for (int k = 0; k < r.a.map->n_kfs; ++k) kfs[k] = make_desc(r.a.kf_frames[k]);
  }
  if ((rc = st.send())) return rc;
  const int blocks = (E_total + kRpWarps - 1) / kRpWarps;
  if ((rc = launch_kernels(ctx, 1, [&] {
         reproject_match_kernel<<<blocks, kRpWarps * 32, 0, ctx->stream>>>(d_tab, d_off, A, E_total);
       })))
    return rc;
  if ((rc = st.receive())) return rc;
  for (int j = 0; j < A; ++j) reproject_replay(st, tab[j].out, *act[j]);
  return 0;
}

}  // namespace

extern "C" int svo_b200_reproject_map(svo_b200_ctx* ctx, const svo_b200_map_view* m, const svo_b200_frame* const* kf_frames,
                                      const svo_b200_frame* cur, const double* cur_T_f_w, const svo_b200_camera* cam,
                                      const svo_b200_reproject_options* opt, const int* cell_order, int* pt_type_io,
                                      int* pt_n_failed_io, int* pt_n_succeeded_io, uint8_t* pt_action_out,
                                      int* overlap_kf_out, int64_t* overlap_count_out, int* new_point_out,
                                      double* new_px_out, int* new_level_out, int* new_type_out, double* new_grad_out,
                                      svo_b200_reproject_stats* stats) {
  std::vector<ReprojCall> call(1);
  ReprojCall& r = call[0];
  r.a = {m, kf_frames, cur, cur_T_f_w, cam, opt, cell_order, pt_type_io, pt_n_failed_io, pt_n_succeeded_io, pt_action_out,
         overlap_kf_out, overlap_count_out, new_point_out, new_px_out, new_level_out, new_type_out, new_grad_out, stats};
  int rc = reproject_check(ctx, r.a);
  if (rc) return rc;
  std::memset(stats, 0, sizeof(*stats));
  for (int p = 0; p < m->n_points; ++p) pt_action_out[p] = SVO_B200_PT_NONE;
  if ((rc = reproject_grid(ctx, r))) return rc;
  reproject_enumerate(r);
  return reproject_run(ctx, call);
}

extern "C" int svo_b200_reproject_map_streams(svo_b200_ctx* ctx, int S, const svo_b200_reproject_stream* streams) {
  if (!ctx || S < 0 || (S > 0 && !streams))
    return set_err(ctx, SVO_B200_EINVAL, "reproject_map_streams: bad arguments (S %d)", S);
  // every stream is checked before anything is written
  std::vector<ReprojCall> calls((size_t)S);
  int64_t e_bound = 0;  // a stream enumerates at most its keyframe features and candidates
  for (int s = 0; s < S; ++s) {
    ReprojCall& r = calls[s];
    r.a = streams[s];
    int rc = reproject_check(ctx, r.a);
    if (!rc) rc = reproject_grid(ctx, r);
    if (rc) return entry_err(ctx, rc, "reproject_map_streams", "stream", s);
    e_bound += (int64_t)(r.a.map->n_kfs ? r.a.map->kf_fts_offset[r.a.map->n_kfs] : 0) + r.a.map->n_candidates;
  }
  if (e_bound > INT32_MAX) return set_err(ctx, SVO_B200_ELIMIT, "reproject_map_streams: more than 2^31-1 points in one launch");
  for (ReprojCall& r : calls) {
    std::memset(r.a.stats, 0, sizeof(*r.a.stats));
    for (int p = 0; p < r.a.map->n_points; ++p) r.a.pt_action_out[p] = SVO_B200_PT_NONE;
    reproject_enumerate(r);
  }
  return reproject_run(ctx, calls);
}
