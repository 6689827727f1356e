"""Map views for the reprojector's edge tests (test_reproject_edges_gpu.py, test_edge_pins.py), built on
synth.make_map_case: maps with thousands of keyframes, points with more than 32 observations and exactly equal viewing
angles, and points that every keyframe sees from more than 60 degrees away."""
from __future__ import annotations

import numpy as np

from rpg_svo_b200 import synth


def kf_positions(view) -> np.ndarray:
    """Frame::pos() of every keyframe: -R^T t."""
    T = np.asarray(view["kf_T_f_w"]).reshape(-1, 3, 4)
    return -np.einsum("kji,kj->ki", T[:, :, :3], T[:, :, 3])


def pad_keyframes(c: dict, n_kfs: int) -> dict:
    """The map of `c` with n_kfs keyframes: the added ones come first, have no key points and no features, and share
    the first keyframe's images; the original keyframes (the ones the points observe) become the last ones."""
    v = dict(c["view"])
    nk = v["n_kfs"]
    pad = n_kfs - nk
    T = np.asarray(v["kf_T_f_w"]).reshape(nk, 3, 4)
    dummy = np.repeat(T[:1], pad, axis=0)
    dummy[:, :, 3] += np.linspace(-1.0, 1.0, pad)[:, None]                  # distinct positions
    v.update(n_kfs=n_kfs, kf_T_f_w=np.concatenate([dummy, T]),
             kf_keypt_pos=np.concatenate([np.zeros((pad, 5, 3)), v["kf_keypt_pos"]]),
             kf_keypt_valid=np.concatenate([np.zeros((pad, 5), np.uint8), v["kf_keypt_valid"]]),
             kf_fts_offset=np.concatenate([np.zeros(pad, np.int32), v["kf_fts_offset"]]).astype(np.int32),
             ftr_kf=(np.asarray(v["ftr_kf"]) + pad).astype(np.int32))
    return dict(c, view=v, kf_pyr=[c["kf_pyr"][0]] * pad + list(c["kf_pyr"]))


def with_obs_lists(c: dict, lists: dict) -> dict:
    """The map of `c` with the observation lists of some points replaced (lists: point -> feature indices)."""
    v = dict(c["view"])
    off, obs = v["pt_obs_offset"], v["pt_obs"]
    per = [list(obs[off[p]:off[p + 1]]) for p in range(v["n_points"])]
    for p, l in lists.items():
        per[p] = list(l)
    ooff = np.zeros(v["n_points"] + 1, np.int32)
    ooff[1:] = np.cumsum([len(x) for x in per])
    v.update(pt_obs_offset=ooff, pt_obs=np.array([i for x in per for i in x], np.int32))
    return dict(c, view=v)


def many_obs_case(seed: int = 21) -> dict:
    """70 keyframes that each observe a point with probability 0.95, so points have up to ~70 observations.  Keyframes
    32..47 repeat the poses of 0..15 (equal angles 32 observations apart: the same lane of the warp's strided loop) and
    17, 19, .., 29 repeat 16, 18, .., 28 (equal angles in neighbouring lanes).  Four points (c["trimmed"]) keep exactly 32,
    33, 64 and 65 of their observations.  Three keyframes 20 m behind the points (as the current frame sees them)
    observe six points (c["far"]), and nothing else does: every cosine is negative.  Three more points (c["wide"]) are
    observed only by a keyframe of their own that sees them 70 degrees away from the current frame (cosine ~0.34): positive,
    but below getCloseViewObs's 0.5.  Both kinds must never be matched."""
    same = tuple((j, j + 32) for j in range(16)) + tuple((j, j + 1) for j in range(16, 30, 2))
    c = synth.make_map_case(seed, n_kfs=70, n_points=250, width=376, height=240, obs_prob=0.95, same_pose=same)
    v = c["view"]
    off, obs = v["pt_obs_offset"], v["pt_obs"]
    lists = {}
    trimmed = [p for p in range(v["n_points"]) if off[p + 1] - off[p] >= 65][:4]
    T = np.asarray(c["cur_T_f_w"]).reshape(3, 4)
    cam = c["cam"]
    pc = np.asarray(v["pt_pos"]) @ T[:, :3].T + T[:, 3]
    u, vv = cam.fx * pc[:, 0] / pc[:, 2] + cam.cx, cam.fy * pc[:, 1] / pc[:, 2] + cam.cy
    seen = [p for p in range(v["n_points"]) if p not in trimmed and off[p + 1] - off[p] >= 40 and pc[p, 2] > 0
            and 20 < u[p] < cam.width - 20 and 20 < vv[p] < cam.height - 20]  # projected and in the overlap keyframes
    far_pts, wide_pts = seen[:6], seen[6:9]
    for p, n in zip(trimmed, (32, 33, 64, 65)):
        lists[p] = obs[off[p]:off[p] + n]
    # three far keyframes
    nk, nf = v["n_kfs"], v["n_ftrs"]
    R = synth.base_pose()[:, :3]
    mean = np.asarray(v["pt_pos"]).mean(axis=0)
    w = -T[:, :3].T @ T[:, 3] - mean
    w /= np.linalg.norm(w)
    u = np.cross(w, [1.0, 0.0, 0.0])
    u /= np.linalg.norm(u)
    far = []
    for d in (-10.0, 0.0, 10.0):                                            # behind the points, seen from the current frame
        centre = mean - 20.0 * w + d * u
        far.append(np.concatenate([R, (-R @ centre)[:, None]], axis=1))
    cur = -T[:, :3].T @ T[:, 3]
    for p in wide_pts:                                                      # 70 degrees away from the current view
        pos = np.asarray(v["pt_pos"])[p]
        wp = (cur - pos) / np.linalg.norm(cur - pos)
        up = np.cross(wp, [0.0, 1.0, 0.0])
        up /= np.linalg.norm(up)
        centre = pos + 5.0 * (np.cos(np.deg2rad(70)) * wp + np.sin(np.deg2rad(70)) * up)
        far.append(np.concatenate([R, (-R @ centre)[:, None]], axis=1))
    n_far = len(far)
    v = dict(v, n_kfs=nk + n_far, kf_T_f_w=np.concatenate([np.asarray(v["kf_T_f_w"]).reshape(nk, 3, 4), np.stack(far)]),
             kf_keypt_pos=np.concatenate([v["kf_keypt_pos"], np.zeros((n_far, 5, 3))]),
             kf_keypt_valid=np.concatenate([v["kf_keypt_valid"], np.zeros((n_far, 5), np.uint8)]),
             kf_fts_offset=np.concatenate([v["kf_fts_offset"], [v["kf_fts_offset"][-1]] * n_far]).astype(np.int32))
    add = dict(ftr_kf=[], ftr_px=[], ftr_f=[], ftr_level=[], ftr_type=[], ftr_grad=[], ftr_point=[])
    for p, kfs in [(p, range(3)) for p in far_pts] + [(p, [3 + i]) for i, p in enumerate(wide_pts)]:
        lists[p] = []
        for j in kfs:
            lists[p].append(nf + len(add["ftr_kf"]))
            add["ftr_kf"].append(nk + j); add["ftr_px"].append([100.0, 80.0]); add["ftr_f"].append([0.0, 0.0, 1.0])
            add["ftr_level"].append(0); add["ftr_type"].append(0); add["ftr_grad"].append([1.0, 0.0]); add["ftr_point"].append(p)
    for k, a in add.items():
        v[k] = np.concatenate([np.asarray(v[k]), np.asarray(a, dtype=np.asarray(v[k]).dtype)])
    v["n_ftrs"] = nf + len(add["ftr_kf"])
    pt_type = np.array(c["pt_type"], copy=True)
    pt_type[far_pts + wide_pts] = 3                                         # GOOD: tried first in their cells
    c = dict(c, view=v, kf_pyr=list(c["kf_pyr"]) + [c["kf_pyr"][0]] * n_far, trimmed=trimmed, far=far_pts, wide=wide_pts,
             pt_type=pt_type)
    return with_obs_lists(c, lists)


def close_view_obs(c: dict) -> list:
    """Point::getCloseViewObs of every point in numpy: (best cosine, winning position in the list, positions that reach
    the same cosine exactly)."""
    v = c["view"]
    T = np.asarray(c["cur_T_f_w"]).reshape(3, 4)
    cur = -T[:, :3].T @ T[:, 3]
    kp = kf_positions(v)
    out = []
    for p in range(v["n_points"]):
        pos = np.asarray(v["pt_pos"])[p]
        o = (cur - pos) / np.linalg.norm(cur - pos)
        lst = v["pt_obs"][v["pt_obs_offset"][p]:v["pt_obs_offset"][p + 1]]
        d = kp[np.asarray(v["ftr_kf"])[lst]] - pos
        cos = (d / np.linalg.norm(d, axis=1)[:, None]) @ o
        best, j = 0.0, 0
        for i, x in enumerate(cos):
            if x > best:
                best, j = x, i
        out.append((best, j, [i for i, x in enumerate(cos) if x == best and len(cos)]))
    return out


def _world_of_pixel(T_f_w, cam, u, v, z=3.0) -> np.ndarray:
    """The world point at depth z that an undistorted pinhole frame with pose T_f_w sees at pixel (u, v)."""
    T = np.asarray(T_f_w).reshape(3, 4)
    pc = np.array([(u - cam.cx) / cam.fx * z, (v - cam.cy) / cam.fy * z, z])
    return T[:, :3].T @ (pc - T[:, 3])


def boundary_case(seed: int = 45) -> dict:
    """Candidates without observations that project 1e-7 px to either side of the isInFrame(px.cast<int>(), 8) limits
    ((int)u = 7 / 8 and width-9 / width-8, the same in v) and of cell boundaries; the cell order is the identity and
    find_match_direct is off, so the order of the new features is the order of the cells the candidates fell in.
    Returns the case and, per added candidate, the (u, v) it projects to."""
    c = synth.make_map_case(seed, n_kfs=3, n_points=60, n_candidates=0)
    v, cam = dict(c["view"]), c["cam"]
    W, H, e = cam.width, cam.height, 1e-7
    px = []
    for a in (8 - e, 8 + e, W - 8 - e, W - 8 + e):                          # u edges, v well inside
        px.append((a, 200.5))
    for b in (8 - e, 8 + e, H - 8 - e, H - 8 + e):                          # v edges
        px.append((300.5, b))
    for k in (1, 2, 5, 12, 24):                                             # cell boundaries at multiples of 30 px
        px += [(30 * k - e, 100.5), (30 * k + e, 130.5), (400.5, min(30 * k, H - 30) - e), (430.5, min(30 * k, H - 30) + e)]
    P = v["n_points"]
    v["pt_pos"] = np.concatenate([v["pt_pos"], [_world_of_pixel(c["cur_T_f_w"], cam, a, b) for a, b in px]])
    v["pt_obs_offset"] = np.concatenate([v["pt_obs_offset"], [v["pt_obs_offset"][-1]] * len(px)]).astype(np.int32)
    v["n_points"] = P + len(px)
    v["cand_point"] = np.arange(P, P + len(px), dtype=np.int32)
    v["n_candidates"] = len(px)
    n_cells = int(np.ceil(W / 30)) * int(np.ceil(H / 30))
    c = dict(c, view=v, pt_type=np.concatenate([c["pt_type"], np.ones(len(px), np.int32)]),
             pt_n_failed=np.concatenate([c["pt_n_failed"], np.zeros(len(px), np.int32)]),
             pt_n_succeeded=np.concatenate([c["pt_n_succeeded"], np.zeros(len(px), np.int32)]),
             cell_order=np.arange(n_cells, dtype=np.int32),
             options=dict(c["options"], find_match_direct=0, max_fts=10000))
    return c, np.array(px)


def keypoint_edge_case(seed: int = 46) -> dict:
    """Keyframes whose only valid key point (Frame::isVisible) lies behind the current camera but maps into the image
    through the negative depth, or 1e-7 px to either side of the image edge (u = 0, u = width, v = 0, v = height).
    Returns the case and the keyframes that must be close."""
    c = synth.make_map_case(seed, n_kfs=10, n_points=300)
    v, cam = dict(c["view"]), c["cam"]
    W, H, e = cam.width, cam.height, 1e-7
    kp, valid = np.array(v["kf_keypt_pos"], copy=True), np.zeros_like(v["kf_keypt_valid"])
    T = np.asarray(c["cur_T_f_w"]).reshape(3, 4)
    inside = {}
    spots = [((-e, 200.0), False), ((e, 200.0), True), ((W - e, 200.0), True), ((W + e, 200.0), False),
             ((300.0, -e), False), ((300.0, e), True), ((300.0, H - e), True), ((300.0, H + e), False)]
    for k, ((u, vv), ok) in enumerate(spots, start=1):
        kp[k, 0] = _world_of_pixel(T, cam, u, vv)
        valid[k, 0] = 1
        inside[k] = ok
    behind = _world_of_pixel(T, cam, 300.0, 200.0, z=-3.0)                  # z < 0, but x/z, y/z land in the image
    kp[9, 0], valid[9, 0] = behind, 1
    inside[9] = False
    v.update(kf_keypt_pos=kp, kf_keypt_valid=valid)
    return dict(c, view=v), sorted(k for k, ok in inside.items() if ok)
