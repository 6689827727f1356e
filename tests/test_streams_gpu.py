"""GPU: svo_b200_depth_filter_update_streams and svo_b200_reproject_map_streams -- S streams' updateSeeds / reprojectMap in
one launch each -- against S single-stream calls, bit for bit, over streams that differ in image size, camera model,
keyframes, seed / point counts, batch counters, options and cell orders; shapes up to 257 streams; and every refusal."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

from rpg_svo_b200 import capi, synth

pytestmark = pytest.mark.gpu

SEED_KEYS = ("a", "b", "mu", "z_range", "sigma2", "status", "px_cur", "z", "n_zmssd")
RP_KEYS = ("pt_type", "pt_n_failed", "pt_n_succeeded", "pt_action", "overlap_kf", "overlap_count", "new_point", "new_px",
           "new_level", "new_type", "new_grad", "n_matches", "n_trials", "n_new", "n_overlap", "n_projected", "n_speculative")


def _same_bits(x, y):
    x, y = np.ascontiguousarray(x), np.ascontiguousarray(y)
    return x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes()


# ---- depth filter --------------------------------------------------------------------------------------------------------
# one pixel narrower, shorter, wider, taller than the frames: refused (svo_b200_camera's size is its frames' level 0)
SIZE_OFFSETS = [(-1, 0), (0, -1), (1, 0), (0, 1)]


def _resized(cam, dw, dh):
    return dataclasses.replace(cam, width=cam.width + dw, height=cam.height + dh)


def _cam_644_radtan():
    return synth.Camera(330.0, 329.0, 321.5, 242.5, 644, 484, 0, (-0.28, 0.067, 0.0009, 0.0008, 0.0))


def _subset(c, idx):
    """The seeds idx of a depth case (every per-seed array sliced, the seeds copied)."""
    out = dict(c)
    for k in ("ftr_px", "ftr_f", "ftr_level", "ftr_type", "ftr_grad", "batch_id", "ref_index"):
        out[k] = np.asarray(c[k])[idx]
    out["seeds"] = {k: np.asarray(v)[idx].copy() for k, v in c["seeds"].items()}
    return out


def _depth_streams():
    """A heterogeneous batch: one (case, keyframe pyramids, keyframe poses, batch_counter) per stream."""
    atan = synth.reference_param_camera("atan")
    cases = []
    a = synth.make_depth_case(301, n_seeds=2000, cam=atan)                       # 752x480 ATAN, 1 keyframe, 2000 seeds
    cases.append((a, [a["ref_pyr"]], [a["T_ref_w"]], 6))
    b = synth.make_multi_keyframe_depth_case(302, n_seeds=31, n_kfs=3)          # 752x480 pinhole, 3 keyframes, 31 seeds
    cases.append((b, b["kf_pyr"], b["kf_T"], 7))
    c = synth.make_depth_case(303, n_seeds=400, width=640, height=480)          # 640x480 pinhole, 5 keyframes
    kfs_c = [c["ref_pyr"]]
    T_c = [c["T_ref_w"]]
    rng = np.random.default_rng(5)
    for _ in range(4):
        xi = np.concatenate([rng.uniform(-0.1, 0.1, 3), np.deg2rad(rng.uniform(-2, 2, 3))])
        T = synth.se3_mul(synth.se3_exp(xi), c["T_ref_w"])
        T_c.append(T)
        kfs_c.append(synth.build_pyramid(synth.render(c["cam"], T, c["plane"], synth.make_texture(7)), c["n_levels"]))
    c["ref_index"] = (np.arange(400) % 5).astype(np.int32)
    cases.append((c, kfs_c, T_c, 3))
    d = synth.make_depth_case(304, n_seeds=1, width=644, height=484, cam=_cam_644_radtan())  # radial-tangential, 1 seed
    cases.append((d, [d["ref_pyr"]], [d["T_ref_w"]], 6))
    e = synth.make_seed_status_case(305)                                        # every status
    cases.append((e, [e["ref_pyr"]], [e["T_ref_w"]], 6))
    f = _subset(a, np.arange(0))                                                 # no seeds
    cases.append((f, [a["ref_pyr"]], [a["T_ref_w"]], 6))
    g = _subset(a, np.arange(0, 2000, 7))                                        # shares a's frames, another batch counter
    cases.append((g, [a["ref_pyr"]], [a["T_ref_w"]], 9))
    return cases


def _run_depth(ctx, cases, cur_override=None):
    """Single calls and one streams call over the same frame handles; returns (singles, batched, handles to free)."""
    frames, kf_tab, kf_T, streams, singles = [], [], [], [], []
    kf_cache = {}
    for j, (c, kpyr, kT, bc) in enumerate(cases):
        cur = cur_override[j] if cur_override and cur_override.get(j) is not None else None
        if cur is None:
            cur = ctx.frame(c["cur_pyr"])
            frames.append(cur)
        own = []
        for p, T in zip(kpyr, kT):
            key = id(p)
            if key not in kf_cache:                                              # one handle per distinct keyframe image
                h = ctx.frame(p)
                frames.append(h)
                kf_cache[key] = len(kf_tab)
                kf_tab.append(h)
                kf_T.append(T)
            own.append(kf_cache[key])
        own = np.asarray(own, np.int32)
        ri = np.asarray(c["ref_index"], np.int32)
        args = (c["ftr_px"], c["ftr_f"], c["ftr_level"], c["ftr_type"], c["ftr_grad"], c["batch_id"])
        singles.append(ctx.depth_filter_update([kf_tab[i] for i in own], [kf_T[i] for i in own], cur, c["T_cur_w"], c["cam"],
                                               ri, *args, bc, c["seeds"]))
        streams.append(dict(cur=cur, cur_T_f_w=c["T_cur_w"], cam=c["cam"], batch_counter=bc, ref_index=own[ri] if len(ri) else ri,
                            ftr_px=c["ftr_px"], ftr_f=c["ftr_f"], ftr_level=c["ftr_level"], ftr_type=c["ftr_type"],
                            ftr_grad=c["ftr_grad"], batch_id=c["batch_id"], seeds=c["seeds"]))
    batched = ctx.depth_filter_update_streams(streams, kf_tab, kf_T)
    return singles, batched, frames


def _check_depth(singles, batched):
    assert len(singles) == len(batched)
    for s, (g, b) in enumerate(zip(singles, batched)):
        for k in SEED_KEYS:
            assert _same_bits(g[k], b[k]), (s, k)


def test_depth_streams_heterogeneous_equal_single_calls(ctx, oracle):
    pool = capi.FramePool(ctx, 752, 480, 5, 2)
    cases = _depth_streams()
    pool.upload_array(np.stack([cases[0][0]["cur_pyr"][0], cases[4][0]["cur_pyr"][0]]))
    over = {0: pool.frames[0], 6: pool.frames[0], 4: pool.frames[1]}           # pool frames; streams 0 and 6 share one
    singles, batched, frames = _run_depth(ctx, cases, cur_override=over)
    _check_depth(singles, batched)
    st = np.concatenate([b["status"] for b in batched])
    counts = {s: int((st == s).sum()) for s in range(1, 8)}
    print("statuses across the batch:", counts)
    for s in range(1, 7):                                                        # every status the single-stream tests reach
        assert counts[s] > 0, s
    # statuses against the oracle, stream by stream
    for (c, kpyr, kT, bc), b in zip(cases, batched):
        if not len(c["ref_index"]):
            continue
        o = oracle.depth_filter_update(kpyr, kT, c["cur_pyr"], c["T_cur_w"], c["cam"], c["ref_index"], c["ftr_px"], c["ftr_f"],
                                       c["ftr_level"], c["ftr_type"], c["ftr_grad"], c["batch_id"], bc, c["seeds"])
        assert np.array_equal(o["status"], b["status"])
    for f in frames:
        f.destroy()
    pool.destroy()


@pytest.mark.parametrize("S", [0, 1, 2, 33, 132, 257])
def test_depth_streams_shapes(ctx, S):
    """S streams over three scenes (streams share current frames and keyframe handles), 0..12 seeds each."""
    scenes = [synth.make_depth_case(310 + k, n_seeds=60, width=w, height=h) for k, (w, h) in enumerate([(752, 480), (640, 480), (644, 484)])]
    rng = np.random.default_rng(S)
    cases = []
    for s in range(S):
        c = scenes[s % 3]
        idx = rng.choice(60, int(rng.integers(0, 13)), replace=False)
        cases.append((_subset(c, idx), [c["ref_pyr"]], [c["T_ref_w"]], int(rng.integers(5, 9))))
    shared = {}
    frames_cur = {}
    for s in range(S):
        k = s % 3
        if k not in frames_cur:
            frames_cur[k] = ctx.frame(scenes[k]["cur_pyr"])
        shared[s] = frames_cur[k]
    singles, batched, frames = _run_depth(ctx, cases, cur_override=shared)
    _check_depth(singles, batched)
    for f in frames + list(frames_cur.values()):
        f.destroy()


def _raw_depth_call(ctx, S, curs, cT, cams, bc, off, refs, refT, n_ref, M, ri, lv, seeds):
    opt = capi.DepthOptions(3, 200.0, 2, 10, 1000)
    z = np.zeros(max(M, 1))
    px, f, g = np.zeros((max(M, 1), 2)), np.tile([0.0, 0.0, 1.0], (max(M, 1), 1)), np.tile([1.0, 0.0], (max(M, 1), 1))
    ty, bi = np.zeros(max(M, 1), np.int32), np.zeros(max(M, 1), np.int32)
    st, pc, nz = np.full(max(M, 1), 77, np.uint8), np.full((max(M, 1), 2), 7.0), np.full(max(M, 1), 77, np.int32)
    rc = ctx.lib.svo_b200_depth_filter_update_streams(
        ctx.h, S, curs, capi._p(cT), cams, capi._p(bc), capi._p(off), refs, capi._p(refT), n_ref, C.byref(opt), capi._p(ri),
        capi._p(px), capi._p(f), capi._p(lv), capi._p(ty), capi._p(g), capi._p(bi), *[capi._p(seeds[k]) for k in ("a", "b", "mu", "z_range", "sigma2")],
        capi._p(st), capi._p(pc), capi._p(z), capi._p(nz))
    return rc, st, pc, z, nz


def test_depth_streams_refusals_write_nothing(ctx):
    c = synth.make_depth_case(320, n_seeds=8)
    kf, cur = ctx.frame(c["ref_pyr"]), ctx.frame(c["cur_pyr"])
    small = ctx.frame(c["cur_pyr"][:2])                                          # a 2-level pyramid
    M = 8

    def base():
        return dict(S=2, curs=(C.c_void_p * 2)(cur.h.value, cur.h.value), cT=np.tile(c["T_cur_w"].reshape(12), (2, 1)),
                    cams=(capi.Camera * 2)(capi.cam_struct(c["cam"]), capi.cam_struct(c["cam"])), bc=np.array([6, 6], np.int32),
                    off=np.array([0, 3, 8], np.int32), refs=(C.c_void_p * 1)(kf.h.value), refT=c["T_ref_w"].reshape(12).copy(),
                    n_ref=1, M=M, ri=np.zeros(M, np.int32), lv=np.zeros(M, np.int32),
                    seeds={k: np.full(M, 0.5, np.float32) for k in ("a", "b", "mu", "z_range", "sigma2")})

    bad = []
    x = base(); x["S"] = -1; bad.append(x)
    x = base(); x["curs"] = (C.c_void_p * 2)(cur.h.value, None); bad.append(x)                      # NULL current frame
    x = base(); x["refs"] = (C.c_void_p * 1)(None); bad.append(x)                                  # NULL keyframe
    x = base(); x["off"] = np.array([0, 5, 3], np.int32); bad.append(x)                            # not monotone
    x = base(); x["off"] = np.array([1, 3, 8], np.int32); bad.append(x)                            # does not start at 0
    x = base(); x["ri"] = np.array([0, 0, 0, 0, 0, 0, 0, 1], np.int32); bad.append(x)              # ref_index out of range
    x = base(); x["ri"] = np.array([0, 0, 0, -1, 0, 0, 0, 0], np.int32); bad.append(x)
    x = base(); x["lv"] = np.array([0, 0, 0, 0, 9, 0, 0, 0], np.int32); bad.append(x)              # level outside the pyramid
    x = base(); x["curs"] = (C.c_void_p * 2)(cur.h.value, small.h.value); bad.append(x)             # max_search_level 2 >= 2 levels
    for dw, dh in SIZE_OFFSETS:                                                                    # a camera of another size
        x = base(); x["cams"] = (capi.Camera * 2)(capi.cam_struct(c["cam"]), capi.cam_struct(_resized(c["cam"], dw, dh))); bad.append(x)
    for j, x in enumerate(bad):
        before = {k: v.copy() for k, v in x["seeds"].items()}
        n0 = ctx.launch_count()
        rc, st, pc, z, nz = _raw_depth_call(ctx, **x)
        assert rc == -1, j                                                                          # SVO_B200_EINVAL
        assert ctx.launch_count() == n0, j
        assert np.all(st == 77) and np.all(pc == 7.0) and np.all(z == 0) and np.all(nz == 77), j
        for k in before:
            assert _same_bits(before[k], x["seeds"][k]), (j, k)
    # S == 0 and streams without seeds: no launch, nothing written
    for x in (dict(base(), S=0), dict(base(), off=np.array([0, 0, 0], np.int32))):
        n0 = ctx.launch_count()
        rc, st, *_ = _raw_depth_call(ctx, **x)
        assert rc == 0 and ctx.launch_count() == n0 and np.all(st == 77)
    # the single-stream depth filter and the epipolar matcher refuse the same way; M == 0 launches nothing
    bad_cam = dataclasses.replace(c["cam"], model=7)
    singles = [dict(cur=None), dict(n_ref=0), dict(ri=np.array([0, 0, 0, 0, 0, 0, 0, 1], np.int32)),
               dict(lv=np.array([0, 0, 0, 0, 9, 0, 0, 0], np.int32)), dict(cur=small), dict(cam=bad_cam)]
    singles += [dict(cam=_resized(c["cam"], dw, dh)) for dw, dh in SIZE_OFFSETS]
    for fn in ("update", "match"):
        for j, over in enumerate(singles + [dict(d_min=None)] * (fn == "match") + [dict(M=0, rc=0)]):
            x = dict(_raw_single_args(c, kf, cur, M), **over)
            want = x.pop("rc", -1)
            before = {k: v.copy() for k, v in x["seeds"].items()}
            n0 = ctx.launch_count()
            rc, outs = _raw_single_call(ctx, fn, **x)
            assert rc == want and ctx.launch_count() == n0, (fn, j)
            for k, o in enumerate(outs):
                assert np.all(o == (77 if o.dtype in (np.uint8, np.int32) else 7.0)), (fn, j, k)
            for k in before:
                assert _same_bits(before[k], x["seeds"][k]), (fn, j, k)
    kf.destroy(); cur.destroy(); small.destroy()


def _raw_single_args(c, kf, cur, M):
    return dict(cur=cur, cam=c["cam"], refs=(C.c_void_p * 1)(kf.h.value), refT=c["T_ref_w"].reshape(12).copy(), n_ref=1,
                cT=c["T_cur_w"].reshape(12).copy(), M=M, ri=np.zeros(M, np.int32), lv=np.zeros(M, np.int32), d_min=np.full(M, 0.5),
                seeds={k: np.full(M, 0.5, np.float32) for k in ("a", "b", "mu", "z_range", "sigma2")})


def _raw_single_call(ctx, fn, cur, cam, refs, refT, n_ref, cT, M, ri, lv, d_min, seeds):
    """svo_b200_depth_filter_update (fn "update") or svo_b200_find_epipolar_match_direct ("match") through raw ctypes, every
    output filled with 77 (integers) or 7.0 (doubles) beforehand; returns the return code and the outputs."""
    opt, cs = capi.DepthOptions(3, 200.0, 2, 10, 1000), capi.cam_struct(cam)
    n = max(M, 1)
    px, f, g = np.zeros((n, 2)), np.tile([0.0, 0.0, 1.0], (n, 1)), np.tile([1.0, 0.0], (n, 1))
    ty, bi, d = np.zeros(n, np.int32), np.zeros(n, np.int32), np.full(n, 1.0)
    cur_h = cur.h if cur is not None else C.c_void_p(None)
    head = (ctx.h, refs, capi._p(refT), n_ref, cur_h, capi._p(cT), C.byref(cs), C.byref(opt), M, capi._p(ri), capi._p(px),
            capi._p(f), capi._p(lv), capi._p(ty), capi._p(g))
    if fn == "update":
        outs = [np.full(n, 77, np.uint8), np.full((n, 2), 7.0), np.full(n, 7.0), np.full(n, 77, np.int32)]
        rc = ctx.lib.svo_b200_depth_filter_update(*head, capi._p(bi), 6, *[capi._p(seeds[k]) for k in ("a", "b", "mu", "z_range", "sigma2")],
                                                  *[capi._p(o) for o in outs])
    else:
        outs = [np.full(n, 77, np.uint8), np.full(n, 7.0), np.full((n, 2), 7.0), np.full(n, 77, np.int32), np.full(n, 7.0),
                np.full(n, 77, np.uint8), np.full((n, 4), 7.0), np.full(n, 77, np.int32)]
        rc = ctx.lib.svo_b200_find_epipolar_match_direct(*head, capi._p(d), capi._p(d_min), capi._p(d),
                                                         *[capi._p(o) for o in outs])
    return rc, outs


# ---- reprojector ---------------------------------------------------------------------------------------------------------
def _rp_cases():
    out = []
    c = synth.make_map_case(330, n_kfs=10, n_points=800)                        # more in-frame points than max_fts
    out.append(c)
    out.append(synth.make_map_case(331, n_kfs=1, n_points=150, n_candidates=10))
    out.append(synth.make_map_case(332, n_kfs=12, n_points=900, bad_frac=0.5))   # many failures: deletions
    e = synth.make_map_case(333, n_kfs=3, n_points=60, n_candidates=5)
    v = dict(e["view"]); v["kf_keypt_valid"] = np.zeros_like(v["kf_keypt_valid"]); v["n_candidates"] = 0
    out.append(dict(e, view=v))                                                   # nothing to project
    cand = synth.make_map_case(334, n_kfs=3, n_points=100, n_candidates=120, bad_frac=0.5)
    v = dict(cand["view"]); v["kf_keypt_valid"] = np.zeros_like(v["kf_keypt_valid"])
    pf = np.array(cand["pt_n_failed"], copy=True); pf[100:] = 30                 # one failed match deletes a candidate
    out.append(dict(cand, view=v, pt_n_failed=pf))                               # only candidates
    g = synth.make_map_case(335, width=640, height=480)
    n_cells = int(np.ceil(640 / 60)) * int(np.ceil(480 / 60))
    out.append(dict(g, options=dict(g["options"], grid_size=60, max_search_level=0, max_n_kfs=2),
                    cell_order=np.random.default_rng(2).permutation(n_cells).astype(np.int32)))
    h = synth.make_map_case(336, n_kfs=4, n_points=300)
    out.append(dict(h, options=dict(h["options"], find_match_direct=0, max_fts=40)))
    a = synth.make_map_case(337, n_kfs=5, n_points=300, cam=synth.reference_param_camera("atan"))
    out.append(a)
    return out


def _rp_args(c, kfs, cur):
    return dict(view=c["view"], kf_frames=kfs, cur=cur, cur_T_f_w=c["cur_T_f_w"], cam=c["cam"], options=c["options"],
                cell_order=c["cell_order"], pt_type=c["pt_type"], pt_n_failed=c["pt_n_failed"], pt_n_succeeded=c["pt_n_succeeded"])


def _run_rp(ctx, cases, share=None, pool_cur=None):
    """pool_cur: key -> a FramePool frame to use as that key's current frame instead of a frame of its own."""
    frames, streams = [], []
    made = {}
    for j, c in enumerate(cases):
        key = share[j] if share else j
        if key not in made:
            kfs = [ctx.frame(p) for p in c["kf_pyr"]]
            cur = pool_cur[key] if pool_cur and key in pool_cur else ctx.frame(c["cur_pyr"])
            frames += kfs + ([] if pool_cur and key in pool_cur else [cur])
            made[key] = (kfs, cur)
        kfs, cur = made[key]
        streams.append(_rp_args(c, kfs, cur))
    singles = [ctx.reproject_map(**s) for s in streams]
    batched = ctx.reproject_map_streams(streams)
    assert len(singles) == len(batched)
    for s, (g, b) in enumerate(zip(singles, batched)):
        for k in RP_KEYS:
            if isinstance(g[k], np.ndarray):
                assert _same_bits(g[k], b[k]), (s, k)
            else:
                assert g[k] == b[k], (s, k)
    for f in frames:
        f.destroy()
    return batched


def test_reproject_streams_heterogeneous_equal_single_calls(ctx):
    cases = _rp_cases()
    batched = _run_rp(ctx, cases)
    act = np.concatenate([b["pt_action"] for b in batched])
    print("point actions across the batch:", {a: int((act == a).sum()) for a in range(4)})
    for a in range(4):                                                            # every SVO_B200_PT_* occurs
        assert (act == a).sum() > 0, a
    assert batched[3]["n_projected"] == 0 and batched[3]["n_new"] == 0
    assert batched[0]["n_matches"] == cases[0]["options"]["max_fts"] + 1        # the maxFts stop was reached


@pytest.mark.parametrize("S", [0, 1, 2, 33, 132, 257])
def test_reproject_streams_shapes(ctx, S):
    """S streams over three small maps whose frames the streams share; options and cell orders differ per stream."""
    base = [synth.make_map_case(340 + k, n_kfs=3, n_points=80, n_candidates=10, width=w, height=h)
            for k, (w, h) in enumerate([(752, 480), (640, 480), (644, 484)])]
    rng = np.random.default_rng(S)
    cases, share = [], []
    for s in range(S):
        c = base[s % 3]
        n_cells = int(np.ceil(c["cam"].width / 30)) * int(np.ceil(c["cam"].height / 30))
        cases.append(dict(c, options=dict(c["options"], max_fts=int(rng.integers(5, 60))),
                          cell_order=rng.permutation(n_cells).astype(np.int32)))
        share.append(s % 3)
    pool = capi.FramePool(ctx, 752, 480, 5, 1)                                    # the 752x480 map's current frame
    pool.upload_array(base[0]["cur_pyr"][0][None])
    _run_rp(ctx, cases, share, pool_cur={0: pool.frames[0]})
    pool.destroy()


def test_reproject_streams_refusals_write_nothing(ctx):
    cases = _rp_cases()[:2]
    kfs = [[ctx.frame(p) for p in c["kf_pyr"]] for c in cases]
    curs = [ctx.frame(c["cur_pyr"]) for c in cases]
    bads = []
    v = dict(cases[1]["view"]); v["pt_obs"] = np.full_like(v["pt_obs"], 10 ** 6); bads.append(dict(view=v))   # index out of range
    v = dict(cases[1]["view"]); v["ftr_kf"] = np.full_like(v["ftr_kf"], 5); bads.append(dict(view=v))        # keyframe index
    bads.append(dict(cell_order=np.full_like(cases[1]["cell_order"], -1)))
    bads.append(dict(options=dict(cases[1]["options"], max_search_level=9)))
    bads.append(dict(cur=None))
    bads.append(dict(cam=dataclasses.replace(cases[1]["cam"], model=7)))                                    # unknown camera model
    # offset tables whose last entry is in range but whose interior is not: a point's observation range reaching past
    # pt_obs (then decreasing), and a negative first keyframe-feature offset
    v = dict(cases[1]["view"]); v["pt_obs_offset"] = v["pt_obs_offset"].copy(); v["pt_obs_offset"][1] = v["pt_obs_offset"][-1] + 1000
    bads.append(dict(view=v))
    v = dict(cases[1]["view"]); v["kf_fts_offset"] = v["kf_fts_offset"].copy(); v["kf_fts_offset"][0] = -3; bads.append(dict(view=v))
    bads += [dict(cam=_resized(cases[1]["cam"], dw, dh)) for dw, dh in SIZE_OFFSETS]                       # camera size != frames'
    # a single reproject_map call refused at the camera or cell-order check has already cleared its stats and actions
    clears_single = (False, False, True, False, False, True, False, False) + (False,) * len(SIZE_OFFSETS)
    for j, over in enumerate(bads):
        preps = []
        for i, c in enumerate(cases):
            a = _rp_args(c, kfs[i], curs[i])
            if i == 1:
                a.update(over)
            if a["cur"] is None:
                a["cur"] = type("NullFrame", (), {"h": C.c_void_p(None)})()
            preps.append(capi._reproject_prepare(**a))
        for _, o, st, _ in preps:
            for k in o:
                o[k][...] = 7 if o[k].dtype != np.uint8 else 77
            st.n_matches = st.n_trials = 99
        snap = [{k: v.copy() for k, v in o.items()} for _, o, _, _ in preps]
        arr = (capi.ReprojectStream * 2)(*[p[0] for p in preps])
        n0 = ctx.launch_count()
        assert ctx.lib.svo_b200_reproject_map_streams(ctx.h, 2, arr) == -1, j
        assert ctx.launch_count() == n0, j
        for (_, o, st, _), sn in zip(preps, snap):
            assert st.n_matches == 99 and st.n_trials == 99, j
            for k in o:
                assert _same_bits(o[k], sn[k]), (j, k)
        rs, o, st, _ = preps[1]
        st.n_new = st.n_overlap = st.n_projected = st.n_speculative = 99
        n0 = ctx.launch_count()
        assert ctx.lib.svo_b200_reproject_map(ctx.h, *[C.c_void_p(getattr(rs, f)) for f, _ in capi.ReprojectStream._fields_]) == -1, j
        assert ctx.launch_count() == n0, j
        stats = [getattr(st, f) for f, _ in capi.ReprojectStats._fields_]
        assert stats == ([0] * 6 if clears_single[j] else [99] * 6), (j, stats)
        for k in o:
            want = np.zeros_like(snap[1][k]) if k == "pt_action" and clears_single[j] else snap[1][k]   # SVO_B200_PT_NONE
            assert _same_bits(o[k], want), (j, k)
    assert ctx.lib.svo_b200_reproject_map_streams(ctx.h, -1, None) == -1
    assert ctx.lib.svo_b200_reproject_map_streams(ctx.h, 0, None) == 0
    for f in [f for k in kfs for f in k] + curs:
        f.destroy()
