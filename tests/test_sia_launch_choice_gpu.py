"""GPU: the alignment kernel's launch choice, pinned field by field.

Every field of svo_b200_sia_last_launch -- the instantiation, its shared memory and staging region, the resident clusters
and the staging mode of every level -- over the configurations of test_sia_geometry_gpu.GEOMETRIES, feature counts at the
capacity edges of every geometry, batch sizes around the occupancy and SM-count thresholds, one and five pyramid levels,
the plain-pinhole and a general camera, and the residual pass, against a recording (tests/golden/sia_launch_choice.npz).
The other alignment tests check what each geometry computes; this one checks that the host keeps choosing and sizing the
same geometry for the same request.

The choice depends on a batch only through its size and its largest feature count, so the first pair of a batch carries
the N features and the others none.  Launch failures are part of the recording (their messages).  The recording keeps the
SM count of the device it was made on; on a device with another count the test is skipped.  Record with

    python -m tests.test_sia_launch_choice_gpu tests/golden/sia_launch_choice.npz
"""
import os
import sys

import numpy as np
import pytest

from rpg_svo_b200 import capi, synth
from tests import sia_cases as sc
from tests.test_sia_geometry_gpu import GEOMETRIES

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sia_launch_choice.npz")
N_FEAT = [0, 1, 96, 97, 159, 160, 192, 193, 304, 305, 320, 321, 384, 385, 512, 513, 768, 769, 1024]
BATCH = [1, 30, 31, 33, 264, 265, 3168]
LEVELS = [1, 5]  # the alignment runs levels 0 .. n - 1, the residual pass level n - 1
CAMERAS = ["pinhole", "atan"]
GRID = ["config", "camera", "levels", "B", "N", "residuals"]
FIELDS = [name for name, _ in capi.SiaLaunch._fields_ if name != "level_stage"] + \
         [f"level_stage[{lv}]" for lv in range(capi.MAX_LEVELS)]
STAGE_CODE = {name: code for code, name in capi.SIA_STAGE_NAMES.items()}


def _report(ctx):
    L = ctx.sia_last_launch()
    return [L[f] for f in FIELDS[:-capi.MAX_LEVELS]] + [STAGE_CODE[L["stages"].get(lv)] for lv in range(capi.MAX_LEVELS)]


def _align(ctx, d, ref, cur, n_lvl, B, N):
    off = np.full(B + 1, N, np.int32)
    off[0] = 0
    ctx.sia_batch_stage([ref] * B, [cur] * B, d["cam"], np.tile(synth.se3_identity(), (B, 1, 1)), off, d["px"][:N],
                        d["f"][:N], d["pos"][:N], d["has_point"][:N], np.tile(d["ref_pos"], (B, 1)), n_lvl - 1, 0, n_iter=1)
    ctx.sia_batch_run()
    ctx.sia_batch_fetch()


def _residuals(ctx, d, ref, cur, n_lvl, N):
    ctx.sparse_residuals(ref, cur, d["cam"], n_lvl - 1, synth.se3_identity(), d["px"][:N], d["f"][:N], d["pos"][:N],
                         d["has_point"][:N], d["ref_pos"])


def sweep():
    """The grid (GRID columns), the launch reports (FIELDS columns, zero where the call failed) and the error messages, in a
    fresh context: the resident-cluster figure it reports is cached per context."""
    ctx = capi.Context(0)
    pairs = {"pinhole": sc.base_pair(),
             "atan": synth.make_frame_pair(1000, width=752, height=480, n_feat=1100, n_levels=5,
                                           cam=synth.reference_param_camera("atan"))}
    frames = {k: (ctx.frame(d["ref_pyr"]), ctx.frame(d["cur_pyr"])) for k, d in pairs.items()}
    grid, rows, errors = [], [], []

    def run(key, call):
        grid.append(key)
        try:
            call()
        except capi.SvoB200Error as e:
            rows.append([0] * len(FIELDS))
            errors.append(str(e))
            return
        rows.append(_report(ctx))
        errors.append("")

    try:
        for ci, cfg in enumerate(GEOMETRIES.values()):
            ctx.sia_config(cfg[0], cfg[1])
            ctx.sia_upfront(cfg[2])
            for ki, kind in enumerate(CAMERAS):
                d, (ref, cur) = pairs[kind], frames[kind]
                for n_lvl in LEVELS:
                    for N in N_FEAT:
                        for B in BATCH:
                            run((ci, ki, n_lvl, B, N, 0), lambda: _align(ctx, d, ref, cur, n_lvl, B, N))
                        run((ci, ki, n_lvl, 1, N, 1), lambda: _residuals(ctx, d, ref, cur, n_lvl, N))
    finally:
        for r, c in frames.values():
            r.destroy(); c.destroy()
        ctx.close()
    return np.array(grid, np.int32), np.array(rows, np.int32), np.array(errors)


def _sm_count(rows):
    return int(rows[:, FIELDS.index("sm_count")].max())  # (failed launches report 0)


def test_launch_choice_is_the_recorded_one():
    with np.load(GOLDEN, allow_pickle=False) as z:
        want = {k: z[k] for k in z.files}
    assert list(want["grid_columns"]) == GRID and list(want["fields"]) == FIELDS
    grid, rows, errors = sweep()
    if _sm_count(rows) != int(want["sm_count"]):
        pytest.skip(f"recorded on a device with {int(want['sm_count'])} SMs, this one has {_sm_count(rows)}")
    assert np.array_equal(grid, want["grid"]), "the swept grid differs from the recorded one"
    bad = [i for i in range(len(grid)) if not np.array_equal(rows[i], want["launch"][i]) or errors[i] != want["error"][i]]
    detail = [(dict(zip(GRID, grid[i].tolist())),
               {f: (int(g), int(w)) for f, g, w in zip(FIELDS, rows[i], want["launch"][i]) if g != w},
               (errors[i], str(want["error"][i]))) for i in bad[:5]]
    assert not bad, f"{len(bad)} of {len(grid)} launches differ, e.g. {detail}"


if __name__ == "__main__":
    grid, rows, errors = sweep()
    np.savez_compressed(sys.argv[1], grid=grid, launch=rows, error=errors, grid_columns=np.array(GRID),
                        fields=np.array(FIELDS), sm_count=np.array(_sm_count(rows)))
    print(f"{len(grid)} launches ({int((errors != '').sum())} failed) recorded in {sys.argv[1]}")
