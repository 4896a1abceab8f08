"""The host scheduler of rayn_b200/csrc/api.cu (pass sizing, the pass loop, graph capture and replay, moment planes, the
albedo and motion passes, an accumulator round) against RaynStats recorded from an earlier build:
tests/golden/host_driver_stats.json, written by tests/golden/make_golden_stats.py.  Every case fixes max_paths_per_pass, so
its pass size does not depend on the GPU's free memory; a change of pass sizing or of the launch sequence shows as a
different pass or launch count."""
import json
import os

import pytest

from rayn_b200 import _lib as L
from rayn_b200 import configs
from rayn_b200.film import Renderer, make_frame_desc
from rayn_b200.scene import OrbitTrapAlbedo

from helpers import small_config
from test_cpu_trap import ALBEDO_HI, ALBEDO_LO, TRAP_HI, TRAP_LO, with_fractal_albedo

pytestmark = pytest.mark.gpu
TR = configs.frame_time_range(1)
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "host_driver_stats.json")
STRUCTURE = ("passes", "launches", "kernel_launches", "paths", "reserved_")
# recorded only where two runs of the recording build agree (tests/golden/make_golden_stats.py)
COUNTERS = ("extend_rays", "shade_lanes", "shadow_rays", "sdf_evals_extend", "sdf_evals_shadow", "sdf_evals_normals", "bulb_iters_extend",
            "bulb_iters_shadow", "march_trips_extend", "march_trips_shadow")
RES, TILE = (40, 36), (8, 8)  # 5 x 5 tiles (the last row partly outside the film)
MAX_PATHS = 2000  # 7 tiles of 8 x 8 pixels at 4 spp per pass: 4 passes


def stats_fields(r):
    s = r.stats()
    return {k: list(getattr(s, k)) if k == "kernel_launches" else int(getattr(s, k)) for k in STRUCTURE + COUNTERS}


def frame_for(inp, integrator):
    ptrs = tuple(a.ctypes.data for a in inp.arrays())
    return make_frame_desc(inp.width, inp.height, TILE, inp.samples, integrator, inp.frame, TR, ptrs, L.MEM_HOST,
                           sets=(inp.sets_1d, inp.sets_2d))


def trap_config(n):
    c, inp = small_config(n, RES, 1, 3)
    return with_fractal_albedo(c, OrbitTrapAlbedo(TRAP_LO, TRAP_HI, ALBEDO_LO, ALBEDO_HI)), inp


def with_renderer(max_paths, c, run):
    """run(renderer) on a fresh context with the scene of config c uploaded; returns the stats after each of its calls"""
    r = Renderer(0, max_paths_per_pass=max_paths)
    try:
        r.upload_scene(c["world"], c["camera"])
        return run(r)
    finally:
        r.close()


def render_case(c, inp, max_paths=MAX_PATHS, renders=1, moments=False):
    def run(r):
        out = []
        for _ in range(renders):
            r.render_host(inp, TILE, c["integrator"], TR, moments=moments)
            out.append(stats_fields(r))
        return out
    return with_renderer(max_paths, c, run)


def albedo_case():
    c, inp = trap_config(3)

    def run(r):
        r.render_albedo(inp, TILE, c["integrator"], TR)
        return [stats_fields(r)]
    return with_renderer(MAX_PATHS, c, run)


def motion_case(albedo=False, prev=False):
    """render_motion, or with prev render_motion_prev against the uploaded scene's own description"""
    c, inp = trap_config(3)

    def run(r):
        desc = r.upload_scene(c["world"], c["camera"]) if prev else None
        r.render_motion(inp, TILE, c["integrator"], TR, 0.5, albedo=albedo, prev=None if desc is None else desc[0])
        return [stats_fields(r)]
    return with_renderer(MAX_PATHS, c, run)


def accum_case():
    c, inp = small_config(4, RES, 1, 3)

    def run(r):
        acc = r.accum_create(RES[0], RES[1], TILE)
        try:
            r.accum_round(acc, frame_for(inp, c["integrator"]), 2, 4, -1.0)
        finally:
            acc.close()
        return [stats_fields(r)]
    return with_renderer(MAX_PATHS, c, run)


# case name -> () -> the stats after each call of the case
CASES = {
    **{f"render_cfg{n}": (lambda n=n: render_case(*small_config(n, RES, 1, 3))) for n in (1, 2, 3, 4)},
    "render_cfg3_trap_fold_all": lambda: render_case(*trap_config(3)),
    # a small single-pass frame: the first render captures the pass as a graph, the second replays it
    "render_cfg3_graph_replay": lambda: render_case(*small_config(3, (33, 27), 1, 3), max_paths=1 << 20, renders=2),
    "render_moments_cfg3": lambda: render_case(*small_config(3, RES, 1, 3), moments=True),
    "render_moments_cfg3_graph_replay": lambda: render_case(*small_config(3, (33, 27), 1, 3), max_paths=1 << 20, renders=2, moments=True),
    "render_albedo_cfg3_trap": albedo_case,
    "render_motion_cfg3_trap": motion_case,
    "render_motion_albedo_cfg3_trap": lambda: motion_case(albedo=True),
    "render_motion_prev_cfg3_trap": lambda: motion_case(prev=True),
    "render_motion_prev_albedo_cfg3_trap": lambda: motion_case(albedo=True, prev=True),
    "accum_round_cfg4": accum_case,
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_stats_equal_recorded(case):
    with open(GOLDEN) as fh:
        recorded = json.load(fh).get(L.LIB_NAME)
    if recorded is None:
        pytest.skip(f"no stats recorded for {L.LIB_NAME}")
    got, want = CASES[case](), recorded[case]
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        assert set(STRUCTURE) <= set(w), f"{case}: the fixture lacks structural fields"
        for k, v in w.items():
            assert g[k] == v, f"{case}, call {i}: {k} = {g[k]}, recorded {v}"
    if case.endswith("graph_replay"):
        assert [g["reserved_"] for g in got] == [1, 1] and got[0]["passes"] == 1
    else:
        assert all(g["passes"] > 1 for g in got)
