"""The CUDA path at the limits of include/rayn_b200.h (16 hitables, 16 materials, 16 lights), at exact ties, on boundary
sample tables and against the closed form of many-light direct illumination.

Every per-object, per-light and per-SDF path of the kernels (the per-SDF work counters, slot_prefix rows, shadow-segment
queues and the owner packing with all 12 light-sample bits, 16 bins, the 8-bit light-index packing, the compact sphere table
and fold-all over 15 spheres, pass sizing with 180 shadow segments per path) runs here with every index it can take, bit for
bit against the oracle, through several passes, graph replay, the queue log and the fused mul_add build.  The scenes are
built by tests/limits_scenes.py; test_cpu_limits.py checks their oracle side."""
import numpy as np
import pytest

from rayn_b200 import _lib as L
from rayn_b200 import Emissive, Srgb
from rayn_b200.film import Renderer, tile_grid

import limits_scenes as S
import mirrors
from helpers import CH, assert_bit_equal, random_rays, small_config
from test_cpu_limits import FAMILIES, K_FRAMES, check_sphere_closest_hit, closed_form_films, sphere_rays

pytestmark = pytest.mark.gpu
TR = S.TR


def assert_film(g, o, what):
    for ch in CH:
        assert_bit_equal(g[ch], o[ch], f"{what} {ch}")


def gpu_render(r, world, cam, inp, integ, tile, **kw):
    r.upload_scene(world, cam)
    return r.render_host(inp, tile, integ, TR, **kw)


def oracle_render(oracle, world, cam, inp, integ, tile, **kw):
    """the trap oracle for worlds with orbit-trap albedos, the plain oracle otherwise"""
    if world.albedo_traps():
        return mirrors.render(world, cam, inp, tile, integ, TR, **kw)
    return oracle.render(world, cam, inp, tile, integ, TR, **kw)


def with_renderer(fn, **cfg):
    r = Renderer(0, **cfg)
    try:
        return fn(r)
    finally:
        r.close()


# (shape, volume, resolution, tile, samples): every shape with volume on (ns = 12) and off, at 32x24 and 40x40
SHAPE_CASES = [("A", True, (32, 24), (8, 8), 1), ("A", False, (40, 40), (16, 16), 2),
               ("B", True, (40, 40), (16, 16), 1), ("B", False, (32, 24), (8, 8), 2),
               ("B16", True, (32, 24), (16, 16), 1), ("B16", False, (40, 40), (8, 8), 1),
               ("C", True, (40, 40), (8, 8), 2), ("C", False, (32, 24), (16, 16), 1)]
IDS = [f"{s}-vol{int(v)}-{r[0]}x{r[1]}-t{t[0]}" for s, v, r, t, _ in SHAPE_CASES]


def _case(case, traps=False):
    shape, volume, res, tile, samples = case
    cam, world = S.SHAPES[shape](res, volume, traps=traps) if traps else S.SHAPES[shape](res, volume)
    integ, inp = S.inputs(res, samples, 3)
    return cam, world, integ, inp, tile


@pytest.mark.parametrize("case", SHAPE_CASES, ids=IDS)
def test_limit_shapes_bit_exact(renderer, oracle, case):
    cam, world, integ, inp, tile = _case(case)
    g = gpu_render(renderer, world, cam, inp, integ, tile)
    st = renderer.stats()
    o, info = oracle.render(world, cam, inp, tile, integ, TR)
    assert_film(g, o, str(case))
    assert st.extend_rays == info["extend_rays"] and st.shade_lanes == info["shade_lanes"]
    assert float(o["color"].sum()) > 0 and float(o["alpha"].sum()) > 0
    if case[0] == "A":  # one Mandelbox (reference constants: the three-operation division) among static spheres: fold-all
        assert renderer.sdf_variant(8) == 4
    if case[0].startswith("B"):
        sky = case[0] == "B"
        got = {i: renderer.sdf_variant(i) for i, _ in S.b_kinds(sky)}
        for i, kind in S.b_kinds(sky):
            assert got[i] in S.B_VARIANTS[kind], (i, kind, got[i])
        v = set(got.values())
        assert {0, 3} <= v and v & {1, 4} and v & {2, 5}, v  # generic, Mandelbulb, 12-iteration and N-iteration Mandelboxes


def test_shape_a_without_fold_all(oracle):
    """[spheres] Mandelbox [spheres] folds all 15 spheres into the producing kernel by default; RAYN_FLAG_NO_FOLD_ALL keeps
    the insertion-order fold.  Both give the oracle's film."""
    for case in SHAPE_CASES[:2]:
        cam, world, integ, inp, tile = _case(case)
        o, _ = oracle.render(world, cam, inp, tile, integ, TR)
        g, v = with_renderer(lambda r: (gpu_render(r, world, cam, inp, integ, tile), r.sdf_variant(8)), flags=L.FLAG_NO_FOLD_ALL)
        assert v == 4
        assert_film(g, o, f"no fold-all {case}")


@pytest.mark.parametrize("case", [SHAPE_CASES[0], SHAPE_CASES[2], SHAPE_CASES[4], SHAPE_CASES[6]], ids=["A", "B", "B16", "C"])
def test_limit_shapes_in_several_passes(oracle, case):
    cam, world, integ, inp, tile = _case(case)
    o, _ = oracle.render(world, cam, inp, tile, integ, TR)
    ntx, nty = tile_grid(inp.width, inp.height, *tile)
    per_tile = tile[0] * tile[1] * inp.spp

    def run(r):
        g = gpu_render(r, world, cam, inp, integ, tile)
        return g, r.stats().passes
    g, passes = with_renderer(run, max_paths_per_pass=per_tile * max(1, ntx * nty // 3))
    assert passes >= 3
    assert_film(g, o, f"multi-pass {case}")


@pytest.mark.parametrize("case", [SHAPE_CASES[0], SHAPE_CASES[2], SHAPE_CASES[6]], ids=["A", "B", "C"])
def test_limit_shapes_graph_replay_and_direct_launches(oracle, case):
    """two frames with default flags, each run as one CUDA-graph launch (reserved_ == 1 marks a frame that was captured or
    replayed: the stats do not say which), and every kernel launched directly (RAYN_FLAG_NO_GRAPH)"""
    cam, world, integ, inp, tile = _case(case)
    o, _ = oracle.render(world, cam, inp, tile, integ, TR)

    def twice(r):
        out = []
        for _ in range(2):
            out.append((gpu_render(r, world, cam, inp, integ, tile), r.stats().reserved_))
        return out
    for rep, (g, graph) in enumerate(with_renderer(twice)):
        assert graph == 1, f"frame {rep} did not run as one graph launch"
        assert_film(g, o, f"graph frame {rep} {case}")
    g, graph = with_renderer(twice, flags=L.FLAG_NO_GRAPH)[0]
    assert graph == 0
    assert_film(g, o, f"direct {case}")


def _parse_queue_log(log):
    out, i = {}, 0
    while i < len(log):
        depth, tile, ns = log[i:i + 3]
        out[(int(depth), int(tile))] = log[i + 3:i + 3 + ns].copy()
        i += 3 + ns
    return {k: v for k, v in out.items() if len(v)}


@pytest.mark.parametrize("case", [SHAPE_CASES[0], SHAPE_CASES[3], SHAPE_CASES[4], SHAPE_CASES[6]], ids=["A", "B", "B16", "C"])
def test_limit_shapes_queue_log(oracle, case):
    """the shading queue, slot for slot, per depth and tile: 16 bins, each padded to a multiple of 4"""
    cam, world, integ, inp, tile = _case(case)

    def run(r):
        r.upload_scene(world, cam)
        r.enable_queue_log(True)
        r.render_host(inp, tile, integ, TR)
        return r.read_queue_log()
    g = _parse_queue_log(with_renderer(run))
    _, info = oracle.render(world, cam, inp, tile, integ, TR, n_threads=1, queue_log=True)
    o = _parse_queue_log(info["queue_log"])
    assert set(g) == set(o)
    for k in o:
        assert np.array_equal(g[k], o[k]), f"shading queue differs at depth/tile {k}"
    assert any((v < 0).any() for v in o.values())


@pytest.mark.parametrize("shape", ["A", "B"])
def test_orbit_traps_on_every_trappable_material(renderer, oracle, shape):
    """shape D: every Lambertian and Dielectric material (material 15 included) has an orbit-trap albedo, against the trap
    oracle; the first-hit albedo plane against its mirror"""
    case = SHAPE_CASES[0] if shape == "A" else SHAPE_CASES[2]
    cam, world, integ, inp, tile = _case(case, traps=True)
    traps = world.albedo_traps()
    assert [t.material for t in traps] == S.TRAPPABLE and max(S.TRAPPABLE) == S.N - 1
    g = gpu_render(renderer, world, cam, inp, integ, tile)
    o, _ = oracle_render(oracle, world, cam, inp, integ, tile)
    assert_film(g, o, f"traps {shape}")
    plain, _ = oracle.render(world, cam, inp, tile, integ, TR)
    assert not np.array_equal(o["color"], plain["color"])

    def albedo(r):
        r.upload_scene(world, cam)
        return r.render_albedo(inp, tile, integ, TR)
    want = mirrors.render_albedo(world, cam, inp, tile, integ, TR)[0]
    for flags in (0, L.FLAG_NO_FOLD_ALL):
        assert_bit_equal(with_renderer(albedo, flags=flags), want, f"albedo {shape} flags {flags}")


def test_full_size_many_sdfs_several_passes_sampled_tiles(oracle):
    """shape B (15 SDFs, volume on: 180 shadow segments per path and depth) at 1920x1080 and 8 spp, with the pass sized by
    free device memory alone: more than one pass.  Six sampled tiles agree with the oracle."""
    res = (1920, 1080)
    cam, world = S.shape_b(res, True)
    integ, inp = S.inputs(res, 2, 3)
    ntx, nty = tile_grid(*res, 16, 16)
    tiles = sorted({int(fx * ntx) * nty + int(fy * nty) for fx, fy in ((0.5, 0.5), (0.4, 0.55), (0.62, 0.45), (0.05, 0.9),
                                                                        (0.33, 0.37), (0.7, 0.62))})

    def run(r):
        g = gpu_render(r, world, cam, inp, integ, (16, 16))
        return g, r.stats()
    g, st = with_renderer(run)
    assert st.passes > 1 and st.paths == res[0] * res[1] * inp.spp
    o, info = oracle.render(world, cam, inp, (16, 16), integ, TR, tile_list=tiles)
    assert info["tiles"] == len(tiles)
    mask = np.zeros((res[1], res[0]), bool)
    for t in tiles:
        x0, y0 = (t // nty) * 16, (t % nty) * 16
        mask[y0:y0 + 16, x0:x0 + 16] = True
    m = mask.reshape(-1)
    for ch in CH:
        n = 1 if ch == "alpha" else 3
        assert_bit_equal(g[ch].reshape(-1, n)[m], o[ch].reshape(-1, n)[m], f"full-size shape B {ch}")
    assert np.isfinite(g["color"]).all() and g["alpha"].max() > 0


# ---- stage KATs on the limit scenes --------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", ["A", "B", "C"])
def test_stage_kats_at_the_limits(renderer, oracle, shape):
    cam, world = S.SHAPES[shape]((32, 24), True)
    desc, keep = world.flatten(cam)
    renderer.upload_scene_desc(desc)
    for depth in (0, 1, 3):
        o, d = random_rays(20_000, seed=40 + depth, spread=1.5)
        gt, gobj = renderer.kat_closest_hit(depth, o, d)
        rt, robj = oracle.kat_closest_hit(desc, depth, o, d)
        assert np.array_equal(gobj, robj), f"closest-hit object, depth {depth}"
        assert_bit_equal(gt, rt, f"closest-hit t, depth {depth}")
        assert len(np.unique(robj)) >= 8
    rng = np.random.default_rng(41)
    s = rng.uniform(-2.0, 2.0, size=(20_000, 3)).astype(np.float32)
    e = np.array([l.pos for l in world.lights], np.float32)[rng.integers(0, S.N, 20_000)]
    g = renderer.kat_occluded(s, e)
    r = oracle.kat_occluded(desc, s, e)
    assert_bit_equal(g, r, "occluded")
    assert 0.02 < r.mean() < 0.98


def test_closest_hit_of_16_spheres_matches_float64_roots(renderer):
    cam, world = S.spheres_only()
    desc, _ = world.flatten(cam)
    renderer.upload_scene_desc(desc)
    o, d = sphere_rays()
    t, obj = renderer.kat_closest_hit(0, o, d)
    check_sphere_closest_hit(t, obj, world, o, d)


# ---- exact ties -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["spheres_before", "spheres_after", "spheres_across", "boxes_adjacent", "boxes_separated"])
@pytest.mark.parametrize("flags", [0, L.FLAG_NO_FOLD_ALL])
def test_first_copy_wins_exact_ties(oracle, kind, flags):
    """two identical hitables: the first index owns every hit (hitable.rs:170-210, `<` in the fold), so the later copy's
    material never shows - the film equals the oracle's and a render with that material changed"""
    integ, inp = S.inputs((32, 32), 1, 3)
    cam, world, later = S.tie_scene(kind, (32, 32))
    cam2, world2, _ = S.tie_scene(kind, (32, 32), second_material=Emissive.new_splat(Srgb(9.0, 0.1, 0.1)))
    o, _ = oracle.render(world, cam, inp, (16, 16), integ, TR)

    def run(r):
        return gpu_render(r, world, cam, inp, integ, (16, 16)), gpu_render(r, world2, cam2, inp, integ, (16, 16))
    g, g2 = with_renderer(run, flags=flags)
    assert_film(g, o, f"tie {kind}")
    assert_film(g2, g, f"tie {kind}, later copy re-materialed")


def test_sphere_on_a_light_and_duplicate_lights(renderer, oracle):
    integ, inp = S.inputs((32, 32), 2, 3)
    cam, world = S.light_tie_scene((32, 32))
    assert len(world.lights) == 10
    g = gpu_render(renderer, world, cam, inp, integ, (16, 16))
    o, _ = oracle.render(world, cam, inp, (16, 16), integ, TR)
    assert_film(g, o, "light ties")


# ---- boundary sample tables -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 3, 4])
@pytest.mark.parametrize("scramble", [None, 0.0, S.ONE_MINUS], ids=["rng", "zero", "one_minus"])
def test_boundary_tables_configs(renderer, oracle, n, scramble):
    c, inp = small_config(n, (32, 32), 2, 4)
    S.boundary_tables(inp, S.boundary_values(c["world"].materials.items), 10 + n, scramble=scramble)
    g = gpu_render(renderer, c["world"], c["camera"], inp, c["integrator"], (16, 16))
    o, _ = oracle.render(c["world"], c["camera"], inp, (16, 16), c["integrator"], TR)
    assert_film(g, o, f"cfg{n} boundary tables, scramble {scramble}")


@pytest.mark.parametrize("shape", ["A", "B"])
@pytest.mark.parametrize("scramble", [None, 0.0, S.ONE_MINUS], ids=["rng", "zero", "one_minus"])
def test_boundary_tables_limit_shapes(renderer, oracle, shape, scramble):
    cam, world = S.SHAPES[shape]((32, 24), True)
    integ, inp = S.inputs((32, 24), 1, 3)
    S.boundary_tables(inp, S.boundary_values(world.materials.items), 30, scramble=scramble)
    g = gpu_render(renderer, world, cam, inp, integ, (8, 8))
    o, _ = oracle.render(world, cam, inp, (8, 8), integ, TR)
    assert_film(g, o, f"shape {shape} boundary tables, scramble {scramble}")


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("scramble", S.EXTREME_TABLE_VALUES, ids=["zero", "one_minus"])
def test_one_dimension_family_at_its_extremes(renderer, oracle, family, scramble):
    """one family of sample dimensions reads only 0 and 1 - 2^-24 (a constant scramble plane, so that fract(table +
    scramble) is exactly that; test_cpu_limits.py checks the reads), the others read their R_d values: config 4 (thin lens,
    volume, roulette at depth 3) and shape A (16 lights)"""
    c, inp = small_config(4, (32, 32), 2, 4)
    cam, world = S.shape_a((32, 24), True)
    integ, inp_a = S.inputs((32, 24), 1, 4)
    for what, w, cm, ig, ip in (("cfg4", c["world"], c["camera"], c["integrator"], inp), ("A", world, cam, integ, inp_a)):
        S.extreme_family_tables(ip, family, ig, scramble, 20)
        g = gpu_render(renderer, w, cm, ip, ig, (16, 16))
        o, _ = oracle.render(w, cm, ip, (16, 16), ig, TR)
        assert_film(g, o, f"{what} family {family} scramble {scramble}")


# ---- many-light direct illumination against its closed form ---------------------------------------------------------------
def test_many_light_direct_illumination_matches_closed_form(renderer):
    """16 lights, NEE only (max_bounces 0, no sky sphere, the lit sphere fills the view): the device's K-frame mean lies
    within 5 standard errors of (albedo / pi) sum_j pi L_j (r_j / d_j)^2 cos(theta_j) in every pixel, and the film-wide mean
    within 3.  The only check here that does not lean on the oracle: a wrong light index, a wrong n / 4 correction or a
    mis-shuffled light choice shifts the mean."""
    def render(world, cam, inp, integ):
        return gpu_render(renderer, world, cam, inp, integ, (8, 8))
    films, expected = closed_form_films(render)
    assert len(films) == K_FRAMES and all(np.isfinite(f).all() and (f > 0).all() for f in films)
    z_px, z_all = S.closed_form_check(films, expected)
    assert z_px < 5 and z_all < 3, (z_px, z_all)


# ---- the fused mul_add build ----------------------------------------------------------------------------------------------
@pytest.mark.skipif(L.MULADD_FUSED or L.LEGACY, reason="already inside a variant run")
def test_fused_mul_add_variant_passes_the_limit_tests():
    """the limit, tie and boundary-table tests again with librayn_b200_fma.so against the fused oracle"""
    from test_gpu_parity import _run_suite_variant
    out = _run_suite_variant({"RAYN_MULADD_FUSED": "1"}, ["tests/test_gpu_limits.py", "-k", "not full_size and not variant"])
    assert " passed" in out
