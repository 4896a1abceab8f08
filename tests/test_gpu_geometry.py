"""The film resolve and the tile-level kernels at launch geometries the other suites do not reach: tiles of 1x1 to 64x64 and
larger than the image, 16384 spp, 254 bounces, a job of 65536 tiles, and both sides of every render limit at RaynFrameDesc.

k_resolve is checked on its own through rayn_b200_kat_resolve against the numpy statement in tests/resolve_ref.py, bit for
bit, for both instances: every significant key width of both sort orders (one to four radix passes), 1, 2, 5 and 8 warps per
CTA, and keys built to take each branch of the sort (skipped passes, uniform digits, ties, sortedness across 32-key chunks).
The plans the hook returns are the coverage record.  The renders are checked bit for bit against the oracle and the CPU
mirrors (films, moments, several passes, the albedo and motion planes, accumulator E and K)."""
import numpy as np
import pytest

from rayn_b200 import _lib as L
from rayn_b200 import CameraStore, HitableStore, Lambertian, MaterialStore, PathTracingIntegrator, PinholeCamera, Sky, Sphere
from rayn_b200 import SphereLight, Srgb, Vec3, VolumeParams, World, configs
from rayn_b200.film import FrameInputs, Renderer, make_frame_desc, tile_grid

import accum_mirror as am
import mirrors
import resolve_ref as rr
from helpers import CH, assert_bit_equal, bits, small_config

pytestmark = pytest.mark.gpu
TR = configs.frame_time_range(1)
DT = 1.0 / 24.0

# ---- k_resolve against the numpy statement ----------------------------------------------------------------------------
KAT = rr.kat_cases()
PLANS = {}  # (case id, moments) -> (np, wpc, slot_bits, depth_bits), as rayn_b200_kat_resolve returned it


def assert_resolved(got, want, what):
    """bit for bit (NaN payloads aside); the sentinel left wherever the reference writes nothing"""
    for k in want:
        g, w = np.asarray(got[k]), np.asarray(want[k])
        untouched = bits(w) == bits(np.full(1, rr.SENTINEL))
        assert (bits(g)[untouched] == bits(w)[untouched]).all(), f"{what} {k}: written outside the resolved tiles"
        assert_bit_equal(g, w, f"{what} {k}")


def kat(r, case, planes, moments=None):
    return r.kat_resolve(case["width"], case["height"], case["tile"], case["samples"], case["max_bounces"], case["n_hitables"], case["tile_ids"],
                         case["term"], case["nrm0"], case["rad"], planes, moments)


@pytest.mark.parametrize("i", range(len(KAT)), ids=[c for c, _ in KAT])
def test_resolve_matches_the_numpy_statement(renderer, i):
    cid, args = KAT[i]
    case = rr.make_case(seed=1000 + i, **args)
    w, h = case["width"], case["height"]
    want, want_m = rr.fresh_planes(w, h)
    rr.resolve(case, want, want_m)
    for mom in (False, True):
        got, got_m = rr.fresh_planes(w, h)
        plan = kat(renderer, case, got, got_m if mom else None)
        p = (plan.np, plan.wpc, plan.slot_bits, plan.depth_bits)
        assert p == rr.expected_plan(case, mom), (cid, mom, p)
        assert plan.smem_bytes <= 227 * 1024
        PLANS[(cid, mom)] = p
        assert_resolved(got, want, f"{cid} moments={mom}")
        if mom:
            assert_resolved({"color_lum2": got_m[0], "background_lum2": got_m[1]}, {"color_lum2": want_m[0], "background_lum2": want_m[1]}, cid)
        else:
            assert (bits(got_m) == bits(np.full(1, rr.SENTINEL))).all()


def test_resolve_cases_cover_every_sort_and_cta_shape():
    """after test_resolve_matches_the_numpy_statement: the plans the hook returned"""
    assert len(PLANS) == 2 * len(KAT), "every resolve case must have run in this session"
    colour = {p[2] + p[3] for p in PLANS.values()}
    normal = {p[2] + 1 for p in PLANS.values()}
    assert colour == set(range(6, 31)), sorted(colour)
    assert normal == set(range(6, 24)), sorted(normal)
    assert {rr.sort_plan(k) for k in colour} == {rr.sort_plan(k) for k in range(6, 31)}
    assert {rr.sort_plan(k)[0] for k in colour} == {1, 2, 3, 4}
    assert (3, 9) in {rr.sort_plan(k) for k in colour}
    for mom in (False, True):
        assert {p[1] for (c, m), p in PLANS.items() if m == mom} == {1, 2, 5, 8}, mom


def test_resolve_hook_applies_the_render_limits(renderer):
    one = np.zeros(4 * 16, np.float32)
    planes, _ = rr.fresh_planes(4, 4)
    # (tile, samples, max_bounces, n_hitables): the first value past each limit
    for tile, samples, mb, n_hit, what in [((1, 1), 4097, 0, 0, "16384 spp"), ((1, 1), 1, 255, 0, "max_bounces"),
                                           ((1, (1 << 20) - 2), 1, 0, 2, "2^22")]:
        with pytest.raises(L.RaynError) as e:
            renderer.kat_resolve(4, 4, tile, samples, mb, n_hit, [0], np.zeros(4, np.uint32), one, one, planes)
        assert e.value.code == L.RAYN_ERR_UNSUPPORTED, what
        assert what in str(e.value), str(e.value)
    with pytest.raises(L.RaynError) as e:
        renderer.kat_resolve(4, 4, (2, 2), 1, 0, 0, [4], np.zeros(16, np.uint32), one, one, planes)  # tile 4 of a 2 x 2 grid
    assert e.value.code == L.RAYN_ERR_INVALID_ARG


# ---- renders at the new tile shapes ------------------------------------------------------------------------------------
SHAPES = [(1, 1), (2, 2), (3, 5), (1, 16), (16, 1), (7, 7), (64, 64)]
# (config, resolution, samples, max_bounces, tile): config 1 at every shape, configs 3 and 4 at some; 64x64 is larger than
# every image here
SHAPE_CASES = [(1, (48, 40), 1, 2, t) for t in SHAPES] + [(3, (40, 36), 1, 3, t) for t in ((3, 5), (1, 16), (64, 64))] + \
              [(4, (40, 36), 1, 2, t) for t in ((16, 1), (7, 7), (2, 2))]


def assert_film(g, o, what, chans=CH):
    for ch in chans:
        assert_bit_equal(g[ch], o[ch], f"{what} {ch}")


@pytest.mark.parametrize("n,res,samples,mb,tile", SHAPE_CASES, ids=[f"cfg{c[0]}-{c[4][0]}x{c[4][1]}" for c in SHAPE_CASES])
def test_tile_shape_renders_equal_the_oracle_and_the_mirrors(oracle, n, res, samples, mb, tile):
    c, inp = small_config(n, res, samples, mb)
    integ, world, cam = c["integrator"], c["world"], c["camera"]
    ntx, nty = tile_grid(*res, *tile)
    assert ntx * nty >= 1
    o, _ = oracle.render(world, cam, inp, tile, integ, TR)
    om, _ = mirrors.render(world, cam, inp, tile, integ, TR, moments=True)
    r = Renderer(0)
    try:
        d, keep = r.upload_scene(world, cam)
        assert_film(r.render_host(inp, tile, integ, TR), o, f"{tile} frame")
        assert_film(r.render_host(inp, tile, integ, TR, moments=True), om, f"{tile} moments", CH + ("moments",))
        assert_bit_equal(r.render_albedo(inp, tile, integ, TR), mirrors.render_albedo(world, cam, inp, tile, integ, TR)[0], f"{tile} albedo")
        assert_bit_equal(r.render_motion(inp, tile, integ, TR, DT), mirrors.render_motion(d, inp, tile, integ, TR, DT)[0], f"{tile} motion")
    finally:
        r.close()
    # several passes: about a third of the tiles per pass
    R = tile[0] * tile[1] * inp.spp
    r = Renderer(0, max_paths_per_pass=max(1, (ntx * nty) // 3) * R)
    try:
        r.upload_scene(world, cam)
        assert_film(r.render_host(inp, tile, integ, TR), o, f"{tile} passes")
        assert r.stats().passes >= min(3, ntx * nty)
    finally:
        r.close()


def frame_for(inp, integrator, tile):
    ptrs = tuple(a.ctypes.data for a in inp.arrays())
    return make_frame_desc(inp.width, inp.height, tile, inp.samples, integrator, inp.frame, TR, ptrs, L.MEM_HOST, sets=(inp.sets_1d, inp.sets_2d))


@pytest.mark.parametrize("res,tile", [((100, 80), (64, 64)), ((96, 80), (40, 40))])
def test_accumulator_tiles_of_several_error_chunks(renderer, oracle, res, tile):
    """k_accum_fold sums a tile's errors in chunks of 1024 pixels: 64x64 (4 chunks) beside a clipped 36x64 tile (2304
    pixels: a partial last chunk), and 40x40 (1600 pixels)"""
    c, _ = small_config(1, res, 1, 2)
    integ = c["integrator"]
    renderer.upload_scene(c["world"], c["camera"])
    acc = renderer.accum_create(*res, tile)
    m = am.AccumMirror(*res, *tile)
    assert max(len(m.tile_pixels(t)) for t in range(m.n_tiles)) > 1024
    assert any(len(m.tile_pixels(t)) % 1024 for t in range(m.n_tiles))
    for rnd in range(3):
        inp = FrameInputs(*res, 1, integ, first_sample=4 * rnd)
        assert renderer.accum_round(acc, frame_for(inp, integ, tile), 2, 8, -1.0) == m.n_tiles
        o, _ = oracle.render(c["world"], c["camera"], inp, tile, integ, TR)
        m.fold(o, list(range(m.n_tiles)), 1)
        err, k = renderer.accum_tiles(acc)
        assert np.array_equal(k, m.K), f"round {rnd}: K"
        assert np.array_equal(err.view(np.uint64), m.E.view(np.uint64)), f"round {rnd}: E {err} vs {m.E}"
    assert_film(renderer.accum_resolve(acc), m.resolve(), "accumulated")


# ---- sample counts and depths --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mb", [2, 20])
def test_16384_spp_on_one_8x8_tile(oracle, mb):
    """np 16384: one warp per CTA; slot_bits 21, so max_bounces 20 gives 26-bit colour keys (three 9-bit radix passes)"""
    c, inp = small_config(1, (8, 8), 4096, mb)
    assert inp.spp == 16384
    r = Renderer(0)
    try:
        r.upload_scene(c["world"], c["camera"])
        o, _ = oracle.render(c["world"], c["camera"], inp, (8, 8), c["integrator"], TR)
        assert_film(r.render_host(inp, (8, 8), c["integrator"], TR), o, f"16384 spp, {mb} bounces")
        if mb == 2:
            om, _ = mirrors.render(c["world"], c["camera"], inp, (8, 8), c["integrator"], TR, moments=True)
            assert_film(r.render_host(inp, (8, 8), c["integrator"], TR, moments=True), om, "16384 spp moments", CH + ("moments",))
    finally:
        r.close()


def test_4000_spp_on_4x4_tiles(renderer, oracle):
    """np 4096: five warps per CTA, for both resolve instances"""
    c, inp = small_config(1, (8, 6), 1000, 2)
    renderer.upload_scene(c["world"], c["camera"])
    o, _ = oracle.render(c["world"], c["camera"], inp, (4, 4), c["integrator"], TR)
    assert_film(renderer.render_host(inp, (4, 4), c["integrator"], TR), o, "4000 spp")
    om, _ = mirrors.render(c["world"], c["camera"], inp, (4, 4), c["integrator"], TR, moments=True)
    assert_film(renderer.render_host(inp, (4, 4), c["integrator"], TR, moments=True), om, "4000 spp moments", CH + ("moments",))


def closed_scene(res):
    """the camera inside a closed white Lambertian box - six spheres of radius 1000 whose near faces bound the cube |x|, |y|,
    |z| <= 1 (sphere normals point outwards, so the box is made of the spheres' outsides) - with a light inside: paths stay
    alive for tens of bounces"""
    mats, hits = MaterialStore(), HitableStore()
    mats.add_material(Sky(Srgb(0.3, 0.4, 0.6), Srgb(0.2, 0.3, 0.6) * 0.05))
    white = mats.add_material(Lambertian(Srgb(0.95, 0.95, 0.95)))
    for axis in range(3):
        for sign in (-1.0, 1.0):
            c = [0.0, 0.0, 0.0]
            c[axis] = sign * 1001.0
            hits.push(Sphere(Vec3(*c), 1000.0, white))
    lights = [SphereLight(Vec3(0.3, 0.5, -0.4), 0.1, Srgb(1.0, 1.0, 1.0) * 20.0)]
    cams = CameraStore()
    cam = cams.add_camera(PinholeCamera(res, 70.0, Vec3(0.0, 0.0, 0.8), Vec3(0.0, 0.0, 0.0), Vec3(0.0, 1.0, 0.0)))
    return cam, World(hits, lights, mats, cams, VolumeParams(None, None))


def test_254_bounces_in_a_closed_scene(renderer, oracle):
    res, tile = (16, 16), (8, 8)
    cam, world = closed_scene(res)
    integ = PathTracingIntegrator(254, 2)
    inp = FrameInputs(*res, 1, integ)
    renderer.upload_scene(world, cam)
    o, _ = oracle.render(world, cam, inp, tile, integ, TR)
    assert_film(renderer.render_host(inp, tile, integ, TR), o, "254 bounces")
    om, _ = mirrors.render(world, cam, inp, tile, integ, TR, moments=True)
    assert_film(renderer.render_host(inp, tile, integ, TR, moments=True), om, "254 bounces moments", CH + ("moments",))
    # the renders reach deep: the shading lanes per depth, from the queue log, go well past depth 10
    renderer.enable_queue_log(True)
    try:
        renderer.render_host(inp, tile, integ, TR)
        log = renderer.read_queue_log()
    finally:
        renderer.enable_queue_log(False)
    depths, i = set(), 0
    while i < len(log):
        if log[i + 2] > 0:
            depths.add(int(log[i]))
        i += 3 + int(log[i + 2])
    assert max(depths) >= 20, max(depths)


# ---- the 65535-tile pass ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("flags", [L.FLAG_TIMING, 0], ids=["serial", "two-sets"])
def test_65536_one_pixel_tiles(oracle, flags):
    """256x256 with 1x1 tiles: more tiles than one launch's grid.y holds (65535), so two passes in either driver - 65535 + 1
    on one set (RAYN_FLAG_TIMING), 32768 + 32768 on two - and the one-CTA scans walk tens of thousands of tiles"""
    c, inp = small_config(1, (256, 256), 1, 2)
    o, _ = oracle.render(c["world"], c["camera"], inp, (1, 1), c["integrator"], TR)
    r = Renderer(0, flags=flags)
    try:
        r.upload_scene(c["world"], c["camera"])
        assert_film(r.render_host(inp, (1, 1), c["integrator"], TR), o, f"65536 tiles flags={flags}")
        assert r.stats().passes == 2
    finally:
        r.close()


# ---- both sides of every render limit --------------------------------------------------------------------------------
def test_largest_slot_key_space_renders(oracle):
    """tile_w*tile_h*spp + 4*n_hitables = 2^22 - 4: a 1 x (2^20 - n - 1) tile at 4 spp.  No bounces and no lights, since
    the oracle renders one tile on one thread."""
    n = 2
    h = (1 << 20) - n - 1
    c, inp = small_config(1, (1, h), 1, 0)
    world = c["world"]
    assert len(world.hitables.items) == n
    world.lights = []
    assert 4 * h + 4 * n == (1 << 22) - 4
    r = Renderer(0)
    try:
        r.upload_scene(world, c["camera"])
        g = r.render_host(inp, (1, h), c["integrator"], TR)
    finally:
        r.close()
    o, _ = oracle.render(world, c["camera"], inp, (1, h), c["integrator"], TR)
    assert_film(g, o, "2^22 - 4 slots")
    assert float(o["alpha"].sum()) > 0


def test_the_first_value_past_each_limit_is_refused(renderer):
    c, _ = small_config(1, (8, 8), 1, 0)
    renderer.upload_scene(c["world"], c["camera"])
    cases = [("16384 spp", FrameInputs(4, 4, 4097, c["integrator"]), (4, 4), c["integrator"]),
             ("max_bounces", FrameInputs(4, 4, 1, PathTracingIntegrator(255, 2)), (4, 4), PathTracingIntegrator(255, 2))]
    h = (1 << 20) - 2  # 4 * h + 4 * 2 = 2^22
    cases.append(("2^22", FrameInputs(1, h, 1, c["integrator"]), (1, h), c["integrator"]))
    for what, inp, tile, integ in cases:
        for moments in (False, True):
            with pytest.raises(L.RaynError) as e:
                renderer.render_host(inp, tile, integ, TR, moments=moments)
            assert e.value.code == L.RAYN_ERR_UNSUPPORTED, what
            assert what in str(e.value), str(e.value)
    # the context still renders
    ok = FrameInputs(8, 8, 1, c["integrator"])
    assert float(renderer.render_host(ok, (8, 8), c["integrator"], TR)["alpha"].sum()) > 0


@pytest.mark.skipif(L.MULADD_FUSED or L.LEGACY, reason="already inside a variant run")
def test_fused_mul_add_variant_passes_this_suite():
    from test_gpu_parity import _run_suite_variant
    assert " passed" in _run_suite_variant({"RAYN_MULADD_FUSED": "1"}, ["tests/test_gpu_geometry.py", "-k", "not variant"])
