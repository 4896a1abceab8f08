"""Motion against an explicit previous scene (rayn_b200_render_motion_prev, k_motion_paths_prev) on the device against its
CPU mirror (tests/render_mirror.cpp) bit for bit: configs 1, 3 and 4, orthographic and thin-lens cameras, an orbit, a cut and
a zoom, limits_scenes.shape_c (15 moving spheres) with displaced previous centres and changed velocities, several passes,
sampled tiles of a 1080p film, host and device planes, and the albedo plane of the same pass against render_albedo.  Also the
identity with render_motion, the argument errors, Film.render_sequence on a world with closure parameters against the explicit
Renderer pipeline, and exact zero motion for a static closure world uploaded every frame."""
import ctypes as C
import math

import numpy as np
import pytest

from rayn_b200 import _lib as L
from rayn_b200 import configs
from rayn_b200.film import FrameInputs, Renderer, make_frame_desc
from rayn_b200.scene import Linear, OrthographicCamera, PinholeCamera, Sphere, ThinLensCamera, Vec3

import limits_scenes as ls
import mirrors
from helpers import assert_bit_equal, small_config
from test_cpu_albedo import trap_config
from test_cpu_motion_prev import changed_kind, rot_y

pytestmark = pytest.mark.gpu
DT = 1.0 / 24.0
TR = configs.frame_time_range(1)
ORIGIN = np.array([-0.45, 0.2, 2.0]) * 2.25


def both(r, world, cam, prev_desc, inp, tile, integ, albedo=False):
    """(device plane [, albedo], mirror plane) against prev_desc; the uploaded scene is world with cam"""
    d, keep = r.upload_scene(world, cam, TR)
    g = r.render_motion(inp, tile, integ, TR, DT, albedo=albedo, prev=prev_desc)
    o = mirrors.render_motion(d, inp, tile, integ, TR, DT, prev=prev_desc)[0]
    return g, o


def cams(c, res):
    """pairs (current, previous) of camera handles: an orbit, a cut, a zoom, an orthographic pan and a thin lens"""
    k = c["world"].cameras
    add = k.add_camera
    o2 = rot_y(ORIGIN, -3.0)
    return {
        "orbit": (add(PinholeCamera(res, 60.0, Vec3(*ORIGIN), Vec3(0, 0, 0), Vec3(0, 1, 0))),
                  add(PinholeCamera(res, 60.0, Vec3(*o2), Vec3(0, 0, 0), Vec3(0, 1, 0)))),
        "cut": (add(PinholeCamera(res, 60.0, Vec3(*ORIGIN), Vec3(0, 0, 0), Vec3(0, 1, 0))),
                add(PinholeCamera(res, 40.0, Vec3(3.0, 4.5, -2.5), Vec3(0.5, 0.2, 0.0), Vec3(0, 1, 0)))),
        "zoom": (add(PinholeCamera(res, 45.0, Vec3(*ORIGIN), Vec3(0, 0, 0), Vec3(0, 1, 0))),
                 add(PinholeCamera(res, 60.0, Linear(Vec3(*ORIGIN), Vec3(0.2, 0.0, 0.0)), Vec3(0, 0, 0), Vec3(0, 1, 0)))),
        "ortho": (add(OrthographicCamera(res, 11.0 / 4.0, Vec3(9.5, -3.5, 9.5), Vec3(0.0, 0.8, 0.0), Vec3(0.0, 1.0, 0.0))),
                  add(OrthographicCamera(res, 3.0, Linear(Vec3(9.3, -3.5, 9.7), Vec3(1.0, 0.5, 0.0)), Vec3(-0.2, 0.8, 0.2), Vec3(0, 1, 0)))),
        "thinlens": (add(ThinLensCamera(res, 60.0, 0.05, Vec3(*ORIGIN), Vec3(0, 0, 0), Vec3(0, 1, 0), Vec3(0, 0, 0))),
                     add(ThinLensCamera(res, 60.0, 0.05, Vec3(*rot_y(ORIGIN, 2.0)), Vec3(0.1, 0, 0), Vec3(0, 1, 0), Vec3(0, 0, 0)))),
    }


@pytest.mark.parametrize("n", [1, 3, 4])
@pytest.mark.parametrize("tile", [(8, 8), (16, 16)])
def test_equals_mirror_and_render_albedo(renderer, n, tile):
    """the configs' own cameras against an orbited copy (config 4's thin lens), with the albedo plane of the same pass"""
    res = (37, 23)
    c, inp = trap_config(n, res, 2)
    cur = c["camera"]
    cd = c["world"].flatten(cur)[0].camera
    prev = c["world"].flatten(cur)
    prev[0].camera.origin[:] = rot_y(np.array(cd.origin[:], np.float64), 2.5).astype(np.float32).tolist()
    (g, a), o = both(renderer, c["world"], cur, prev[0], inp, tile, c["integrator"], albedo=True)
    assert_bit_equal(g, o, f"cfg{n} {tile}")
    assert (g[..., 0] != 0).any()
    assert_bit_equal(a, renderer.render_albedo(inp, tile, c["integrator"], TR), f"cfg{n} albedo")
    assert_bit_equal(renderer.render_motion(inp, tile, c["integrator"], TR, DT, prev=prev[0]), g, "without albedo")


@pytest.mark.parametrize("kind", ["orbit", "cut", "zoom", "ortho", "thinlens"])
def test_camera_pairs(renderer, kind):
    res = (48, 40)
    c, inp = small_config(3, res, 2, 1)
    cur, prv = cams(c, res)[kind]
    p = c["world"].flatten(prv, TR)
    g, o = both(renderer, c["world"], cur, p[0], inp, (16, 16), c["integrator"])
    assert_bit_equal(g, o, kind)
    assert (g[..., 0] != 0).any()


def shape_c_prev(world, cam):
    """shape C's previous scene: every small sphere displaced and with another velocity (the sky sphere unchanged)"""
    d, keep = world.flatten(cam, TR)
    hit = (L.RaynHitable * d.n_hitables)(*[d.hitables[i] for i in range(d.n_hitables)])
    rng = np.random.default_rng(11)
    for i in range(1, d.n_hitables):
        hit[i].center[:] = (np.array(hit[i].center[:], np.float32) + rng.uniform(-0.05, 0.05, 3).astype(np.float32)).tolist()
        hit[i].center_velocity[:] = (np.array(hit[i].center_velocity[:], np.float32) * np.float32(-0.5)
                                     + rng.uniform(-1, 1, 3).astype(np.float32)).tolist()
    p = L.RaynSceneDesc.from_buffer_copy(d)
    p.hitables = C.cast(hit, C.POINTER(L.RaynHitable))
    return p, (keep, hit)


def test_limits_shape_c_moving_spheres(renderer):
    cam, world = ls.shape_c((29, 21), False)
    integ, inp = ls.inputs((29, 21), 2, 1)
    p, keep = shape_c_prev(world, cam)
    g, o = both(renderer, world, cam, p, inp, (8, 8), integ)
    assert_bit_equal(g, o, "shape C")
    assert (g[..., 0] != 0).any()


def test_several_passes():
    res = (61, 45)
    c, inp = small_config(3, res, 2, 1)
    cur, prv = cams(c, res)["orbit"]
    p = c["world"].flatten(prv, TR)
    r = Renderer(0, max_paths_per_pass=8 * 8 * 8 * 3)
    try:
        g, o = both(r, c["world"], cur, p[0], inp, (8, 8), c["integrator"])
        assert r.stats().passes > 1
    finally:
        r.close()
    assert_bit_equal(g, o, "passes")


def test_full_size_cfg3_sampled_tiles(renderer):
    c, _ = small_config(3, (1920, 1080), 1, 1)
    inp = FrameInputs(1920, 1080, 1, c["integrator"])
    cur, prv = cams(c, (1920, 1080))["orbit"]
    d, keep = renderer.upload_scene(c["world"], cur, TR)
    p = c["world"].flatten(prv, TR)
    g = renderer.render_motion(inp, (16, 16), c["integrator"], TR, DT, prev=p[0])
    o = mirrors.render_motion(d, inp, (16, 16), c["integrator"], TR, DT, prev=p[0], subsample_k=97)[0]
    nty = (1080 + 1080 % 16) // 16
    for t in range(0, 120 * nty, 97):
        tx, ty = t // nty, t % nty
        sl = (slice(ty * 16, ty * 16 + 16), slice(tx * 16, tx * 16 + 16))
        assert_bit_equal(g[sl], o[sl], f"tile {t}")


def test_device_planes(renderer):
    torch = pytest.importorskip("torch")
    res = (27, 19)
    c, inp = small_config(3, res, 2, 1)
    cur, prv = cams(c, res)["orbit"]
    d, keep = renderer.upload_scene(c["world"], cur, TR)
    p = c["world"].flatten(prv, TR)
    ptrs = tuple(a.ctypes.data for a in inp.arrays())
    f = make_frame_desc(*res, (8, 8), inp.samples, c["integrator"], inp.frame, TR, ptrs, L.MEM_HOST, sets=(inp.sets_1d, inp.sets_2d))
    m = torch.full((19 * 27 * 4,), 7.0, device="cuda")
    a = torch.full((19 * 27 * 3,), 7.0, device="cuda")
    torch.cuda.synchronize()
    L.check(renderer._lib.rayn_b200_render_motion_prev(renderer.ctx, C.byref(f), DT, C.byref(p[0]), m.data_ptr(), a.data_ptr(), L.MEM_DEVICE),
            renderer.ctx)
    o = mirrors.render_motion(d, inp, (8, 8), c["integrator"], TR, DT, prev=p[0])[0]
    assert_bit_equal(m.cpu().numpy().reshape(19, 27, 4), o, "device motion")
    assert_bit_equal(a.cpu().numpy().reshape(19, 27, 3), renderer.render_albedo(inp, (8, 8), c["integrator"], TR), "device albedo")


@pytest.mark.parametrize("n", [1, 3, 4])
def test_identity_with_render_motion(renderer, n):
    """prev = the uploaded scene, no moving sphere (the camera may move linearly): render_motion's plane bit for bit"""
    from test_cpu_temporal import moving_cameras
    res = (29, 21)
    c, inp = trap_config(n, res, 2)
    handles = [c["camera"]] + (list(moving_cameras(c, res).values()) if n == 3 else [])
    for cam in handles:
        d, keep = renderer.upload_scene(c["world"], cam, TR)
        a, aa = renderer.render_motion(inp, (8, 8), c["integrator"], TR, DT, albedo=True)
        b, ab = renderer.render_motion(inp, (8, 8), c["integrator"], TR, DT, albedo=True, prev=d)
        assert_bit_equal(b, a, f"cfg{n} motion")
        assert_bit_equal(ab, aa, f"cfg{n} albedo")


def test_argument_errors(renderer):
    c, inp = small_config(3, (16, 16), 1, 1)
    d, keep = renderer.upload_scene(c["world"], c["camera"], TR)
    ptrs = tuple(a.ctypes.data for a in inp.arrays())
    f = make_frame_desc(16, 16, (8, 8), inp.samples, c["integrator"], inp.frame, TR, ptrs, L.MEM_HOST, sets=(inp.sets_1d, inp.sets_2d))
    out = np.zeros(4 * 16 * 16, np.float32)
    lib = renderer._lib

    def call(prev, dt=DT):
        return lib.rayn_b200_render_motion_prev(renderer.ctx, C.byref(f), dt, prev, out.ctypes.data, None, L.MEM_HOST)
    ortho = c["world"].cameras.add_camera(OrthographicCamera((16, 16), 2.0, Vec3(9.5, -3.5, 9.5), Vec3(0, 0, 0), Vec3(0, 1, 0)))
    p_cam = c["world"].flatten(ortho, TR)
    c2, _ = small_config(3, (16, 16), 1, 1)
    from test_cpu_trap import FRACTAL_MATERIAL
    c2["world"].hitables.push(Sphere(Vec3(0, 0, 0), 0.1, FRACTAL_MATERIAL))
    p_n = c2["world"].flatten(c2["camera"], TR)
    p_kind = changed_kind(d)
    assert call(None) == L.RAYN_ERR_INVALID_ARG
    for dt in (np.inf, -np.inf, np.nan):
        assert call(C.byref(d), dt) == L.RAYN_ERR_INVALID_ARG
    for bad in (p_cam[0], p_n[0], p_kind[0]):
        assert call(C.byref(bad)) == L.RAYN_ERR_INVALID_ARG
    assert call(C.byref(d)) == L.RAYN_OK  # the context is usable after the errors


@pytest.mark.skipif(not L.LEGACY, reason="the legacy test kernels exist only in librayn_b200_legacy.so")
def test_simple_march_is_unsupported():
    c, inp = small_config(3, (16, 16), 1, 1)
    r = Renderer(0, flags=L.FLAG_SIMPLE_MARCH)
    try:
        d, keep = r.upload_scene(c["world"], c["camera"])
        with pytest.raises(L.RaynError) as e:
            r.render_motion(inp, (8, 8), c["integrator"], TR, DT, prev=d)
        assert e.value.code == L.RAYN_ERR_UNSUPPORTED
    finally:
        r.close()


# ---- closure worlds through Film.render_sequence ----
def orbit_camera(res, deg_per_s=60.0):
    r0 = np.linalg.norm(ORIGIN[[0, 2]])
    a0 = math.atan2(ORIGIN[2], ORIGIN[0])

    def origin(t):
        a = a0 + math.radians(deg_per_s) * t
        return (r0 * math.cos(a), ORIGIN[1], r0 * math.sin(a))
    return PinholeCamera(res, 60.0, origin, Vec3(0, 0, 0), Vec3(0, 1, 0))


def circling_sphere(world):
    from test_cpu_trap import FRACTAL_MATERIAL
    world.hitables.push(Sphere(lambda t: (1.1 * math.cos(4.0 * t), 0.9, 1.1 * math.sin(4.0 * t)), 0.3, FRACTAL_MATERIAL))


@pytest.mark.parametrize("shutter", [0.0, 1.0 / 24.0])
def test_film_render_sequence_with_closures(shutter):
    """6 frames of an orbiting camera and a sphere on a circle equal the explicit Renderer pipeline: per frame upload_scene
    with the frame's time range, render_host(moments=True), render_motion (first frame) or render_motion_prev against the
    previous frame's scene, temporal_push and the scaled denoise"""
    from rayn_b200.film import ALBEDO_SAMPLES, TEMPORAL_DEFAULTS, Film
    res = (32, 24)
    c, _ = small_config(3, res, 2, 1)
    circling_sphere(c["world"])
    cam = c["world"].cameras.add_camera(orbit_camera(res))
    assert c["world"].has_closures(cam)
    film = Film(["color", "alpha", "background", "normal", "albedo", "motion"], res)
    seen = []
    frames = range(1, 7)
    n = film.render_sequence(c["world"], cam, c["integrator"], None, (16, 16), frames, 24, shutter, 2, iterations=3,
                             on_frame=lambda f: seen.append({k: np.copy(v) for k, v in f.channels.items()}))
    assert n == 6
    frame_dt = float(np.float32(1.0) / np.float32(24))
    r = Renderer(0)
    t = r.temporal_create(*res)
    prev = None
    try:
        for i, k in enumerate(frames):
            start = np.float32(k) * np.float32(frame_dt)
            tr = (float(start), float(start + np.float32(shutter)))
            scene = r.upload_scene(c["world"], cam, tr)
            inp = FrameInputs(res[0], res[1], 2, c["integrator"], frame=k)
            p = r.render_host(inp, (16, 16), c["integrator"], tr, moments=True)
            g_inp = FrameInputs(res[0], res[1], min(2, ALBEDO_SAMPLES), c["integrator"], frame=k)
            mv, alb = r.render_motion(g_inp, (16, 16), c["integrator"], tr, frame_dt, albedo=True, prev=None if prev is None else prev[0])
            blend, m, s = r.temporal_push(t, p, p["moments"], mv, reset=(i == 0), **TEMPORAL_DEFAULTS)
            out = r.denoise(res[0], res[1], dict(p, color=blend["color"], background=blend["background"]), 3, albedo=alb.reshape(-1),
                            moments=m, spp=inp.spp, var_scale=s)
            for ch in ("color", "background"):
                assert_bit_equal(seen[i][ch], out[ch].reshape(res[1], res[0], 3), f"frame {k} {ch}")
            assert_bit_equal(seen[i]["motion"], mv, f"frame {k} motion")
            assert_bit_equal(seen[i]["albedo"], alb, f"frame {k} albedo")
            if prev is not None:
                o = mirrors.render_motion(scene[0], g_inp, (16, 16), c["integrator"], tr, frame_dt, prev=prev[0])[0]
                assert_bit_equal(mv, o, f"frame {k} motion mirror")
                assert (np.abs(mv[..., 0][np.isfinite(mv[..., 2])]) > 0.1).mean() > 0.5  # the orbit moves the image
            prev = scene
    finally:
        t.close()
        r.close()


def test_static_closure_world_gives_exact_zero_motion():
    """closures that return constants, uploaded again every frame: dx = dy = +0 and z_prev == z on every frame"""
    from rayn_b200.film import Film
    res = (24, 18)
    c, _ = small_config(3, res, 1, 1)
    from test_cpu_trap import FRACTAL_MATERIAL
    c["world"].hitables.push(Sphere(lambda t: (-1.0, 0.4, 0.9), 0.35, FRACTAL_MATERIAL))
    cam = c["world"].cameras.add_camera(PinholeCamera(res, 60.0, lambda t: tuple(ORIGIN), Vec3(0, 0, 0), Vec3(0, 1, 0)))
    film = Film(["color", "alpha", "background", "normal", "motion"], res)
    seen = []
    film.render_sequence(c["world"], cam, c["integrator"], None, (8, 8), range(1, 5), 24, 1.0 / 24.0, 1,
                         on_frame=lambda f: seen.append(np.copy(f.channels["motion"])))
    assert len(seen) == 4
    for k, mv in enumerate(seen):
        assert (mv[..., :2].view(np.uint32) == 0).all(), k
        assert_bit_equal(mv[..., 3], mv[..., 2], f"frame {k} z_prev")
        assert np.isfinite(mv[..., 2]).any()
