"""Motion plane (rayn_b200_render_motion, rt_first_hit.cuh), temporal push (rayn_b200_temporal_push, rt_temporal.cuh) and the
scaled variance denoise (rayn_b200_film_denoise_variance_scaled) on the device against their CPU mirrors
(tests/render_mirror.cpp, tests/film_mirror.cpp) bit for bit: configs 1, 3 and 4 (thin lens), an orthographic and a
moving pinhole camera, 15 moving spheres, odd sizes, 8x8 and 16x16 tiles, several passes, sampled tiles of a 1080p film, the
albedo plane of the same pass against render_albedo, exact zero motion on static scenes, a rendered camera-dolly sequence and a
moving-sphere sequence through push (history ping-pong, reset, disocclusion, aliased planes, host and device planes) and the
scaled denoise, and argument errors."""
import ctypes as C

import numpy as np
import pytest

from rayn_b200 import _lib as L
from rayn_b200 import configs
from rayn_b200.film import FrameInputs, Renderer, denoise_desc
from rayn_b200.scene import Linear, OrthographicCamera, PinholeCamera, Vec3

import limits_scenes as ls
import mirrors
from helpers import assert_bit_equal, small_config
from test_cpu_albedo import trap_config

pytestmark = pytest.mark.gpu
DT = 1.0 / 24.0
TR = configs.frame_time_range(1)
ORIGIN = np.array([-0.45, 0.2, 2.0]) * 2.25


def gpu_motion(r, c, inp, tile, camera=None, albedo=False):
    r.upload_scene(c["world"], camera if camera is not None else c["camera"])
    return r.render_motion(inp, tile, c["integrator"], TR, DT, albedo=albedo)


def mirror(c, inp, tile, camera=None, **kw):
    return mirrors.render_motion(c["world"].flatten(camera if camera is not None else c["camera"])[0], inp, tile, c["integrator"], TR, DT, **kw)[0]


def dolly(c, res, speed=1.5):
    """config 3's camera moving towards the fractal with its look-at point fixed"""
    d = -ORIGIN / np.linalg.norm(ORIGIN) * speed
    return c["world"].cameras.add_camera(PinholeCamera(res, 60.0, Linear(Vec3(*ORIGIN), Vec3(*d)), Vec3(0, 0, 0), Vec3(0, 1, 0)))


@pytest.mark.parametrize("n", [1, 3, 4])
@pytest.mark.parametrize("tile", [(8, 8), (16, 16)])
def test_motion_equals_mirror(renderer, n, tile):
    c, inp = trap_config(n, (37, 23), 2)
    cam = dolly(c, (37, 23)) if n == 3 else None
    m, a = gpu_motion(renderer, c, inp, tile, cam, albedo=True)
    assert_bit_equal(m, mirror(c, inp, tile, cam), f"cfg{n} {tile}")
    renderer.upload_scene(c["world"], cam if cam is not None else c["camera"])
    assert_bit_equal(a, renderer.render_albedo(inp, tile, c["integrator"], TR), f"cfg{n} albedo")
    assert_bit_equal(renderer.render_motion(inp, tile, c["integrator"], TR, DT), m, "without albedo")


def test_moving_cameras_and_spheres(renderer):
    from rayn_b200 import Sphere
    from test_cpu_trap import FRACTAL_MATERIAL
    res = (48, 40)
    c, inp = trap_config(3, res, 2)
    w = c["world"]
    w.hitables.push(Sphere(Linear(Vec3(-1.2, 0.9, 0.5), Vec3(30.0, 0.0, 0.0)), 0.4, FRACTAL_MATERIAL))
    cams = [c["camera"],
            w.cameras.add_camera(OrthographicCamera(res, 11.0 / 4.0, Linear(Vec3(9.5, -3.5, 9.5), Vec3(1.0, 0.5, 0.0)), Vec3(0.0, 0.8, 0.0),
                                                    Vec3(0.0, 1.0, 0.0))),
            w.cameras.add_camera(PinholeCamera(res, 60.0, Vec3(*ORIGIN), Linear(Vec3(0, 0, 0), Vec3(0.6, 0.0, 0.0)), Vec3(0, 1, 0)))]  # a pan
    for i, cam in enumerate(cams):
        assert_bit_equal(gpu_motion(renderer, c, inp, (16, 16), cam), mirror(c, inp, (16, 16), cam), f"camera {i}")


def test_limits_shape_c_moving_spheres(renderer):
    cam, world = ls.shape_c((29, 21), False)
    integ, inp = ls.inputs((29, 21), 2, 1)
    renderer.upload_scene(world, cam)
    g = renderer.render_motion(inp, (8, 8), integ, TR, DT)
    o = mirrors.render_motion(world.flatten(cam)[0], inp, (8, 8), integ, TR, DT)[0]
    assert_bit_equal(g, o, "shape C")
    assert (g[..., 0] != 0).any()


def test_several_passes():
    c, inp = small_config(3, (61, 45), 2, 1)
    cam = dolly(c, (61, 45))
    r = Renderer(0, max_paths_per_pass=8 * 8 * 8 * 3)
    try:
        g = gpu_motion(r, c, inp, (8, 8), cam)
        assert r.stats().passes > 1
    finally:
        r.close()
    assert_bit_equal(g, mirror(c, inp, (8, 8), cam), "passes")


def test_static_scene_is_exactly_zero(renderer):
    c, inp = small_config(3, (33, 19), 2, 1)
    g = gpu_motion(renderer, c, inp, (16, 16))
    assert (g[..., :2].view(np.uint32) == 0).all()
    assert_bit_equal(g[..., 3], g[..., 2], "z_prev")


def test_full_size_cfg3_sampled_tiles(renderer):
    c, _ = small_config(3, (1920, 1080), 1, 1)
    inp = FrameInputs(1920, 1080, 1, c["integrator"])
    cam = dolly(c, (1920, 1080))
    g = gpu_motion(renderer, c, inp, (16, 16), cam)
    o = mirrors.render_motion(c["world"].flatten(cam)[0], inp, (16, 16), c["integrator"], TR, DT, subsample_k=97)[0]
    nty = (1080 + 1080 % 16) // 16
    for t in range(0, 120 * nty, 97):
        tx, ty = t // nty, t % nty
        sl = (slice(ty * 16, ty * 16 + 16), slice(tx * 16, tx * 16 + 16))
        assert_bit_equal(g[sl], o[sl], f"tile {t}")


def test_device_planes(renderer):
    torch = pytest.importorskip("torch")
    c, inp = small_config(3, (27, 19), 2, 1)
    cam = dolly(c, (27, 19))
    renderer.upload_scene(c["world"], cam)
    from rayn_b200.film import make_frame_desc
    ptrs = tuple(a.ctypes.data for a in inp.arrays())
    f = make_frame_desc(27, 19, (8, 8), inp.samples, c["integrator"], inp.frame, TR, ptrs, L.MEM_HOST, sets=(inp.sets_1d, inp.sets_2d))
    m = torch.full((19 * 27 * 4,), 7.0, device="cuda")
    a = torch.full((19 * 27 * 3,), 7.0, device="cuda")
    torch.cuda.synchronize()
    L.check(renderer._lib.rayn_b200_render_motion(renderer.ctx, C.byref(f), DT, m.data_ptr(), a.data_ptr(), L.MEM_DEVICE), renderer.ctx)
    assert_bit_equal(m.cpu().numpy().reshape(19, 27, 4), mirror(c, inp, (8, 8), cam), "device motion")
    assert_bit_equal(a.cpu().numpy().reshape(19, 27, 3), renderer.render_albedo(inp, (8, 8), c["integrator"], TR), "device albedo")


# ---- sequences through the temporal push and the scaled denoise ----
def sequence(r, c, cam, res, samples, n_frames):
    """per frame: (film planes with moments, motion) rendered with the frame's own seed and time range"""
    out = []
    for k in range(1, n_frames + 1):
        inp = FrameInputs(res[0], res[1], samples, c["integrator"], frame=k)
        tr = configs.frame_time_range(k)
        r.upload_scene(c["world"], cam)
        p = r.render_host(inp, (16, 16), c["integrator"], tr, moments=True)
        mv = r.render_motion(inp, (16, 16), c["integrator"], tr, DT)
        out.append((p, mv))
    return out


def push_both(r, t, tm, p, mv, kw, reset):
    h, w = mv.shape[:2]
    planes = {k: p[k] for k in ("color", "background", "normal")}
    g = r.temporal_push(t, planes, p["moments"], mv, reset=reset, **kw)
    rc, oc, om, s = tm.push(planes, p["moments"], mv, reset=reset, **kw)
    assert rc == 0
    assert_bit_equal(g[0]["color"], oc["color"], "color")
    assert_bit_equal(g[0]["background"], oc["background"], "background")
    assert_bit_equal(g[1], om, "moments")
    assert_bit_equal(g[2], s, "var_scale")
    return g


@pytest.mark.parametrize("scene", ["dolly", "moving_sphere"])
def test_sequence_push_and_scaled_denoise(renderer, scene):
    res = (40, 30)
    c, _ = small_config(3, res, 2, 1)
    if scene == "dolly":
        cam = dolly(c, res)
    else:
        from rayn_b200 import Sphere
        from test_cpu_trap import FRACTAL_MATERIAL
        c["world"].hitables.push(Sphere(Linear(Vec3(-1.0, 0.3, 0.8), Vec3(6.0, 0.0, 0.0)), 0.35, FRACTAL_MATERIAL))
        cam = c["camera"]
    frames = sequence(renderer, c, cam, res, 2, 6)
    kw = dict(alpha_min=0.2, sigma_depth=0.05, normal_cos=0.8)
    t = renderer.temporal_create(*res)
    tm = mirrors.TemporalMirror(*res)
    spp = 8
    d = denoise_desc(3, np.inf, 0.3, 0.2)
    try:
        for k, (p, mv) in enumerate(frames):
            g = push_both(renderer, t, tm, p, mv, kw, reset=(k == 3))
            if k == 0 or k == 3:
                assert (g[2] == 1).all()
            elif k in (2, 5):
                assert (g[2] < 1).any()
            planes = dict(p, color=g[0]["color"], background=g[0]["background"])
            dn = renderer.denoise(res[0], res[1], planes, 3, np.inf, 0.3, 0.2, moments=g[1], spp=spp, sigma_luminance=4.0, var_scale=g[2])
            rc, o = mirrors.denoise(res[0], res[1], planes, d, moments=g[1], spp=spp, sigma_luminance=4.0, var_scale=g[2])
            assert rc == 0
            for ch in ("color", "background"):
                assert_bit_equal(dn[ch], o[ch].reshape(dn[ch].shape), f"frame {k} denoise {ch}")
    finally:
        t.close()


def test_alpha_one_and_unit_scale_identities(renderer):
    res = (24, 18)
    c, _ = small_config(3, res, 1, 1)
    frames = sequence(renderer, c, dolly(c, res), res, 1, 3)
    t = renderer.temporal_create(*res)
    try:
        for p, mv in frames:
            planes = {k: p[k] for k in ("color", "background", "normal")}
            out, om, s = renderer.temporal_push(t, planes, p["moments"], mv, 1.0, 0.05, 0.5)
            assert_bit_equal(out["color"], p["color"]), assert_bit_equal(om, p["moments"])
            assert (s == 1).all()
            a = renderer.denoise(*res, p, 3, moments=p["moments"], spp=4)
            b = renderer.denoise(*res, p, 3, moments=p["moments"], spp=4, var_scale=s)
            for ch in a:
                assert_bit_equal(b[ch], a[ch], ch)
    finally:
        t.close()


def test_device_planes_and_aliasing(renderer):
    """device planes, with out aliasing in, give the host result"""
    torch = pytest.importorskip("torch")
    res = (31, 17)
    w, h = res
    c, _ = small_config(3, res, 1, 1)
    frames = sequence(renderer, c, dolly(c, res), res, 1, 3)
    kw = dict(alpha_min=0.3, sigma_depth=0.05, normal_cos=0.5)
    th, td = renderer.temporal_create(*res), renderer.temporal_create(*res)
    try:
        for p, mv in frames:
            planes = {k: p[k] for k in ("color", "background", "normal")}
            ref = renderer.temporal_push(th, planes, p["moments"], mv, **kw)
            dev = {k: torch.from_numpy(np.ascontiguousarray(v, np.float32).reshape(-1)).cuda() for k, v in planes.items()}
            m = torch.from_numpy(np.ascontiguousarray(p["moments"].transpose(2, 0, 1)).reshape(2, -1)).cuda()
            mvd = torch.from_numpy(np.ascontiguousarray(mv).reshape(-1)).cuda()
            s = torch.empty(w * h, device="cuda")
            torch.cuda.synchronize()
            pin = L.RaynFilmPlanes(dev["color"].data_ptr(), None, dev["background"].data_ptr(), dev["normal"].data_ptr(), L.MEM_DEVICE)
            mp = L.RaynMomentPlanes(m[0].data_ptr(), m[1].data_ptr(), L.MEM_DEVICE)
            d = L.RaynTemporalDesc(kw["alpha_min"], kw["sigma_depth"], kw["normal_cos"], 0)
            L.check(renderer._lib.rayn_b200_temporal_push(renderer.ctx, td.handle, C.byref(d), C.byref(pin), C.byref(mp), mvd.data_ptr(), C.byref(pin),
                                                          C.byref(mp), s.data_ptr()), renderer.ctx)
            L.check(renderer._lib.rayn_b200_sync(renderer.ctx), renderer.ctx)
            assert_bit_equal(dev["color"].cpu().numpy(), ref[0]["color"].reshape(-1), "device color")
            assert_bit_equal(m.cpu().numpy().reshape(2, h, w).transpose(1, 2, 0), ref[1], "device moments")
            assert_bit_equal(s.cpu().numpy().reshape(h, w), ref[2], "device var_scale")
    finally:
        th.close(), td.close()


def test_argument_errors(renderer):
    c, inp = small_config(3, (16, 16), 1, 1)
    renderer.upload_scene(c["world"], c["camera"])
    with pytest.raises(L.RaynError):
        renderer.render_motion(inp, (8, 8), c["integrator"], TR, np.inf)
    t = renderer.temporal_create(16, 16)
    try:
        p = renderer.render_host(inp, (8, 8), c["integrator"], TR, moments=True)
        mv = renderer.render_motion(inp, (8, 8), c["integrator"], TR, DT)
        planes = {k: p[k] for k in ("color", "background", "normal")}
        for bad in (dict(alpha_min=0.0, sigma_depth=0.1, normal_cos=0.5), dict(alpha_min=0.5, sigma_depth=-1.0, normal_cos=0.5),
                    dict(alpha_min=0.5, sigma_depth=0.1, normal_cos=2.0)):
            with pytest.raises(L.RaynError):
                renderer.temporal_push(t, planes, p["moments"], mv, **bad)
        pin = L.RaynFilmPlanes(None, None, None, None, L.MEM_HOST)
        d = L.RaynTemporalDesc(0.5, 0.1, 0.5, 0)
        assert renderer._lib.rayn_b200_temporal_push(renderer.ctx, t.handle, C.byref(d), C.byref(pin), None, None, C.byref(pin), None,
                                                     None) == L.RAYN_ERR_INVALID_ARG
        mp = L.RaynMomentPlanes(None, None, L.MEM_HOST)
        assert renderer._lib.rayn_b200_film_denoise_variance_scaled(renderer.ctx, C.byref(denoise_desc(3)), 4.0, 4, C.byref(mp), None, np.inf, None,
                                                                    16, 16, C.byref(pin), C.byref(pin)) == L.RAYN_ERR_INVALID_ARG
    finally:
        t.close()
    with pytest.raises(L.RaynError):
        renderer.temporal_create(0, 16)


def test_pixel_without_a_hit_takes_no_history(renderer):
    """synthetic frames: a pixel whose motion is (0, 0, +inf, +inf) takes the current frame, on the device as in the mirror"""
    from test_cpu_temporal import frame
    w, h = 11, 8
    t, tm = renderer.temporal_create(w, h), mirrors.TemporalMirror(w, h)
    try:
        for k, (p, m, mv) in enumerate([frame(w, h, 120), frame(w, h, 121, static=False)]):
            if k == 1:
                p["normal"][:4] = 0.0
                mv[:4, :, 2:] = np.inf
            p["moments"] = m
            g = push_both(renderer, t, tm, p, mv, dict(alpha_min=0.5, sigma_depth=0.1, normal_cos=-1.0), False)
            if k == 1:
                assert (g[2][:4] == 1).all() and (g[2][4:] < 1).any()
                assert_bit_equal(g[0]["color"][:4], p["color"][:4])
    finally:
        t.close()


def test_film_render_sequence(renderer, tmp_path):
    """Film.render_sequence equals the explicit Renderer pipeline frame by frame, and its motion channel is the mirror's"""
    from rayn_b200.film import ALBEDO_SAMPLES, TEMPORAL_DEFAULTS, Film
    res = (32, 24)
    c, _ = small_config(3, res, 2, 1)
    cam = dolly(c, res)
    film = Film(["color", "alpha", "background", "normal", "albedo", "motion"], res)
    seen = []
    n = film.render_sequence(c["world"], cam, c["integrator"], None, (16, 16), range(3, 6), 24, 1.0 / 24.0, 2, iterations=3,
                             on_frame=lambda f: seen.append({k: np.copy(v) for k, v in f.channels.items()}))
    assert n == 3 and len(seen) == 3
    r = Renderer(0)
    t = r.temporal_create(*res)
    try:
        r.upload_scene(c["world"], cam)
        for i, k in enumerate(range(3, 6)):
            tr = configs.frame_time_range(k)
            inp = FrameInputs(res[0], res[1], 2, c["integrator"], frame=k)
            p = r.render_host(inp, (16, 16), c["integrator"], tr, moments=True)
            mv, alb = r.render_motion(FrameInputs(res[0], res[1], min(2, ALBEDO_SAMPLES), c["integrator"], frame=k), (16, 16), c["integrator"],
                                      tr, DT, albedo=True)
            blend, m, s = r.temporal_push(t, p, p["moments"], mv, reset=(i == 0), **TEMPORAL_DEFAULTS)
            out = r.denoise(res[0], res[1], dict(p, color=blend["color"], background=blend["background"]), 3, albedo=alb.reshape(-1),
                            moments=m, spp=inp.spp, var_scale=s)
            for ch in ("color", "background"):
                assert_bit_equal(seen[i][ch], out[ch].reshape(res[1], res[0], 3), f"frame {k} {ch}")
            assert_bit_equal(seen[i]["motion"], mv, f"frame {k} motion")
            assert_bit_equal(seen[i]["albedo"], alb, f"frame {k} albedo")
            assert_bit_equal(mv, mirrors.render_motion(c["world"].flatten(cam)[0], FrameInputs(res[0], res[1], 2, c["integrator"], frame=k),
                                                       (16, 16), c["integrator"], tr, DT)[0], f"frame {k} motion mirror")
    finally:
        t.close()
        r.close()
    with pytest.raises(ValueError):
        film.save_to(["motion"], str(tmp_path), "x")
