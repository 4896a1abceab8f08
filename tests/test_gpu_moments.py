"""Luminance moments on the device (rayn_b200_render_frame_moments, k_resolve<true>) against their CPU mirror
(tests/moments_oracle.cpp) bit for bit, and the variance-guided denoise (rayn_b200_film_denoise_variance) against its mirror
(tests/denoise_variance_oracle.cpp): configs 1-5 at odd sizes and two tile shapes, traps, fold-all on and off, moving spheres and
the thin-lens / orthographic cameras, several passes, sampled tiles of a full-size film, host and device planes, NULL planes,
film planes equal to render_frame's, render_frame and render_frame_moments alternated through the graph cache, the golden
fixture, argument errors and the Film / Renderer interfaces."""
import ctypes as C
import os

import numpy as np
import pytest

from rayn_b200 import _lib as L
from rayn_b200 import configs
from rayn_b200.film import Film, FrameInputs, Renderer, denoise_desc, make_frame_desc
from rayn_b200.scene import Lambertian, Sphere, Vec3

import moments_oracle as mo
from helpers import CH, assert_bit_equal, small_config
from test_cpu_albedo import trap_config
from test_cpu_moments import moment_film
from test_cpu_trap import FRACTAL_MATERIAL

pytestmark = pytest.mark.gpu
TR = configs.frame_time_range(1)
COLOR_CH = ("color", "background")
GOLDEN = "cfg3_moments_32x32_8spp"


def gpu(r, c, inp, tile, camera=None):
    r.upload_scene(c["world"], camera if camera is not None else c["camera"])
    return r.render_host(inp, tile, c["integrator"], TR, moments=True)


def mirror(c, inp, tile, camera=None, **kw):
    return mo.render(c["world"], camera if camera is not None else c["camera"], inp, tile, c["integrator"], TR, **kw)


def check(g, o, what):
    for k in CH + ("moments",):
        assert_bit_equal(g[k], o[k], f"{what} {k}")


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5])
@pytest.mark.parametrize("res", [(37, 23), (64, 48)])
@pytest.mark.parametrize("tile", [(8, 8), (16, 16)])
def test_moments_equal_mirror(renderer, n, res, tile):
    c, inp = small_config(n, res, 2, 3)
    g = gpu(renderer, c, inp, tile)
    check(g, mirror(c, inp, tile), f"cfg{n} {res} {tile}")
    plain = renderer.render_host(inp, tile, c["integrator"], TR)
    for k in CH:
        assert_bit_equal(g[k], plain[k], f"cfg{n} film planes equal render_frame's {k}")


@pytest.mark.parametrize("flags", [0, L.FLAG_NO_FOLD_ALL])
def test_traps_and_fold_all(flags):
    c, inp = trap_config(3, (40, 36), 2, 3)
    w = c["world"]
    plain = w.materials.add_material(Lambertian((0.6, 0.5, 0.4)))
    w.hitables.push(Sphere(Vec3(0.9, -0.7, 0.6), 0.35, FRACTAL_MATERIAL))
    w.hitables.push(Sphere(Vec3(-0.8, 0.6, 0.9), 0.3, plain))
    r = Renderer(0, flags=flags)
    try:
        check(gpu(r, c, inp, (8, 8)), mirror(c, inp, (8, 8)), f"traps flags {flags}")
    finally:
        r.close()


def test_moving_spheres_and_cameras(renderer):
    from rayn_b200 import Linear, OrthographicCamera, ThinLensCamera
    c, inp = trap_config(3, (48, 40), 2, 3)
    w = c["world"]
    w.hitables.push(Sphere(Linear(Vec3(-1.2, 0.9, 0.5), Vec3(30.0, 0.0, 0.0)), 0.4, FRACTAL_MATERIAL))
    res = (48, 40)
    cams = [c["camera"],
            w.cameras.add_camera(ThinLensCamera(res, 60.0, Linear(0.02, 0.2), Linear(Vec3(-1.0, 0.45, 4.5), Vec3(2.0, 0.0, 0.0)),
                                                Vec3(0, 0, 0), Linear(Vec3(0, 1, 0), Vec3(0.5, 0, 0)), Linear(Vec3(0, 0, 0), Vec3(0, 1, 0)))),
            w.cameras.add_camera(OrthographicCamera(res, 11.0 / 4.0, Vec3(9.5, -3.5, 9.5), Vec3(0.0, 0.8, 0.0), Vec3(0.0, 1.0, 0.0)))]
    for i, cam in enumerate(cams):
        check(gpu(renderer, c, inp, (16, 16), cam), mirror(c, inp, (16, 16), cam), f"camera {i}")


def test_several_passes():
    c, inp = small_config(3, (45, 37), 2, 3)
    r = Renderer(0, max_paths_per_pass=4 * 64 * inp.spp)
    try:
        g = gpu(r, c, inp, (8, 8))
        assert r.stats().passes > 1
        check(g, mirror(c, inp, (8, 8)), "multi-pass")
    finally:
        r.close()


def test_full_size_cfg3_sampled_tiles(renderer):
    c, _ = small_config(3, (1920, 1080), 1, 3)
    inp = FrameInputs(1920, 1080, 1, c["integrator"])
    g = gpu(renderer, c, inp, (16, 16))
    o = mirror(c, inp, (16, 16), subsample_k=97)
    nty = (1080 + 1080 % 16) // 16
    gm = {k: (g[k].reshape(1080, 1920, -1) if k != "moments" else g[k]) for k in CH + ("moments",)}
    om = {k: (o[k].reshape(1080, 1920, -1) if k != "moments" else o[k]) for k in CH + ("moments",)}
    for t in range(0, 120 * nty, 97):
        tx, ty = t // nty, t % nty
        sl = (slice(ty * 16, ty * 16 + 16), slice(tx * 16, tx * 16 + 16))
        for k in gm:
            assert_bit_equal(gm[k][sl], om[k][sl], f"tile {t} {k}")


def golden_config():
    from test_cpu_trap import trap_golden_config
    return trap_golden_config()


def test_golden(renderer):
    from test_cpu_oracle import GOLD, GOLD_SUFFIX
    c, inp = golden_config()
    gold = np.load(os.path.join(GOLD, GOLDEN + GOLD_SUFFIX + ".npz"))
    g = gpu(renderer, c, inp, (16, 16))
    for k in CH + ("moments",):
        assert_bit_equal(g[k], gold[k], f"golden {k}")


def _dev_frame(c, inp, w, h, tile, tabs):
    return make_frame_desc(w, h, tile, inp.samples, c["integrator"], inp.frame, TR, tuple(t.data_ptr() for t in tabs), L.MEM_DEVICE,
                           sets=(inp.sets_1d, inp.sets_2d))


def test_device_and_null_planes(renderer):
    """device planes (NaN-filled: uncovered pixels are cleared), and every combination of absent film / moment planes"""
    import torch
    w, h = 45, 33  # 33 rows: row 32 is outside the tile grid
    c, inp = small_config(3, (w, h), 2, 3)
    ref = mirror(c, inp, (16, 16))
    renderer.upload_scene(c["world"], c["camera"])
    dev = torch.device("cuda", 0)
    tabs = [torch.from_numpy(a.copy()).to(dev) for a in inp.arrays()]
    f = _dev_frame(c, inp, w, h, (16, 16), tabs)
    lib = L.lib()
    for film_on, mc_on, mb_on in ((True, True, True), (False, True, False), (False, False, True), (True, False, False)):
        planes = {k: torch.full(((1 if k == "alpha" else 3) * w * h,), float("nan"), device=dev) for k in CH}
        m = torch.full((2, w * h), float("nan"), device=dev)
        pf = L.RaynFilmPlanes(*(planes[k].data_ptr() if film_on else None for k in CH), L.MEM_DEVICE)
        pm = L.RaynMomentPlanes(m[0].data_ptr() if mc_on else None, m[1].data_ptr() if mb_on else None, L.MEM_DEVICE)
        torch.cuda.synchronize()
        L.check(lib.rayn_b200_render_frame_moments(renderer.ctx, C.byref(f), C.byref(pf), C.byref(pm)), renderer.ctx)
        what = f"film={film_on} mc={mc_on} mb={mb_on}"
        if film_on:
            for k in CH:
                assert_bit_equal(planes[k].cpu().numpy(), ref[k], f"{what} {k}")
        mm = m.cpu().numpy()
        for i, on in enumerate((mc_on, mb_on)):
            if on:
                assert_bit_equal(mm[i].reshape(h, w), ref["moments"][:, :, i], f"{what} moments {i}")
            else:
                assert np.isnan(mm[i]).all()
    # host space with NULL film planes
    mh = np.zeros((2, w * h), np.float32)
    ptrs = tuple(a.ctypes.data for a in inp.arrays())
    fh = make_frame_desc(w, h, (16, 16), inp.samples, c["integrator"], inp.frame, TR, ptrs, L.MEM_HOST, sets=(inp.sets_1d, inp.sets_2d))
    pm = L.RaynMomentPlanes(mh[0].ctypes.data, mh[1].ctypes.data, L.MEM_HOST)
    L.check(lib.rayn_b200_render_frame_moments(renderer.ctx, C.byref(fh), C.byref(L.RaynFilmPlanes(None, None, None, None, L.MEM_HOST)),
                                               C.byref(pm)), renderer.ctx)
    assert_bit_equal(mh.reshape(2, h, w).transpose(1, 2, 0), ref["moments"], "host moments, NULL film planes")


def test_alternating_with_render_frame_through_the_graph_cache():
    """render_frame and render_frame_moments on one context, each captured and replayed, each still equal to its mirror"""
    c, inp = small_config(1, (32, 32), 2, 2)
    ref = mirror(c, inp, (16, 16))
    r = Renderer(0)
    try:
        r.upload_scene(c["world"], c["camera"])
        for i in range(3):
            g = r.render_host(inp, (16, 16), c["integrator"], TR)
            assert r.stats().reserved_ == 1
            for k in CH:
                assert_bit_equal(g[k], ref[k], f"round {i} render_frame {k}")
            g = r.render_host(inp, (16, 16), c["integrator"], TR, moments=True)
            assert r.stats().reserved_ == 1
            check(g, ref, f"round {i} moments")
        for i in range(2):  # the same call twice in a row replays its own graph
            check(r.render_host(inp, (16, 16), c["integrator"], TR, moments=True), ref, f"replay {i}")
    finally:
        r.close()


def test_plain_render_never_replays_a_moments_graph(renderer):
    """Device planes and device inputs, one context: render_frame_moments captures its graph, then render_frame with the same
    film planes must not replay it (it would write the moment planes); each call is checked against its mirror, and the moment
    buffer, refilled with NaN before every plain call, must stay NaN."""
    import torch
    w, h = 32, 32
    c, inp = small_config(1, (w, h), 2, 2)
    ref = mirror(c, inp, (16, 16))
    renderer.upload_scene(c["world"], c["camera"])
    dev = torch.device("cuda", 0)
    tabs = [torch.from_numpy(a.copy()).to(dev) for a in inp.arrays()]
    f = _dev_frame(c, inp, w, h, (16, 16), tabs)
    planes = {k: torch.zeros((1 if k == "alpha" else 3) * w * h, device=dev) for k in CH}
    m = torch.zeros((2, w * h), device=dev)
    pf = L.RaynFilmPlanes(*(planes[k].data_ptr() for k in CH), L.MEM_DEVICE)
    pm = L.RaynMomentPlanes(m[0].data_ptr(), m[1].data_ptr(), L.MEM_DEVICE)
    lib = L.lib()
    for i in range(3):
        m.fill_(float("nan"))
        torch.cuda.synchronize()
        L.check(lib.rayn_b200_render_frame_moments(renderer.ctx, C.byref(f), C.byref(pf), C.byref(pm)), renderer.ctx)
        assert renderer.stats().reserved_ == 1
        assert_bit_equal(m.cpu().numpy().reshape(2, h, w).transpose(1, 2, 0), ref["moments"], f"round {i} moments")
        for _ in range(2):  # a capture, then a replay of the plain graph
            for k in CH:
                planes[k].fill_(float("nan"))
            m.fill_(float("nan"))
            torch.cuda.synchronize()
            L.check(lib.rayn_b200_render_frame(renderer.ctx, C.byref(f), C.byref(pf)), renderer.ctx)
            assert renderer.stats().reserved_ == 1
            for k in CH:
                assert_bit_equal(planes[k].cpu().numpy(), ref[k], f"round {i} render_frame {k}")
            assert torch.isnan(m).all(), f"round {i}: render_frame wrote the moment planes"


def test_argument_errors():
    lib = L.lib()
    r = Renderer(0)
    try:
        c, inp = small_config(3, (16, 16), 1, 1)
        p = {k: np.zeros((1 if k == "alpha" else 3) * 256, np.float32) for k in CH}
        m = np.zeros((2, 256), np.float32)
        ptrs = tuple(a.ctypes.data for a in inp.arrays())
        f = make_frame_desc(16, 16, (8, 8), inp.samples, c["integrator"], inp.frame, TR, ptrs, L.MEM_HOST, sets=(inp.sets_1d, inp.sets_2d))
        pf = L.RaynFilmPlanes(*(p[k].ctypes.data for k in CH), L.MEM_HOST)
        pm = L.RaynMomentPlanes(m[0].ctypes.data, m[1].ctypes.data, L.MEM_HOST)
        call = lambda pf=pf, pm=pm: lib.rayn_b200_render_frame_moments(r.ctx, C.byref(f), C.byref(pf) if pf is not None else None,  # noqa: E731
                                                                       C.byref(pm) if pm is not None else None)
        assert call() == L.RAYN_ERR_NO_SCENE
        r.upload_scene(c["world"], c["camera"])
        assert call() == L.RAYN_OK
        assert call(pm=None) == L.RAYN_ERR_INVALID_ARG
        assert call(pf=None) == L.RAYN_ERR_INVALID_ARG
        assert call(pm=L.RaynMomentPlanes(m[0].ctypes.data, None, L.MEM_DEVICE)) == L.RAYN_ERR_INVALID_ARG  # mixed spaces
        assert call(pf=L.RaynFilmPlanes(None, None, None, None, L.MEM_HOST), pm=L.RaynMomentPlanes(None, None, L.MEM_HOST)) == L.RAYN_ERR_INVALID_ARG
        # the variance denoise
        fp = moment_film(4, 4, 1)[0]
        flat = {k: np.ascontiguousarray(v).reshape(-1) for k, v in fp.items()}
        mm = np.ones((2, 16), np.float32)
        pin = L.RaynFilmPlanes(flat["color"].ctypes.data, flat["alpha"].ctypes.data, flat["background"].ctypes.data, flat["normal"].ctypes.data,
                               L.MEM_HOST)
        o = {k: np.zeros(48, np.float32) for k in COLOR_CH}
        pout = L.RaynFilmPlanes(o["color"].ctypes.data, None, o["background"].ctypes.data, None, L.MEM_HOST)
        d = denoise_desc(2)
        dv = lambda sl=1.0, spp=4, pm=L.RaynMomentPlanes(mm[0].ctypes.data, mm[1].ctypes.data, L.MEM_HOST), sa=1.0, alb=None: \
            lib.rayn_b200_film_denoise_variance(r.ctx, C.byref(d), sl, spp, C.byref(pm) if pm is not None else None, sa, alb, 4, 4,  # noqa: E731
                                                C.byref(pin), C.byref(pout))
        assert dv() == L.RAYN_OK and dv(sl=float("inf")) == L.RAYN_OK
        assert dv(pm=None) == L.RAYN_ERR_INVALID_ARG
        assert dv(pm=L.RaynMomentPlanes(mm[0].ctypes.data, None, L.MEM_HOST)) == L.RAYN_ERR_INVALID_ARG  # background without moments
        assert dv(pm=L.RaynMomentPlanes(mm[0].ctypes.data, mm[1].ctypes.data, L.MEM_DEVICE)) == L.RAYN_ERR_INVALID_ARG  # mixed spaces
        for spp in (0, -3):
            assert dv(spp=spp) == L.RAYN_ERR_INVALID_ARG
        for s in (0.0, -1.0, float("nan")):
            assert dv(sl=s) == L.RAYN_ERR_INVALID_ARG
        assert dv(sa=0.0, alb=mm.ctypes.data) == L.RAYN_ERR_INVALID_ARG
    finally:
        r.close()


@pytest.mark.skipif(not L.LEGACY, reason="the legacy test kernels exist only in librayn_b200_legacy.so")
def test_simple_march_is_unsupported_inner():
    c, inp = small_config(3, (16, 16), 1, 1)
    r = Renderer(0, flags=L.FLAG_SIMPLE_MARCH)
    try:
        r.upload_scene(c["world"], c["camera"])
        with pytest.raises(L.RaynError) as e:
            r.render_host(inp, (8, 8), c["integrator"], TR, moments=True)
        assert e.value.code == L.RAYN_ERR_UNSUPPORTED
    finally:
        r.close()


# ---- the variance-guided filter ---------------------------------------------------------------------------------------
def check_var(r, planes, desc, sl, spp, m, w, h, what, albedo=None, sa=np.inf):
    g = r.denoise(w, h, planes, desc.iterations, desc.sigma_color, desc.sigma_normal, desc.sigma_alpha, albedo=albedo,
                  sigma_albedo=None if albedo is None else sa, moments=m, spp=spp, sigma_luminance=sl)
    rc, o = mo.denoise(w, h, planes, desc, sl, spp, m, sa if albedo is not None else np.inf, albedo)
    assert rc == L.RAYN_OK and set(g) == set(o)
    for k in g:
        assert_bit_equal(g[k].reshape(-1), o[k], f"{what} {k}")
    return g


@pytest.mark.parametrize("w,h", [(1, 1), (3, 5), (37, 23), (129, 67)])
def test_variance_random_planes(renderer, w, h):
    p, m = moment_film(w, h, 300 + w)
    p["color"][h // 2, w // 2, 1] = np.nan
    alb = np.random.default_rng(w * h).uniform(0, 1, (h, w, 3)).astype(np.float32)
    for it in range(1, 9):
        for sl in (0.5, 4.0):
            check_var(renderer, p, denoise_desc(it, 2.5, 0.4, 0.5), sl, 16, m, w, h, f"{w}x{h} L={it} sl={sl}")
        check_var(renderer, p, denoise_desc(it, 2.5, 0.4, 0.5), 2.0, 4, m, w, h, f"{w}x{h} L={it} albedo", alb, 0.2)


@pytest.mark.parametrize("n", [1, 3, 4])
def test_variance_rendered_films(renderer, n):
    c, inp = trap_config(n, (64, 48), 2, 3)
    g = gpu(renderer, c, inp, (16, 16))
    planes = {k: g[k].reshape((48, 64, 3) if k != "alpha" else (48, 64)) for k in CH}
    alb = renderer.render_albedo(inp, (16, 16), c["integrator"], TR)
    for sl in (1.0, 4.0):
        check_var(renderer, planes, denoise_desc(5), sl, inp.spp, g["moments"], 64, 48, f"cfg{n} sl={sl}")
    check_var(renderer, planes, denoise_desc(5), 2.0, inp.spp, g["moments"], 64, 48, f"cfg{n} albedo", alb, 0.2)
    # +inf: the device's own film_denoise / film_denoise_albedo
    d = denoise_desc(5)
    u = renderer.denoise(64, 48, planes, 5, moments=g["moments"], spp=inp.spp, sigma_luminance=np.inf, sigma_color=d.sigma_color)
    ref = renderer.denoise(64, 48, planes, 5, sigma_color=d.sigma_color)
    ua = renderer.denoise(64, 48, planes, 5, albedo=alb, moments=g["moments"], spp=inp.spp, sigma_luminance=np.inf, sigma_color=d.sigma_color)
    refa = renderer.denoise(64, 48, planes, 5, albedo=alb, sigma_color=d.sigma_color)
    for k in COLOR_CH:
        assert_bit_equal(u[k], ref[k], f"cfg{n} +inf {k}")
        assert_bit_equal(ua[k], refa[k], f"cfg{n} +inf albedo {k}")


def test_variance_full_size_cfg3(renderer):
    c, _ = small_config(3, (1920, 1080), 1, 3)
    inp = FrameInputs(1920, 1080, 1, c["integrator"])
    g = gpu(renderer, c, inp, (16, 16))
    planes = {k: g[k].reshape((1080, 1920, 3) if k != "alpha" else (1080, 1920)) for k in CH}
    check_var(renderer, planes, denoise_desc(3), 4.0, inp.spp, g["moments"], 1920, 1080, "1080p")


def test_variance_spaces_and_aliasing(renderer):
    import torch
    w, h = 67, 45
    p, m = moment_film(w, h, 21)
    d = denoise_desc(5, 2.5, 0.4, 0.5)
    rc, ref = mo.denoise(w, h, p, d, 2.0, 8, m)
    assert rc == L.RAYN_OK
    flat = {k: np.ascontiguousarray(v).reshape(-1) for k, v in p.items()}
    mflat = np.ascontiguousarray(m.transpose(2, 0, 1)).reshape(2, -1)
    lib = L.lib()
    for in_dev in (False, True):
        for out_dev in (False, True):
            for alias in (False, True):
                if alias and in_dev != out_dev:
                    continue
                src = {k: (torch.from_numpy(v.copy()).cuda() if in_dev else v.copy()) for k, v in flat.items()}
                ms = torch.from_numpy(mflat.copy()).cuda() if in_dev else mflat.copy()
                dst = src if alias else {k: (torch.full((v.size,), float("nan"), device="cuda") if out_dev else np.full_like(v, np.nan))
                                         for k, v in flat.items() if k in COLOR_CH}

                def ptr(t):
                    return t.data_ptr() if isinstance(t, torch.Tensor) else t.ctypes.data
                sp = L.MEM_DEVICE if in_dev else L.MEM_HOST
                pin = L.RaynFilmPlanes(ptr(src["color"]), ptr(src["alpha"]), ptr(src["background"]), ptr(src["normal"]), sp)
                pout = L.RaynFilmPlanes(ptr(dst["color"]), None, ptr(dst["background"]), None, L.MEM_DEVICE if out_dev else L.MEM_HOST)
                pm = L.RaynMomentPlanes(ptr(ms[0]), ptr(ms[1]), sp)
                torch.cuda.synchronize()
                L.check(lib.rayn_b200_film_denoise_variance(renderer.ctx, C.byref(d), 2.0, 8, C.byref(pm), 1.0, None, w, h, C.byref(pin),
                                                            C.byref(pout)), renderer.ctx)
                L.check(lib.rayn_b200_sync(renderer.ctx), renderer.ctx)
                for k in COLOR_CH:
                    got = dst[k].cpu().numpy() if isinstance(dst[k], torch.Tensor) else dst[k]
                    assert_bit_equal(got, ref[k], f"in_dev={in_dev} out_dev={out_dev} alias={alias} {k}")


# ---- interfaces -----------------------------------------------------------------------------------------------------
def test_film_moments_channel():
    c, inp = small_config(3, (48, 32), 2, 3)
    film = Film(["color", "alpha", "background", "normal", "moments"], (48, 32))
    film.render_frame_into(c["world"], c["camera"], c["integrator"], None, (16, 16), 1, TR, 2)
    plain = Film(list(CH), (48, 32))
    plain.render_frame_into(c["world"], c["camera"], c["integrator"], None, (16, 16), 1, TR, 2)
    for k in CH:
        assert_bit_equal(film.channels[k], plain.channels[k], f"render_frame_into {k}")
    assert film.last_stats.paths == plain.last_stats.paths
    ref = mirror(c, inp, (16, 16))
    assert_bit_equal(film.channels["moments"], ref["moments"], "Film moments channel")
    before = {k: film.channels[k].copy() for k in COLOR_CH}
    moments = film.channels["moments"]
    film.denoise(3)
    from rayn_b200.film import DENOISE_LUMINANCE_SIGMA, DENOISE_VARIANCE_SIGMA_COLOR
    rc, o = mo.denoise(48, 32, {**before, "normal": film.channels["normal"], "alpha": film.channels["alpha"]},
                       denoise_desc(3, DENOISE_VARIANCE_SIGMA_COLOR), DENOISE_LUMINANCE_SIGMA, inp.spp, moments)
    for k in COLOR_CH:
        assert_bit_equal(film.channels[k].reshape(-1), o[k], f"Film.denoise {k}")
    # the moments describe the unfiltered render: they leave with the first filter, and a second call is the unguided one
    assert "moments" not in film.channels
    once = {k: film.channels[k].copy() for k in COLOR_CH}
    film.denoise(2)
    ref = film._renderer.denoise(48, 32, {**once, "normal": film.channels["normal"], "alpha": film.channels["alpha"]}, 2)
    for k in COLOR_CH:
        assert_bit_equal(film.channels[k], ref[k], f"second Film.denoise {k}")
    film.render_frame_into(c["world"], c["camera"], c["integrator"], None, (16, 16), 1, TR, 2)
    assert_bit_equal(film.channels["moments"], moments, "render_frame_into fills the moments again")


@pytest.mark.skipif(L.MULADD_FUSED, reason="rayn_host links the unfused product library")
@pytest.mark.parametrize("albedo", [False, True])
def test_cpp_host_denoise_variance(renderer, tmp_path, albedo):
    """rayn_host --denoise 5 --denoise-variance [--denoise-albedo] writes the image of the Python path (render with moments,
    render_albedo with the film's first 4 * min(samples, ALBEDO_SAMPLES) samples, variance-guided denoise with the library
    defaults), and its dumped planes are that path's bit for bit"""
    import subprocess
    from rayn_b200 import build
    from rayn_b200.film import ALBEDO_SAMPLES
    exe = os.path.join(os.path.dirname(build.OUT), "rayn_host")
    w, h, npx = 48, 32, 48 * 32
    args = [exe, "--config", "3", "--res", str(w), str(h), "--samples", "2", "--bounces", "3", "--denoise", "5", "--denoise-variance"]
    args += ["--denoise-albedo"] if albedo else []
    r = subprocess.run(args + ["--dump", str(tmp_path / "a.bin"), "--out", str(tmp_path / "a.ppm")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    raw = np.fromfile(tmp_path / "a.bin", np.float32)
    c, inp = small_config(3, (w, h), 2, 3)
    g = gpu(renderer, c, inp, (16, 16))
    alb = renderer.render_albedo(FrameInputs(w, h, min(2, ALBEDO_SAMPLES), c["integrator"]), (16, 16), c["integrator"], TR) if albedo else None
    den = renderer.denoise(w, h, {k: g[k] for k in CH}, 5, albedo=alb, moments=g["moments"], spp=inp.spp)
    assert_bit_equal(raw[:3 * npx], den["color"], "rayn_host --denoise-variance color")
    assert_bit_equal(raw[4 * npx:7 * npx], den["background"], "rayn_host --denoise-variance background")
    img = (tmp_path / "a.ppm").read_bytes()
    head = f"P6\n{w} {h}\n255\n".encode()
    assert img.startswith(head) and len(img) == len(head) + 3 * npx
    px = np.frombuffer(img[len(head):], np.uint8).reshape(h, w, 3)
    v = np.clip(den["color"] + den["background"], 0.0, 1.0).reshape(h, w, 3).astype(np.float64) ** (1.0 / 2.2)
    expect = np.clip(np.floor(v * 255.0), 0, 255)[::-1]  # y flipped, as save_to writes it
    assert np.abs(px.astype(np.int32) - expect.astype(np.int32)).max() <= 1
    plain = subprocess.run([a for a in args if a != "--denoise-variance"] + ["--dump", str(tmp_path / "b.bin")], capture_output=True, text=True)
    assert plain.returncode == 0, plain.stderr
    assert not np.array_equal(np.fromfile(tmp_path / "b.bin", np.float32), raw)  # the variance guide changed the image


@pytest.mark.skipif(L.MULADD_FUSED or L.LEGACY, reason="already inside a variant run")
def test_fused_and_legacy_variants():
    from test_gpu_parity import _run_suite_variant
    assert " passed" in _run_suite_variant({"RAYN_MULADD_FUSED": "1"}, ["tests/test_gpu_moments.py", "-k",
                                                                        "not full_size and not variants and not random_planes and not cpp_host"])
    assert " passed" in _run_suite_variant({"RAYN_B200_LEGACY": "1"}, ["tests/test_gpu_moments.py", "-k", "simple_march"])
