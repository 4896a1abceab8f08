"""First-hit albedo plane on the device (rayn_b200_render_albedo, rt_first_hit.cuh) against its CPU mirror
(tests/render_mirror.cpp) bit for bit, and the albedo-guided denoise (rayn_b200_film_denoise_albedo) against its mirror
(tests/film_mirror.cpp): odd sizes and tile shapes with and without traps, a trap material shared by a sphere and the
Mandelbox, fold-all on and off, moving spheres, thin-lens and orthographic cameras, sampled tiles of a full-size film, host and
device planes, the alpha identity at full size, the golden fixture, no side effects on later renders, argument errors and the
Film / Renderer interfaces."""
import ctypes as C
import os

import numpy as np
import pytest

from rayn_b200 import _lib as L
from rayn_b200 import configs
from rayn_b200.film import ALBEDO_SAMPLES, DENOISE_ALBEDO_SIGMA, Film, FrameInputs, Renderer, denoise_desc, make_frame_desc
from rayn_b200.scene import Lambertian, Sphere, Vec3

import mirrors
from helpers import CH, assert_bit_equal, small_config
from test_cpu_albedo import trap_config, white
from test_cpu_denoise import random_film
from test_cpu_trap import FRACTAL_MATERIAL

pytestmark = pytest.mark.gpu
TR = configs.frame_time_range(1)
COLOR_CH = ("color", "background")
ALBEDO_GOLDEN = "cfg3_trap_albedo_32x32_8spp"


def gpu_albedo(r, c, inp, tile, camera=None):
    r.upload_scene(c["world"], camera if camera is not None else c["camera"])
    return r.render_albedo(inp, tile, c["integrator"], TR)


def mirror(c, inp, tile, camera=None):
    return mirrors.render_albedo(c["world"], camera if camera is not None else c["camera"], inp, tile, c["integrator"], TR)[0]


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5])
@pytest.mark.parametrize("tile", [(8, 8), (16, 16)])
@pytest.mark.parametrize("trap", [False, True])
def test_albedo_equals_mirror(renderer, n, tile, trap):
    c, inp = trap_config(n, (37, 23), 2) if trap else small_config(n, (37, 23), 2, 1)
    assert_bit_equal(gpu_albedo(renderer, c, inp, tile), mirror(c, inp, tile), f"cfg{n} {tile} trap={trap}")


@pytest.mark.parametrize("flags", [0, L.FLAG_NO_FOLD_ALL])
def test_shared_trap_material_and_fold_all(flags):
    """config 3 plus two spheres: one shares the Mandelbox's trap material (s = 1 there), one has a plain Lambertian"""
    c, inp = trap_config(3, (40, 36), 2)
    w = c["world"]
    plain = w.materials.add_material(Lambertian((0.6, 0.5, 0.4)))
    w.hitables.push(Sphere(Vec3(0.9, -0.7, 0.6), 0.35, FRACTAL_MATERIAL))
    w.hitables.push(Sphere(Vec3(-0.8, 0.6, 0.9), 0.3, plain))
    r = Renderer(0, flags=flags)
    try:
        assert_bit_equal(gpu_albedo(r, c, inp, (8, 8)), mirror(c, inp, (8, 8)), f"shared material flags {flags}")
    finally:
        r.close()


def test_moving_spheres_and_cameras(renderer):
    """time-varying sphere centres (lane-0 time of the depth-0 packet), a moving thin-lens and an orthographic camera"""
    from rayn_b200 import Linear, OrthographicCamera, ThinLensCamera
    c, inp = trap_config(3, (48, 40), 2)
    w = c["world"]
    w.hitables.push(Sphere(Linear(Vec3(-1.2, 0.9, 0.5), Vec3(30.0, 0.0, 0.0)), 0.4, FRACTAL_MATERIAL))
    res = (48, 40)
    cams = [c["camera"],
            w.cameras.add_camera(ThinLensCamera(res, 60.0, Linear(0.02, 0.2), Linear(Vec3(-1.0, 0.45, 4.5), Vec3(2.0, 0.0, 0.0)),
                                                Vec3(0, 0, 0), Linear(Vec3(0, 1, 0), Vec3(0.5, 0, 0)), Linear(Vec3(0, 0, 0), Vec3(0, 1, 0)))),
            w.cameras.add_camera(OrthographicCamera(res, 11.0 / 4.0, Vec3(9.5, -3.5, 9.5), Vec3(0.0, 0.8, 0.0), Vec3(0.0, 1.0, 0.0)))]
    for i, cam in enumerate(cams):
        assert_bit_equal(gpu_albedo(renderer, c, inp, (16, 16), cam), mirror(c, inp, (16, 16), cam), f"camera {i}")


def test_full_size_cfg3_trap_sampled_tiles(renderer):
    c, _ = trap_config(3, (1920, 1080), 1)
    inp = FrameInputs(1920, 1080, 1, c["integrator"])
    g = gpu_albedo(renderer, c, inp, (16, 16))
    o = mirrors.render_albedo(c["world"], c["camera"], inp, (16, 16), c["integrator"], TR, subsample_k=97)[0]  # every 97th tile
    nty = (1080 + 1080 % 16) // 16
    for t in range(0, 120 * nty, 97):
        tx, ty = t // nty, t % nty
        sl = (slice(ty * 16, ty * 16 + 16), slice(tx * 16, tx * 16 + 16))
        assert_bit_equal(g[sl], o[sl], f"tile {t}")


@pytest.mark.parametrize("n,samples", [(3, 1), (2, 2)])
def test_alpha_identity_full_size(renderer, n, samples):
    """albedo (1, 1, 1) everywhere, no traps: every channel equals render_frame's alpha plane for the same frame"""
    c, _ = small_config(n, (1920, 1080), samples, 3)
    inp = FrameInputs(1920, 1080, samples, c["integrator"])
    white(c)
    a = gpu_albedo(renderer, c, inp, (16, 16))
    g = renderer.render_host(inp, (16, 16), c["integrator"], TR)
    for ch in range(3):
        assert_bit_equal(a[:, :, ch], g["alpha"].reshape(1080, 1920), f"cfg{n} channel {ch}")


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5])
def test_alpha_identity_downscaled(renderer, n):
    c, inp = small_config(n, (53, 29), 2, 2)
    white(c)
    a = gpu_albedo(renderer, c, inp, (8, 8))
    g = renderer.render_host(inp, (8, 8), c["integrator"], TR)
    for ch in range(3):
        assert_bit_equal(a[:, :, ch], g["alpha"].reshape(29, 53), f"cfg{n} channel {ch}")


def test_golden(renderer):
    from test_cpu_oracle import GOLD, GOLD_SUFFIX
    from test_cpu_trap import trap_golden_config
    c, inp = trap_golden_config()
    gold = np.load(os.path.join(GOLD, ALBEDO_GOLDEN + GOLD_SUFFIX + ".npz"))["albedo"]
    assert_bit_equal(gpu_albedo(renderer, c, inp, (16, 16)), gold, "albedo golden")


def test_device_planes_and_stats(renderer):
    import torch
    c, inp = trap_config(3, (45, 33), 2)
    ref = mirror(c, inp, (16, 16))
    renderer.upload_scene(c["world"], c["camera"])
    dev = torch.device("cuda", 0)
    tabs = [torch.from_numpy(a.copy()).to(dev) for a in inp.arrays()]
    out = torch.full((3 * 45 * 33,), float("nan"), device=dev)
    f = make_frame_desc(45, 33, (16, 16), inp.samples, c["integrator"], inp.frame, TR, tuple(t.data_ptr() for t in tabs), L.MEM_DEVICE,
                        sets=(inp.sets_1d, inp.sets_2d))
    torch.cuda.synchronize()
    L.check(L.lib().rayn_b200_render_albedo(renderer.ctx, C.byref(f), out.data_ptr(), L.MEM_DEVICE), renderer.ctx)
    assert_bit_equal(out.cpu().numpy().reshape(33, 45, 3), ref, "device planes")
    st = renderer.stats()
    assert st.passes >= 1 and st.paths == 45 * 32 * inp.spp  # film.rs:399-404: 33 rows make two 16-row tiles, row 32 is not rendered
    assert st.kernel_launches[L.KERNEL_NAMES.index("resolve")] == st.passes and st.reserved_ == 0


def test_no_side_effects_on_goldens():
    """the committed golden films render bit for bit after albedo passes (graph cache, pass buffers, staging)"""
    from test_cpu_oracle import GOLD, GOLD_SUFFIX, GOLDEN_CASES
    r = Renderer(0)
    try:
        for name, (n, res, samples, mb) in list(GOLDEN_CASES.items())[:2]:
            c, inp = small_config(n, res, samples, mb)
            gold = np.load(os.path.join(GOLD, name + GOLD_SUFFIX + ".npz"))
            r.upload_scene(c["world"], c["camera"])
            r.render_host(inp, (16, 16), c["integrator"], TR)  # captures the graph
            for tile in ((16, 16), (8, 8)):
                r.render_albedo(inp, tile, c["integrator"], TR)
                g = r.render_host(inp, (16, 16), c["integrator"], TR)
                for ch in CH:
                    assert_bit_equal(g[ch], gold[ch], f"golden {name} after albedo {tile} {ch}")
    finally:
        r.close()


def test_argument_errors():
    lib = L.lib()
    r = Renderer(0)
    try:
        c, inp = small_config(3, (16, 16), 1, 1)
        out = np.zeros(3 * 16 * 16, np.float32)
        ptrs = tuple(a.ctypes.data for a in inp.arrays())

        def frame(**kw):
            f = make_frame_desc(16, 16, (8, 8), inp.samples, c["integrator"], inp.frame, TR, ptrs, L.MEM_HOST, sets=(inp.sets_1d, inp.sets_2d))
            for k, v in kw.items():
                setattr(f, k, v)
            return f
        call = lambda f, o=out.ctypes.data, sp=L.MEM_HOST: lib.rayn_b200_render_albedo(r.ctx, C.byref(f), o, sp)  # noqa: E731
        assert call(frame()) == L.RAYN_ERR_NO_SCENE
        r.upload_scene(c["world"], c["camera"])
        assert call(frame(), o=None) == L.RAYN_ERR_INVALID_ARG
        assert call(frame(), sp=7) == L.RAYN_ERR_INVALID_ARG
        assert call(frame(width=0)) == L.RAYN_ERR_INVALID_ARG
        assert call(frame(samples=0)) == L.RAYN_ERR_INVALID_ARG
        assert call(frame(volume_marches=3)) == L.RAYN_ERR_UNSUPPORTED
        assert call(frame(sets_1d=1)) == L.RAYN_ERR_INVALID_ARG
        assert call(frame(samples_1d=None)) == L.RAYN_ERR_INVALID_ARG
        assert call(frame(tile_offset=5, tile_stride=2)) == L.RAYN_OK  # tile selection is ignored
        assert lib.rayn_b200_render_albedo(None, C.byref(frame()), out.ctypes.data, L.MEM_HOST) == L.RAYN_ERR_INVALID_ARG
        p = random_film(4, 4, 1)
        pin = L.RaynFilmPlanes(p["color"].ctypes.data, p["alpha"].ctypes.data, None, p["normal"].ctypes.data, L.MEM_HOST)
        o4 = np.zeros(48, np.float32)
        pout = L.RaynFilmPlanes(o4.ctypes.data, None, None, None, L.MEM_HOST)
        d = denoise_desc(2)
        alb = np.zeros(48, np.float32)
        assert lib.rayn_b200_film_denoise_albedo(r.ctx, C.byref(d), 0.1, None, 4, 4, C.byref(pin), C.byref(pout)) == L.RAYN_ERR_INVALID_ARG
        assert lib.rayn_b200_film_denoise_albedo(r.ctx, C.byref(d), float("inf"), None, 4, 4, C.byref(pin), C.byref(pout)) == L.RAYN_ERR_INVALID_ARG
        for s in (0.0, -1.0, float("nan"), 1e-30):
            assert lib.rayn_b200_film_denoise_albedo(r.ctx, C.byref(d), s, alb.ctypes.data, 4, 4, C.byref(pin), C.byref(pout)) == L.RAYN_ERR_INVALID_ARG
    finally:
        r.close()


@pytest.mark.skipif(not L.LEGACY, reason="the legacy test kernels exist only in librayn_b200_legacy.so")
def test_simple_march_is_unsupported_inner():
    c, inp = small_config(3, (16, 16), 1, 1)
    r = Renderer(0, flags=L.FLAG_SIMPLE_MARCH)
    try:
        r.upload_scene(c["world"], c["camera"])
        with pytest.raises(L.RaynError) as e:
            r.render_albedo(inp, (8, 8), c["integrator"], TR)
        assert e.value.code == L.RAYN_ERR_UNSUPPORTED
    finally:
        r.close()


# ---- the albedo-guided filter ---------------------------------------------------------------------------------------
def gpu_guided(r, planes, desc, albedo, sigma, w, h):
    return {k: v.reshape(-1) for k, v in r.denoise(w, h, planes, desc.iterations, desc.sigma_color, desc.sigma_normal, desc.sigma_alpha,
                                                   albedo=albedo, sigma_albedo=sigma).items()}


def check_guided(r, planes, desc, albedo, sigma, w, h, what):
    g = gpu_guided(r, planes, desc, albedo, sigma, w, h)
    rc, o = mirrors.denoise(w, h, planes, desc, albedo, sigma)
    assert rc == L.RAYN_OK and set(g) == set(o)
    for k in g:
        assert_bit_equal(g[k], o[k], f"{what} {k}")
    return g


@pytest.mark.parametrize("w,h", [(1, 1), (3, 5), (37, 23), (129, 67)])
def test_guided_random_planes(renderer, w, h):
    p = random_film(w, h, 200 + w)
    alb = np.random.default_rng(w * h).uniform(0, 1, (h, w, 3)).astype(np.float32)
    alb[h // 2, w // 2, 0] = np.nan
    alb[0, w - 1, 2] = np.inf
    for it in range(1, 9):
        for sigma in (0.05, 0.3):
            check_guided(renderer, p, denoise_desc(it, 0.5, 0.3, 0.4), alb, sigma, w, h, f"{w}x{h} L={it} s={sigma}")


def test_guided_absent_planes_spaces_and_aliasing(renderer):
    import torch
    w, h = 67, 45
    p = random_film(w, h, 11)
    alb = np.random.default_rng(3).uniform(0, 1, (h, w, 3)).astype(np.float32)
    d = denoise_desc(5, 0.5, 0.3, 0.3)
    check_guided(renderer, {k: v for k, v in p.items() if k != "background"}, d, alb, 0.1, w, h, "NULL background")
    check_guided(renderer, {k: v for k, v in p.items() if k != "color"}, d, alb, 0.1, w, h, "NULL color")
    rc, ref = mirrors.denoise(w, h, p, d, alb, 0.1)
    assert rc == L.RAYN_OK
    flat = {k: np.ascontiguousarray(v).reshape(-1) for k, v in p.items()}
    flat["albedo"] = alb.reshape(-1)
    lib = L.lib()
    for in_dev in (False, True):
        for out_dev in (False, True):
            for alias in (False, True):
                if alias and in_dev != out_dev:
                    continue
                src = {k: (torch.from_numpy(v.copy()).cuda() if in_dev else v.copy()) for k, v in flat.items()}
                dst = src if alias else {k: (torch.full((v.size,), float("nan"), device="cuda") if out_dev else np.full_like(v, np.nan))
                                         for k, v in flat.items() if k in COLOR_CH}

                def ptr(t):
                    return t.data_ptr() if isinstance(t, torch.Tensor) else t.ctypes.data
                pin = L.RaynFilmPlanes(ptr(src["color"]), ptr(src["alpha"]), ptr(src["background"]), ptr(src["normal"]),
                                       L.MEM_DEVICE if in_dev else L.MEM_HOST)
                pout = L.RaynFilmPlanes(ptr(dst["color"]), None, ptr(dst["background"]), None, L.MEM_DEVICE if out_dev else L.MEM_HOST)
                torch.cuda.synchronize()
                L.check(lib.rayn_b200_film_denoise_albedo(renderer.ctx, C.byref(d), 0.1, ptr(src["albedo"]), w, h, C.byref(pin), C.byref(pout)),
                        renderer.ctx)
                L.check(lib.rayn_b200_sync(renderer.ctx), renderer.ctx)
                for k in COLOR_CH:
                    got = dst[k].cpu().numpy() if isinstance(dst[k], torch.Tensor) else dst[k]
                    assert_bit_equal(got, ref[k], f"in_dev={in_dev} out_dev={out_dev} alias={alias} {k}")


@pytest.mark.parametrize("n", [1, 3, 4])
def test_infinite_sigma_equals_unguided_on_rendered_films(renderer, n):
    c, inp = trap_config(n, (64, 48), 1, 3)
    renderer.upload_scene(c["world"], c["camera"])
    film = renderer.render_host(inp, (16, 16), c["integrator"], TR)
    alb = renderer.render_albedo(inp, (16, 16), c["integrator"], TR)
    planes = {k: film[k].reshape((48, 64, 3) if k != "alpha" else (48, 64)) for k in CH}
    d = denoise_desc(5)
    g = gpu_guided(renderer, planes, d, alb, np.inf, 64, 48)
    u = renderer.denoise(64, 48, planes, 5)
    for k in COLOR_CH:
        assert_bit_equal(g[k], u[k].reshape(-1), f"cfg{n} {k}")


def test_guided_rendered_trap_film(renderer):
    c, inp = trap_config(3, (96, 96), 1, 3)
    renderer.upload_scene(c["world"], c["camera"])
    film = renderer.render_host(inp, (16, 16), c["integrator"], TR)
    alb = renderer.render_albedo(inp, (16, 16), c["integrator"], TR)
    planes = {k: film[k].reshape((96, 96, 3) if k != "alpha" else (96, 96)) for k in CH}
    for sigma in (0.02, 0.1, 0.5):
        check_guided(renderer, planes, denoise_desc(5), alb, sigma, 96, 96, f"trap film sigma {sigma}")


def test_guided_quality_at_the_default(renderer):
    """tools/bench_albedo.py (DESIGN.md §4e): on config 3 with the README palette at 96x96, the 4 spp film filtered with the
    default sigmas and a 4 * ALBEDO_SAMPLES spp albedo plane is closer (col+bg MSE) to a 256 spp film of another frame than
    the unguided filter (measured: 0.94 of its MSE)"""
    from rayn_b200.scene import Dielectric, OrbitTrapAlbedo
    c = configs.baseline_config(3, res=(96, 96), samples=1)
    c["world"].materials.items[1] = Dielectric.new_remap(OrbitTrapAlbedo(0.6676, 1.45, (0.9, 0.35, 0.1), (0.1, 0.3, 0.8)), 0.6)
    renderer.upload_scene(c["world"], c["camera"])
    lo = renderer.render_host(FrameInputs(96, 96, 1, c["integrator"]), (16, 16), c["integrator"], TR)
    hi = renderer.render_host(FrameInputs(96, 96, 64, c["integrator"], frame=2), (16, 16), c["integrator"], TR)
    alb = renderer.render_albedo(FrameInputs(96, 96, ALBEDO_SAMPLES, c["integrator"]), (16, 16), c["integrator"], TR)
    target = (hi["color"] + hi["background"]).astype(np.float64)

    def mse(d):
        return float(np.mean((d["color"].reshape(-1) + d["background"].reshape(-1) - target) ** 2))
    assert mse(renderer.denoise(96, 96, lo, 5, albedo=alb)) < 0.97 * mse(renderer.denoise(96, 96, lo, 5))


# ---- interfaces -----------------------------------------------------------------------------------------------------
def test_film_albedo_channel(tmp_path):
    c, _ = trap_config(3, (48, 32), 2)
    film = Film(["color", "alpha", "background", "normal", "albedo"], (48, 32))
    film.render_frame_into(c["world"], c["camera"], c["integrator"], None, (16, 16), 1, TR, 2)
    plain = Film(list(CH), (48, 32))
    plain.render_frame_into(c["world"], c["camera"], c["integrator"], None, (16, 16), 1, TR, 2)
    for k in CH:
        assert_bit_equal(film.channels[k], plain.channels[k], f"render_frame_into {k}")
    assert film.last_stats.paths == plain.last_stats.paths and film.last_stats.launches == plain.last_stats.launches
    inp = FrameInputs(48, 32, min(2, ALBEDO_SAMPLES), c["integrator"])
    assert_bit_equal(film.channels["albedo"], mirror(c, inp, (16, 16)), "Film albedo channel")
    before = {k: film.channels[k].copy() for k in COLOR_CH}
    film.denoise(3)
    plain.denoise(3)
    if np.isinf(DENOISE_ALBEDO_SIGMA):
        for k in COLOR_CH:
            assert_bit_equal(film.channels[k], plain.channels[k], f"Film.denoise at the default sigma {k}")
    else:
        rc, ref = mirrors.denoise(48, 32, {**before, "normal": film.channels["normal"], "alpha": film.channels["alpha"]}, denoise_desc(3),
                             film.channels["albedo"], DENOISE_ALBEDO_SIGMA)
        for k in COLOR_CH:
            assert_bit_equal(film.channels[k].reshape(-1), ref[k], f"Film.denoise {k}")
    paths = film.save_to(["albedo"], str(tmp_path), "t")
    from PIL import Image
    img = np.asarray(Image.open(paths[0]))
    expect = film._renderer.postprocess(L.POST_BACKGROUND, 48, 32, {"background": film.channels["albedo"].reshape(-1)})
    assert img.shape == (32, 48, 3) and np.array_equal(img, expect)


def test_film_render_adaptive_albedo():
    c, _ = trap_config(3, (40, 24), 1)
    film = Film(["color", "alpha", "background", "normal", "albedo"], (40, 24))
    film.render_adaptive(c["world"], c["camera"], c["integrator"], None, (16, 16), 1, TR, 1, max_rounds=3, threshold=-1.0)
    inp = FrameInputs(40, 24, min(3, ALBEDO_SAMPLES), c["integrator"])
    assert_bit_equal(film.channels["albedo"], mirror(c, inp, (16, 16)), "render_adaptive albedo")
    film.denoise(2)


@pytest.mark.skipif(L.MULADD_FUSED or L.LEGACY, reason="already inside a variant run")
def test_fused_and_legacy_variants():
    from test_gpu_parity import _run_suite_variant
    assert " passed" in _run_suite_variant({"RAYN_MULADD_FUSED": "1"}, ["tests/test_gpu_albedo.py", "-k",
                                                                        "not full_size and not variants and not cpp_host"])
    assert " passed" in _run_suite_variant({"RAYN_B200_LEGACY": "1"}, ["tests/test_gpu_albedo.py", "-k", "simple_march"])


@pytest.mark.skipif(L.MULADD_FUSED, reason="rayn_host links the unfused product library")
def test_cpp_host_denoise_albedo(renderer, tmp_path):
    """rayn_host --denoise L --denoise-albedo gives the Python path (render, render_albedo with the film's first
    4 * min(samples, ALBEDO_SAMPLES) samples, albedo-guided denoise with the library defaults) bit for bit"""
    import subprocess
    from rayn_b200 import build
    from test_cpu_trap import ALBEDO_HI, ALBEDO_LO, TRAP_HI, TRAP_LO
    exe = os.path.join(os.path.dirname(build.OUT), "rayn_host")
    trap = [str(v) for v in (TRAP_LO, TRAP_HI) + ALBEDO_LO + ALBEDO_HI]
    args = [exe, "--config", "3", "--res", "48", "32", "--samples", "2", "--bounces", "3", "--orbit-trap"] + trap + ["--denoise", "3"]
    r = subprocess.run(args + ["--denoise-albedo", "--dump", str(tmp_path / "a.bin")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    raw = np.fromfile(tmp_path / "a.bin", np.float32)
    npx = 48 * 32
    c, inp = trap_config(3, (48, 32), 2, 3)
    renderer.upload_scene(c["world"], c["camera"])
    film = renderer.render_host(inp, (16, 16), c["integrator"], TR)
    alb = renderer.render_albedo(FrameInputs(48, 32, min(2, ALBEDO_SAMPLES), c["integrator"]), (16, 16), c["integrator"], TR)
    den = renderer.denoise(48, 32, film, 3, albedo=alb)
    assert_bit_equal(raw[:3 * npx], den["color"], "rayn_host --denoise-albedo color")
    assert_bit_equal(raw[4 * npx:7 * npx], den["background"], "rayn_host --denoise-albedo background")
    assert subprocess.run([exe, "--config", "3", "--denoise-albedo"], capture_output=True, text=True).returncode == 2
