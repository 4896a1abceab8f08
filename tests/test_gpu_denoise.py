"""GPU film denoiser (rayn_b200_film_denoise, rt_denoise.cuh) against its CPU mirror (tests/film_mirror.cpp), bit for
bit: random planes, rendered films, every level count, host and device spaces, aliasing, absent planes; argument
errors; the exact zero-weight cutoff of dm::exp on the device; image quality; and that rendering is unaffected."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from rayn_b200 import _lib as L
from rayn_b200 import configs
from rayn_b200.film import Film, denoise_desc

import mirrors
from helpers import CH, assert_bit_equal, small_config
from test_cpu_denoise import random_film

pytestmark = pytest.mark.gpu
TR = configs.frame_time_range(1)
COLOR_CH = ("color", "background")


def gpu(renderer, planes, desc, w, h):
    rc = _call(renderer, planes, desc, w, h)
    assert rc == L.RAYN_OK, L.lib().rayn_b200_last_error(renderer.ctx)
    return _call.outs


def _call(renderer, planes, desc, w, h):
    flat = {k: np.ascontiguousarray(v, np.float32).reshape(-1) for k, v in planes.items() if v is not None}
    outs = {k: np.full_like(flat[k], np.nan) for k in COLOR_CH if k in flat}

    def ptr(d, k):
        return d[k].ctypes.data if k in d else None
    pin = L.RaynFilmPlanes(ptr(flat, "color"), ptr(flat, "alpha"), ptr(flat, "background"), ptr(flat, "normal"), L.MEM_HOST)
    pout = L.RaynFilmPlanes(ptr(outs, "color"), None, ptr(outs, "background"), None, L.MEM_HOST)
    _call.outs = outs
    return L.lib().rayn_b200_film_denoise(renderer.ctx, C.byref(desc), w, h, C.byref(pin), C.byref(pout))


def check_against_mirror(renderer, planes, desc, w, h, what):
    g = gpu(renderer, planes, desc, w, h)
    rc, o = mirrors.denoise(w, h, planes, desc)
    assert rc == L.RAYN_OK
    assert set(g) == set(o)
    for k in g:
        assert_bit_equal(g[k], o[k], f"{what} {k}")
    return g


@pytest.mark.parametrize("w,h", [(1, 1), (3, 5), (37, 23), (129, 67), (1, 53), (53, 1)])
def test_random_planes_bit_equal(renderer, w, h):
    p = random_film(w, h, 100 + w * h)
    for it, s in ((1, (0.3, 0.2, 0.2)), (3, (0.5, 0.1, np.inf)), (5, (1.0, 0.5, 0.3))):
        check_against_mirror(renderer, p, denoise_desc(it, *s), w, h, f"{w}x{h} L={it}")


def test_every_level_count(renderer):
    p = random_film(261, 133, 7)
    for it in range(1, 9):
        check_against_mirror(renderer, p, denoise_desc(it, 0.4, 0.3, 0.3), 261, 133, f"L={it}")


def test_non_finite_pixels_bit_equal(renderer):
    p = random_film(45, 33, 8)
    for y, x, ch, v in [(3, 4, 0, np.nan), (10, 10, 1, np.inf), (20, 5, 2, -np.inf), (32, 44, 0, np.nan), (0, 0, 1, np.inf)]:
        p["color"][y, x, ch] = v
        p["background"][x % 33, y, ch] = v
    check_against_mirror(renderer, p, denoise_desc(5, 0.5, 0.3, 0.3), 45, 33, "non-finite")


def test_absent_colour_planes(renderer):
    p = random_film(40, 30, 9)
    d = denoise_desc(4, 0.5, 0.3, 0.3)
    full = check_against_mirror(renderer, p, d, 40, 30, "both")
    only_c = check_against_mirror(renderer, {k: v for k, v in p.items() if k != "background"}, d, 40, 30, "NULL background")
    only_b = check_against_mirror(renderer, {k: v for k, v in p.items() if k != "color"}, d, 40, 30, "NULL color")
    assert_bit_equal(only_c["color"], full["color"], "channels are filtered independently")
    assert_bit_equal(only_b["background"], full["background"], "channels are filtered independently")


def test_device_spaces_and_aliasing(renderer):
    import torch
    w, h = 67, 45
    p = random_film(w, h, 10)
    d = denoise_desc(5, 0.5, 0.3, 0.3)
    rc, ref = mirrors.denoise(w, h, p, d)
    assert rc == L.RAYN_OK
    flat = {k: np.ascontiguousarray(v).reshape(-1) for k, v in p.items()}
    lib = L.lib()
    for in_dev in (False, True):
        for out_dev in (False, True):
            for alias in (False, True):
                src = {k: (torch.from_numpy(v.copy()).cuda() if in_dev else v.copy()) for k, v in flat.items()}
                if alias and in_dev == out_dev:
                    dst = src
                elif alias:
                    continue
                else:
                    dst = {k: (torch.full((v.size,), float("nan"), device="cuda") if out_dev else np.full_like(v, np.nan))
                           for k, v in flat.items() if k in COLOR_CH}

                def ptr(t):
                    return t.data_ptr() if isinstance(t, torch.Tensor) else t.ctypes.data
                pin = L.RaynFilmPlanes(ptr(src["color"]), ptr(src["alpha"]), ptr(src["background"]), ptr(src["normal"]),
                                       L.MEM_DEVICE if in_dev else L.MEM_HOST)
                pout = L.RaynFilmPlanes(ptr(dst["color"]), None, ptr(dst["background"]), None, L.MEM_DEVICE if out_dev else L.MEM_HOST)
                torch.cuda.synchronize()
                L.check(lib.rayn_b200_film_denoise(renderer.ctx, C.byref(d), w, h, C.byref(pin), C.byref(pout)), renderer.ctx)
                L.check(lib.rayn_b200_sync(renderer.ctx), renderer.ctx)
                for k in COLOR_CH:
                    got = dst[k].cpu().numpy() if isinstance(dst[k], torch.Tensor) else dst[k]
                    assert_bit_equal(got, ref[k], f"in_dev={in_dev} out_dev={out_dev} alias={alias} {k}")


@pytest.mark.parametrize("n,res,samples,mb", [(1, (64, 48), 1, 2), (3, (64, 48), 2, 4), (4, (48, 40), 1, 3)])
def test_rendered_films_bit_equal(renderer, n, res, samples, mb):
    c, inp = small_config(n, res, samples, mb)
    renderer.upload_scene(c["world"], c["camera"])
    g = renderer.render_host(inp, (16, 16), c["integrator"], TR)
    check_against_mirror(renderer, g, denoise_desc(5), res[0], res[1], f"cfg{n}")


def test_full_size_config3_film_bit_equal(renderer):
    """A full-size 1920x1080 config 3 film rendered on the GPU at 4 spp; the mirror only filters it."""
    c, inp = small_config(3, (1920, 1080), 1, 8)
    renderer.upload_scene(c["world"], c["camera"])
    g = renderer.render_host(inp, (16, 16), c["integrator"], TR)
    check_against_mirror(renderer, g, denoise_desc(5), 1920, 1080, "cfg3 1920x1080")


def test_film_denoise_in_place(renderer):
    c = configs.baseline_config(3, res=(40, 32), samples=1, max_bounces=3)
    f = Film(("color", "alpha", "background", "normal"), (40, 32))
    f.render_frame_into(c["world"], c["camera"], c["integrator"], None, (16, 16), 1, TR, c["samples"])
    before = {k: v.copy() for k, v in f.channels.items()}
    f.denoise(3, sigma_color=0.4)
    rc, o = mirrors.denoise(40, 32, before, denoise_desc(3, 0.4))
    for k in COLOR_CH:
        assert f.channels[k].shape == (32, 40, 3)
        assert_bit_equal(f.channels[k].reshape(-1), o[k], f"Film.denoise {k}")
    for k in ("alpha", "normal"):
        assert_bit_equal(f.channels[k], before[k], f"guide {k} untouched")


def test_bad_arguments_are_rejected(renderer):
    p = random_film(8, 8, 11)
    good = denoise_desc(3, 0.5, 0.5, 0.5)
    assert _call(renderer, p, good, 8, 8) == L.RAYN_OK
    for missing in ("normal", "alpha"):
        assert _call(renderer, {k: v for k, v in p.items() if k != missing}, good, 8, 8) == L.RAYN_ERR_INVALID_ARG
    for field, value in [("iterations", 0), ("iterations", 9), ("iterations", -1), ("sigma_color", 0.0), ("sigma_color", -0.5),
                         ("sigma_normal", float("nan")), ("sigma_alpha", 0.0), ("sigma_alpha", -np.inf), ("sigma_color", 1e-30)]:
        d = denoise_desc(3, 0.5, 0.5, 0.5)
        setattr(d, field, value)
        assert _call(renderer, p, d, 8, 8) == L.RAYN_ERR_INVALID_ARG, (field, value)
    assert _call(renderer, p, good, 0, 8) == L.RAYN_ERR_INVALID_ARG
    pin = L.RaynFilmPlanes(p["color"].ctypes.data, p["alpha"].ctypes.data, None, p["normal"].ctypes.data, L.MEM_HOST)
    pout = L.RaynFilmPlanes(None, None, None, None, L.MEM_HOST)  # color given without an output plane
    assert L.lib().rayn_b200_film_denoise(renderer.ctx, C.byref(good), 8, 8, C.byref(pin), C.byref(pout)) == L.RAYN_ERR_INVALID_ARG
    assert _call(renderer, p, good, 8, 8) == L.RAYN_OK  # the context still works


def test_exp_zero_weight_cutoff_on_the_device(renderer):
    """rt_denoise.cuh skips taps with e > 103.972076f as weight +0: dm::exp must return +0 for EVERY float argument at or
    below -103.972084f.  Every float in [-111, -103.972084] is evaluated on the device (below -110 dm::exp clamps to -110)."""
    lo, hi = np.float32(-103.972084).view(np.uint32), np.float32(-111.0).view(np.uint32)
    assert lo == 0xc2cff1b5
    x = np.arange(lo, hi + 1, dtype=np.uint32).view(np.float32)
    x = np.concatenate([x, np.float32([-np.inf, -3.4e38, -1e30, -200.0])])
    out = renderer.kat_detmath(0, x)
    assert (out.view(np.uint32) == 0).all(), x[out.view(np.uint32) != 0][:5]
    edge = renderer.kat_detmath(0, np.float32([-103.972076, -0.0, 0.0]))
    assert edge[0] > 0  # the cutoff is tight: the next float up gives the smallest denormal
    assert (edge[1:].view(np.uint32) == np.float32(1.0).view(np.uint32)).all()  # the centre tap's weight is exactly h*h


def test_denoised_low_spp_is_closer_to_high_spp(renderer):
    """Config 3 at 96x96: col+bg denoised at 4 spp has lower MSE against a 256 spp render than the raw 4 spp image."""
    def render(samples):
        c, inp = small_config(3, (96, 96), samples, 8)
        renderer.upload_scene(c["world"], c["camera"])
        return renderer.render_host(inp, (16, 16), c["integrator"], TR)
    lo, hi = render(1), render(64)
    den = renderer.denoise(96, 96, lo)
    target = hi["color"] + hi["background"]
    mse_raw = float(np.mean((lo["color"] + lo["background"] - target).astype(np.float64) ** 2))
    mse_den = float(np.mean((den["color"] + den["background"] - target).astype(np.float64) ** 2))
    print(f"cfg3 96x96: MSE vs 256 spp raw 4 spp {mse_raw:.6g}, denoised {mse_den:.6g}, ratio {mse_den / mse_raw:.4f}")
    assert mse_den < mse_raw


def test_rendering_is_unchanged_by_a_denoise(renderer):
    from test_cpu_oracle import GOLD, GOLD_SUFFIX, GOLDEN_CASES
    name = "cfg3_32x32_8spp_3b"
    n, res, samples, mb = GOLDEN_CASES[name]
    gold = np.load(os.path.join(GOLD, name + GOLD_SUFFIX + ".npz"))
    c, inp = small_config(n, res, samples, mb)
    renderer.upload_scene(c["world"], c["camera"])
    before = renderer.render_host(inp, (16, 16), c["integrator"], TR)
    renderer.denoise(res[0], res[1], before)
    renderer.denoise(513, 257, random_film(513, 257, 12))
    after = renderer.render_host(inp, (16, 16), c["integrator"], TR)
    for ch in CH:
        assert_bit_equal(before[ch], gold[ch], f"before {ch}")
        assert_bit_equal(after[ch], gold[ch], f"after {ch}")


def test_cpp_host_denoise_flag(tmp_path):
    from rayn_b200 import build
    exe = os.path.join(os.path.dirname(build.OUT), "rayn_host")
    args = [exe, "--config", "3", "--res", "48", "32", "--samples", "1", "--bounces", "3"]
    subprocess.run(args + ["--dump", str(tmp_path / "raw.bin")], capture_output=True, text=True, check=True)
    subprocess.run(args + ["--denoise", "4", "--dump", str(tmp_path / "den.bin")], capture_output=True, text=True, check=True)
    npx = 48 * 32

    def planes(path):
        raw = np.fromfile(path, np.float32)
        return {"color": raw[:3 * npx], "alpha": raw[3 * npx:4 * npx], "background": raw[4 * npx:7 * npx], "normal": raw[7 * npx:]}
    raw, den = planes(tmp_path / "raw.bin"), planes(tmp_path / "den.bin")
    rc, o = mirrors.denoise(48, 32, raw, denoise_desc(4))
    assert rc == L.RAYN_OK
    for k in COLOR_CH:
        assert_bit_equal(den[k], o[k], f"rayn_host --denoise {k}")
    for k in ("alpha", "normal"):
        assert_bit_equal(den[k], raw[k], f"rayn_host --denoise leaves {k}")


@pytest.mark.skipif(L.MULADD_FUSED or L.LEGACY, reason="already inside a variant run")
def test_fused_mul_add_variant_denoise_bit_equal():
    """librayn_b200_fma.so against the mirror built in the same mul_add mode."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "pytest", "-x", "-q", "-m", "gpu", "-p", "no:cacheprovider", "tests/test_gpu_denoise.py",
                        "-k", "not variant and not full_size and not cpp_host"], cwd=root, env=dict(os.environ, RAYN_MULADD_FUSED="1"),
                       capture_output=True, text=True)
    assert r.returncode == 0 and " passed" in r.stdout, r.stdout[-3000:] + r.stderr[-1500:]
