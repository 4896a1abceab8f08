"""CPU mirrors of the luminance-moment render (tests/render_mirror.cpp) and of the variance-guided denoise
(tests/film_mirror.cpp): the mirror's film planes against the render oracle, lum2 >= lum(mean)^2, every denoise entry point
against a numpy float32 restatement of the header's statement, the +inf identity against the plain and albedo-guided entry
points, the argument rules, the RaynMomentPlanes layout and the Film checks that need no GPU."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from rayn_b200 import _lib as L
from rayn_b200 import configs
from rayn_b200.film import Film, denoise_desc
from rayn_b200.scene import OrbitTrapAlbedo

import mirrors
from helpers import assert_bit_equal, small_config
from test_cpu_denoise import random_film
from test_cpu_trap import ALBEDO_HI, ALBEDO_LO, TRAP_HI, TRAP_LO, with_fractal_albedo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TR = configs.frame_time_range(1)
f32 = np.float32


def lum(x):
    x = np.asarray(x, f32)
    return (f32(0.2126) * x[..., 0] + f32(0.7152) * x[..., 1]) + f32(0.0722) * x[..., 2]


@pytest.mark.parametrize("n", [1, 2, 3, 4])
def test_film_planes_equal_the_oracle(oracle, n):
    """the mirror only adds the lum^2 fold: its film planes are the render oracle's bit for bit"""
    c, inp = small_config(n, (19, 11), 2, 2)
    m = mirrors.render(c["world"], c["camera"], inp, (8, 8), c["integrator"], TR, moments=True)[0]
    o, _ = oracle.render(c["world"], c["camera"], inp, (8, 8), c["integrator"], TR)
    for k in ("color", "alpha", "background", "normal"):
        assert_bit_equal(m[k], o[k], f"cfg{n} {k}")
    assert m["moments"].shape == (11, 19, 2)


def test_film_planes_equal_the_oracle_under_motion(oracle):
    """a panning camera and a moving sphere over the frame's shutter: the camera packets' times are the oracle's, so the
    films are equal bit for bit, and the motion shows in them"""
    from rayn_b200.scene import Linear, Vec3
    from test_cpu_motion_prev import sphere_world
    from test_cpu_temporal import moving_cameras
    c, inp = small_config(3, (19, 11), 2, 2)
    sphere_world(c, Linear(Vec3(-1.0, 0.4, 0.9), Vec3(4.0, 0.0, 1.0)), 0.35)
    pan = moving_cameras(c, (19, 11))["pan"]
    m = mirrors.render(c["world"], pan, inp, (8, 8), c["integrator"], TR, moments=True)[0]
    o, _ = oracle.render(c["world"], pan, inp, (8, 8), c["integrator"], TR)
    for k in ("color", "alpha", "background", "normal"):
        assert_bit_equal(m[k], o[k], f"moving {k}")
    still, _ = oracle.render(c["world"], pan, inp, (8, 8), c["integrator"], (TR[0], TR[0]))
    assert not np.array_equal(o["color"], still["color"])


@pytest.mark.parametrize("n", [1, 2, 3, 4])
def test_second_moment_bounds_the_squared_mean(n):
    """mean of squares >= square of the mean (Jensen), within float rounding, on every pixel of colour and background"""
    c, inp = small_config(n, (21, 13), 4, 2)
    if n == 3:
        with_fractal_albedo(c, OrbitTrapAlbedo(TRAP_LO, TRAP_HI, ALBEDO_LO, ALBEDO_HI))
    m = mirrors.render(c["world"], c["camera"], inp, (8, 8), c["integrator"], TR, moments=True)[0]
    for i, k in enumerate(("color", "background")):
        lm = lum(m[k].reshape(13, 21, 3)).astype(np.float64)
        l2 = m["moments"][:, :, i].astype(np.float64)
        assert (l2 >= 0).all()
        assert (l2 >= lm * lm * (1 - 2e-6) - 1e-30).all(), f"cfg{n} {k}"
    assert m["moments"][:, :, 0].any() or m["moments"][:, :, 1].any()


def test_tile_grid_quirk_leaves_zeros():
    """film.rs:399-404: a 20-wide film with 16-wide tiles has one tile column; pixels 16..19 stay 0"""
    c, inp = small_config(3, (20, 9), 1, 1)
    m = mirrors.render(c["world"], c["camera"], inp, (16, 16), c["integrator"], TR, moments=True)[0]
    assert (m["moments"][:, 16:] == 0).all() and m["moments"][:, :16].any()


def test_golden_film_planes_are_the_trap_golden():
    """the moments golden holds the same film as cfg3_trap_32x32_8spp_3b (same scene, same mirror family)"""
    from test_cpu_oracle import GOLD, GOLD_SUFFIX
    g = np.load(os.path.join(GOLD, "cfg3_moments_32x32_8spp" + GOLD_SUFFIX + ".npz"))
    t = np.load(os.path.join(GOLD, "cfg3_trap_32x32_8spp_3b" + GOLD_SUFFIX + ".npz"))
    for k in ("color", "alpha", "background", "normal"):
        assert_bit_equal(g[k], t[k], k)
    assert g["moments"].shape == (32, 32, 2) and g["moments"].any()


# ---- the variance-guided filter -------------------------------------------------------------------------------------
def moment_film(w, h, seed):
    """random_film plus moment planes: lum(c)^2 plus a random spread, a few pixels below lum(c)^2 (clamped to v = 0)"""
    p = random_film(w, h, seed)
    rng = np.random.default_rng(seed + 1)
    m = np.empty((h, w, 2), f32)
    for i, k in enumerate(("color", "background")):
        l = lum(p[k])
        m[:, :, i] = l * l + rng.uniform(-0.05, 1.0, (h, w)).astype(f32) * rng.uniform(0, 1, (h, w)).astype(f32)
    return p, m


def np_variance(planes, key, moments, spp, iters, sc, sn, sa, sl, albedo=None, sal=np.inf, scale=None):
    """The header's statement of rayn_b200_film_denoise_variance in numpy float32, per tap in tap order.  scale (float32
    [H, W]): rayn_b200_film_denoise_variance_scaled's per-pixel variance scale of level 0.  sl = +inf: the luminance term is
    not added, which with albedo None is rayn_b200_film_denoise's statement and with albedo rayn_b200_film_denoise_albedo's
    (moments may then be None)."""
    vexp = np.vectorize(lambda x: mirrors.exp(f32(x)), otypes=[f32])
    c = np.asarray(planes[key], f32).copy()
    H, W = c.shape[:2]
    nrm, a = np.asarray(planes["normal"], f32), np.asarray(planes["alpha"], f32)
    ic0, in_, ia = (f32(1) / (f32(s) * f32(s)) for s in (sc, sn, sa))
    il = f32(0) if albedo is None or np.isinf(sal) else f32(1) / (f32(sal) * f32(sal))
    alb = None if albedo is None else np.asarray(albedo, f32).reshape(H, W, 3)
    var = not np.isinf(sl)
    l0 = lum(c)
    v = np.zeros((H, W), f32) if moments is None else np.fmax(np.asarray(moments, f32)[:, :, 0 if key == "color" else 1] - l0 * l0, f32(0))
    v = (v if scale is None else v * np.asarray(scale, f32).reshape(H, W)) / f32(spp)
    yy, xx = np.mgrid[0:H, 0:W]
    h5, k3 = [f32(x) for x in (0.0625, 0.25, 0.375, 0.25, 0.0625)], [f32(0.25), f32(0.5), f32(0.25)]

    def tap(step, dy, dx):
        qy, qx = yy + step * dy, xx + step * dx
        inside = (qy >= 0) & (qy < H) & (qx >= 0) & (qx < W)
        qy, qx = np.clip(qy, 0, H - 1), np.clip(qx, 0, W - 1)
        return inside & np.isfinite(c[qy, qx]).all(axis=2), qy, qx

    with np.errstate(all="ignore"):
        for i in range(iters):
            step, ic = 1 << i, f32(ic0 * f32(2.0 ** i))
            fin = np.isfinite(c).all(axis=2)
            gs, gw = np.zeros((H, W), f32), np.zeros((H, W), f32)
            for dy in (-1, 0, 1):
                for dx in (-1, 0, 1):
                    ok, qy, qx = tap(1, dy, dx)
                    kk = k3[dy + 1] * k3[dx + 1]
                    gs, gw = np.where(ok, gs + kk * v[qy, qx], gs), np.where(ok, gw + kk, gw)
            ilp = f32(1) / (f32(sl) * np.sqrt(gs / gw) + f32(1e-10))
            lp = lum(c)
            sr, sg, sb, sw, sv = (np.zeros((H, W), f32) for _ in range(5))
            for dy in range(-2, 3):
                for dx in range(-2, 3):
                    ok, qy, qx = tap(step, dy, dx)
                    cq = c[qy, qx]
                    d = cq - c
                    dc2 = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
                    dn = nrm[qy, qx] - nrm
                    dn2 = (dn[..., 0] * dn[..., 0] + dn[..., 1] * dn[..., 1]) + dn[..., 2] * dn[..., 2]
                    da = a[qy, qx] - a
                    e = (dc2 * ic + dn2 * in_) + (da * da) * ia
                    if il != 0:
                        dl = alb[qy, qx] - alb
                        e = e + ((dl[..., 0] * dl[..., 0] + dl[..., 1] * dl[..., 1]) + dl[..., 2] * dl[..., 2]) * il
                    if var:
                        e = e + np.abs(lum(cq) - lp) * ilp
                    ok = ok & ~np.isnan(e)
                    w = (h5[dy + 2] * h5[dx + 2]) * vexp(np.where(ok, -e, f32(0)))
                    sr, sg, sb = (np.where(ok, s + w * cq[..., j], s) for j, s in enumerate((sr, sg, sb)))
                    sw = np.where(ok, sw + w, sw)
                    ww = w * w
                    sv = np.where(ok & (ww != 0), sv + ww * v[qy, qx], sv)
            new = np.stack([sr / sw, sg / sw, sb / sw], axis=2)
            c = np.where(fin[..., None], new, c)
            v = np.where(fin, sv / (sw * sw), v)
    return c


@pytest.mark.parametrize("w,h,iters,sl,with_albedo", [(9, 7, 3, 2.0, False), (6, 11, 2, 0.5, True), (1, 1, 1, 1.0, False),
                                                      (13, 5, 4, 8.0, True)])
def test_mirror_matches_the_numpy_statement(w, h, iters, sl, with_albedo):
    p, m = moment_film(w, h, 7 + w)
    p["color"][h // 2, w // 2, 1] = np.nan  # a non-finite pixel is copied and skipped as a tap
    alb = np.random.default_rng(3).uniform(0, 1, (h, w, 3)).astype(f32) if with_albedo else None
    desc = denoise_desc(iters, 2.5, 0.4, 0.5)
    rc, out = mirrors.denoise(w, h, p, desc, alb, 0.3, moments=m, spp=16, sigma_luminance=sl)
    assert rc == L.RAYN_OK
    for k in ("color", "background"):
        ref = np_variance(p, k, m, 16, iters, 2.5, 0.4, 0.5, sl, alb, 0.3)
        assert_bit_equal(out[k].reshape(h, w, 3), ref, f"{k} {w}x{h} L={iters}")


@pytest.mark.parametrize("w,h,iters,with_albedo", [(9, 7, 3, False), (13, 5, 4, True), (1, 1, 1, False)])
def test_scaled_mirror_matches_the_numpy_statement(w, h, iters, with_albedo):
    """rayn_b200_film_denoise_variance_scaled's mirror against the numpy statement with a per-pixel scale: random scales,
    0, 1e-30 and 1e30 next to unit ones"""
    p, m = moment_film(w, h, 31 + w)
    p["color"][h // 2, w // 2, 0] = np.inf
    rng = np.random.default_rng(w * h)
    scale = rng.choice(np.array([0.0, 1e-30, 1e30, 1.0, 1.0], f32), (h, w))
    scale = np.where(rng.uniform(size=(h, w)) < 0.4, rng.uniform(0.0, 3.0, (h, w)).astype(f32), scale).astype(f32)
    alb = rng.uniform(0, 1, (h, w, 3)).astype(f32) if with_albedo else None
    desc = denoise_desc(iters, 2.5, 0.4, 0.5)
    rc, out = mirrors.denoise(w, h, p, desc, alb, 0.3, moments=m, spp=16, sigma_luminance=1.5, var_scale=scale)
    assert rc == L.RAYN_OK
    for k in ("color", "background"):
        ref = np_variance(p, k, m, 16, iters, 2.5, 0.4, 0.5, 1.5, alb, 0.3, scale=scale)
        assert_bit_equal(out[k].reshape(h, w, 3), ref, f"{k} {w}x{h} L={iters}")
        if w * h > 1:  # the scale reaches the result
            assert not np.array_equal(ref, np_variance(p, k, m, 16, iters, 2.5, 0.4, 0.5, 1.5, alb, 0.3)), k


@pytest.mark.parametrize("w,h,iters", [(9, 7, 3), (13, 5, 4), (1, 1, 1)])
@pytest.mark.parametrize("with_albedo", [False, True])
def test_plain_and_albedo_mirrors_match_the_numpy_statement(w, h, iters, with_albedo):
    """rayn_b200_film_denoise's and rayn_b200_film_denoise_albedo's mirrors against np_variance without the luminance term,
    bit for bit, with non-finite pixels (the variance entry points are checked above)"""
    p, _ = moment_film(w, h, 41 + w)
    p["color"][h // 2, w // 2, 1] = np.nan
    p["background"][0, w - 1, 2] = -np.inf
    alb = np.random.default_rng(w * h + iters).uniform(0, 1, (h, w, 3)).astype(f32) if with_albedo else None
    rc, out = mirrors.denoise(w, h, p, denoise_desc(iters, 2.5, 0.4, 0.5), alb, 0.3)
    assert rc == L.RAYN_OK
    for k in ("color", "background"):
        ref = np_variance(p, k, None, 1, iters, 2.5, 0.4, 0.5, np.inf, alb, 0.3)
        assert_bit_equal(out[k].reshape(h, w, 3), ref, f"{k} {w}x{h} L={iters} albedo={with_albedo}")


def test_variance_term_changes_the_result():
    p, m = moment_film(12, 10, 5)
    desc = denoise_desc(3, 2.5, 0.4, 0.5)
    _, a = mirrors.denoise(12, 10, p, desc, moments=m, spp=4, sigma_luminance=1.0)
    _, b = mirrors.denoise(12, 10, p, desc, moments=m, spp=4, sigma_luminance=np.inf)
    assert not np.array_equal(a["color"], b["color"])


@pytest.mark.parametrize("iters", [1, 5])
def test_infinite_sigma_luminance_is_the_existing_filters(iters):
    """sigma_luminance = +inf: film_denoise (albedo NULL) or film_denoise_albedo bit for bit"""
    p, m = moment_film(15, 9, 11)
    alb = np.random.default_rng(2).uniform(0, 1, (9, 15, 3)).astype(f32)
    desc = denoise_desc(iters)
    rc, out = mirrors.denoise(15, 9, p, desc, moments=m, spp=4, sigma_luminance=np.inf)
    assert rc == L.RAYN_OK
    rc0, ref = mirrors.denoise(15, 9, p, desc)
    assert rc0 == L.RAYN_OK
    rc, out_a = mirrors.denoise(15, 9, p, desc, alb, 0.2, moments=m, spp=4, sigma_luminance=np.inf)
    rc1, ref_a = mirrors.denoise(15, 9, p, desc, alb, 0.2)
    assert rc == rc1 == L.RAYN_OK
    for k in ("color", "background"):
        assert_bit_equal(out[k], ref[k], k)
        assert_bit_equal(out_a[k], ref_a[k], k + " albedo")


def test_mirror_argument_rules():
    p, m = moment_film(5, 4, 1)
    desc = denoise_desc(2)
    assert mirrors.denoise(5, 4, p, desc, moments=m, spp=0, sigma_luminance=1.0)[0] == L.RAYN_ERR_INVALID_ARG  # spp < 1
    for bad in (0.0, -1.0, np.nan):
        assert mirrors.denoise(5, 4, p, desc, moments=m, spp=4, sigma_luminance=bad)[0] == L.RAYN_ERR_INVALID_ARG
    assert mirrors.denoise(5, 4, p, desc, np.zeros((4, 5, 3), f32), 0.0, moments=m, spp=4, sigma_luminance=1.0)[0] == L.RAYN_ERR_INVALID_ARG  # bad sigma_albedo
    # a colour plane without its moment plane
    flat = {k: np.ascontiguousarray(v, f32).reshape(-1) for k, v in p.items()}
    out = {k: np.empty_like(flat[k]) for k in ("color", "background")}
    pin = L.RaynFilmPlanes(flat["color"].ctypes.data, flat["alpha"].ctypes.data, flat["background"].ctypes.data, flat["normal"].ctypes.data, 0)
    pout = L.RaynFilmPlanes(out["color"].ctypes.data, None, out["background"].ctypes.data, None, 0)
    mc = np.ascontiguousarray(m[:, :, 0]).reshape(-1)
    mp = L.RaynMomentPlanes(mc.ctypes.data, None, 0)
    rc = mirrors.film_lib().rayn_oracle_film_denoise_variance(C.byref(desc), 1.0, 4, C.byref(mp), 1.0, None, 5, 4, C.byref(pin), C.byref(pout))
    assert rc == L.RAYN_ERR_INVALID_ARG


def test_moment_planes_layout_matches_the_c_compiler(tmp_path):
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "rayn_b200.h"\nint main(){'
                   'printf("%zu %zu %zu %zu\\n", sizeof(RaynMomentPlanes), offsetof(RaynMomentPlanes, color_lum2),'
                   'offsetof(RaynMomentPlanes, background_lum2), offsetof(RaynMomentPlanes, space));return 0;}')
    exe = tmp_path / "sz"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    M = L.RaynMomentPlanes
    assert got == [C.sizeof(M), M.color_lum2.offset, M.background_lum2.offset, M.space.offset]


def test_film_moments_channel_rules(tmp_path):
    """the accumulator does not fold moments, and the moments channel is not an image"""
    film = Film(["color", "alpha", "moments"], (8, 8))
    with pytest.raises(ValueError):
        film.render_adaptive(None, None, None, None, (8, 8), 1, (0.0, 1.0), 1)
    film.channels["moments"] = np.zeros((8, 8, 2), f32)
    with pytest.raises(ValueError):
        film.save_to(["moments"], str(tmp_path), "x")


def test_cpp_host_denoise_variance_argument_rules():
    """rayn_host rejects --denoise-variance without --denoise L and together with --adaptive (before any GPU work)"""
    from rayn_b200 import build
    exe = os.path.join(os.path.dirname(build.OUT), "rayn_host")
    for extra in (["--denoise-variance"], ["--denoise", "3", "--denoise-variance", "--adaptive", "0.05"],
                  ["--denoise-albedo", "--denoise-variance"]):
        r = subprocess.run([exe, "--config", "3"] + extra, capture_output=True, text=True)
        assert r.returncode == 2, (extra, r.stderr)
