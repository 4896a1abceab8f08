"""CPU mirrors of the first-hit albedo plane (tests/render_mirror.cpp) and of the albedo-guided denoise
(tests/film_mirror.cpp): the resolve against numpy, the alpha identity against the render oracle, the guided filter
against the unguided entry point at sigma_albedo = +inf, albedo edges that do not mix, and the skip rules for non-finite albedo."""
import numpy as np
import pytest

from rayn_b200 import _lib as L
from rayn_b200 import configs
from rayn_b200.film import denoise_desc
from rayn_b200.scene import Dielectric, Lambertian, OrbitTrapAlbedo

import mirrors
from helpers import assert_bit_equal, small_config
from test_cpu_denoise import random_film
from test_cpu_trap import ALBEDO_HI, ALBEDO_LO, TRAP_HI, TRAP_LO, with_fractal_albedo

TR = configs.frame_time_range(1)
COLOR_CH = ("color", "background")


def white(c):
    """every Lambertian / Dielectric material with albedo (1, 1, 1) and no trap: the albedo plane is the alpha plane"""
    for m in c["world"].materials.items:
        if isinstance(m, (Lambertian, Dielectric)):
            m.albedo, m.albedo_gen = np.ones(3, np.float32), None
    return c


def trap_config(n, res, samples, mb=1):
    c, inp = small_config(n, res, samples, mb)
    return with_fractal_albedo(c, OrbitTrapAlbedo(TRAP_LO, TRAP_HI, ALBEDO_LO, ALBEDO_HI)), inp


def mirror_albedo(c, inp, tile=(16, 16)):
    return mirrors.render_albedo(c["world"], c["camera"], inp, tile, c["integrator"], TR)


@pytest.mark.parametrize("n", [1, 3, 4])
def test_resolve_matches_numpy(n):
    """the plane is the float32 sum of the per-sample albedos in ascending sample order / spp (float64: within rounding)"""
    c, inp = trap_config(n, (21, 13), 2)
    plane, per = mirror_albedo(c, inp, (8, 8))
    spp = inp.spp
    seq = np.add.accumulate(per, axis=2, dtype=np.float32)[:, :, -1, :] / np.float32(spp)  # sequential float32 sums
    assert_bit_equal(plane, seq, f"cfg{n} float32 statement")
    np.testing.assert_allclose(plane.astype(np.float64), per.astype(np.float64).mean(axis=2), rtol=1e-6, atol=1e-7)
    assert (per >= 0).all() and (per <= 1).all()


def test_tile_grid_quirk_leaves_zeros():
    """film.rs:399-404: a 20-wide film with 16-wide tiles has one tile column; pixels 16..19 stay 0"""
    c, inp = trap_config(3, (20, 9), 1)
    plane, per = mirror_albedo(c, inp, (16, 16))
    assert (plane[:, 16:] == 0).all() and (per[:, 16:] == 0).all()
    assert plane[:, :16].any()


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5])
def test_white_albedo_equals_oracle_alpha(oracle, n):
    """with albedo (1, 1, 1) everywhere and no traps, every channel is the render oracle's alpha plane bit for bit"""
    c, inp = small_config(n, (19, 11), 1, 1)
    white(c)
    plane, _ = mirror_albedo(c, inp, (8, 8))
    o, _ = oracle.render(c["world"], c["camera"], inp, (8, 8), c["integrator"], TR)
    alpha = o["alpha"].reshape(11, 19)
    for ch in range(3):
        assert_bit_equal(plane[:, :, ch], alpha, f"cfg{n} channel {ch}")


def test_trap_changes_only_fractal_hits():
    """a trap palette changes a sample's albedo only where the constant-albedo plane saw the fractal's material"""
    c, inp = trap_config(3, (24, 16), 2)
    _, per_trap = mirror_albedo(c, inp)
    c2, _ = small_config(3, (24, 16), 2, 1)
    _, per_const = mirror_albedo(c2, inp)
    changed = (per_trap != per_const).any(axis=3)
    fractal = (per_const == np.asarray(c2["world"].materials.items[1].albedo, np.float32)).all(axis=3)
    assert changed.any() and not (changed & ~fractal).any()


# ---- the albedo-guided filter ---------------------------------------------------------------------------------------
def guided(planes, desc, albedo, sigma):
    h, w = planes["normal"].shape[:2]
    rc, out = mirrors.denoise(w, h, planes, desc, albedo, sigma)
    assert rc == L.RAYN_OK
    return {k: v.reshape(h, w, 3) for k, v in out.items()}


@pytest.mark.parametrize("w,h", [(1, 1), (7, 5), (33, 21)])
def test_infinite_sigma_equals_unguided_mirror(w, h):
    p = random_film(w, h, 30 + w)
    alb = np.random.default_rng(w).uniform(0, 1, (h, w, 3)).astype(np.float32)
    alb[0, 0, 0] = np.nan  # not even a non-finite albedo matters: the term is not added
    for it in (1, 3, 5):
        d = denoise_desc(it, 0.5, 0.3, 0.4)
        rc, ref = mirrors.denoise(w, h, p, d)
        assert rc == L.RAYN_OK
        got = guided(p, d, alb, np.inf)
        for k in COLOR_CH:
            assert_bit_equal(got[k].reshape(-1), ref[k], f"{w}x{h} L={it} {k}")


def test_albedo_edges_do_not_mix():
    """two halves with identical colour statistics, normal and alpha but different albedo: a sharp albedo sigma keeps them
    apart (each half's result is the one of the half filtered alone), the unguided filter mixes them"""
    w, h = 24, 16
    rng = np.random.default_rng(5)
    p = {"color": rng.uniform(0.2, 0.8, (h, w, 3)).astype(np.float32), "background": rng.uniform(0.2, 0.8, (h, w, 3)).astype(np.float32),
         "normal": np.tile(np.float32([0, 0, 1]), (h, w, 1)), "alpha": np.ones((h, w), np.float32)}
    alb = np.zeros((h, w, 3), np.float32)
    alb[:, w // 2:] = (0.9, 0.35, 0.1)
    d = denoise_desc(3, 10.0, 1.0, 1.0)
    both = guided(p, d, alb, 0.01)
    for half in (slice(0, w // 2), slice(w // 2, w)):
        alone = guided({k: np.ascontiguousarray(v[:, half]) for k, v in p.items()}, d, np.ascontiguousarray(alb[:, half]), 0.01)
        for k in COLOR_CH:
            assert_bit_equal(both[k][:, half], alone[k], f"half {half} {k}")
    unguided = guided(p, d, alb, np.inf)
    assert not np.array_equal(unguided["color"][:, : w // 2], both["color"][:, : w // 2])


def test_non_finite_albedo_taps():
    """a tap whose albedo is NaN is skipped (e is NaN), one whose albedo is +inf has weight +0 (e = +inf): with every
    other albedo equal, the result is the filter without those taps; a NaN albedo at the centre skips every tap -> NaN"""
    w, h = 9, 9
    p = random_film(w, h, 3)
    alb = np.full((h, w, 3), 0.5, np.float32)
    d = denoise_desc(1, 0.7, 0.5, 0.5)
    base = guided(p, d, alb, 0.2)
    ref = mirrors.denoise(w, h, p, d)[1]
    for k in COLOR_CH:  # equal albedo everywhere: the term is 0, the unguided result
        assert_bit_equal(base[k].reshape(-1), ref[k], f"equal albedo {k}")
    alb[4, 4, 1] = np.nan
    got = guided(p, d, alb, 0.2)
    assert np.isnan(got["color"][4, 4]).all()
    alb[4, 4, 1] = np.inf
    got_inf = guided(p, d, alb, 0.2)
    assert np.isnan(got_inf["color"][4, 4]).all()  # the centre is dead to every tap but itself: e = inf - inf = NaN there too
    assert_bit_equal(got["color"][0, 0], base["color"][0, 0], "taps out of reach are unchanged")
    changed = ~(got["color"] == base["color"]).all(axis=2)
    assert changed[3:6, 3:6].any() and not changed[:2].any()


def test_argument_errors():
    p = random_film(4, 4, 1)
    alb = np.zeros((4, 4, 3), np.float32)
    for sigma in (0.0, -1.0, np.nan, 1e-30):
        rc, _ = mirrors.denoise(4, 4, p, denoise_desc(2, 0.5, 0.5, 0.5), alb, sigma)
        assert rc == L.RAYN_ERR_INVALID_ARG, sigma
