"""The film denoiser's CPU mirror (tests/film_mirror.cpp) against the properties of the a-trous statement and an
independent float64 numpy restatement; the ABI struct layout; Film.denoise's argument check.  No GPU needed."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from rayn_b200 import _lib as L
from rayn_b200.film import Film, denoise_desc

import mirrors

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H5 = np.array([0.0625, 0.25, 0.375, 0.25, 0.0625])


def random_film(w, h, seed):
    rng = np.random.default_rng(seed)
    n = rng.normal(size=(h, w, 3))
    n /= np.linalg.norm(n, axis=2, keepdims=True)
    return {"color": rng.uniform(0.1, 1.0, (h, w, 3)).astype(np.float32), "background": rng.uniform(0.1, 2.0, (h, w, 3)).astype(np.float32),
            "normal": n.astype(np.float32), "alpha": (rng.uniform(size=(h, w)) < 0.7).astype(np.float32)}


def mirror(planes, desc):
    h, w = planes["normal"].shape[:2]
    rc, out = mirrors.denoise(w, h, planes, desc)
    assert rc == L.RAYN_OK
    return {k: v.reshape(h, w, 3) for k, v in out.items()}


def numpy_f64(planes, key, iterations, sc, sn, sa):
    """The statement in float64: weights h*h*exp(-e), taps outside the image dropped (all inputs finite)."""
    c = planes[key].astype(np.float64)
    n, a = planes["normal"].astype(np.float64), planes["alpha"].astype(np.float64)
    hh, ww = a.shape
    for i in range(iterations):
        s = 2 ** i
        ic, inn, ia = 2.0 ** i / sc ** 2, 1.0 / sn ** 2, 1.0 / sa ** 2
        num, den = np.zeros_like(c), np.zeros((hh, ww))
        for dy in range(-2, 3):
            for dx in range(-2, 3):
                ys, xs = np.arange(hh) + s * dy, np.arange(ww) + s * dx
                vy, vx = (ys >= 0) & (ys < hh), (xs >= 0) & (xs < ww)
                valid = vy[:, None] & vx[None, :]
                yq, xq = np.clip(ys, 0, hh - 1), np.clip(xs, 0, ww - 1)
                cq, nq, aq = c[yq][:, xq], n[yq][:, xq], a[yq][:, xq]
                e = ((cq - c) ** 2).sum(2) * ic + ((nq - n) ** 2).sum(2) * inn + (aq - a) ** 2 * ia
                wgt = np.where(valid, H5[dy + 2] * H5[dx + 2] * np.exp(-e), 0.0)
                num += wgt[:, :, None] * cq
                den += wgt
        c = num / den[:, :, None]
    return c


def test_exp_of_minus_zero_is_exactly_one():
    """The centre tap has e = 0; dm::exp(-0.0f) must be exactly 1.0f, so the centre weight is h*h and sum w > 0."""
    assert mirrors.exp(np.float32(-0.0)).view(np.uint32) == np.float32(1.0).view(np.uint32)
    assert mirrors.exp(np.float32(0.0)).view(np.uint32) == np.float32(1.0).view(np.uint32)


def test_constant_image_stays_constant():
    p = random_film(29, 17, 1)
    p["color"][:] = np.float32([0.3, 0.7, 1.9])
    p["background"][:] = np.float32(0.05)
    out = mirror(p, denoise_desc(5, 0.2, 0.3, 0.4))
    for k in ("color", "background"):
        np.testing.assert_allclose(out[k], p[k], rtol=1e-6, atol=0)


def _split_matches_halves(p, axis, desc):
    full = mirror(p, desc)
    k = p["alpha"].shape[axis] // 2 + 1
    for sl in ((slice(None, k),), (slice(k, None),)):
        idx = sl if axis == 0 else (slice(None),) + sl
        part = mirror({c: np.ascontiguousarray(v[idx]) for c, v in p.items()}, desc)
        for c in ("color", "background"):
            assert np.array_equal(full[c][idx].view(np.uint32), part[c].view(np.uint32)), (axis, sl, c)


@pytest.mark.parametrize("iterations", [1, 3, 5])
def test_normal_edge_does_not_mix(iterations):
    """Opposite normals on either side of a vertical edge: with sigma_normal = 0.1, e >= 4 * 100 across it, every
    cross-edge weight is +0, so each side is exactly the filter of that side alone."""
    p = random_film(23, 19, 2)
    p["alpha"][:] = 1.0
    p["normal"][:] = [0.0, 0.0, 1.0]
    p["normal"][:, 23 // 2 + 1:] = [0.0, 0.0, -1.0]
    _split_matches_halves(p, 1, denoise_desc(iterations, 0.5, 0.1, np.inf))


@pytest.mark.parametrize("iterations", [1, 3, 5])
def test_alpha_edge_does_not_mix(iterations):
    p = random_film(21, 26, 3)
    p["normal"][:] = [0.0, 1.0, 0.0]
    p["alpha"][:] = 0.0
    p["alpha"][26 // 2 + 1:] = 1.0
    _split_matches_halves(p, 0, denoise_desc(iterations, 0.5, np.inf, 0.05))


def test_non_finite_pixels_pass_through_and_do_not_leak():
    p = random_film(31, 27, 4)
    bad = [(3, 4, 0, np.nan), (10, 10, 1, np.inf), (20, 5, 2, -np.inf), (26, 30, 0, np.nan), (0, 0, 1, np.inf)]
    for y, x, ch, v in bad:
        p["color"][y, x, ch] = v
        p["background"][y, x, ch] = v
    out = mirror(p, denoise_desc(5, 0.5, 0.3, 0.3))
    mask = np.zeros((27, 31), bool)
    for y, x, _, _ in bad:
        mask[y, x] = True
    for k in ("color", "background"):
        assert np.array_equal(out[k][mask].view(np.uint32), p[k][mask].view(np.uint32))
        assert np.isfinite(out[k][~mask]).all()


@pytest.mark.parametrize("w,h", [(37, 23), (1, 41), (41, 1), (1, 1)])
def test_mirror_agrees_with_float64_numpy(w, h):
    p = random_film(w, h, 5 + w)
    sc, sn, sa = 0.5, 0.4, 0.6
    out = mirror(p, denoise_desc(3, sc, sn, sa))
    for k in ("color", "background"):
        ref = numpy_f64(p, k, 3, sc, sn, sa)
        np.testing.assert_allclose(out[k], ref, rtol=1e-5, atol=0)


def test_infinite_sigmas_give_the_plain_a_trous_smoothing():
    p = random_film(19, 13, 6)
    out = mirror(p, denoise_desc(2, np.inf, np.inf, np.inf))
    ref = numpy_f64(p, "color", 2, np.inf, np.inf, np.inf)
    np.testing.assert_allclose(out["color"], ref, rtol=1e-6, atol=0)


@pytest.mark.parametrize("field,value", [("iterations", 0), ("iterations", 9), ("sigma_color", 0.0), ("sigma_normal", -1.0),
                                         ("sigma_alpha", float("nan")), ("sigma_color", 1e-30)])
def test_mirror_rejects_bad_descriptors(field, value):
    d = denoise_desc(3, 0.5, 0.5, 0.5)
    setattr(d, field, value)
    rc, _ = mirrors.denoise(4, 4, random_film(4, 4, 7), d)
    assert rc == L.RAYN_ERR_INVALID_ARG


def test_denoise_desc_layout_matches_the_c_compiler(tmp_path):
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "rayn_b200.h"\nint main(){'
                   'printf("%zu %zu %zu %zu %zu\\n", sizeof(RaynDenoiseDesc), offsetof(RaynDenoiseDesc, iterations), '
                   'offsetof(RaynDenoiseDesc, sigma_color), offsetof(RaynDenoiseDesc, sigma_normal), offsetof(RaynDenoiseDesc, sigma_alpha));'
                   'return 0;}')
    exe = tmp_path / "sz"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    D = L.RaynDenoiseDesc
    assert got == [C.sizeof(D), D.iterations.offset, D.sigma_color.offset, D.sigma_normal.offset, D.sigma_alpha.offset]


def test_film_denoise_needs_the_guide_channels():
    f = Film(("color", "background"), (8, 8))
    f.channels = {"color": np.zeros((8, 8, 3), np.float32), "background": np.zeros((8, 8, 3), np.float32)}
    with pytest.raises(ValueError):
        f.denoise()
