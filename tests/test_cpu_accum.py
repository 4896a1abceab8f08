"""Sample-range tables (rayn_b200_host_rd_tables_at), the RaynAdaptiveDesc layout, and the numpy mirror of the film
accumulator (tests/accum_mirror.py) against a float64 restatement of the tile error.  No GPU needed."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from rayn_b200 import _lib as L
from rayn_b200.film import FrameInputs, adaptive_desc
from rayn_b200.scene import PathTracingIntegrator

import accum_mirror as am

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _fp(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def tables_at(spp, s1, s2, offset, first):
    a, b = np.full(spp * s1, np.nan, np.float32), np.full(2 * spp * s2, np.nan, np.float32)
    rc = L.host_lib().rayn_b200_host_rd_tables_at(spp, s1, s2, offset, first, _fp(a), _fp(b))
    return rc, a, b


@pytest.mark.parametrize("spp,s1,s2,offset", [(4, 3, 5, 1), (16, 1, 2, 1000), (1, 7, 0, 0), (12, 0, 4, 3)])
def test_first_sample_zero_is_rd_tables(spp, s1, s2, offset):
    a, b = np.empty(spp * s1, np.float32), np.empty(2 * spp * s2, np.float32)
    assert L.host_lib().rayn_b200_host_rd_tables(spp, s1, s2, offset, _fp(a), _fp(b)) == L.RAYN_OK
    rc, a0, b0 = tables_at(spp, s1, s2, offset, 0)
    assert rc == L.RAYN_OK
    assert np.array_equal(a.view(np.uint32), a0.view(np.uint32)) and np.array_equal(b.view(np.uint32), b0.view(np.uint32))


@pytest.mark.parametrize("s0,n", [(4, 4), (8, 16), (48, 12), (3, 5)])
def test_a_range_is_a_slice_of_the_longer_table(s0, n):
    s1, s2, offset = 4, 3, 7
    rc, full1, full2 = tables_at(s0 + n, s1, s2, offset, 0)
    assert rc == L.RAYN_OK
    rc, a, b = tables_at(n, s1, s2, offset, s0)
    assert rc == L.RAYN_OK
    full1, full2 = full1.reshape(s1, s0 + n), full2.reshape(s2, s0 + n, 2)
    for i in range(s1):
        assert np.array_equal(a.reshape(s1, n)[i].view(np.uint32), full1[i, s0:].view(np.uint32)), i
    for i in range(s2):
        assert np.array_equal(b.reshape(s2, n, 2)[i].view(np.uint32), full2[i, s0:].view(np.uint32)), i


def test_the_range_must_end_within_2_pow_32():
    assert tables_at(4, 2, 2, 1, 2 ** 32 - 4)[0] == L.RAYN_OK
    assert tables_at(4, 2, 2, 1, 2 ** 32 - 3)[0] == L.RAYN_ERR_INVALID_ARG
    assert tables_at(1, 1, 1, 1, 2 ** 32)[0] == L.RAYN_ERR_INVALID_ARG
    assert tables_at(1, 1, 1, 1, 2 ** 63)[0] == L.RAYN_ERR_INVALID_ARG


def test_the_last_sample_before_2_pow_32_is_index_2_pow_32():
    """Element n of set i is index ((offset + i) << 32) + first + n + 1: at first + spp = 2^32 the last element of set i
    has index (offset + i + 1) << 32."""
    rc, a, _ = tables_at(2, 2, 0, 5, 2 ** 32 - 2)
    assert rc == L.RAYN_OK
    rc, d, _ = tables_at(1, 1, 0, 5, 2 ** 32 - 1)  # index (5 << 32) + 2^32 = 6 << 32
    rc, c, _ = tables_at(1, 1, 0, 6, 2 ** 32 - 1)  # index 7 << 32
    assert a[1].view(np.uint32) == d[0].view(np.uint32)  # set 0, element 1 of [2^32 - 2, 2^32): index 6 << 32
    assert a[3].view(np.uint32) == c[0].view(np.uint32)  # set 1: index 7 << 32


def test_frame_inputs_first_sample():
    integ = PathTracingIntegrator(3, 2)
    full = FrameInputs(8, 8, 3, integ, frame=2)
    later = FrameInputs(8, 8, 1, integ, frame=2, first_sample=8)
    assert later.first_sample == 8 and FrameInputs(8, 8, 1, integ).first_sample == 0
    f1 = full.samples_1d.reshape(full.sets_1d, 12)[:, 8:]
    assert np.array_equal(later.samples_1d.reshape(later.sets_1d, 4).view(np.uint32), f1.view(np.uint32))
    f2 = full.samples_2d.reshape(full.sets_2d, 12, 2)[:, 8:]
    assert np.array_equal(later.samples_2d.reshape(later.sets_2d, 4, 2).view(np.uint32), f2.view(np.uint32))
    assert np.array_equal(later.scramble, full.scramble)


def test_adaptive_desc_layout_matches_the_c_compiler(tmp_path):
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "rayn_b200.h"\nint main(){'
                   'printf("%zu %zu %zu %zu\\n", sizeof(RaynAdaptiveDesc), offsetof(RaynAdaptiveDesc, min_rounds), '
                   'offsetof(RaynAdaptiveDesc, max_rounds), offsetof(RaynAdaptiveDesc, threshold));return 0;}')
    exe = tmp_path / "sz"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    D = L.RaynAdaptiveDesc
    assert got == [C.sizeof(D), D.min_rounds.offset, D.max_rounds.offset, D.threshold.offset]
    d = adaptive_desc(3, 9, -1.0)
    assert (d.min_rounds, d.max_rounds, d.threshold) == (3, 9, -1.0)


def _random_planes(npx, rng, lo=0.0, hi=2.0):
    return {k: rng.uniform(lo, hi, npx * c).astype(np.float32) for k, c in am.NC.items()}


def _tile_error_f64(m, t):
    """E restated in float64 from the mirror's state (no float32 rounding, plain pairwise sum)."""
    p = m.tile_pixels(t)
    idx3 = (p[:, None] * 3 + np.arange(3)).ravel()
    i = (m.S["color"][idx3].astype(np.float64) + m.S["background"][idx3]).reshape(-1, 3) / m.K[t]
    a = m.H[idx3].astype(np.float64).reshape(-1, 3) / m.Kh[t]
    e = np.abs(i - a).sum(1) / np.sqrt(np.maximum(i.sum(1), 2.0 ** -10))
    return float(e.mean())


@pytest.mark.parametrize("w,h,tw,th", [(37, 23, 16, 16), (64, 48, 8, 8), (40, 24, 16, 16), (5, 3, 2, 2)])
def test_mirror_error_agrees_with_float64(w, h, tw, th):
    rng = np.random.default_rng(w * h)
    m = am.AccumMirror(w, h, tw, th)
    for r in range(5):
        m.fold(_random_planes(w * h, rng), list(range(m.n_tiles)), 1 + r % 2)
        for t in range(m.n_tiles):
            if r == 0:
                assert m.E[t] == np.inf
            else:
                assert m.E[t] == pytest.approx(_tile_error_f64(m, t), rel=1e-5)
    assert (m.K == 4 + 8 + 4 + 8 + 4).all() and (m.Kh == 4 + 4 + 4).all() and (m.rounds == 5).all()


def test_mirror_identical_halves_give_zero_error():
    """Rounds 2k and 2k+1 bring the same film: I = A exactly, so E = 0."""
    rng = np.random.default_rng(1)
    m = am.AccumMirror(32, 32, 16, 16)
    p = _random_planes(32 * 32, rng)
    m.fold(p, list(range(4)), 1)
    m.fold(p, list(range(4)), 1)
    assert (m.E == 0.0).all()


def test_mirror_nan_and_inf_rules():
    m = am.AccumMirror(16, 16, 16, 16)
    rng = np.random.default_rng(2)
    a, b = _random_planes(256, rng), _random_planes(256, rng)
    a["color"][5] = np.nan  # one NaN e: +inf, and the tile's E is +inf
    m.fold(a, [0], 1)
    m.fold(b, [0], 1)
    assert m.E[0] == np.inf
    # s <= 0 is clamped to 2^-10 by fmax (NaN-ignoring): negative radiance still gives a finite e
    m2 = am.AccumMirror(16, 16, 16, 16)
    c, d = _random_planes(256, rng, -1.0, -0.5), _random_planes(256, rng, -1.0, -0.5)
    m2.fold(c, [0], 1)
    m2.fold(d, [0], 1)
    assert np.isfinite(m2.E[0]) and m2.E[0] > 0
    assert am.tile_error(np.float32([[0, 0, 0]]), np.float32([[0, 0, 0]]), np.float32([[0, 0, 0]]), 4, 4) == 0.0


def test_mirror_active_rule():
    m = am.AccumMirror(32, 16, 16, 16)  # 2 tiles
    m.rounds[:] = [2, 2]
    m.E[:] = [0.5, 0.1]
    assert m.active(2, 4, 0.2) == [0]
    assert m.active(3, 4, 0.2) == [0, 1]  # below min_rounds
    assert m.active(2, 2, 10.0) == []     # max_rounds reached
    assert m.active(2, 4, -1.0) == [0, 1]  # negative: never stops
    m.E[:] = [np.inf, np.inf]
    assert m.active(2, 4, np.inf) == []    # +inf <= +inf
    m.E[:] = [np.nan, 0.0]
    assert m.active(2, 4, 0.0) == [0]      # NaN E never satisfies E <= threshold


def test_mirror_one_power_of_two_round_resolves_to_the_planes():
    rng = np.random.default_rng(3)
    m = am.AccumMirror(37, 23, 16, 16)  # 37 % 16 = 5, 23 % 16 = 7 (< 8): the last partial tiles are dropped (film.rs:399-404)
    assert (m.ntx, m.nty) == (2, 1)
    p = _random_planes(37 * 23, rng)
    m.fold(p, list(range(m.n_tiles)), 4)
    out = m.resolve()
    x = np.arange(37 * 23) % 37
    y = np.arange(37 * 23) // 37
    cov = (x < 32) & (y < 16)
    for k, c in am.NC.items():
        got, want = out[k].reshape(-1, c), p[k].reshape(-1, c)
        assert np.array_equal(got[cov].view(np.uint32), want[cov].view(np.uint32)), k
        assert (got[~cov] == 0).all(), k
