"""Orbit-trap albedo on the CPU (include/rayn_b200.h, RaynAlbedoTrap): the trap oracle's trap and palette (tests/render_mirror.cpp)
against the numpy restatement in tests/trap_mirror.py bit for bit, identity films against the render oracle that pin the trap
plumbing, and the ABI."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from rayn_b200 import _lib as L
from rayn_b200 import configs
from rayn_b200.scene import Dielectric, Lambertian, OrbitTrapAlbedo

import trap_mirror as tm
from helpers import CH, assert_bit_equal, small_config

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TR = configs.frame_time_range(1)
ALBEDO_LO, ALBEDO_HI = (0.9, 0.35, 0.1), (0.1, 0.3, 0.8)
FRACTAL_MATERIAL = 1  # configs.setup(): sky, then the fractal's grey Dielectric
TRAP_LO, TRAP_HI = 0.6676, 1.45  # the example range (tools/trap_range.py)
TRAP_GOLDEN = "cfg3_trap_32x32_8spp_3b"  # tests/golden/make_golden_trap.py


def trap_golden_config():
    c, inp = small_config(3, (32, 32), 2, 3)
    return with_fractal_albedo(c, OrbitTrapAlbedo(TRAP_LO, TRAP_HI, ALBEDO_LO, ALBEDO_HI)), inp


def fractal(n, **kw):
    h = configs.baseline_config(n, res=(8, 8), samples=1, max_bounces=1)["world"].hitables.items[1].flatten()
    for k, v in kw.items():
        setattr(h, k, v)
    return h


def trap_points(seed, n=4000):
    """random points, points near the surfaces (on rays through the origin at the radii where the fractals sit) and specials"""
    rng = np.random.default_rng(seed)
    a = rng.uniform(-3, 3, size=(n, 3))
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    b = d * rng.uniform(0.3, 2.2, size=(n, 1))
    spec = np.array([[np.nan, 0, 0], [0, np.nan, 1], [np.inf, 0, 0], [0, 0, 0], [1e30, -1e30, 0], [-0.0, 0, 0], [1e-40, 0, 0]])
    return np.concatenate([a, b, spec]).astype(np.float32)


@pytest.fixture(scope="module")
def toracle():
    """the orbit-trap oracle (tests/mirrors.py): the render oracle of oracle/ plus trap, palette and per-lane albedo"""
    import mirrors
    mirrors.render_lib()
    return mirrors


def unfused_only():
    if L.MULADD_FUSED:
        pytest.skip("the numpy restatement is of the unfused mul_add build; the fused one is compared GPU against oracle")


@pytest.mark.parametrize("n", [2, 3, 4, 5])
def test_trap_kat_equals_numpy(toracle, n):
    unfused_only()
    h = fractal(n)
    p = trap_points(n)
    assert_bit_equal(toracle.kat_sdf_trap(h, p), tm.sdf_trap(h, p), f"cfg{n} trap")


@pytest.mark.parametrize("kind", ["box_generic", "box_7", "bulb_3", "bulb_small_bailout"])
def test_trap_kat_other_constants(toracle, kind):
    unfused_only()
    h = {"box_generic": lambda: fractal(3, box_l=0.0, min_rad_sq=0.0),  # constants of the generic estimator (variant 0)
         "box_7": lambda: fractal(3, iterations=7, scale=2.3),
         "bulb_3": lambda: fractal(2, iterations=3),
         "bulb_small_bailout": lambda: fractal(2, bulb_bailout=0.9)}[kind]()
    p = trap_points(11)
    assert_bit_equal(toracle.kat_sdf_trap(h, p), tm.sdf_trap(h, p), kind)


@pytest.mark.parametrize("n", [2, 3])
def test_trap_zero_iterations_and_nan(toracle, n):
    h = fractal(n, iterations=0)
    assert np.all(toracle.kat_sdf_trap(h, trap_points(3, 50)) == np.inf)
    h = fractal(n)
    t = toracle.kat_sdf_trap(h, np.array([[np.nan, np.nan, np.nan]] * 5, np.float32))
    assert np.all(t == np.inf)  # a NaN never replaces the running minimum


def test_palette_equals_numpy(toracle):
    lo, hi = np.float32(0.25), np.float32(3.5)
    d = L.RaynAlbedoTrap(FRACTAL_MATERIAL, float(lo), float(hi), (C.c_float * 3)(*ALBEDO_LO), (C.c_float * 3)(*ALBEDO_HI))
    inside = np.random.default_rng(5).uniform(lo, hi, 3000).astype(np.float32)
    edges = np.array([lo, hi, np.nextafter(lo, np.float32(0)), np.nextafter(lo, np.float32(9)), np.nextafter(hi, np.float32(0)),
                      np.nextafter(hi, np.float32(9)), -1, 0, -0.0, 1e30, np.inf, -np.inf, np.nan], np.float32)
    t = np.concatenate([inside, edges])
    s, a = toracle.kat_trap_albedo(d, t)
    ws, wa = tm.palette(lo, hi, ALBEDO_LO, ALBEDO_HI, t)
    assert_bit_equal(s, ws, "s")
    assert_bit_equal(a, wa, "albedo")
    n = len(inside)
    assert list(s[n:n + 2]) == [0, 1] and s[-3] == 1 and s[-2] == 0 and s[-1] == 0  # lo, hi, +inf, -inf, NaN
    assert np.all((s[:n] >= 0) & (s[:n] <= 1))


def with_fractal_albedo(c, albedo):
    """the config's world with the fractal's Dielectric given another albedo (constant or OrbitTrapAlbedo)"""
    mats = c["world"].materials.items
    mats[FRACTAL_MATERIAL] = Dielectric(albedo, mats[FRACTAL_MATERIAL].roughness)
    return c


def render_with(binding, c, inp):
    """the film of the render oracle (oracle.binding, constant albedos) or of the trap oracle (the world's traps), 8x8 tiles"""
    return binding.render(c["world"], c["camera"], inp, (8, 8), c["integrator"], TR)[0]


@pytest.mark.parametrize("n", [3, 4])
@pytest.mark.parametrize("lo,hi,which", [(-2.0, -1.0, "hi"), (1e30, 2e30, "lo")])
def test_identity_films(oracle, toracle, n, lo, hi, which):
    """s == 1 (every trap >= 0 > trap_hi) gives albedo_hi exactly, s == 0 (every finite trap < trap_lo) albedo_lo: the trap
    oracle's film equals the render oracle's constant-albedo film bit for bit, so the trap plumbing (the per-lane split of
    integrate in tests/render_mirror.cpp) moved no sample."""
    c, inp = small_config(n, (21, 13), 1, 3)
    with_fractal_albedo(c, OrbitTrapAlbedo(lo, hi, ALBEDO_LO, ALBEDO_HI))
    assert len(c["world"].albedo_traps()) == 1
    got = render_with(toracle, c, inp)
    ref = render_with(oracle, with_fractal_albedo(c, ALBEDO_HI if which == "hi" else ALBEDO_LO), inp)
    for ch in CH:
        assert_bit_equal(got[ch], ref[ch], f"cfg{n} s={which} {ch}")


def test_trap_changes_only_albedo_pixels(oracle, toracle):
    """A real trap range changes the config-3 film, and only pixels whose paths read the fractal's albedo: the pixels that
    also change when the fractal's constant albedo changes (paths that hit the SDF at some depth)."""
    c, inp = small_config(3, (24, 24), 1, 3)
    base = render_with(oracle, c, inp)
    with_fractal_albedo(c, OrbitTrapAlbedo(0.4, 3.0, ALBEDO_LO, ALBEDO_HI))
    trap = render_with(toracle, c, inp)
    dark = render_with(oracle, with_fractal_albedo(c, (0.0, 0.0, 0.0)), inp)
    px = lambda a, b: (a["color"].reshape(-1, 3) != b["color"].reshape(-1, 3)).any(axis=1)
    changed, sdf_px = px(trap, base), px(dark, base)
    assert changed.sum() > 0.1 * changed.size, changed.sum()
    assert not (changed & ~sdf_px).any()
    for ch in ("alpha", "normal", "background"):
        assert_bit_equal(trap[ch], base[ch], ch)


def test_oracle_reproduces_trap_golden(toracle):
    from test_cpu_oracle import GOLD, GOLD_SUFFIX
    c, inp = trap_golden_config()
    o = toracle.render(c["world"], c["camera"], inp, (16, 16), c["integrator"], TR)[0]
    g = np.load(os.path.join(GOLD, TRAP_GOLDEN + GOLD_SUFFIX + ".npz"))
    for ch in CH:
        assert_bit_equal(o[ch], g[ch], ch)


def test_traps_list_and_materials():
    t = OrbitTrapAlbedo(0.5, 2.0, ALBEDO_LO, ALBEDO_HI)
    for m in (Lambertian(t), Dielectric(t, 10.0), Dielectric.new_remap(t, 0.6)):
        assert m.albedo_gen is t and np.array_equal(m.albedo, np.float32(ALBEDO_HI))
    c = configs.baseline_config(3, res=(8, 8), samples=1, max_bounces=1)
    assert c["world"].albedo_traps() == []
    desc, keep = c["world"].flatten(c["camera"])  # the shape tests, bench.py and the oracle binding unpack
    with_fractal_albedo(c, t)
    (d,) = c["world"].albedo_traps()
    assert (d.material, d.trap_lo, d.trap_hi, tuple(d.albedo_lo), tuple(d.albedo_hi)) == (
        FRACTAL_MATERIAL, 0.5, 2.0, tuple(np.float32(ALBEDO_LO)), tuple(np.float32(ALBEDO_HI)))
    for bad in ((1.0, 1.0), (2.0, 1.0), (np.nan, 1.0), (0.0, np.inf)):
        with pytest.raises(ValueError):
            OrbitTrapAlbedo(*bad, ALBEDO_LO, ALBEDO_HI)


def test_albedo_trap_layout_matches_gcc(tmp_path):
    src = tmp_path / "l.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "rayn_b200.h"\nint main(void){printf("%zu %zu %zu %zu %zu %zu\\n",'
                   'sizeof(RaynAlbedoTrap), offsetof(RaynAlbedoTrap, material), offsetof(RaynAlbedoTrap, trap_lo),'
                   'offsetof(RaynAlbedoTrap, trap_hi), offsetof(RaynAlbedoTrap, albedo_lo), offsetof(RaynAlbedoTrap, albedo_hi));return 0;}\n')
    exe = tmp_path / "l"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    T = L.RaynAlbedoTrap
    assert got == [C.sizeof(T), T.material.offset, T.trap_lo.offset, T.trap_hi.offset, T.albedo_lo.offset, T.albedo_hi.offset]


def test_new_symbols_declared_and_exported():
    hdr = open(os.path.join(ROOT, "include", "rayn_b200.h")).read()
    for name in ("rayn_b200_set_albedo_traps", "rayn_b200_kat_sdf_trap"):
        assert re.search(r"\b" + name + r"\s*\(", hdr), name
        assert name in L.SYMBOLS, name
    lib = os.path.join(ROOT, "rayn_b200", "_build", "librayn_b200.so")
    if not os.path.exists(lib):
        pytest.skip("library not built")
    syms = subprocess.run(["nm", "-D", "--defined-only", lib], check=True, capture_output=True, text=True).stdout
    for name in ("rayn_b200_set_albedo_traps", "rayn_b200_kat_sdf_trap"):
        assert re.search(r"\bT " + name + r"\b", syms), name
