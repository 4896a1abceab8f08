"""The Metallic material on the CPU (include/rayn_b200.h, RAYN_MATERIAL_METALLIC): the metal mirror's f and scatter
(tests/metallic_mirror.cpp) against a float64 restatement of the statement, the two identities that tie it to the Dielectric, a
furnace check of the sampled lobe, the mirror's films of scenes without metals against the oracle's, the remap and the
flattening in Python and in rayn_host, and the orbit-trap path on a metal."""
import os
import subprocess

import numpy as np
import pytest

from rayn_b200 import _lib as L
from rayn_b200 import configs
from rayn_b200.scene import Dielectric, Lambertian, Metallic, OrbitTrapAlbedo, Srgb

import metallic_mirrors
from helpers import CH, assert_bit_equal, small_config

TR = configs.frame_time_range(1)
FRACTAL_MATERIAL = 1  # configs.setup() / setup_single_sphere(): sky, then the fractal's (the sphere's) grey Dielectric
COPPER = (0.95, 0.64, 0.54)
PI32, TWO_PI32 = float(np.float32(np.pi)), float(np.float32(2 * np.pi))


def metal(f0, rough):
    return Metallic(Srgb(*f0), rough).flatten()


def with_fractal_material(c, material):
    c["world"].materials.items[FRACTAL_MATERIAL] = material
    return c


def metal_config(n, res, samples, mb, f0=COPPER, roughness=0.3):
    c, inp = small_config(n, res, samples, mb)
    return with_fractal_material(c, Metallic.new_remap(f0, roughness)), inp


@pytest.fixture(scope="module")
def moracle():
    """the metal mirror: the oracle and the render mirror, unchanged, with the metal's f and scatter (tests/metallic_mirror.cpp)"""
    metallic_mirrors.lib()
    return metallic_mirrors


# ---- float64 restatement of the statement ---------------------------------------------------------------------------------
def _dot(a, b):
    return (a * b).sum(-1)


def _normalized(a):
    return a / np.linalg.norm(a, axis=-1, keepdims=True)


def _onb(n):  # math.rs:49-59, as rt_device.cuh::onb
    ks = np.where(n[:, 2] >= 0, 1.0, -1.0)
    ka = 1.0 / (1.0 + np.abs(n[:, 2]))
    kb = -ks * n[:, 0] * n[:, 1] * ka
    u = np.stack([1.0 - n[:, 0] ** 2 * ka, ks * kb, -ks * n[:, 0]], -1)
    v = np.stack([kb, ks - n[:, 1] ** 2 * ka * ks, -n[:, 1]], -1)
    return u, v, n


def _schlick(c, f0):
    return f0 + (1.0 - f0) * (1.0 - c) ** 5


def f64_f(f0, rough, first, second, n):
    dotv = np.maximum(0.0, _dot(first, n))
    half = _normalized(second + first)
    spec = np.maximum(0.0, _dot(half, n)) ** rough * (rough + 2.0) / (2.0 * np.pi)
    return spec[:, None] * _schlick(dotv[:, None], np.asarray(f0, np.float64)[None, :])


def f64_scatter(f0, rough, wo, n, u2, u3):
    """-> wi, f, pdf, cos(n, wi), b = sin of the lobe angle.  cosine_power with rayn's 2u azimuth (math.rs:106-113)."""
    a = u2 ** (1.0 / (rough + 1.0))
    b = np.sqrt(1.0 - a * a)
    s = np.stack([b * np.cos(2.0 * u3), b * np.sin(2.0 * u3), a], -1)
    r = wo - n * (2.0 * _dot(wo, n))[:, None]
    bu, bv, bw = _onb(r)
    wi = _normalized(bu * s[:, :1] + bv * s[:, 1:2] + bw * s[:, 2:])
    cap = np.maximum(a ** rough, float(np.finfo(np.float32).eps))
    pdf = (rough + 1.0) / (2.0 * np.pi) * cap
    coeff = (rough + 2.0) / (2.0 * np.pi) * cap
    cos_n = _dot(n, wi)
    coeff = np.where(cos_n < 0, 0.0, coeff)
    cosv = np.abs(_dot(n, wo))
    return wi, coeff[:, None] * _schlick(cosv[:, None], np.asarray(f0, np.float64)[None, :]), pdf, cos_n, b


def inputs(n, seed):
    """unit normals and outgoing directions on the normal's side, random samples, with the edge cases appended: normal
    incidence, grazing and exactly perpendicular wo (a zero normal dot), and samples at 0 and 1"""
    rng = np.random.default_rng(seed)
    nrm = _normalized(rng.normal(size=(n, 3)))
    wo = _normalized(rng.normal(size=(n, 3)))
    wo = np.where((_dot(wo, nrm) < 0)[:, None], -wo, wo)
    u = rng.random((n, 4))
    z = np.array([0.0, 0.0, 1.0])
    edge_wo = [z, _normalized(np.array([1.0, 0.0, 1e-3])), _normalized(np.array([0.0, 1.0, 1e-6])), np.array([1.0, 0.0, 0.0]),
               np.array([0.0, -1.0, 0.0]), _normalized(np.array([1.0, 1.0, 1.0]))]
    edge_u = [[0.5, 0.5, 0.0, 0.0], [0.5, 0.5, 1.0, 0.0], [0.5, 0.5, 0.999999, 0.999999], [0.5, 0.5, 0.5, 0.25],
              [0.5, 0.5, 1e-7, 0.75], [0.5, 0.5, 0.3, 0.0]]
    nrm = np.concatenate([nrm, np.tile(z, (len(edge_wo), 1))])
    wo = np.concatenate([wo, np.array(edge_wo)])
    u = np.concatenate([u, np.array(edge_u)])
    s1d = rng.random(len(nrm))
    return nrm.astype(np.float32), wo.astype(np.float32), s1d.astype(np.float32), u.astype(np.float32)


MATERIALS = [((0.95, 0.64, 0.54), 1.0), (COPPER, 301.0), ((0.0, 0.0, 0.0), 7.5), ((1.0, 1.0, 1.0), 73.03), ((0.04, 0.5, 1.0), 11.2)]


@pytest.mark.parametrize("f0,rough", MATERIALS)
def test_metal_mirror_equals_float64_statement(moracle, f0, rough):
    """scatter's wi, f, pdf and f(wo, wi, n) against float64, within float32 rounding: the lobe's sine b = sqrt(1 - a^2)
    cancels as a -> 1 (an absolute error of about 1.2e-7 / b in wi), and pow amplifies a relative error of its base by the
    exponent.  Bounces within 1e-4 of the horizon are left out of the zero test, where float32 and float64 may fall on
    different sides."""
    m = metal(f0, rough)
    nrm, wo, s1d, u = inputs(4000, int(rough))
    wi, f, pdf, fe = moracle.kat_bsdf(m, nrm, wo, s1d, u)
    n64, wo64 = nrm.astype(np.float64), wo.astype(np.float64)
    rwi, rf, rpdf, cos_n, b = f64_scatter(f0, rough, wo64, n64, u[:, 2].astype(np.float64), u[:, 3].astype(np.float64))
    tol = 2e-6 * (rough + 4.0)
    wi_err = 1e-5 + 1.2e-7 / np.maximum(b, 1e-7)
    assert (np.abs(wi - rwi).max(1) <= wi_err).all()
    assert np.allclose(pdf, rpdf, rtol=tol, atol=1e-30)
    clear = np.abs(cos_n) > 1e-4
    assert np.allclose(f[clear], rf[clear], rtol=tol, atol=1e-6 * (rough + 2.0))
    assert (f[cos_n < -1e-4] == 0).all() and (f[cos_n > 1e-4] >= 0).all()
    rfe = f64_f(f0, rough, wo64, wi.astype(np.float64), n64)
    assert np.allclose(fe, rfe, rtol=tol, atol=1e-6 * (rough + 2.0))
    if f0 == (0.0, 0.0, 0.0):  # F0 = 0: f is the Schlick tail (1 - c)^5 alone, zero at normal incidence
        assert (fe[-6] == 0).all() and (f[-6] == 0).all()
    if f0 == (1.0, 1.0, 1.0):  # F0 = 1: the Fresnel factor is exactly 1
        assert_bit_equal(f[:, 0], f[:, 1]) and assert_bit_equal(f[:, 1], f[:, 2])


def test_zero_normal_dot_and_below_horizon(moracle):
    """wo perpendicular to n: dotv = 0 so F = F0 + (1 - F0); a bounce below the horizon has f = 0 and keeps its pdf"""
    m = metal((0.3, 0.6, 0.9), 1.0)
    nrm = np.array([[0, 0, 1]] * 3, np.float32)
    wo = np.array([[1, 0, 0], [0, 1, 0], [0.6, 0, 0.8]], np.float32)
    u = np.array([[0.5, 0.5, 0.9, 0.0]] * 3, np.float32)
    wi, f, pdf, fe = moracle.kat_bsdf(m, nrm, wo, np.zeros(3, np.float32), u)
    below = (wi * nrm).sum(1) < 0
    assert below[:2].any()
    assert (f[below] == 0).all() and (pdf > 0).all()


def test_identity_a_f0_004_is_the_black_dielectric(moracle):
    """(a): F0 = 0.04 gives the f of a Dielectric with albedo 0 and the same exponent, bit for bit, at the same (wo, wi, n):
    with s1d = 0 the Dielectric's scatter takes its specular bounce, which is the metal's wi"""
    nrm, wo, _, u = inputs(6000, 11)
    zero = np.zeros(len(nrm), np.float32)
    for rough in (1.0, 5.0, 73.03, 301.0):
        gm = moracle.kat_bsdf(metal((0.04, 0.04, 0.04), rough), nrm, wo, zero, u)
        gd = moracle.kat_bsdf(Dielectric(Srgb(0, 0, 0), rough).flatten(), nrm, wo, zero, u)
        assert_bit_equal(gm[0], gd[0], f"wi {rough}")
        assert_bit_equal(gm[3], gd[3], f"f(wo, wi, n) {rough}")


def test_identity_b_f0_one_is_the_dielectric_specular_lobe(moracle):
    """(b): F0 = 1 gives the wi and f of the Dielectric's scatter with s1d = 0, bit for bit; the pdf differs"""
    nrm, wo, s1d, u = inputs(6000, 12)
    zero = np.zeros(len(nrm), np.float32)
    for rough in (1.0, 5.0, 73.03, 301.0):
        gm = moracle.kat_bsdf(metal((1.0, 1.0, 1.0), rough), nrm, wo, s1d, u)  # the metal reads no s1d
        gd = moracle.kat_bsdf(Dielectric(Srgb(0.3, 0.2, 0.1), rough).flatten(), nrm, wo, zero, u)
        assert_bit_equal(gm[0], gd[0], f"wi {rough}")
        assert_bit_equal(gm[1], gd[1], f"f {rough}")
        assert not np.array_equal(gm[2], gd[2])


def test_metal_reads_neither_s1d_nor_u0_u1(moracle):
    m = metal(COPPER, 12.0)
    nrm, wo, s1d, u = inputs(2000, 13)
    a = moracle.kat_bsdf(m, nrm, wo, s1d, u)
    v = u.copy()
    v[:, :2] = np.random.default_rng(3).random((len(u), 2))
    b = moracle.kat_bsdf(m, nrm, wo, 1.0 - s1d, v)
    for x, y in zip(a, b):
        assert_bit_equal(x, y, "samples the metal does not read")


def _rd2(n):
    """R_d (Roberts) points in [0, 1)^2: frac(0.5 + alpha * i) with alpha = (1/g, 1/g^2), g the plastic number"""
    g = 1.32471795724474602596
    i = np.arange(1, n + 1, dtype=np.float64)[:, None]
    return np.mod(0.5 + i * np.array([1.0 / g, 1.0 / (g * g)]), 1.0)


@pytest.mark.parametrize("rough", [1.0, 7.5, 73.03])
@pytest.mark.parametrize("theta", [0.0, 0.8, 1.4])
def test_furnace_f0_one(moracle, rough, theta):
    """F0 = 1: the mean of f |n.wi| / pdf over R_d samples is the lobe's directional albedo as scatter samples it, that is the
    expectation over (u2, u3) of (rough + 2) / (rough + 1) * max(0, n.wi(u2, u3)) (the below-horizon zero; rayn's 2u
    azimuth), by float64 midpoint quadrature on a 1200 x 1200 grid.  Tolerance: 5 standard errors of the samples' spread,
    which bounds a quasi-random mean's error as loosely as a random one's."""
    N = 200000
    u23 = _rd2(N).astype(np.float32)
    u = np.concatenate([np.full((N, 2), 0.5, np.float32), u23], 1)
    nrm = np.tile(np.array([0, 0, 1], np.float32), (N, 1))
    wo = np.tile(np.array([np.sin(theta), 0, np.cos(theta)], np.float32), (N, 1))
    wi, f, pdf, _ = moracle.kat_bsdf(metal((1, 1, 1), rough), nrm, wo, np.zeros(N, np.float32), u)
    est = f[:, 0].astype(np.float64) * np.abs(wi[:, 2].astype(np.float64)) / pdf.astype(np.float64)
    K = 1200
    g = (np.arange(K) + 0.5) / K
    q2, q3 = np.meshgrid(g, g, indexing="ij")
    w64 = np.tile(wo[:1].astype(np.float64), (K * K, 1))
    n64 = np.tile(np.array([[0.0, 0.0, 1.0]]), (K * K, 1))
    _, _, _, cos_n, _ = f64_scatter((1, 1, 1), rough, w64, n64, q2.ravel(), q3.ravel())
    want = ((rough + 2.0) / (rough + 1.0) * np.maximum(cos_n, 0.0)).mean()
    se = est.std() / np.sqrt(N)
    assert abs(est.mean() - want) <= 5 * se + 1e-6, (est.mean(), want, se)
    # the lobe is centred on reflected(wo, n), the mirror image of the OUTGOING direction, which lies below the surface (the
    # Dielectric's reference quirk, oracle/README.md): only the part that reaches above the horizon carries energy
    if theta == 0.0 and rough >= 7.5:
        assert want < 1e-6 and (f == 0).mean() > 0.999
    if theta == 1.4:  # near grazing the lobe straddles the horizon
        assert want > 0.005


def test_new_remap_is_the_dielectrics():
    r = np.concatenate([np.linspace(0, 1, 1001), [0.6, 0.2, 0.3, 1e-8, 0.999999]]).astype(np.float32)
    for x in r:
        assert np.float32(Metallic.new_remap(COPPER, x).roughness).view(np.uint32) == \
            np.float32(Dielectric.new_remap(COPPER, x).roughness).view(np.uint32)
    m = Metallic.new_remap(OrbitTrapAlbedo(0.5, 1.5, (0.1, 0.2, 0.3), (0.9, 0.8, 0.7)), 0.2)
    assert m.albedo_gen is not None and np.array_equal(m.f0, np.float32([0.9, 0.8, 0.7]))
    d = m.flatten()
    assert d.kind == L.MATERIAL_METALLIC == 4 and d.roughness == Dielectric.new_remap((0, 0, 0), 0.2).roughness


def test_cpp_host_flattens_the_same_metal_scene(tmp_path):
    """rayn_host --metallic R G B ROUGHNESS (with and without --orbit-trap) hands the C ABI the descriptors scene.py makes"""
    from rayn_b200 import build
    build.build()
    exe = os.path.join(os.path.dirname(build.OUT), "rayn_host")
    for n in (1, 2, 3, 4, 5):
        for rough, trap in ((0.3, False), (0.6, False), (0.2, True)):
            if trap and n == 1:
                continue
            out = tmp_path / f"scene{n}.bin"
            args = [exe, "--config", str(n), "--res", "160", "90", "--metallic", *map(str, COPPER), str(rough)]
            if trap:
                args += ["--orbit-trap", "0.6676", "1.45", "0.9", "0.35", "0.1", "0.1", "0.3", "0.8"]
            subprocess.run(args + ["--dump-scene", str(out)], check=True)
            c = configs.baseline_config(n, res=(160, 90))
            f0 = OrbitTrapAlbedo(0.6676, 1.45, (0.9, 0.35, 0.1), (0.1, 0.3, 0.8)) if trap else COPPER
            with_fractal_material(c, Metallic.new_remap(f0, rough))
            d, keep = c["world"].flatten(c["camera"])
            want = b"".join(bytes(d.hitables[i]) for i in range(d.n_hitables)) + b"".join(bytes(d.materials[i]) for i in range(d.n_materials)) + \
                b"".join(bytes(d.lights[i]) for i in range(d.n_lights)) + bytes(d.camera) + bytes(d.volume)
            assert out.read_bytes() == want, f"config {n} roughness {rough} trap {trap}"


@pytest.mark.parametrize("n", [3, 4])
@pytest.mark.parametrize("lo,hi,which", [(-2.0, -1.0, "hi"), (1e30, 2e30, "lo")])
def test_trap_palette_replaces_f0(moracle, n, lo, hi, which):
    """the render mirror's trap path on a metal: with s = 1 (every trap above trap_hi) the film is the film of a constant
    metal with F0 = albedo_hi, with s = 0 that of F0 = albedo_lo, bit for bit; and a palette in between changes the film"""
    alo, ahi = (0.9, 0.35, 0.1), (0.1, 0.3, 0.8)
    c, inp = metal_config(n, (21, 13), 1, 3)
    with_fractal_material(c, Metallic.new_remap(OrbitTrapAlbedo(lo, hi, alo, ahi), 0.3))
    g = moracle.render(c["world"], c["camera"], inp, (8, 8), c["integrator"], TR)
    c0, _ = metal_config(n, (21, 13), 1, 3, f0=ahi if which == "hi" else alo)
    o = moracle.oracle_render(c0["world"], c0["camera"], inp, (8, 8), c0["integrator"], TR)
    for ch in CH:
        assert_bit_equal(g[ch], o[ch], f"cfg{n} s={which} {ch}")
    with_fractal_material(c, Metallic.new_remap(OrbitTrapAlbedo(0.6676, 1.45, alo, ahi), 0.3))
    t = moracle.render(c["world"], c["camera"], inp, (8, 8), c["integrator"], TR)
    assert not np.array_equal(t["color"], o["color"])


def test_metal_film_renders_and_differs_from_the_dielectric(oracle, moracle):
    """the metal mirror renders a metal Mandelbox: finite, lit, with the alpha and normal channels of a surface that receives
    light, the same as the oracle's Dielectric film has"""
    c, inp = metal_config(3, (24, 16), 1, 3)
    m = moracle.oracle_render(c["world"], c["camera"], inp, (8, 8), c["integrator"], TR)
    c0, _ = small_config(3, (24, 16), 1, 3)
    d = oracle.render(c0["world"], c0["camera"], inp, (8, 8), c0["integrator"], TR)[0]
    assert np.isfinite(m["color"]).all() and m["color"].sum() > 0
    assert_bit_equal(m["alpha"], d["alpha"], "alpha: the same surfaces receive light")
    assert_bit_equal(m["normal"], d["normal"], "normal")
    assert not np.array_equal(m["color"], d["color"])


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5])
def test_metal_mirror_leaves_every_other_kind_as_the_oracle_has_it(oracle, moracle, n):
    """scenes without a metal: the metal mirror's oracle loop equals the oracle's film, its render mirror (with a trap) the
    render mirror's, its albedo plane the render mirror's, and its BSDF KAT the oracle's, bit for bit"""
    import mirrors
    c, inp = small_config(n, (23, 17), 1, 3)
    o = oracle.render(c["world"], c["camera"], inp, (8, 8), c["integrator"], TR)[0]
    m = moracle.oracle_render(c["world"], c["camera"], inp, (8, 8), c["integrator"], TR)
    for ch in CH:
        assert_bit_equal(m[ch], o[ch], f"cfg{n} oracle loop {ch}")
    if n > 1:
        c["world"].materials.items[FRACTAL_MATERIAL] = Dielectric.new_remap(OrbitTrapAlbedo(0.6676, 1.45, (0.9, 0.35, 0.1), (0.1, 0.3, 0.8)), 0.6)
    r = mirrors.render(c["world"], c["camera"], inp, (8, 8), c["integrator"], TR, moments=True)[0]
    m = moracle.render(c["world"], c["camera"], inp, (8, 8), c["integrator"], TR, moments=True)
    for ch in CH + ("moments",):
        assert_bit_equal(m[ch], r[ch], f"cfg{n} render mirror {ch}")
    assert_bit_equal(moracle.render_albedo(c["world"], c["camera"], inp, (8, 8), c["integrator"], TR),
                     mirrors.render_albedo(c["world"], c["camera"], inp, (8, 8), c["integrator"], TR)[0], f"cfg{n} albedo")
    nrm, wo, s1d, u = inputs(2000, n)
    for mat in (Lambertian(Srgb(0.6, 0.4, 0.2)).flatten(), Dielectric.new_remap(Srgb(0.2, 0.2, 0.2), 0.6).flatten()):
        for a, b in zip(moracle.kat_bsdf(mat, nrm, wo, s1d, u), oracle.kat_bsdf(mat, nrm, wo, s1d, u)):
            assert_bit_equal(a, b, f"kat kind {mat.kind}")
