"""The Metallic material on the device (include/rayn_b200.h, RAYN_MATERIAL_METALLIC; the METAL shading kernels) against the metal
mirror (tests/metallic_mirror.cpp: the oracle and the render mirror with the metal's f and scatter) bit for bit: the argument checks, the BSDF KAT with specials, films of every kind of scene a metal can sit
in (sphere, Mandelbox smooth and rough, an orbit-trap palette, volume and depth of field, a mixed scene) through passes, graph
replay, moments and accumulator rounds, the albedo plane, the legacy kernels, and rayn_host --metallic."""
import os
import subprocess

import numpy as np
import pytest

from rayn_b200 import _lib as L
from rayn_b200 import configs
from rayn_b200.film import Film, FrameInputs, Renderer
from rayn_b200.scene import Dielectric, Lambertian, Metallic, OrbitTrapAlbedo, Sphere, Srgb, Vec3

import accum_mirror as am
import metallic_mirrors as mm
from helpers import CH, assert_bit_equal, small_config
from test_cpu_metallic import COPPER, FRACTAL_MATERIAL, inputs, metal, metal_config, with_fractal_material

pytestmark = pytest.mark.gpu
TR = configs.frame_time_range(1)
TRAP = OrbitTrapAlbedo(0.6676, 1.45, (0.9, 0.35, 0.1), (0.1, 0.3, 0.8))


def gpu_film(r, c, inp, tile, **kw):
    r.upload_scene(c["world"], c["camera"])
    return r.render_host(inp, tile, c["integrator"], TR, **kw)


def mirror_film(c, inp, tile, **kw):
    """the render mirror's film (orbit-trap albedos, moments) with the metal's BSDF"""
    return mm.render(c["world"], c["camera"], inp, tile, c["integrator"], TR, **kw)


def assert_film(g, o, what, channels=CH):
    for ch in channels:
        assert_bit_equal(g[ch], o[ch], f"{what} {ch}")


def test_upload_rejects_bad_metals_and_traps_accept_them(renderer):
    lib = L.lib()
    c, _ = metal_config(3, (16, 16), 1, 2)
    nan, inf = float("nan"), float("inf")
    for f0, rough in [((nan, 0.5, 0.5), 10.0), ((0.5, inf, 0.5), 10.0), ((0.5, 0.5, -inf), 10.0), (COPPER, nan), (COPPER, inf),
                      (COPPER, 0.0), (COPPER, -0.0), (COPPER, -3.0)]:
        with_fractal_material(c, Metallic(f0, rough))
        d, keep = c["world"].flatten(c["camera"])
        assert lib.rayn_b200_upload_scene(renderer.ctx, d) == L.RAYN_ERR_INVALID_ARG, (f0, rough)
    d, keep = c["world"].flatten(c["camera"])
    d.materials[FRACTAL_MATERIAL].kind = 5
    assert lib.rayn_b200_upload_scene(renderer.ctx, d) == L.RAYN_ERR_INVALID_ARG
    with_fractal_material(c, Metallic(COPPER, 1e-30))  # any finite exponent > 0
    renderer.upload_scene(c["world"], c["camera"])
    with_fractal_material(c, Metallic.new_remap(TRAP, 0.3))
    renderer.upload_scene(c["world"], c["camera"])
    renderer.set_albedo_traps(c["world"].albedo_traps())  # a metal takes a trap


def test_bsdf_kat_equals_mirror(renderer):
    nrm, wo, s1d, u = inputs(20000, 5)
    spec_n = np.array([[np.nan, 0, 1], [0, 0, 0], [0, 0, 1], [0, 0, -1], [1e-30, 0, 1], [np.inf, 0, 0]], np.float32)
    spec_wo = np.array([[0, 0, 1], [0, 1, 0], [np.nan, 0, 0], [0, 0, 1], [-0.0, 0, 1], [0, 0, 1]], np.float32)
    nrm, wo = np.concatenate([nrm, spec_n]), np.concatenate([wo, spec_wo])
    s1d = np.concatenate([s1d, np.zeros(6, np.float32)])
    u = np.concatenate([u, np.array([[0.5, 0.5, 0.5, 0.5]] * 6, np.float32)])
    mats = [metal(f0, r) for f0, r in [(COPPER, 1.0), (COPPER, 301.0), ((0, 0, 0), 7.5), ((1, 1, 1), 73.03), ((0.04, 0.04, 0.04), 2.5),
                                       ((-0.5, 2.0, 1e-30), 12.0)]]
    for m in mats:
        g = renderer.kat_bsdf(m, nrm, wo, s1d, u)
        r = mm.kat_bsdf(m, nrm, wo, s1d, u)
        for a, b, what in zip(g, r, ("wi", "f", "pdf", "f(wo,wi,n)")):
            assert_bit_equal(a, b, f"metal f0={list(m.albedo)} rough={m.roughness} {what}")


@pytest.mark.parametrize("n,res,tile,mb,rough", [(1, (37, 23), (8, 8), 3, 0.3), (3, (48, 40), (16, 16), 4, 0.2), (3, (41, 27), (8, 8), 3, 0.6),
                                                 (2, (40, 24), (16, 16), 3, 0.4), (4, (29, 31), (8, 8), 2, 0.3), (5, (32, 24), (16, 16), 3, 0.5)])
def test_metal_film_equals_mirror(renderer, n, res, tile, mb, rough):
    """config 1 with the sphere metallic, config 3 smooth and rough, the Mandelbulb configs, config 4 (volume and depth of field)"""
    c, inp = metal_config(n, res, 1, mb, roughness=rough)
    g = gpu_film(renderer, c, inp, tile)
    o = mm.oracle_render(c["world"], c["camera"], inp, tile, c["integrator"], TR)
    assert_film(g, o, f"cfg{n} {res} rough {rough}")
    assert g["color"].sum() > 0


@pytest.mark.parametrize("n", [3, 4])
def test_trap_tinted_metal_equals_mirror(renderer, n):
    c, inp = metal_config(n, (40, 32), 1, 3)
    with_fractal_material(c, Metallic.new_remap(TRAP, 0.3))
    g = gpu_film(renderer, c, inp, (8, 8))
    assert_film(g, mirror_film(c, inp, (8, 8)), f"cfg{n} trap metal")
    c0, _ = metal_config(n, (40, 32), 1, 3, f0=(0.1, 0.3, 0.8))
    assert not np.array_equal(g["color"], gpu_film(renderer, c0, inp, (8, 8))["color"])


def mixed_scene(res):
    """config 3 with a metal Mandelbox plus a Lambertian, a Dielectric and a second metal sphere, and a trap on the fractal"""
    c, inp = metal_config(3, res, 1, 4)
    w = c["world"]
    with_fractal_material(c, Metallic.new_remap(TRAP, 0.25))
    lam = w.materials.add_material(Lambertian((0.6, 0.5, 0.4)))
    die = w.materials.add_material(Dielectric.new_remap(Srgb(0.3, 0.5, 0.2), 0.4))
    gold = w.materials.add_material(Metallic.new_remap((1.0, 0.78, 0.34), 0.1))
    w.hitables.push(Sphere(Vec3(0.9, -0.7, 0.6), 0.35, lam))
    w.hitables.push(Sphere(Vec3(-0.8, 0.6, 0.9), 0.3, die))
    w.hitables.push(Sphere(Vec3(0.7, 0.8, -0.6), 0.3, gold))
    w.hitables.push(Sphere(Vec3(-0.6, -0.8, 0.5), 0.25, FRACTAL_MATERIAL))  # shares the trap metal: s = 1 there
    return c, inp


@pytest.mark.parametrize("flags,max_paths", [(0, 0), (L.FLAG_NO_FOLD_ALL, 0), (0, 3000), (L.FLAG_NO_GRAPH, 3000)])
def test_mixed_scene_passes_and_graph_replay(flags, max_paths):
    c, inp = mixed_scene((36, 28))
    o = mirror_film(c, inp, (8, 8))
    r = Renderer(0, max_paths_per_pass=max_paths, flags=flags)
    try:
        for rep in range(2):  # the second small single-pass frame replays the captured graph (unless disabled)
            assert_film(gpu_film(r, c, inp, (8, 8)), o, f"flags {flags} max_paths {max_paths} run {rep}")
        st = r.stats()
        assert st.passes > 1 if max_paths else st.passes == 1
        if max_paths == 0:
            assert st.reserved_ == 1  # replayed from the captured graph
    finally:
        r.close()


def test_mixed_scene_without_traps_and_plain_scene_after_it(renderer, oracle):
    """the METAL kernels without traps, then a scene without metals on the same context renders the oracle's film again"""
    c, inp = mixed_scene((33, 21))
    c["world"].materials.items[FRACTAL_MATERIAL] = Metallic.new_remap(COPPER, 0.25)
    assert_film(gpu_film(renderer, c, inp, (8, 8)), mm.oracle_render(c["world"], c["camera"], inp, (8, 8), c["integrator"], TR), "mixed, no trap")
    c0, _ = small_config(3, (33, 21), 1, 4)
    assert_film(gpu_film(renderer, c0, inp, (8, 8)), oracle.render(c0["world"], c0["camera"], inp, (8, 8), c0["integrator"], TR)[0], "no metal after")


@pytest.mark.parametrize("trap", [False, True])
def test_moments_equal_mirror(renderer, trap):
    c, inp = mixed_scene((31, 27))
    if not trap:
        c["world"].materials.items[FRACTAL_MATERIAL] = Metallic.new_remap(COPPER, 0.25)
    g = gpu_film(renderer, c, inp, (8, 8), moments=True)
    assert_film(g, mirror_film(c, inp, (8, 8), moments=True), f"moments trap={trap}", CH + ("moments",))


def test_full_size_cfg3_sampled_tiles(renderer):
    c, _ = metal_config(3, (1920, 1080), 1, 3)
    inp = FrameInputs(1920, 1080, 1, c["integrator"])
    k = 97
    ntx, nty = (1920 + 1920 % 16) // 16, (1080 + 1080 % 16) // 16
    tiles = [t for t in range(ntx * nty) if t % k == 0]
    g = gpu_film(renderer, c, inp, (16, 16), tile_list=tiles)
    o = mm.oracle_render(c["world"], c["camera"], inp, (16, 16), c["integrator"], TR, subsample_k=k)
    assert_film(g, o, "full size sampled tiles")


def test_render_adaptive_rounds():
    c, inp = mixed_scene((40, 32))
    (w, h), tile, integ = (40, 32), (8, 8), c["integrator"]
    f = Film(CH, (w, h))
    rounds = f.render_adaptive(c["world"], c["camera"], integ, None, tile, 1, TR, 1, min_rounds=2, max_rounds=4, threshold=0.3)
    m = am.AccumMirror(w, h, *tile)
    ref_rounds = 0
    while True:
        act = m.active(2, 4, 0.3)
        if not act:
            break
        inp = FrameInputs(w, h, 1, integ, frame=1, first_sample=int(m.K[act[0]]))
        m.fold(mm.render(c["world"], c["camera"], inp, tile, integ, TR, tile_list=act), act, 1)
        ref_rounds += 1
    assert rounds == ref_rounds >= 2
    want = m.resolve()
    for ch in CH:
        assert_bit_equal(f.channels[ch].reshape(-1), want[ch], f"adaptive {ch}")


@pytest.mark.parametrize("n,trap", [(1, False), (3, False), (3, True), (4, True)])
def test_albedo_plane_equals_mirror(renderer, n, trap):
    c, inp = metal_config(n, (37, 23), 2, 1)
    if trap:
        with_fractal_material(c, Metallic.new_remap(TRAP, 0.3))
    renderer.upload_scene(c["world"], c["camera"])
    g = renderer.render_albedo(inp, (8, 8), c["integrator"], TR)
    o = mm.render_albedo(c["world"], c["camera"], inp, (8, 8), c["integrator"], TR)
    assert_bit_equal(g, o, f"cfg{n} trap={trap}")
    if not trap:  # a pixel wholly on the metal gives its F0 (up to the rounding of the sum over samples)
        assert abs(g[..., 0].max() - COPPER[0]) < 1e-6 and abs(g[..., 2].max() - COPPER[2]) < 1e-6


@pytest.mark.parametrize("n", [1, 3, 4])
def test_all_ones_albedo_is_alpha(renderer, n):
    """every Lambertian / Dielectric albedo and every metal's F0 is (1, 1, 1), no traps: every channel is the alpha plane"""
    c, inp = metal_config(n, (53, 29), 2, 2, f0=(1.0, 1.0, 1.0))
    for m in c["world"].materials.items:
        if isinstance(m, (Lambertian, Dielectric, Metallic)):
            m.albedo, m.albedo_gen = np.ones(3, np.float32), None
    renderer.upload_scene(c["world"], c["camera"])
    a = renderer.render_albedo(inp, (8, 8), c["integrator"], TR)
    g = renderer.render_host(inp, (8, 8), c["integrator"], TR)
    assert g["alpha"].sum() > 0
    for ch in range(3):
        assert_bit_equal(a[:, :, ch], g["alpha"].reshape(29, 53), f"cfg{n} channel {ch}")


@pytest.mark.skipif(not L.LEGACY, reason="the legacy test kernels exist only in librayn_b200_legacy.so")
def test_legacy_kernels_on_a_metal_scene_inner():
    """the one-thread-per-ray legacy kernels give the metal mirror's film on metal scenes, as the product kernels do above"""
    for n, res, mb in [(3, (40, 32), 4), (1, (32, 24), 3), (4, (24, 24), 2)]:
        c, inp = metal_config(n, res, 1, mb)
        if n == 3:
            c, inp = mixed_scene(res)
            c["world"].materials.items[FRACTAL_MATERIAL] = Metallic.new_remap(COPPER, 0.25)
        r = Renderer(0, flags=L.FLAG_SIMPLE_MARCH)
        try:
            g = gpu_film(r, c, inp, (16, 16))
        finally:
            r.close()
        assert_film(g, mm.oracle_render(c["world"], c["camera"], inp, (16, 16), c["integrator"], TR), f"legacy cfg{n}")


@pytest.mark.skipif(L.MULADD_FUSED or L.LEGACY, reason="already inside a variant run")
def test_fused_and_legacy_variants():
    from test_gpu_parity import _run_suite_variant
    assert " passed" in _run_suite_variant({"RAYN_MULADD_FUSED": "1"}, ["tests/test_gpu_metallic.py", "-k", "not full_size and not variants and not rayn_host"])
    assert " passed" in _run_suite_variant({"RAYN_B200_LEGACY": "1"}, ["tests/test_gpu_metallic.py", "-k", "legacy_kernels"])


@pytest.mark.skipif(L.MULADD_FUSED, reason="rayn_host links the unfused product library")
def test_rayn_host_metallic(renderer, tmp_path):
    """rayn_host --metallic gives the Python film bit for bit, and composes with --orbit-trap, --denoise, --adaptive and --panorama"""
    from rayn_b200 import build
    exe = os.path.join(os.path.dirname(build.OUT), "rayn_host")
    base = [exe, "--config", "3", "--res", "48", "32", "--samples", "1", "--bounces", "3"]
    metal_args = ["--metallic", *map(str, COPPER), "0.3"]
    r = subprocess.run(base + metal_args + ["--dump", str(tmp_path / "m.bin")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    npx = 48 * 32
    raw = np.fromfile(tmp_path / "m.bin", np.float32)
    c, inp = metal_config(3, (48, 32), 1, 3)
    start = np.float32(1) * (np.float32(1.0) / np.float32(24))
    tr = (float(start), float(start + np.float32(1.0) / np.float32(24.0)))
    renderer.upload_scene(c["world"], c["camera"])
    ref = renderer.render_host(inp, (16, 16), c["integrator"], tr)
    for i, ch in enumerate(CH):
        lo = {0: 0, 1: 3, 2: 4, 3: 7}[i] * npx
        assert_bit_equal(raw[lo:lo + ref[ch].size], ref[ch], f"rayn_host --metallic {ch}")
    trap = ["--orbit-trap", "0.6676", "1.45", "0.9", "0.35", "0.1", "0.1", "0.3", "0.8"]
    for extra in (trap, ["--denoise", "2"], ["--adaptive", "0.3", "--rounds", "3"], ["--panorama"], trap + ["--panorama", "--denoise", "2"]):
        r = subprocess.run(base + metal_args + extra + ["--dump", str(tmp_path / "x.bin")], capture_output=True, text=True)
        assert r.returncode == 0, (extra, r.stderr)
        plain = subprocess.run(base + extra + ["--dump", str(tmp_path / "p.bin")], capture_output=True, text=True)
        assert plain.returncode == 0, plain.stderr
        x = np.fromfile(tmp_path / "x.bin", np.float32)[:3 * npx]
        assert np.isfinite(x).all() and not np.array_equal(x, np.fromfile(tmp_path / "p.bin", np.float32)[:3 * npx]), extra
    out = tmp_path / "copper.ppm"
    r = subprocess.run([exe, "--config", "3", "--samples", "4", "--metallic", "0.95", "0.64", "0.54", "0.3", "--out", str(out)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert out.stat().st_size == len(b"P6\n1920 1080\n255\n") + 1920 * 1080 * 3
