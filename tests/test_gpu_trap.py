"""Orbit-trap albedo on the device (rayn_b200_set_albedo_traps, k_normals<V, true>, the TRAP shading kernels) against the CPU
trap oracle (tests/trap_oracle.cpp) bit for bit: the trap KAT, films at odd sizes and tile shapes, a material shared by a sphere
and the Mandelbox, sampled tiles of a full-size film, fold-all on and off, graph replay, pass sizes, host and device planes, the identity films, the
golden fixture, the existing goldens after a clear, adaptive rounds and argument errors."""
import ctypes as C
import os

import numpy as np
import pytest

from rayn_b200 import _lib as L
from rayn_b200 import configs
from rayn_b200.film import Film, FrameInputs, Renderer, make_frame_desc
from rayn_b200.scene import Lambertian, OrbitTrapAlbedo, Sphere, Vec3

import accum_mirror as am
from helpers import CH, assert_bit_equal, small_config
from test_cpu_trap import (ALBEDO_HI, ALBEDO_LO, FRACTAL_MATERIAL, TRAP_GOLDEN, TRAP_HI, TRAP_LO, fractal, toracle,  # noqa: F401
                           trap_golden_config, trap_points, with_fractal_albedo)

pytestmark = pytest.mark.gpu
TR = configs.frame_time_range(1)


def trap_config(n, res, samples, mb, lo=TRAP_LO, hi=TRAP_HI):
    c, inp = small_config(n, res, samples, mb)
    return with_fractal_albedo(c, OrbitTrapAlbedo(lo, hi, ALBEDO_LO, ALBEDO_HI)), inp


def gpu_film(r, c, inp, tile, **kw):
    r.upload_scene(c["world"], c["camera"])
    return r.render_host(inp, tile, c["integrator"], TR, **kw)


def oracle_film(binding, c, inp, tile, **kw):
    return binding.render(c["world"], c["camera"], inp, tile, c["integrator"], TR, **kw)[0]


def assert_film(g, o, what):
    for ch in CH:
        assert_bit_equal(g[ch], o[ch], f"{what} {ch}")


@pytest.mark.parametrize("n", [2, 3, 4, 5])
def test_trap_kat_equals_oracle(renderer, toracle, n):
    h = fractal(n)
    p = trap_points(20 + n, 20000)
    assert_bit_equal(renderer.kat_sdf_trap(h, p), toracle.kat_sdf_trap(h, p), f"cfg{n}")


def test_trap_kat_generic_mandelbox(renderer, toracle):
    """constants that select the generic per-point estimator (variant 0) for the march kernels"""
    c = configs.baseline_config(3, res=(8, 8), samples=1, max_bounces=1)
    c["world"].hitables.items[1].sdf.box_fold.l = np.float32(0.0)
    renderer.upload_scene(c["world"], c["camera"])
    assert renderer.sdf_variant(1) == 0
    h = c["world"].hitables.items[1].flatten()
    p = trap_points(7, 20000)
    assert_bit_equal(renderer.kat_sdf_trap(h, p), toracle.kat_sdf_trap(h, p), "generic")


@pytest.mark.parametrize("n,res,tile,mb", [(3, (37, 23), (8, 8), 3), (3, (48, 40), (16, 16), 4), (4, (29, 31), (8, 8), 2),
                                           (4, (40, 24), (16, 16), 3)])
def test_trap_film_equals_oracle(renderer, toracle, n, res, tile, mb):
    c, inp = trap_config(n, res, 1, mb)
    g = gpu_film(renderer, c, inp, tile)
    o = oracle_film(toracle, c, inp, tile)
    assert_film(g, o, f"cfg{n} {res} {tile}")
    c0, _ = small_config(n, res, 1, mb)
    assert not np.array_equal(g["color"], gpu_film(renderer, c0, inp, tile)["color"])  # the trap shows


def shared_material_scene(res):
    """config 3 plus two spheres: one shares the Mandelbox's trap material (s = 1 there), one has a Lambertian without a trap"""
    c, inp = trap_config(3, res, 1, 3)
    w = c["world"]
    plain = w.materials.add_material(Lambertian((0.6, 0.5, 0.4)))
    w.hitables.push(Sphere(Vec3(0.9, -0.7, 0.6), 0.35, FRACTAL_MATERIAL))
    w.hitables.push(Sphere(Vec3(-0.8, 0.6, 0.9), 0.3, plain))
    return c, inp


@pytest.mark.parametrize("flags", [0, L.FLAG_NO_FOLD_ALL])
def test_shared_trap_material_sphere_and_sdf(toracle, flags):
    c, inp = shared_material_scene((40, 36))
    r = Renderer(0, flags=flags)
    try:
        g = gpu_film(r, c, inp, (8, 8))
    finally:
        r.close()
    assert_film(g, oracle_film(toracle, c, inp, (8, 8)), f"shared material flags {flags}")


def test_full_size_cfg3_sampled_tiles(renderer, toracle):
    c, _ = trap_config(3, (1920, 1080), 1, 3)
    inp = FrameInputs(1920, 1080, 1, c["integrator"])
    k = 97
    ntx, nty = (1920 + 1920 % 16) // 16, (1080 + 1080 % 16) // 16
    tiles = [t for t in range(ntx * nty) if t % k == 0]
    g = gpu_film(renderer, c, inp, (16, 16), tile_list=tiles)
    o = oracle_film(toracle, c, inp, (16, 16), subsample_k=k)
    assert_film(g, o, "full size sampled tiles")


@pytest.mark.parametrize("flags,max_paths", [(0, 0), (L.FLAG_NO_FOLD_ALL, 0), (0, 3000), (L.FLAG_NO_GRAPH, 3000)])
def test_fold_all_pass_size_and_graph_replay(toracle, flags, max_paths):
    c, inp = trap_config(3, (33, 27), 1, 3)
    o = oracle_film(toracle, c, inp, (8, 8))
    r = Renderer(0, max_paths_per_pass=max_paths, flags=flags)
    try:
        for rep in range(2):  # the second small single-pass frame replays the captured graph (unless disabled)
            g = gpu_film(r, c, inp, (8, 8))
            assert_film(g, o, f"flags {flags} max_paths {max_paths} run {rep}")
        st = r.stats()
        assert st.passes > 1 if max_paths else st.passes == 1
        if max_paths == 0:
            assert st.reserved_ == 1  # replayed from the captured graph
    finally:
        r.close()


def test_device_planes(renderer, toracle):
    import torch
    c, inp = trap_config(4, (24, 20), 1, 2)
    renderer.upload_scene(c["world"], c["camera"])
    w, h = inp.width, inp.height
    dev = {k: torch.zeros((1 if k == "alpha" else 3) * w * h, dtype=torch.float32, device="cuda") for k in CH}
    torch.cuda.synchronize()
    ptrs = tuple(a.ctypes.data for a in inp.arrays())
    f = make_frame_desc(w, h, (8, 8), inp.samples, c["integrator"], inp.frame, TR, ptrs, L.MEM_HOST, sets=(inp.sets_1d, inp.sets_2d))
    renderer.render(f, L.RaynFilmPlanes(*(dev[k].data_ptr() for k in CH), L.MEM_DEVICE))
    L.check(L.lib().rayn_b200_sync(renderer.ctx), renderer.ctx)
    assert_film({k: v.cpu().numpy() for k, v in dev.items()}, oracle_film(toracle, c, inp, (8, 8)), "device planes")


@pytest.mark.parametrize("n", [3, 4])
@pytest.mark.parametrize("lo,hi,which", [(-2.0, -1.0, "hi"), (1e30, 2e30, "lo")])
def test_identity_films_on_device(renderer, n, lo, hi, which):
    c, inp = trap_config(n, (21, 13), 1, 3, lo, hi)
    g = gpu_film(renderer, c, inp, (8, 8))
    st_trap = renderer.stats()
    ref = gpu_film(renderer, with_fractal_albedo(c, ALBEDO_HI if which == "hi" else ALBEDO_LO), inp, (8, 8))
    st = renderer.stats()
    assert_film(g, ref, f"cfg{n} s={which}")
    assert st_trap.sdf_evals_normals == st.sdf_evals_normals > 0  # 4 per SDF shading lane, traps not counted


def test_trap_golden(renderer):
    from test_cpu_oracle import GOLD, GOLD_SUFFIX
    c, inp = trap_golden_config()
    g = gpu_film(renderer, c, inp, (16, 16))
    assert_film(g, np.load(os.path.join(GOLD, TRAP_GOLDEN + GOLD_SUFFIX + ".npz")), "trap golden")


@pytest.mark.parametrize("clear", ["set_empty", "upload"])
def test_existing_goldens_after_clear(renderer, clear):
    """a trap set on the golden scene's Dielectric (material 1) and rendered with, then cleared by set_albedo_traps([]) or by a
    fresh upload_scene: the committed golden films render bit for bit"""
    from test_cpu_oracle import GOLD, GOLD_SUFFIX, GOLDEN_CASES
    for name, (n, res, samples, mb) in sorted(GOLDEN_CASES.items()):
        c, inp = small_config(n, res, samples, mb)
        renderer.upload_scene(c["world"], c["camera"])
        renderer.set_albedo_traps([trap_desc()])
        t = renderer.render_host(inp, (16, 16), c["integrator"], TR)  # allocates the trap buffer, leaves the list set
        if clear == "set_empty":
            renderer.set_albedo_traps([])
        else:
            renderer.upload_scene(c["world"], c["camera"])
        g = renderer.render_host(inp, (16, 16), c["integrator"], TR)
        gold = np.load(os.path.join(GOLD, name + GOLD_SUFFIX + ".npz"))
        assert_film(g, gold, f"golden {name} after {clear}")
        assert n == 1 or not np.array_equal(t["color"], gold["color"])  # the trap did show before the clear


def test_set_empty_list_restores_constant_albedo(renderer):
    """the trap world uploaded, then its list cleared: the film is the constant-albedo (albedo_hi) film"""
    c, inp = trap_config(3, (24, 24), 1, 3)
    renderer.upload_scene(c["world"], c["camera"])
    renderer.set_albedo_traps([])
    g = renderer.render_host(inp, (8, 8), c["integrator"], TR)
    ref = gpu_film(renderer, with_fractal_albedo(c, ALBEDO_HI), inp, (8, 8))
    assert_film(g, ref, "cleared list")


def test_render_adaptive_with_trap(toracle):
    c, _ = trap_config(3, (40, 32), 1, 3)
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
        m.fold(toracle.render(c["world"], c["camera"], inp, tile, integ, TR, tile_list=act)[0], act, 1)
        ref_rounds += 1
    assert rounds == ref_rounds >= 2
    want = m.resolve()
    for ch in CH:
        assert_bit_equal(f.channels[ch].reshape(-1), want[ch], f"adaptive {ch}")


def trap_desc(material=FRACTAL_MATERIAL, lo=TRAP_LO, hi=TRAP_HI, alo=ALBEDO_LO, ahi=ALBEDO_HI):
    return L.RaynAlbedoTrap(material, lo, hi, (C.c_float * 3)(*alo), (C.c_float * 3)(*ahi))


def test_argument_errors():
    lib = L.lib()
    r = Renderer(0)
    try:
        ctx = r.ctx
        one = (L.RaynAlbedoTrap * 1)(trap_desc())
        assert lib.rayn_b200_set_albedo_traps(ctx, 1, one) == L.RAYN_ERR_NO_SCENE
        c, inp = small_config(3, (16, 16), 1, 2)
        r.upload_scene(c["world"], c["camera"])  # materials: 0 sky, 1 grey Dielectric, 2 / 3 emissive

        def status(*traps, n=None):
            arr = (L.RaynAlbedoTrap * max(len(traps), 1))(*traps)
            return lib.rayn_b200_set_albedo_traps(ctx, len(traps) if n is None else n, arr)
        bad = [trap_desc(material=-1), trap_desc(material=4), trap_desc(material=0), trap_desc(material=2),
               trap_desc(lo=1.0, hi=1.0), trap_desc(lo=2.0, hi=1.0), trap_desc(lo=float("nan")), trap_desc(hi=float("inf")),
               trap_desc(alo=(0.1, float("nan"), 0.1)), trap_desc(ahi=(0.1, 0.1, float("-inf")))]
        for t in bad:
            assert status(t) == L.RAYN_ERR_INVALID_ARG, (t.material, t.trap_lo, t.trap_hi, list(t.albedo_lo), list(t.albedo_hi))
        assert status(trap_desc(), trap_desc()) == L.RAYN_ERR_INVALID_ARG  # duplicate material
        assert status(trap_desc(), n=-1) == L.RAYN_ERR_INVALID_ARG
        assert status(trap_desc(), n=L.RAYN_MAX_MATERIALS + 1) == L.RAYN_ERR_INVALID_ARG
        assert lib.rayn_b200_set_albedo_traps(ctx, 1, None) == L.RAYN_ERR_INVALID_ARG
        assert status(trap_desc()) == L.RAYN_OK
        assert lib.rayn_b200_set_albedo_traps(ctx, 0, None) == L.RAYN_OK
        assert lib.rayn_b200_set_albedo_traps(None, 0, None) == L.RAYN_ERR_INVALID_ARG
        sphere = L.RaynHitable()
        p = np.zeros(3, np.float32)
        fp = C.POINTER(C.c_float)
        assert lib.rayn_b200_kat_sdf_trap(ctx, C.byref(sphere), 1, p.ctypes.data_as(fp), p.ctypes.data_as(fp)) == L.RAYN_ERR_INVALID_ARG
    finally:
        r.close()


@pytest.mark.skipif(not L.LEGACY, reason="the legacy test kernels exist only in librayn_b200_legacy.so")
def test_legacy_flag_with_traps_is_unsupported_inner():
    c, inp = trap_config(3, (16, 16), 1, 2)
    r = Renderer(0, flags=L.FLAG_SIMPLE_MARCH)
    try:
        r.upload_scene(c["world"], c["camera"])
        with pytest.raises(L.RaynError) as e:
            r.render_host(inp, (8, 8), c["integrator"], TR)
        assert e.value.code == L.RAYN_ERR_UNSUPPORTED
        r.set_albedo_traps([])
        r.render_host(inp, (8, 8), c["integrator"], TR)  # without traps the legacy kernels still render
    finally:
        r.close()


@pytest.mark.skipif(L.MULADD_FUSED or L.LEGACY, reason="already inside a variant run")
def test_fused_and_legacy_variants():
    from test_gpu_parity import _run_suite_variant
    assert " passed" in _run_suite_variant({"RAYN_MULADD_FUSED": "1"}, ["tests/test_gpu_trap.py", "-k", "not full_size and not variants and not cpp_host"])
    assert " passed" in _run_suite_variant({"RAYN_B200_LEGACY": "1"}, ["tests/test_gpu_trap.py", "-k", "legacy_flag"])


@pytest.mark.skipif(L.MULADD_FUSED, reason="rayn_host links the unfused product library")
def test_cpp_host_orbit_trap_flag(renderer, tmp_path):
    """rayn_host --orbit-trap gives the Python film bit for bit, and composes with --denoise and --adaptive"""
    import subprocess
    from rayn_b200 import build
    exe = os.path.join(os.path.dirname(build.OUT), "rayn_host")
    trap = [str(v) for v in (TRAP_LO, TRAP_HI) + ALBEDO_LO + ALBEDO_HI]
    args = [exe, "--config", "3", "--res", "48", "32", "--samples", "1", "--bounces", "3", "--orbit-trap"] + trap
    r = subprocess.run(args + ["--dump", str(tmp_path / "t.bin")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    npx = 48 * 32
    raw = np.fromfile(tmp_path / "t.bin", np.float32)
    c, inp = trap_config(3, (48, 32), 1, 3)
    ref = gpu_film(renderer, c, inp, (16, 16))
    assert_bit_equal(raw[:3 * npx], ref["color"], "rayn_host --orbit-trap color")
    assert_bit_equal(raw[4 * npx:7 * npx], ref["background"], "rayn_host --orbit-trap background")
    for extra in (["--denoise", "2"], ["--adaptive", "0.3", "--rounds", "3"], ["--adaptive", "0.3", "--rounds", "3", "--denoise", "2"]):
        r = subprocess.run(args + extra + ["--dump", str(tmp_path / "x.bin")], capture_output=True, text=True)
        assert r.returncode == 0, (extra, r.stderr)
        plain = subprocess.run(args[:args.index("--orbit-trap")] + extra + ["--dump", str(tmp_path / "p.bin")], capture_output=True, text=True)
        assert plain.returncode == 0, plain.stderr
        assert not np.array_equal(np.fromfile(tmp_path / "x.bin", np.float32)[:3 * npx], np.fromfile(tmp_path / "p.bin", np.float32)[:3 * npx])
    r = subprocess.run([exe, "--config", "1", "--orbit-trap"] + trap, capture_output=True, text=True)
    assert r.returncode == 2
