"""The equirectangular (360-degree panorama) camera on the device: films bit for bit against the oracle through the render paths,
the albedo and motion planes against the render mirror, the wrapped denoise and push against the film mirror, a sequence whose
denoised seam is continuous, and rayn_host --panorama against the Python path."""
import math
import os
import subprocess

import numpy as np
import pytest

from rayn_b200 import _lib as L
from rayn_b200 import configs
from rayn_b200.film import Film, FrameInputs, Renderer, denoise_desc
from rayn_b200.scene import EquirectangularCamera, Lambertian, Linear, Sphere, Srgb, Vec3

import panorama_mirrors as pm
from helpers import CH, assert_bit_equal
from test_cpu_panorama import (GUIDES, T_KW, TR, DT, denoise_mirror, film_with_guides, panorama_config, push_frame, run_push, tile_x,
                               yaw_scenes)

pytestmark = pytest.mark.gpu
TILE = (16, 16)


def oracle_film(c, cam, inp):
    """the oracle's render_tile with the panorama's camera branch (tests/panorama_mirror.cpp)"""
    return pm.oracle_render(c["world"], cam, inp, TILE, c["integrator"], TR)


def check_film(g, o, what):
    for k in CH:
        assert_bit_equal(g[k], o[k], f"{what}: {k}")


def moving_scene():
    """config 1 with a panorama whose origin and at move, and a second sphere moving across the seam"""
    c, _, inp = panorama_config(1, (64, 32), 1, 2)
    w = c["world"]
    src = w.cameras.get(c["camera"])
    cam = w.cameras.add_camera(EquirectangularCamera((64, 32), Linear(src.origin[0], np.float32([0.3, 0.0, -0.2])), Linear(src.at[0], np.float32([0.0, 0.5, 0.0])),
                                                     Linear(*src.up)))
    mat = w.materials.add_material(Lambertian(Srgb(0.6, 0.3, 0.2)))
    w.hitables.push(Sphere(Linear(Vec3(-1.0, 0.2, 6.0), Vec3(4.0, 0.0, 0.0)), 0.5, mat))
    return c, cam, inp


def test_films_bit_equal_the_oracle(renderer):
    cases = [("config 1", *panorama_config(1, (64, 32), 1, 2)),
             ("config 3 inside the light ring", *panorama_config(3, (64, 32), 1, 3, origin=(0.0, 0.0, 1.3))),
             ("moving camera and sphere", *moving_scene())]
    for what, c, cam, inp in cases:
        renderer.upload_scene(c["world"], cam, TR)
        g = renderer.render_host(inp, TILE, c["integrator"], TR)
        check_film(g, oracle_film(c, cam, inp), what)


def test_passes_graph_replay_and_moments():
    c, cam, inp = panorama_config(3, (64, 32), 1, 3, origin=(0.0, 0.0, 1.3))
    want = oracle_film(c, cam, inp)
    m = pm.render(c["world"], cam, inp, TILE, c["integrator"], TR, moments=True)
    for max_paths in (0, 1500):  # one pass (graph captured, then replayed), and several passes
        r = Renderer(0, max_paths_per_pass=max_paths)
        try:
            r.upload_scene(c["world"], cam)
            for rep in range(2):
                g = r.render_host(inp, TILE, c["integrator"], TR)
                check_film(g, want, f"max_paths {max_paths}, render {rep}")
            if max_paths:
                assert r.stats().passes > 1
            g = r.render_host(inp, TILE, c["integrator"], TR, moments=True)
            check_film(g, want, "with moments")
            assert_bit_equal(g["moments"], m["moments"], "moments")
        finally:
            r.close()


def test_adaptive_rounds_and_shards(renderer):
    c, cam, inp = panorama_config(1, (64, 32), 1, 2)
    want = oracle_film(c, cam, inp)
    renderer.upload_scene(c["world"], cam)
    acc = renderer.accum_create(64, 32, TILE)
    try:
        from rayn_b200.film import make_frame_desc
        f = make_frame_desc(64, 32, TILE, inp.samples, c["integrator"], inp.frame, TR, tuple(a.ctypes.data for a in inp.arrays()), L.MEM_HOST,
                            sets=(inp.sets_1d, inp.sets_2d))
        renderer.accum_round(acc, f, threshold=-1.0)
        check_film(renderer.accum_resolve(acc), want, "one accumulator round")
    finally:
        acc.close()
    parts = [renderer.render_host(inp, TILE, c["integrator"], TR, tile_offset=k, tile_stride=3) for k in range(3)]
    for k in CH:
        assert_bit_equal(parts[0][k] + parts[1][k] + parts[2][k], want[k], f"three shards: {k}")


def test_albedo_and_motion_planes_bit_equal_the_mirror(renderer):
    c, cam, inp = moving_scene()
    desc = renderer.upload_scene(c["world"], cam, TR)[0]
    alb = renderer.render_albedo(inp, TILE, c["integrator"], TR)
    want_alb = pm.render_albedo(c["world"], cam, inp, TILE, c["integrator"], TR)
    assert_bit_equal(alb, want_alb, "albedo")
    motion = renderer.render_motion(inp, TILE, c["integrator"], TR, DT)
    want, _ = pm.render_motion(desc, inp, TILE, c["integrator"], TR, DT)
    assert_bit_equal(motion, want, "motion")
    prev = c["world"].flatten(cam, (TR[0] - DT, TR[1] - DT))
    motion = renderer.render_motion(inp, TILE, c["integrator"], TR, DT, prev=prev[0])
    want, _ = pm.render_motion(desc, inp, TILE, c["integrator"], TR, DT, prev=prev[0])
    assert_bit_equal(motion, want, "motion against prev")


def test_static_scene_gives_exact_zero_motion(renderer):
    c, cam, inp = panorama_config(3, (64, 32), 1, 3)
    renderer.upload_scene(c["world"], cam)
    m = renderer.render_motion(inp, TILE, c["integrator"], TR, DT)
    ok = np.isfinite(m[..., 2])
    assert ok.all()
    assert (m[..., :2].view(np.uint32) == 0).all()  # +0 exactly
    assert_bit_equal(m[..., 3], m[..., 2], "z_prev == z")


def test_yaw_closed_form_on_the_device(renderer):
    W, H, k = 64, 32, 3
    c, cur, prev = yaw_scenes(W, H, k)
    inp = FrameInputs(W, H, 1, c["integrator"])
    desc = renderer.upload_scene(c["world"], cur)[0]
    pdesc = c["world"].flatten(prev)
    m = renderer.render_motion(inp, TILE, c["integrator"], TR, DT, prev=pdesc[0])
    np.testing.assert_allclose(m[..., 0], -k, atol=1e-3)
    np.testing.assert_allclose(m[..., 1], 0.0, atol=1e-3)
    want, _ = pm.render_motion(desc, inp, TILE, c["integrator"], TR, DT, prev=pdesc[0])
    assert_bit_equal(m, want, "yaw motion")


def test_unknown_camera_kind_is_rejected(renderer):
    c, cam, _ = panorama_config(1, (16, 16), 1, 1)
    d, keep = c["world"].flatten(cam)
    d.camera.kind = 4
    import ctypes as C
    assert renderer._lib.rayn_b200_upload_scene(renderer.ctx, C.byref(d)) == L.RAYN_ERR_INVALID_ARG
    prev = c["world"].flatten(c["camera"])  # a pinhole: a cut, not motion
    renderer.upload_scene(c["world"], cam)
    inp = FrameInputs(16, 16, 1, c["integrator"])
    with pytest.raises(L.RaynError):
        renderer.render_motion(inp, TILE, c["integrator"], TR, DT, prev=prev[0])


# ---- wrapped denoise and push --------------------------------------------------------------------------------------------
def gpu_denoise(r, planes, extra, levels, alb, var, device=False):
    h, w = planes["normal"].shape[:2]
    kw = {}
    if alb:
        kw.update(albedo=extra["albedo"].reshape(-1), sigma_albedo=0.2)
    if var:
        kw.update(moments=extra["moments"], spp=4, sigma_luminance=4.0, var_scale=extra["scale"] if var == "scaled" else None)
    if not device:
        return r.denoise(w, h, planes, levels, sigma_color=2.5, wrap=True, **kw)
    import ctypes as C
    import torch
    dev = {k: torch.from_numpy(np.ascontiguousarray(v, np.float32).reshape(-1)).cuda() for k, v in planes.items()}
    out = {k: torch.full_like(dev[k], float("nan")) for k in ("color", "background")}
    m = torch.from_numpy(np.ascontiguousarray(extra["moments"].transpose(2, 0, 1)).reshape(2, -1)).cuda()
    a = torch.from_numpy(extra["albedo"].reshape(-1)).cuda()
    s = torch.from_numpy(extra["scale"].reshape(-1)).cuda()
    pin = L.RaynFilmPlanes(dev["color"].data_ptr(), dev["alpha"].data_ptr(), dev["background"].data_ptr(), dev["normal"].data_ptr(), L.MEM_DEVICE)
    pout = L.RaynFilmPlanes(out["color"].data_ptr(), None, out["background"].data_ptr(), None, L.MEM_DEVICE)
    mp = L.RaynMomentPlanes(m[0].data_ptr(), m[1].data_ptr(), L.MEM_DEVICE)
    rc = r._lib.rayn_b200_film_denoise_wrap(r.ctx, C.byref(denoise_desc(levels, sigma_color=2.5)), 4.0 if var else float("inf"), 4,
                                            C.byref(mp) if var else None, s.data_ptr() if var == "scaled" else None, 0.2,
                                            a.data_ptr() if alb else None, w, h, C.byref(pin), C.byref(pout))
    L.check(rc, r.ctx)
    L.check(r._lib.rayn_b200_sync(r.ctx), r.ctx)
    return {k: v.cpu().numpy().reshape(h, w, 3) for k, v in out.items()}


@pytest.mark.parametrize("alb,var", GUIDES)
def test_denoise_wrap_bit_equal_the_mirror(renderer, alb, var):
    W, H = 40, 18
    planes, extra = film_with_guides(W, H, 21)
    for levels in (1, 3, 6):
        want = denoise_mirror(planes, extra, levels, alb, var, True)
        for device in (False, True):
            got = gpu_denoise(renderer, planes, extra, levels, alb, var, device)
            for k in ("color", "background"):
                assert_bit_equal(got[k].reshape(H, W, 3), want[k], f"{k}, {levels} levels, device {device}")


def test_denoise_wrap_tiling_identity_on_the_device(renderer):
    W, H, levels = 24, 10, 3
    planes, extra = film_with_guides(W, H, 9)
    n = 2 * -(-(2 ** (levels + 1) - 2) // W) + 1
    tiled = {k: tile_x(v, n) for k, v in planes.items()}
    textra = {k: tile_x(v, n) for k, v in extra.items()}
    want = renderer.denoise(W * n, H, tiled, levels, sigma_color=2.5, albedo=textra["albedo"].reshape(-1), sigma_albedo=0.2,
                            moments=textra["moments"], spp=4, sigma_luminance=4.0, var_scale=textra["scale"])
    got = gpu_denoise(renderer, planes, extra, levels, True, "scaled")
    m = n // 2
    for k in ("color", "background"):
        assert_bit_equal(got[k], want[k][:, m * W:(m + 1) * W], k)


def test_push_wrap_bit_equal_the_mirror(renderer):
    W, H = 32, 12
    (a, ma, va), (b, mb, vb) = push_frame(W, H, 1, W / 2), push_frame(W, H, 2, W / 2)
    vb[1, :3, 0] = [np.nan, np.inf, 3e9]
    vb[4:8, :, 0] += np.float32(0.1234567)  # tap positions that round
    want = run_push(a, ma, va, b, mb, vb, True)
    t = renderer.temporal_create(W, H)
    try:
        renderer.temporal_push(t, a, ma, va, reset=True, wrap=True, **T_KW)
        got = renderer.temporal_push(t, b, mb, vb, wrap=True, **T_KW)
    finally:
        t.close()
    for k in ("color", "background"):
        assert_bit_equal(got[0][k], want[0][k], k)
    assert_bit_equal(got[1], want[1], "moments")
    assert_bit_equal(got[2], want[2], "var_scale")
    # device planes
    import ctypes as C
    import torch
    t = renderer.temporal_create(W, H)
    try:
        outs = []
        for planes, mom, mv, reset in ((a, ma, va, 1), (b, mb, vb, 0)):
            d = {k: torch.from_numpy(np.ascontiguousarray(planes[k], np.float32).reshape(-1)).cuda() for k in ("color", "background", "normal")}
            m = torch.from_numpy(np.ascontiguousarray(mom.transpose(2, 0, 1)).reshape(2, -1)).cuda()
            mvd = torch.from_numpy(mv.reshape(-1)).cuda()
            oc, ob, om, sc = torch.empty_like(d["color"]), torch.empty_like(d["background"]), torch.empty_like(m), torch.empty(W * H, device="cuda")
            pin = L.RaynFilmPlanes(d["color"].data_ptr(), None, d["background"].data_ptr(), d["normal"].data_ptr(), L.MEM_DEVICE)
            pout = L.RaynFilmPlanes(oc.data_ptr(), None, ob.data_ptr(), None, L.MEM_DEVICE)
            mi = L.RaynMomentPlanes(m[0].data_ptr(), m[1].data_ptr(), L.MEM_DEVICE)
            mo = L.RaynMomentPlanes(om[0].data_ptr(), om[1].data_ptr(), L.MEM_DEVICE)
            desc = L.RaynTemporalDesc(T_KW["alpha_min"], T_KW["sigma_depth"], T_KW["normal_cos"], reset)
            L.check(renderer._lib.rayn_b200_temporal_push_wrap(renderer.ctx, t.handle, C.byref(desc), C.byref(pin), C.byref(mi), mvd.data_ptr(),
                                                               C.byref(pout), C.byref(mo), sc.data_ptr()), renderer.ctx)
            L.check(renderer._lib.rayn_b200_sync(renderer.ctx), renderer.ctx)
            outs.append((oc.cpu().numpy(), sc.cpu().numpy()))
    finally:
        t.close()
    assert_bit_equal(outs[1][0].reshape(H, W, 3), want[0]["color"], "device colour")
    assert_bit_equal(outs[1][1].reshape(H, W), want[2], "device var_scale")


def test_wrap_entry_points_reject_bad_arguments(renderer):
    import ctypes as C
    W, H = 8, 8
    planes, extra = film_with_guides(W, H, 1)
    for bad in (dict(iterations=0), dict(sigma_luminance=0.0), dict(sigma_luminance=float("nan")), dict(spp=0)):
        kw = dict(moments=extra["moments"], spp=bad.get("spp", 4), sigma_luminance=bad.get("sigma_luminance", 4.0))
        with pytest.raises(L.RaynError):
            renderer.denoise(W, H, planes, bad.get("iterations", 3), wrap=True, **kw)
    t = renderer.temporal_create(W, H)
    try:
        desc = L.RaynTemporalDesc(0.0, 0.1, 0.5, 0)  # alpha_min 0 is out of range
        assert renderer._lib.rayn_b200_temporal_push_wrap(renderer.ctx, t.handle, C.byref(desc), None, None, None, None, None, None) == \
            L.RAYN_ERR_INVALID_ARG
    finally:
        t.close()


# ---- sequences and the host ----------------------------------------------------------------------------------------------
def seam_ratio(img):
    """mean |column 0 - column W-1| over the mean |column x+1 - column x| of the six interior pairs next to the seam (the
    same part of the scene, so the ratio compares the seam with its neighbourhood, not with the rest of the picture)"""
    seam = np.abs(img[:, 0] - img[:, -1]).mean()
    w = img.shape[1]
    inner = np.mean([np.abs(img[:, x + 1] - img[:, x]).mean() for x in (0, 1, 2, w - 4, w - 3, w - 2)])
    return seam / inner


def orbit_sequence(monkeypatch, wrap_allowed):
    """config 3 seen by a panorama orbiting the fractal and looking outwards, so the seam looks at the fractal; the wrapped
    calls are recorded, and with wrap_allowed False forced off"""
    W, H = 96, 48
    c = configs.baseline_config(3, res=(W, H), samples=1, max_bounces=3)

    def origin(t):
        return Vec3(4.0 * math.sin(0.3 * t), 0.4, 4.0 * math.cos(0.3 * t))

    def at(t):
        return Vec3(8.0 * math.sin(0.3 * t), 0.8, 8.0 * math.cos(0.3 * t))
    cam = c["world"].cameras.add_camera(EquirectangularCamera((W, H), origin, at, Vec3(0.0, 1.0, 0.0)))
    calls = []
    for name in ("temporal_push", "denoise"):
        orig = getattr(Renderer, name)

        def rec(self, *a, _orig=orig, _name=name, **kw):
            calls.append((_name, kw.get("wrap")))
            if not wrap_allowed:
                kw["wrap"] = False
            return _orig(self, *a, **kw)
        monkeypatch.setattr(Renderer, name, rec)
    f = Film(["color", "alpha", "background", "normal"], (W, H))
    ratios = []
    f.render_sequence(c["world"], cam, c["integrator"], None, TILE, range(1, 5), 24, 1 / 48, 1,
                      on_frame=lambda film: ratios.append(seam_ratio(film.channels["color"] + film.channels["background"])))
    monkeypatch.undo()
    return calls, ratios, f


# The seam may differ no more than its neighbouring column pairs do, on average over frames 2-4.  The films are bit-exact
# functions of the scene (they match the oracle), so the ratios do not move between runs: 0.79 wrapped, 1.13 without the wrap
# (H100, both mul_add builds).
SEAM_FACTOR = 1.0


def test_sequence_denoises_across_the_seam(monkeypatch):
    """over frames 2-4 (the history in use), the seam of the wrapped sequence is no rougher than its neighbourhood, and the same
    sequence pushed and filtered without the wrap fails that; frame by frame its seam is rougher than the wrapped one's"""
    calls, ratios, f = orbit_sequence(monkeypatch, True)
    assert f.panorama and calls and all(w is True for _, w in calls)
    calls, plain, _ = orbit_sequence(monkeypatch, False)
    assert np.mean(ratios[1:]) <= SEAM_FACTOR < np.mean(plain[1:]), (ratios, plain)
    assert all(a < b for a, b in zip(ratios[1:], plain[1:])), (ratios, plain)


@pytest.mark.skipif(L.MULADD_FUSED, reason="rayn_host links the product library, the unfused mul_add build")
def test_rayn_host_panorama_writes_the_python_planes(tmp_path):
    from rayn_b200 import build
    from rayn_b200.scene import BlackmanHarrisFilter
    exe = os.path.join(os.path.dirname(build.build()), "rayn_host")
    W, H = 64, 32
    out = tmp_path / "pano.bin"
    subprocess.run([exe, "--config", "1", "--res", str(W), str(H), "--samples", "1", "--bounces", "2", "--panorama", "--denoise", "3",
                    "--dump", str(out)], check=True, capture_output=True)
    got = np.fromfile(out, np.float32)
    c, cam, _ = panorama_config(1, (W, H), 1, 2)
    start = np.float32(1) * (np.float32(1.0) / np.float32(24))
    tr = (float(start), float(start + np.float32(1.0) / np.float32(24.0)))
    f = Film(["color", "alpha", "background", "normal"], (W, H))
    f.render_frame_into(c["world"], cam, c["integrator"], BlackmanHarrisFilter(1.5), TILE, 1, tr, 1)
    f.denoise(3)
    want = np.concatenate([f.channels[k].reshape(-1) for k in CH])
    assert_bit_equal(got, want, "rayn_host --panorama --denoise 3")
