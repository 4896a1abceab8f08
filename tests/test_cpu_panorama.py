"""The equirectangular (360-degree panorama) camera and the filters that wrap round its seam, on the CPU: the oracle's camera
against a float64 restatement, the motion projection as its inverse, a yaw with a closed-form answer, the wrapped denoise and
push against the non-wrapped filters by tiling and rolling identities, and the scene, host and argument rules."""
import math
import os
import subprocess

import numpy as np
import pytest

from rayn_b200 import _lib as L
from rayn_b200 import configs
from rayn_b200.film import FrameInputs, check_panorama_width, denoise_desc
from rayn_b200.scene import EquirectangularCamera, Linear

import mirrors
import panorama_mirrors as pm
from helpers import assert_bit_equal
from test_cpu_denoise import random_film

TR = configs.frame_time_range(1)
DT = 1.0 / 24.0


def panorama_config(n, res, samples, max_bounces, origin=None):
    """config n with an EquirectangularCamera at its camera's origin (or at `origin`), at and up, added to its world: (config,
    the panorama's camera handle, FrameInputs)"""
    c = configs.baseline_config(n, res=res, samples=samples, max_bounces=max_bounces)
    src = c["world"].cameras.get(c["camera"])
    o = Linear(*src.origin) if origin is None else Linear(np.float32(origin), np.zeros(3))
    cam = c["world"].cameras.add_camera(EquirectangularCamera(res, o, Linear(*src.at), Linear(*src.up)))
    return c, cam, FrameInputs(res[0], res[1], c["samples"], c["integrator"])


def desc_of(world, cam):
    return world.flatten(cam)[0].camera


def directions64(cd, u, v):
    """the camera statement in float64 from the stored float32 origin, at and up"""
    o, at, up = (np.array(getattr(cd, k), np.float64) for k in ("origin", "at", "up"))
    bw = (o - at) / np.linalg.norm(o - at)
    bu = np.cross(up, bw)
    bu /= np.linalg.norm(bu)
    bv = np.cross(bw, bu)
    phi, th = (np.asarray(u, np.float64) - 0.5) * 2 * np.pi, (np.asarray(v, np.float64) - 0.5) * np.pi
    d = bu * (np.cos(th) * np.sin(phi))[:, None] + bv * np.sin(th)[:, None] - bw * (np.cos(th) * np.cos(phi))[:, None]
    return d


def angle(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.arctan2(np.linalg.norm(np.cross(a, b), axis=1), np.sum(a * b, axis=1))


# ---- the camera ----------------------------------------------------------------------------------------------------------
def test_oracle_directions_against_float64():
    """Directions over a (u, v) grid with u outside [0, 1] and both poles: within 1e-6 rad of the float64 statement (the
    float pi and 2 pi, the sincos and the normalisation each cost a few 1e-8 rad), unit length, and u = 0 and u = 1 agree."""
    c, cam, _ = panorama_config(3, (64, 32), 1, 1)
    cd = desc_of(c["world"], cam)
    uu, vv = np.meshgrid(np.linspace(-0.25, 1.25, 61, dtype=np.float32), np.linspace(0.0, 1.0, 33, dtype=np.float32))
    u, v = uu.ravel(), vv.ravel()
    ro, rd = pm.kat_camera_rays(cd, u, v)
    assert (ro == np.float32(cd.origin)).all()
    err = angle(rd, directions64(cd, u, v))
    assert err.max() < 1e-6, err.max()
    assert np.abs(np.linalg.norm(rd.astype(np.float64), axis=1) - 1.0).max() < 1e-6
    v1 = np.linspace(0.0, 1.0, 33, dtype=np.float32)
    _, d0 = pm.kat_camera_rays(cd, np.zeros_like(v1), v1)
    _, d1 = pm.kat_camera_rays(cd, np.ones_like(v1), v1)
    assert angle(d0, d1).max() < 1e-6
    # the screen centre looks at `at`, +u turns towards bu, v = 1 is the up pole
    _, dc = pm.kat_camera_rays(cd, np.float32([0.5, 0.75, 0.5]), np.float32([0.5, 0.5, 1.0]))
    o, at, up = (np.array(getattr(cd, k), np.float64) for k in ("origin", "at", "up"))
    bu = np.cross(up, o - at)
    bu /= np.linalg.norm(bu)
    bv = np.cross(o - at, bu)
    assert angle(dc, np.stack([at - o, bu, bv])).max() < 1e-6


def test_panorama_mirror_keeps_the_reference_cameras():
    """the panorama mirror's oracle renders the reference cameras exactly as the oracle does"""
    from oracle import binding
    c = configs.baseline_config(1, res=(24, 16), samples=1, max_bounces=2)
    inp = FrameInputs(24, 16, 1, c["integrator"])
    want, _ = binding.render(c["world"], c["camera"], inp, (8, 8), c["integrator"], TR)
    got = pm.oracle_render(c["world"], c["camera"], inp, (8, 8), c["integrator"], TR)
    for k in want:
        assert_bit_equal(got[k], want[k], k)


def test_projection_inverts_camera_ray():
    """proj(o + d t) gives back (u W, v H) to 1e-3 px for random rays, the seam columns included (u just below 0 and just
    above 1 project to the other side, so px is compared modulo W), and z = t"""
    W, H = 64, 32
    c, cam, _ = panorama_config(3, (W, H), 1, 1)
    cd = desc_of(c["world"], cam)
    rng = np.random.default_rng(5)
    u = np.concatenate([rng.uniform(0, 1, 3000), rng.uniform(-0.01, 0.01, 500), rng.uniform(0.99, 1.01, 500)]).astype(np.float32)
    v = rng.uniform(0.02, 0.98, len(u)).astype(np.float32)
    t = rng.uniform(0.5, 20.0, len(u))
    ro, rd = pm.kat_camera_rays(cd, u, v)
    X = (ro.astype(np.float64) + rd.astype(np.float64) * t[:, None]).astype(np.float32)
    p = pm.kat_project(cd, W, H, X).astype(np.float64)
    dx = np.mod(p[:, 0] - u.astype(np.float64) * W + W / 2, W) - W / 2
    assert np.abs(dx).max() < 1e-3
    assert np.abs(p[:, 1] - v.astype(np.float64) * H).max() < 1e-3
    np.testing.assert_allclose(p[:, 2], t, rtol=1e-5)
    assert ((u < 0) & (p[:, 0] > W / 2)).any() and ((u > 1) & (p[:, 0] < W / 2)).any()


def yaw_camera(world, res, origin, yaw):
    at = np.asarray(origin, np.float64) + np.array([math.sin(yaw), 0.0, -math.cos(yaw)])
    return world.cameras.add_camera(EquirectangularCamera(res, Linear(np.float32(origin), np.zeros(3)), Linear(at.astype(np.float32), np.zeros(3)),
                                 Linear(np.float32([0, 1, 0]), np.zeros(3))))


def yaw_scenes(W, H, k):
    """config 1 (a sphere inside the sky sphere: every ray hits) seen by two constant panoramas at one origin with world up,
    the previous one turned by 2 pi k / W.  A point at azimuth a is at phi = a - yaw, so the previous frame sees every point
    k pixels to the LEFT: dx = -k, dy = 0."""
    c = configs.baseline_config(1, res=(W, H), samples=1, max_bounces=1)
    origin = (0.0, 0.3, 3.0)
    cur, prev = yaw_camera(c["world"], (W, H), origin, 0.4), yaw_camera(c["world"], (W, H), origin, 0.4 + 2 * math.pi * k / W)
    return c, cur, prev


def test_yaw_closed_form_in_the_mirror():
    W, H, k = 64, 32, 3
    c, cur, prev = yaw_scenes(W, H, k)
    inp = FrameInputs(W, H, 1, c["integrator"])
    scene, pscene = c["world"].flatten(cur)[0], c["world"].flatten(prev)[0]
    plane, per, geo = pm.render_motion(scene, inp, (16, 16), c["integrator"], TR, DT, prev=pscene, geometry=True)
    ok = ~np.isnan(per[..., 2])
    assert ok.all()
    np.testing.assert_allclose(per[..., 0][ok], -k, atol=1e-3)
    np.testing.assert_allclose(per[..., 1][ok], 0.0, atol=1e-3)
    assert (geo[..., 4][ok] * W < k).sum() > 0  # samples whose previous position lies across the seam
    np.testing.assert_allclose(plane[..., 0], -k, atol=1e-3)


# ---- the wrapped filters -------------------------------------------------------------------------------------------------
GUIDES = [(alb, var) for alb in (False, True) for var in (None, "unscaled", "scaled")]


def film_with_guides(w, h, seed):
    rng = np.random.default_rng(seed + 100)
    f = random_film(w, h, seed)
    lum = (0.2126 * f["color"][..., 0] + 0.7152 * f["color"][..., 1]) + 0.0722 * f["color"][..., 2]
    extra = {"albedo": rng.uniform(0, 1, (h, w, 3)).astype(np.float32),
             "moments": np.stack([lum ** 2 + rng.uniform(0, 0.3, (h, w)), rng.uniform(0, 3, (h, w))], axis=2).astype(np.float32),
             "scale": rng.uniform(0.2, 1.0, (h, w)).astype(np.float32)}
    return f, extra


def denoise_mirror(planes, extra, levels, alb, var, wrap):
    h, w = planes["normal"].shape[:2]
    kw = {}
    if alb:
        kw.update(albedo=extra["albedo"], sigma_albedo=0.2)
    if var:
        kw.update(moments=extra["moments"], spp=4, sigma_luminance=4.0, var_scale=extra["scale"] if var == "scaled" else None)
    rc, out = (pm.denoise_wrap if wrap else mirrors.denoise)(w, h, planes, denoise_desc(levels), **kw)
    assert rc == L.RAYN_OK
    return {k: v.reshape(h, w, 3) for k, v in out.items()}


def tile_x(a, n):
    return np.concatenate([a] * n, axis=1)


@pytest.mark.parametrize("alb,var", GUIDES)
def test_denoise_wrap_commutes_with_roll(alb, var):
    W, H = 20, 9
    planes, extra = film_with_guides(W, H, 11)
    base = denoise_mirror(planes, extra, 4, alb, var, True)
    for s in (1, 7, W - 1):
        rolled = denoise_mirror({k: np.roll(v, s, axis=1) for k, v in planes.items()}, {k: np.roll(v, s, axis=1) for k, v in extra.items()},
                                4, alb, var, True)
        for k in ("color", "background"):
            assert_bit_equal(rolled[k], np.roll(base[k], s, axis=1), f"{k}, roll {s}")


def test_denoise_wrap_differs_at_the_seam_only():
    """the wrap changes the columns within reach of the seam and no other"""
    W, H = 40, 8
    planes, extra = film_with_guides(W, H, 3)
    a, b = denoise_mirror(planes, extra, 2, True, "unscaled", True), denoise_mirror(planes, extra, 2, True, "unscaled", False)
    diff = (a["color"] != b["color"]).any(axis=(0, 2))
    assert diff[0] and diff[-1] and not diff[6:W - 6].any()


def push_frame(w, h, seed, dx_range):
    """a frame and a motion plane whose dx, dy are multiples of 2^-8: with W <= 2^12 every tap position
    ((x + 0.5) + dx) - 0.5 of the film tiled three times is then exact in float (at most 14 integer bits and 8 fraction bits),
    so the tiled film's taps are the wrapped film's shifted by exactly W"""
    rng = np.random.default_rng(seed)
    f = random_film(w, h, seed)
    mom = rng.uniform(0, 3, (h, w, 2)).astype(np.float32)
    z = rng.uniform(1.0, 2.0, (h, w)).astype(np.float32)
    mv = np.stack([np.round(rng.uniform(-dx_range, dx_range, (h, w)) * 256) / 256, np.round(rng.uniform(-1.5, 1.5, (h, w)) * 256) / 256,
                   z, z * np.float32(1.01)], axis=2).astype(np.float32)
    mv[0, 0, 3] = np.inf  # a pixel without a hit
    return f, mom, mv


T_KW = dict(alpha_min=0.2, sigma_depth=0.5, normal_cos=-1.0)


def run_push(planes_a, mom_a, mv_a, planes_b, mom_b, mv_b, wrap):
    """a reset push of frame a, then a push of frame b, through pm.PushWrap (wrap) or the C++ mirror of the unwrapped push ->
    (planes, moments, var_scale, history [14, H, W]) of the second push"""
    h, w = planes_a["normal"].shape[:2]
    t = pm.PushWrap(w, h) if wrap else mirrors.TemporalMirror(w, h)
    rc, *_ = t.push(planes_a, mom_a, mv_a, reset=True, **T_KW)
    assert rc == 0
    rc, out, mom, scale = t.push(planes_b, mom_b, mv_b, **T_KW)
    assert rc == 0
    hist = t.hist if wrap else t.hist[t.cur].reshape(mirrors.N_HIST, h, w)
    return out, mom, scale, hist


def test_push_wrap_is_the_middle_of_the_tiled_film():
    """the numpy wrapped push against the C++ mirror of the unwrapped push on the film tiled three times: the middle copy, bit
    for bit (exact tap positions, see push_frame), history included"""
    W, H = 32, 12
    (a, ma, va), (b, mb, vb) = push_frame(W, H, 1, W / 2), push_frame(W, H, 2, W / 2)
    got = run_push(a, ma, va, b, mb, vb, True)
    t3 = [{k: tile_x(v, 3) for k, v in p.items()} if isinstance(p, dict) else tile_x(p, 3) for p in (a, ma, va, b, mb, vb)]
    want = run_push(*t3, False)
    for k in ("color", "background"):
        assert_bit_equal(got[0][k], want[0][k][:, W:2 * W], k)
    assert_bit_equal(got[1], want[1][:, W:2 * W], "moments")
    assert_bit_equal(got[2], want[2][:, W:2 * W], "var_scale")
    assert_bit_equal(got[3], want[3][:, :, W:2 * W], "history")
    # the seam mattered: some pixels take history across it, which the non-wrapped push on the untiled film does not
    plain = run_push(a, ma, va, b, mb, vb, False)
    assert not np.array_equal(plain[2], got[2])


def test_push_wrap_commutes_with_roll():
    W, H = 28, 10
    (a, ma, va), (b, mb, vb) = push_frame(W, H, 3, W / 2), push_frame(W, H, 4, W / 2)
    base = run_push(a, ma, va, b, mb, vb, True)
    for s in (1, 9, W - 1):
        r = [{k: np.roll(v, s, axis=1) for k, v in p.items()} if isinstance(p, dict) else np.roll(p, s, axis=1) for p in (a, ma, va, b, mb, vb)]
        got = run_push(*r, True)
        for k in ("color", "background"):
            assert_bit_equal(got[0][k], np.roll(base[0][k], s, axis=1), f"{k}, roll {s}")
        assert_bit_equal(got[2], np.roll(base[2], s, axis=1), f"var_scale, roll {s}")


def test_push_wrap_survives_non_finite_and_huge_motion():
    """NaN, +-inf and |dx| beyond 2^24 take no history (the current frame passes through); no index leaves the film"""
    W, H = 16, 6
    (a, ma, va), (b, mb, vb) = push_frame(W, H, 5, 4), push_frame(W, H, 6, 4)
    vb[1, :4, 0] = [np.nan, np.inf, -np.inf, 3e9]
    vb[2, :2, 0] = [-(2.0 ** 24) - 4096, 2.0 ** 24 - 64]
    out, _, scale, _ = run_push(a, ma, va, b, mb, vb, True)
    assert (scale[1, :4] == 1.0).all() and (out["color"][1, :4] == b["color"][1, :4]).all()
    assert np.isfinite(out["color"]).all()


# ---- scene, host and argument rules --------------------------------------------------------------------------------------
def test_scene_and_host_flatten_the_same_panorama(tmp_path):
    from rayn_b200 import build
    build.build()
    exe = os.path.join(os.path.dirname(build.OUT), "rayn_host")
    for n in (1, 3):
        out = tmp_path / f"pano{n}.bin"
        subprocess.run([exe, "--config", str(n), "--res", "160", "80", "--panorama", "--dump-scene", str(out)], check=True)
        c, cam, _ = panorama_config(n, (160, 80), 1, 1)
        d, keep = c["world"].flatten(cam)
        assert d.camera.kind == L.CAMERA_EQUIRECTANGULAR
        assert d.camera.half_pixel_size == np.float32(np.float32(np.pi) / np.float32(80)) / np.float32(2)
        want = b"".join(bytes(d.hitables[i]) for i in range(d.n_hitables)) + b"".join(bytes(d.materials[i]) for i in range(d.n_materials)) + \
            b"".join(bytes(d.lights[i]) for i in range(d.n_lights)) + bytes(d.camera) + bytes(d.volume)
        assert out.read_bytes() == want, f"config {n}"


def test_width_the_tile_grid_does_not_cover_is_refused(tmp_path):
    from rayn_b200 import build
    from rayn_b200.film import Film
    c, cam, _ = panorama_config(1, (70, 32), 1, 1)
    with pytest.raises(ValueError):
        check_panorama_width(c["world"], cam, 70, (16, 16))  # 70 % 16 = 6 < 8: the last 6 columns are not rendered
    for w in (64, 72, 79):
        assert check_panorama_width(c["world"], cam, w, (16, 16))
    assert not check_panorama_width(c["world"], c["camera"], 70, (16, 16))  # other cameras keep the reference grid
    f = Film(["color", "alpha", "background", "normal"], (70, 32))
    for call in (lambda: f.render_frame_into(c["world"], cam, c["integrator"], None, (16, 16), 1, TR, 1),
                 lambda: f.render_adaptive(c["world"], cam, c["integrator"], None, (16, 16), 1, TR, 1),
                 lambda: f.render_sequence(c["world"], cam, c["integrator"], None, (16, 16), range(1, 3), 24, 1 / 24, 1)):
        with pytest.raises(ValueError):
            call()
    exe = os.path.join(os.path.dirname(build.build()), "rayn_host")
    r = subprocess.run([exe, "--config", "1", "--res", "70", "32", "--panorama", "--dump-scene", str(tmp_path / "x.bin")], capture_output=True)
    assert r.returncode == 2 and not (tmp_path / "x.bin").exists()


@pytest.mark.parametrize("field,value", [("alpha_min", 0.0), ("alpha_min", 1.5), ("sigma_depth", 0.0), ("sigma_depth", np.nan),
                                         ("normal_cos", 1.5)])
def test_push_wrap_mirror_rejects_what_the_unwrapped_mirror_rejects(field, value):
    W, H = 8, 6
    f, mom, mv = push_frame(W, H, 1, 2)
    kw = dict(T_KW, **{field: value})
    assert pm.PushWrap(W, H).push(f, mom, mv, **kw)[0] == mirrors.TemporalMirror(W, H).push(f, mom, mv, **kw)[0] == L.RAYN_ERR_INVALID_ARG
