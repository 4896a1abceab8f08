"""CPU mirrors of the motion plane (tests/motion_oracle.cpp), the temporal push and the scaled variance denoise
(tests/temporal_oracle.cpp): the motion records against float64 closed forms (a pinhole camera translating sideways past the
scene, a sphere moving in front of a static camera), the identities the header guarantees (static scenes give dx = dy = +0 and
z_prev == z; alpha = 1 returns the frame bit for bit with s = 1; a cumulative mean gives s = 1/n; a unit scale is the unscaled
filter), the argument rules and the RaynTemporalDesc layout."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from rayn_b200 import _lib as L
from rayn_b200 import configs
from rayn_b200.film import denoise_desc
from rayn_b200.scene import Lambertian, Linear, PinholeCamera, Sphere, Vec3

import moments_oracle as mo
import temporal_oracle as to
from helpers import assert_bit_equal, small_config
from test_cpu_denoise import random_film

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TR = configs.frame_time_range(1)
DT = 1.0 / 24.0
ORIGIN = np.array([-0.45, 0.2, 2.0]) * 2.25


def basis(origin, at, up=(0.0, 1.0, 0.0)):
    bw = (origin - at) / np.linalg.norm(origin - at)
    bu = np.cross(up, bw)
    return bu / np.linalg.norm(bu), bw


def camera_desc(world, cam):
    desc, _ = world.flatten(cam)
    return desc.camera


def add_camera(c, cam):
    return c["world"].cameras.add_camera(cam)


def test_static_scene_gives_exact_zero_motion():
    """a static camera and scene: both projections are the same function of the same point, so dx = dy = +0 and z_prev == z"""
    c, inp = small_config(3, (23, 17), 2, 1)
    plane, per = to.render_motion(c["world"], c["camera"], inp, (8, 8), c["integrator"], TR, DT)
    valid = ~np.isnan(per[..., 2])
    assert valid.any()
    assert (per[..., :2][valid].view(np.uint32) == 0).all()
    assert_bit_equal(per[..., 3][valid], per[..., 2][valid], "z_prev")
    assert (plane[..., :2].view(np.uint32) == 0).all()
    assert_bit_equal(plane[..., 3], plane[..., 2], "plane z_prev")


def test_camera_translating_sideways():
    """the camera moves along its own right axis bu (origin and look-at point together): a point at view depth z moves by
    dx = 0.5 W v dt / (z hx) pixels between frames, dy = 0 and z_prev = z (float64 closed form per sample)"""
    W, H = 40, 28
    c, inp = small_config(3, (W, H), 2, 1)
    bu, _ = basis(ORIGIN, np.zeros(3))
    v = 0.8
    vel = Vec3(*(v * bu))
    cam = add_camera(c, PinholeCamera((W, H), 60.0, Linear(Vec3(*ORIGIN), vel), Linear(Vec3(0, 0, 0), vel), Vec3(0, 1, 0)))
    hx = camera_desc(c["world"], cam).half_size[0]
    _, per = to.render_motion(c["world"], cam, inp, (8, 8), c["integrator"], TR, DT)
    valid = ~np.isnan(per[..., 2])
    assert valid.mean() > 0.9
    z = per[..., 2][valid].astype(np.float64)
    expect = 0.5 * W * v * DT / (z * hx)
    np.testing.assert_allclose(per[..., 0][valid], expect, rtol=2e-4, atol=2e-4)
    np.testing.assert_allclose(per[..., 1][valid], 0.0, atol=2e-4)
    np.testing.assert_allclose(per[..., 3][valid], z, rtol=1e-5)


def test_sphere_moving_in_front_of_a_static_camera():
    """a sphere moving along the camera's right axis: its hits move by dx = -0.5 W s dt / (z hx), everything else is exactly 0"""
    W, H = 40, 28
    c, inp = small_config(3, (W, H), 2, 1)
    bu, bw = basis(ORIGIN, np.zeros(3))
    s = 3.0
    centre = ORIGIN - 2.5 * bw
    mat = c["world"].materials.add_material(Lambertian((0.5, 0.5, 0.5)))
    c["world"].hitables.push(Sphere(Linear(Vec3(*centre), Vec3(*(s * bu))), 0.3, mat))
    hx = camera_desc(c["world"], c["camera"]).half_size[0]
    _, per = to.render_motion(c["world"], c["camera"], inp, (8, 8), c["integrator"], TR, DT)
    valid = ~np.isnan(per[..., 2])
    moving = valid & (per[..., 0] != 0)
    assert 0.02 < moving.mean() < 0.9
    assert (per[..., :2][valid & ~moving].view(np.uint32) == 0).all()
    z = per[..., 2][moving].astype(np.float64)
    np.testing.assert_allclose(per[..., 0][moving], -0.5 * W * s * DT / (z * hx), rtol=1e-3, atol=2e-4)
    np.testing.assert_allclose(per[..., 1][moving], 0.0, atol=2e-3)


def test_resolve_is_the_mean_over_valid_samples():
    c, inp = small_config(3, (21, 13), 2, 1)
    bu, _ = basis(ORIGIN, np.zeros(3))
    cam = add_camera(c, PinholeCamera((21, 13), 60.0, Linear(Vec3(*ORIGIN), Vec3(*(0.5 * bu))), Vec3(0, 0, 0), Vec3(0, 1, 0)))
    plane, per = to.render_motion(c["world"], cam, inp, (8, 8), c["integrator"], TR, DT)
    ok = ~np.isnan(per[..., 2])
    n = ok.sum(axis=2)
    s = np.where(ok[..., None], per, 0).astype(np.float64).sum(axis=2)
    has = n > 0
    np.testing.assert_allclose(plane[has], s[has] / n[has][:, None], rtol=1e-6, atol=1e-7)
    assert np.isinf(plane[~has][:, 2:]).all()


def test_tile_grid_quirk_pixels_never_match():
    """film.rs:399-404: a 20-wide film with 16-wide tiles has one tile column; pixels 16..19 get (0, 0, +inf, +inf)"""
    c, inp = small_config(3, (20, 9), 1, 1)
    plane, _ = to.render_motion(c["world"], c["camera"], inp, (16, 16), c["integrator"], TR, DT)
    assert (plane[:, 16:, :2] == 0).all() and np.isposinf(plane[:, 16:, 2:]).all()
    assert np.isfinite(plane[:, :16, 2]).any()


# ---- temporal push ----
def frame(w, h, seed, static=True):
    p = random_film(w, h, seed)
    rng = np.random.default_rng(seed)
    p["color"] = rng.uniform(0, 1, (h, w, 3)).astype(np.float32)
    p["background"] = rng.uniform(0, 0.2, (h, w, 3)).astype(np.float32)
    m = rng.uniform(0, 1, (h, w, 2)).astype(np.float32)
    mv = np.zeros((h, w, 4), np.float32)
    mv[..., 2] = mv[..., 3] = 3.0
    if not static:
        mv[..., 0] = rng.uniform(-1.5, 1.5, (h, w))
        mv[..., 1] = rng.uniform(-1.5, 1.5, (h, w))
        mv[..., 3] = rng.uniform(2.9, 3.1, (h, w))
    return p, m, mv


def test_alpha_one_returns_every_frame_unchanged():
    w, h = 17, 11
    t = to.TemporalMirror(w, h)
    for k in range(4):
        p, m, mv = frame(w, h, 40 + k, static=False)
        rc, out, om, s = t.push(p, m, mv, 1.0, 0.1, -1.0)
        assert rc == L.RAYN_OK
        assert_bit_equal(out["color"], p["color"]), assert_bit_equal(out["background"], p["background"])
        assert_bit_equal(om, m)
        assert (s == 1.0).all()


def test_cumulative_mean_on_a_static_view():
    """alpha_min -> 0, no motion, equal depths and normals: the blend is the running mean, s = 1/n"""
    w, h = 13, 9
    t = to.TemporalMirror(w, h)
    frames = [frame(w, h, 60 + k) for k in range(6)]
    for k, (p, m, mv) in enumerate(frames):
        p["normal"] = frames[0][0]["normal"]
        rc, out, om, s = t.push(p, m, mv, 1e-6, 0.01, 0.9)
        assert rc == L.RAYN_OK
        mean = np.mean([f[0]["color"].astype(np.float64) for f in frames[:k + 1]], axis=0)
        np.testing.assert_allclose(out["color"], mean, rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(om, np.mean([f[1].astype(np.float64) for f in frames[:k + 1]], axis=0), rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(s, 1.0 / (k + 1), rtol=1e-5)


def test_reset_and_disocclusion_take_the_current_frame():
    w, h = 15, 10
    t = to.TemporalMirror(w, h)
    p0, m0, mv0 = frame(w, h, 80)
    t.push(p0, m0, mv0, 0.2, 0.05, 0.5)
    p1, m1, mv1 = frame(w, h, 81)
    p1["normal"] = p0["normal"]
    mv1[:5, :, 3] = 10.0  # depth disagrees with the history: disoccluded
    mv1[5:8, :, 0] = 100.0  # reprojects outside the image
    rc, out, om, s = t.push(p1, m1, mv1, 0.2, 0.05, 0.5)
    assert rc == 0
    assert_bit_equal(out["color"][:8], p1["color"][:8])
    assert (s[:8] == 1).all() and (s[8:] < 1).all()
    rc, out, om, s = t.push(p0, m0, mv0, 0.2, 0.05, 0.5, reset=True)
    assert_bit_equal(out["color"], p0["color"]), assert_bit_equal(om, m0)
    assert (s == 1).all()


@pytest.mark.parametrize("field,value", [("alpha_min", 0.0), ("alpha_min", 1.5), ("alpha_min", np.nan), ("sigma_depth", 0.0),
                                         ("normal_cos", 1.5), ("normal_cos", np.nan), ("reset", 2)])
def test_mirror_rejects_bad_descriptors(field, value):
    t = to.TemporalMirror(4, 4)
    p, m, mv = frame(4, 4, 1)
    kw = dict(alpha_min=0.2, sigma_depth=0.1, normal_cos=0.5, reset=False)
    kw[field] = value
    if field == "reset":
        d = L.RaynTemporalDesc(0.2, 0.1, 0.5, value)
        z = np.zeros(16 * 14, np.float32)
        rc = to.temporal_lib().rayn_oracle_temporal_push(4, 4, C.byref(d), *([z.ctypes.data] * 13))
    else:
        rc = t.push(p, m, mv, **kw)[0]
    assert rc == L.RAYN_ERR_INVALID_ARG


def test_unit_scale_is_the_unscaled_filter():
    w, h = 19, 14
    p = random_film(w, h, 90)
    m = np.random.default_rng(90).uniform(0, 2, (h, w, 2)).astype(np.float32)
    d = denoise_desc(3, np.inf, 0.5, 0.5)
    rc0, a = mo.denoise(w, h, p, d, 4.0, 16, m)
    rc1, b = to.denoise_scaled(w, h, p, d, 4.0, 16, m, np.ones((h, w), np.float32))
    assert rc0 == rc1 == 0
    for k in a:
        assert_bit_equal(b[k], a[k], k)
    rc2, c_ = to.denoise_scaled(w, h, p, d, 4.0, 16, m, np.full((h, w), 0.25, np.float32))
    assert rc2 == 0 and not np.array_equal(c_["color"], a["color"])


def test_temporal_desc_layout_matches_the_c_compiler(tmp_path):
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "rayn_b200.h"\nint main(){'
                   'printf("%zu %zu %zu %zu %zu\\n", sizeof(RaynTemporalDesc), offsetof(RaynTemporalDesc, alpha_min), '
                   'offsetof(RaynTemporalDesc, sigma_depth), offsetof(RaynTemporalDesc, normal_cos), offsetof(RaynTemporalDesc, reset));}')
    exe = tmp_path / "sz"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    T = L.RaynTemporalDesc
    assert got == [C.sizeof(T), T.alpha_min.offset, T.sigma_depth.offset, T.normal_cos.offset, T.reset.offset]


def test_pixel_without_a_hit_takes_no_history():
    """a sky / miss pixel (motion (0, 0, +inf, +inf), normal 0) never matches a history tap, whatever normal_cos"""
    w, h = 9, 7
    t = to.TemporalMirror(w, h)
    p0, m0, mv0 = frame(w, h, 120)
    p0["color"][:] = 1.0
    t.push(p0, m0, mv0, 0.5, 0.1, -1.0)
    p1, m1, mv1 = frame(w, h, 121)
    p1["color"][:] = 0.0
    p1["normal"][:] = 0.0
    mv1[..., 2:] = np.inf
    rc, out, om, s = t.push(p1, m1, mv1, 0.5, 0.1, -1.0)
    assert rc == 0
    assert_bit_equal(out["color"], p1["color"]), assert_bit_equal(om, m1)
    assert (s == 1).all()


def test_orthographic_depths_below_zero_still_match():
    """an orthographic view depth may be <= 0: the depth test compares against |z_prev|"""
    w, h = 9, 7
    t = to.TemporalMirror(w, h)
    for k in range(3):
        p, m, mv = frame(w, h, 130 + k)
        mv[..., 2:] = -3.0
        p["normal"][:] = (0.0, 1.0, 0.0)
        rc, out, om, s = t.push(p, m, mv, 0.25, 0.05, 0.5)
        assert rc == 0
        np.testing.assert_allclose(s, 1.0 if k == 0 else (0.5 if k == 1 else 1.0 / 3.0), rtol=1e-6)


# ---- the projection against float64 geometry ----
def _v(a):
    return np.array(list(a), np.float64)


def proj64(cam, X, t, W, H):
    """float64 projection of points X [..., 3] at times t [...] by the camera's linear-in-time parameters: film pixels and
    view depth of the ray through the pinhole / lens centre (perspective) or along the view direction (orthographic)"""
    t = np.asarray(t, np.float64)[..., None]
    o = _v(cam.origin) + _v(cam.origin_velocity) * t
    at = _v(cam.at) + _v(cam.at_velocity) * t
    up = _v(cam.up) + _v(cam.up_velocity) * t
    nz = lambda a: a / np.linalg.norm(a, axis=-1, keepdims=True)  # noqa: E731
    r = X.astype(np.float64) - o
    hx, hy = cam.half_size[0], cam.half_size[1]
    if cam.kind == L.CAMERA_ORTHOGRAPHIC:
        fwd = nz(at - o)
        right = nz(np.cross(fwd, up))
        upv = np.cross(right, fwd)
        z = (r * fwd).sum(-1)
        return (((r * right).sum(-1) + hx) / cam.full_size[0] * W, ((r * upv).sum(-1) + hy) / cam.full_size[1] * H, z)
    back = nz(o - at)
    right = nz(np.cross(up, back))
    upv = np.cross(back, right)
    z = -(r * back).sum(-1)
    return ((r * right).sum(-1) / (z * hx) * 0.5 + 0.5) * W, ((r * upv).sum(-1) / (z * hy) * 0.5 + 0.5) * H, z


def moving_cameras(c, res):
    from rayn_b200.scene import OrthographicCamera, ThinLensCamera
    cams = c["world"].cameras
    return {
        "pan": cams.add_camera(PinholeCamera(res, 60.0, Vec3(*ORIGIN), Linear(Vec3(0, 0, 0), Vec3(0.9, -0.3, 0.0)), Vec3(0, 1, 0))),
        "dolly": cams.add_camera(PinholeCamera(res, 60.0, Linear(Vec3(*ORIGIN), Vec3(*(-ORIGIN * 0.3))), Vec3(0, 0, 0), Vec3(0, 1, 0))),
        "ortho": cams.add_camera(OrthographicCamera(res, 11.0 / 4.0, Linear(Vec3(9.5, -3.5, 9.5), Vec3(1.0, 0.5, -0.5)),
                                                    Linear(Vec3(0.0, 0.8, 0.0), Vec3(0.3, 0.0, 0.2)), Vec3(0.0, 1.0, 0.0))),
        "thinlens": cams.add_camera(ThinLensCamera(res, 60.0, 0.05, Linear(Vec3(*ORIGIN), Vec3(1.2, 0.0, -0.4)), Vec3(0, 0, 0),
                                                   Linear(Vec3(0, 1, 0), Vec3(0.3, 0, 0)), Vec3(0, 0, 0))),
        "pinhole_lens": cams.add_camera(ThinLensCamera(res, 60.0, 0.0, Linear(Vec3(*ORIGIN), Vec3(1.2, 0.0, -0.4)), Vec3(0, 0, 0),
                                                       Vec3(0, 1, 0), Vec3(0, 0, 0))),
    }


@pytest.mark.parametrize("kind", ["pan", "dolly", "ortho", "pinhole_lens"])
def test_projection_inverts_camera_ray(kind):
    """the current-time projection of every hit point is the film position (u W, v H) of the ray that found it (the thin
    lens through its lens centre, so with aperture 0)"""
    W, H = 36, 26
    c, inp = small_config(3, (W, H), 2, 1)
    cam = moving_cameras(c, (W, H))[kind]
    _, per, geo = to.render_motion(c["world"], cam, inp, (8, 8), c["integrator"], TR, DT, geometry=True)
    ok = ~np.isnan(per[..., 2])
    assert ok.mean() > 0.5
    px, py, z = proj64(camera_desc(c["world"], cam), geo[..., :3][ok], geo[..., 3][ok], W, H)
    np.testing.assert_allclose(px, geo[..., 4][ok].astype(np.float64) * W, atol=2e-3)
    np.testing.assert_allclose(py, geo[..., 5][ok].astype(np.float64) * H, atol=2e-3)
    np.testing.assert_allclose(per[..., 2][ok], z, rtol=2e-5, atol=2e-5)


@pytest.mark.parametrize("kind", ["pan", "dolly", "ortho", "thinlens"])
def test_motion_matches_float64_projection(kind):
    """(dx, dy, z, z_prev) of every valid sample against the float64 projection at tau and tau - frame_dt"""
    W, H = 36, 26
    c, inp = small_config(3, (W, H), 2, 1)
    cam = moving_cameras(c, (W, H))[kind]
    _, per, geo = to.render_motion(c["world"], cam, inp, (8, 8), c["integrator"], TR, DT, geometry=True)
    ok = ~np.isnan(per[..., 2])
    X, t = geo[..., :3][ok], geo[..., 3][ok].astype(np.float64)
    cd = camera_desc(c["world"], cam)
    x1, y1, z1 = proj64(cd, X, t, W, H)
    x0, y0, z0 = proj64(cd, X, t - DT, W, H)
    assert np.abs(x0 - x1).max() > 0.05  # the camera moves
    np.testing.assert_allclose(per[..., 0][ok], x0 - x1, atol=3e-3)
    np.testing.assert_allclose(per[..., 1][ok], y0 - y1, atol=3e-3)
    np.testing.assert_allclose(per[..., 2][ok], z1, rtol=2e-5, atol=2e-5)
    np.testing.assert_allclose(per[..., 3][ok], z0, rtol=2e-5, atol=2e-5)


def test_film_motion_channel_rules(tmp_path):
    """"motion" is a Film channel that render_adaptive and save_to reject, like "moments"; render_sequence needs the four film
    channels"""
    from rayn_b200.film import Film
    f = Film(["color", "alpha", "background", "normal", "motion"], (8, 8))
    f.channels = {"motion": np.zeros((8, 8, 4), np.float32)}
    with pytest.raises(ValueError):
        f.save_to(["motion"], str(tmp_path), "x")
    with pytest.raises(ValueError):
        f.render_adaptive(None, None, None, None, (8, 8), 1, (0.0, 1.0), 1)
    with pytest.raises(ValueError):
        Film(["color", "motion"], (8, 8)).render_sequence(None, None, None, None, (8, 8), range(1, 2), 24, 1 / 24, 1)
