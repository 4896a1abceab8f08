"""CPU mirror of the motion plane against an explicit previous scene (rayn_b200_render_motion_prev, tests/motion_prev_oracle.cpp)
against float64 closed forms: a pinhole camera orbiting a static scene, a cut to an unrelated pose, a zoom, an orthographic pan,
a thin-lens camera, a static sphere displaced between frames and a moving sphere whose velocity changes.  Also the header's
identity with render_motion when prev is the uploaded scene, the argument rules of the mirror, the chord of closure parameters
(Linear.chord), flattening of worlds with and without closures, and render_sequence's argument rules for closure worlds."""
import math

import numpy as np
import pytest

from rayn_b200 import _lib as L
from rayn_b200 import configs
from rayn_b200.scene import Linear, OrthographicCamera, PinholeCamera, Sphere, ThinLensCamera, Vec3

import motion_prev_oracle as mpo
import temporal_oracle as to
from helpers import assert_bit_equal, small_config
from test_cpu_temporal import ORIGIN, basis, proj64

TR = configs.frame_time_range(1)
DT = 1.0 / 24.0
W, H = 36, 26


def rot_y(v, deg):
    a = math.radians(deg)
    c, s = math.cos(a), math.sin(a)
    return np.array([c * v[0] + s * v[2], v[1], -s * v[0] + c * v[2]])


def descs(world, cam, prev_cam, prev_world=None):
    """(uploaded scene, previous scene, keepalives): the previous scene is prev_world (default: world) with prev_cam"""
    d, k = world.flatten(cam)
    p, kp = (prev_world or world).flatten(prev_cam)
    return d, p, (k, kp)


def expect(cur, prev, P, tau, moved=None):
    """float64 (dx, dy, z, z_prev) of hit points P [n, 3] at camera times tau [n]; moved: P' where it is not P"""
    Pp = P if moved is None else moved
    x1, y1, z1 = proj64(cur, P, tau, W, H)
    x0, y0, z0 = proj64(prev, Pp, tau - DT, W, H)
    return x0 - x1, y0 - y1, z1, z0


def check(per, geo, cur, prev, moved_fn=None, min_valid=0.5, min_motion=0.05):
    ok = ~np.isnan(per[..., 2])
    assert ok.mean() > min_valid
    P, tau = geo[..., :3][ok].astype(np.float64), geo[..., 3][ok].astype(np.float64)
    dx, dy, z, zp = expect(cur, prev, P, tau, None if moved_fn is None else moved_fn(P, tau))
    assert np.abs(dx).max() > min_motion or np.abs(dy).max() > min_motion
    # rtol: near the previous camera's plane (a cut) film positions are large and ill-conditioned
    np.testing.assert_allclose(per[..., 0][ok], dx, rtol=1e-4, atol=3e-3)
    np.testing.assert_allclose(per[..., 1][ok], dy, rtol=1e-4, atol=3e-3)
    np.testing.assert_allclose(per[..., 2][ok], z, rtol=2e-5, atol=2e-5)
    np.testing.assert_allclose(per[..., 3][ok], zp, rtol=2e-5, atol=2e-5)
    if cur.kind != L.CAMERA_ORTHOGRAPHIC:
        assert (per[..., 3][ok] > 0).all()
    return ok


def prev_motion(c, cam, prev_cam, prev_world=None, inp=None):
    d, p, keep = descs(c["world"], cam, prev_cam, prev_world)
    _, per, geo = mpo.render_motion_prev(d, p, inp, (8, 8), c["integrator"], TR, DT, geometry=True)
    return per, geo, d.camera, p.camera


def test_orbit_of_a_static_scene():
    """the camera origin orbits the fractal about the y axis by 3 degrees between frames, looking at the centre"""
    c, inp = small_config(3, (W, H), 2, 1)
    cams = c["world"].cameras
    cur = cams.add_camera(PinholeCamera((W, H), 60.0, Vec3(*ORIGIN), Vec3(0, 0, 0), Vec3(0, 1, 0)))
    prv = cams.add_camera(PinholeCamera((W, H), 60.0, Vec3(*rot_y(ORIGIN, -3.0)), Vec3(0, 0, 0), Vec3(0, 1, 0)))
    per, geo, cd, pd = prev_motion(c, cur, prv, inp=inp)
    ok = check(per, geo, cd, pd, min_valid=0.9, min_motion=0.5)
    assert (per[..., 0][ok] != 0).mean() > 0.9


def test_cut_to_an_unrelated_pose():
    """the previous camera looks at the scene from the other side and above: points behind it are invalid samples"""
    c, inp = small_config(3, (W, H), 2, 1)
    cams = c["world"].cameras
    cur = cams.add_camera(PinholeCamera((W, H), 60.0, Vec3(*ORIGIN), Vec3(0, 0, 0), Vec3(0, 1, 0)))
    prv = cams.add_camera(PinholeCamera((W, H), 40.0, Vec3(3.0, 4.5, -2.5), Vec3(0.5, 0.2, 0.0), Vec3(0, 1, 0)))
    per, geo, cd, pd = prev_motion(c, cur, prv, inp=inp)
    check(per, geo, cd, pd, min_valid=0.3, min_motion=2.0)


def test_zoom():
    """only the field of view changes (60 -> 45 degrees): half_size comes from the previous camera"""
    c, inp = small_config(3, (W, H), 2, 1)
    cams = c["world"].cameras
    cur = cams.add_camera(PinholeCamera((W, H), 45.0, Vec3(*ORIGIN), Vec3(0, 0, 0), Vec3(0, 1, 0)))
    prv = cams.add_camera(PinholeCamera((W, H), 60.0, Vec3(*ORIGIN), Vec3(0, 0, 0), Vec3(0, 1, 0)))
    per, geo, cd, pd = prev_motion(c, cur, prv, inp=inp)
    assert pd.half_size[0] != cd.half_size[0]
    ok = check(per, geo, cd, pd, min_valid=0.9, min_motion=1.0)
    # a zoom about the image centre: film positions scale towards it, depths are unchanged
    np.testing.assert_allclose(per[..., 3][ok], per[..., 2][ok], rtol=1e-6)


def test_orthographic_pan():
    c, inp = small_config(3, (W, H), 2, 1)
    cams = c["world"].cameras
    cur = cams.add_camera(OrthographicCamera((W, H), 11.0 / 4.0, Vec3(9.5, -3.5, 9.5), Vec3(0.0, 0.8, 0.0), Vec3(0.0, 1.0, 0.0)))
    prv = cams.add_camera(OrthographicCamera((W, H), 11.0 / 4.0, Vec3(9.3, -3.5, 9.7), Vec3(-0.2, 0.8, 0.2), Vec3(0.0, 1.0, 0.0)))
    per, geo, cd, pd = prev_motion(c, cur, prv, inp=inp)
    check(per, geo, cd, pd, min_valid=0.3, min_motion=0.5)


def test_thin_lens():
    """thin-lens cameras with an aperture: the projection goes through the lens centre, as in render_motion"""
    c, inp = small_config(3, (W, H), 2, 1)
    cams = c["world"].cameras
    cur = cams.add_camera(ThinLensCamera((W, H), 60.0, 0.05, Vec3(*ORIGIN), Vec3(0, 0, 0), Vec3(0, 1, 0), Vec3(0, 0, 0)))
    prv = cams.add_camera(ThinLensCamera((W, H), 60.0, 0.05, Vec3(*rot_y(ORIGIN, 2.0)), Vec3(0.1, 0, 0), Vec3(0, 1, 0), Vec3(0, 0, 0)))
    per, geo, cd, pd = prev_motion(c, cur, prv, inp=inp)
    check(per, geo, cd, pd, min_valid=0.9, min_motion=0.5)


def sphere_world(c, center, radius):
    from test_cpu_trap import FRACTAL_MATERIAL
    c["world"].hitables.push(Sphere(center, radius, FRACTAL_MATERIAL))
    return len(c["world"].hitables) - 1


def sphere_hits(P, centre, radius):
    return np.abs(np.linalg.norm(P - centre, axis=-1) - radius) < 1e-3


def test_static_sphere_displaced():
    """a constant sphere centre moved between frames: its hits move back by the displacement, P' = P + (c_prev - c)"""
    c, inp = small_config(3, (W, H), 2, 1)
    bu, bw = basis(ORIGIN, np.zeros(3))
    c1 = ORIGIN - 2.5 * bw
    c0 = c1 - 0.15 * bu + 0.05 * np.array([0.0, 1.0, 0.0])
    j = sphere_world(c, Vec3(*c1), 0.3)
    prev_world, _ = small_config(3, (W, H), 2, 1)
    sphere_world(prev_world, Vec3(*c0), 0.3)
    d, p, keep = descs(c["world"], c["camera"], prev_world["camera"], prev_world["world"])
    assert p.hitables[j].center[0] != d.hitables[j].center[0]
    _, per, geo = mpo.render_motion_prev(d, p, inp, (8, 8), c["integrator"], TR, DT, geometry=True)
    c1f, c0f = np.array(d.hitables[j].center[:], np.float64), np.array(p.hitables[j].center[:], np.float64)

    def moved(P, tau):
        on = sphere_hits(P, c1f, 0.3)
        assert 0.02 < on.mean() < 0.9
        return np.where(on[:, None], P + (c0f - c1f), P)
    ok = check(per, geo, d.camera, p.camera, moved)
    # everything off the sphere is static: exactly zero
    P = geo[..., :3][ok].astype(np.float64)
    off = ~sphere_hits(P, c1f, 0.3)
    assert (per[..., :2][ok][off].view(np.uint32) == 0).all()


def test_moving_sphere_changes_velocity():
    """c(t) = c1 + v1 t now, c_prev(t) = c0 + v0 t before: P' = P + (c_prev(tau - dt) - c(tau))"""
    c, inp = small_config(3, (W, H), 2, 1)
    bu, bw = basis(ORIGIN, np.zeros(3))
    base = ORIGIN - 2.5 * bw
    v1, v0 = 3.0 * bu, -2.0 * bu + np.array([0.0, 1.5, 0.0])
    j = sphere_world(c, Linear(Vec3(*base), Vec3(*v1)), 0.3)
    prev_world, _ = small_config(3, (W, H), 2, 1)
    sphere_world(prev_world, Linear(Vec3(*(base - 0.1 * bu)), Vec3(*v0)), 0.3)
    d, p, keep = descs(c["world"], c["camera"], prev_world["camera"], prev_world["world"])
    _, per, geo = mpo.render_motion_prev(d, p, inp, (8, 8), c["integrator"], TR, DT, geometry=True)
    h, hp = d.hitables[j], p.hitables[j]
    ctr = lambda hh, t: np.array(hh.center[:], np.float64) + np.array(hh.center_velocity[:], np.float64) * t[:, None]  # noqa: E731

    def moved(P, tau):
        on = sphere_hits(P, ctr(h, tau), 0.3)
        assert 0.02 < on.mean() < 0.9
        return np.where(on[:, None], P + (ctr(hp, tau - DT) - ctr(h, tau)), P)
    check(per, geo, d.camera, p.camera, moved)


# ---- the identity with render_motion ----
@pytest.mark.parametrize("n", [1, 3, 4])
def test_prev_equal_to_the_uploaded_scene_is_render_motion(n):
    """prev = the uploaded scene (its camera may move linearly; no sphere moves): render_motion's plane bit for bit"""
    from test_cpu_temporal import moving_cameras
    c, inp = small_config(n, (29, 21), 2, 1)
    sphere_world(c, Vec3(-1.0, 0.4, 0.9), 0.35)
    cams = [c["camera"]] + ([moving_cameras(c, (29, 21))[k] for k in ("pan", "dolly", "ortho", "thinlens")] if n == 3 else [])
    for cam in cams:
        d, keep = c["world"].flatten(cam)
        a = to.render_motion(c["world"], cam, inp, (8, 8), c["integrator"], TR, DT)
        b = mpo.render_motion_prev(d, d, inp, (8, 8), c["integrator"], TR, DT)
        assert_bit_equal(b[0], a[0], f"cfg{n} plane")
        assert_bit_equal(b[1], a[1], f"cfg{n} records")


def test_moving_sphere_differs_from_render_motion_by_rounding_only():
    c, inp = small_config(3, (29, 21), 2, 1)
    sphere_world(c, Linear(Vec3(-1.0, 0.4, 0.9), Vec3(4.0, 0.0, 1.0)), 0.35)
    d, keep = c["world"].flatten(c["camera"])
    _, a = to.render_motion(c["world"], c["camera"], inp, (8, 8), c["integrator"], TR, DT)
    _, b = mpo.render_motion_prev(d, d, inp, (8, 8), c["integrator"], TR, DT)
    ok = ~np.isnan(a[..., 2])
    assert_bit_equal(np.isnan(b[..., 2]), ~ok)
    assert (a[..., 0][ok] != 0).any()
    np.testing.assert_allclose(b[ok], a[ok], rtol=1e-5, atol=1e-4)


def changed_kind(d):
    """a copy of scene d whose first hitable has another kind (keep the returned array alive with it)"""
    import ctypes as C
    hit = (L.RaynHitable * d.n_hitables)(*[d.hitables[i] for i in range(d.n_hitables)])
    hit[0].kind = L.HITABLE_MANDELBULB if hit[0].kind != L.HITABLE_MANDELBULB else L.HITABLE_SPHERE
    p = L.RaynSceneDesc.from_buffer_copy(d)
    p.hitables = C.cast(hit, C.POINTER(L.RaynHitable))
    return p, hit


def test_mirror_argument_rules():
    """NULL prev, another camera kind, another hitable count or another hitable kind: RAYN_ERR_INVALID_ARG"""
    c, inp = small_config(3, (8, 8), 1, 1)
    d, k = c["world"].flatten(c["camera"])
    ortho = c["world"].cameras.add_camera(OrthographicCamera((8, 8), 2.0, Vec3(9.5, -3.5, 9.5), Vec3(0, 0, 0), Vec3(0, 1, 0)))
    p_cam, kc = c["world"].flatten(ortho)
    c2, _ = small_config(3, (8, 8), 1, 1)
    sphere_world(c2, Vec3(0, 0, 0), 0.1)
    p_n, kn = c2["world"].flatten(c2["camera"])
    p_kind, kk = changed_kind(d)
    for bad in (None, p_cam, p_n, p_kind):
        with pytest.raises(RuntimeError) as e:
            mpo.render_motion_prev(d, bad, inp, (8, 8), c["integrator"], TR, DT)
        assert e.value.args[0] == L.RAYN_ERR_INVALID_ARG


# ---- closures and their chord ----
def orbit(radius=5.0, height=1.0, speed=0.8):
    return lambda t: Vec3(radius * math.cos(speed * t), height, radius * math.sin(speed * t))


@pytest.mark.parametrize("t0,t1", [(0.0, 1.0 / 24.0), (0.375, 0.5), (2.0 / 24.0, 2.0 / 24.0), (-1.5, 3.0)])
def test_chord_matches_the_closure_at_the_shutter_ends(t0, t1):
    f = orbit()
    lin = Linear.chord(f, t0, t1)
    assert lin.base.dtype == np.float32 and lin.velocity.dtype == np.float32
    t0f, t1f = np.float32(t0), np.float32(t1)
    for t in (t0f, t1f):
        got = lin.base + lin.velocity * t  # float32, as seq3 evaluates it
        want = np.asarray(f(float(t)).v, np.float64)
        # base, velocity * t and their sum are each rounded to float32: a few ulp of the largest magnitude involved
        scale = np.abs(lin.base).astype(np.float64) + np.abs(lin.velocity * t).astype(np.float64) + np.abs(want)
        np.testing.assert_array_less(np.abs(got - want), 4 * np.finfo(np.float32).eps * scale + 1e-30)
    if t1f == t0f:
        assert (lin.velocity == 0).all()
        assert_bit_equal(lin.base, f(float(t0f)).v)
    else:
        v = (np.asarray(f(float(t1f)).v, np.float64) - np.asarray(f(float(t0f)).v, np.float64)) / (float(t1f) - float(t0f))
        assert_bit_equal(lin.velocity, v.astype(np.float32))


def test_chord_of_a_linear_closure_is_the_linear():
    base, vel = np.array([0.25, -1.0, 2.0]), np.array([0.5, 0.125, -4.0])
    lin = Linear.chord(lambda t: tuple(base + vel * t), 0.5, 1.5)
    assert_bit_equal(lin.base, base.astype(np.float32)), assert_bit_equal(lin.velocity, vel.astype(np.float32))


def closure_world(res=(16, 12)):
    c, _ = small_config(3, res, 1, 1)
    cam = c["world"].cameras.add_camera(PinholeCamera(res, 60.0, orbit(), Vec3(0, 0, 0), Vec3(0, 1, 0)))
    return c, cam


def test_closure_world_needs_a_time_range():
    c, cam = closure_world()
    assert c["world"].has_closures(cam) and not c["world"].has_closures(c["camera"])
    with pytest.raises(ValueError):
        c["world"].flatten(cam)
    d, keep = c["world"].flatten(cam, (0.5, 0.75))
    lin = Linear.chord(orbit(), 0.5, 0.75)
    assert list(d.camera.origin) == lin.base.tolist() and list(d.camera.origin_velocity) == lin.velocity.tolist()
    c2, _ = small_config(3, (16, 12), 1, 1)
    sphere_world(c2, lambda t: (0.5 * t, 0.0, 1.0), 0.2)
    assert c2["world"].has_closures(c2["camera"])
    with pytest.raises(ValueError):
        c2["world"].flatten(c2["camera"])
    d2, keep2 = c2["world"].flatten(c2["camera"], (1.0, 1.0))
    h = d2.hitables[d2.n_hitables - 1]
    assert list(h.center) == [0.5, 0.0, 1.0] and list(h.center_velocity) == [0.0, 0.0, 0.0]


def _bytes(desc):
    out = [bytes(desc.camera), bytes(desc.volume), bytes(desc.consts)]
    out += [bytes(desc.hitables[i]) for i in range(desc.n_hitables)]
    out += [bytes(desc.materials[i]) for i in range(desc.n_materials)]
    out += [bytes(desc.lights[i]) for i in range(desc.n_lights)]
    return out


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5])
def test_worlds_without_closures_flatten_as_before(n):
    """a time range changes nothing for constant and Linear parameters; Linear spheres and cameras keep base and velocity"""
    from test_cpu_temporal import moving_cameras
    c = configs.baseline_config(n, res=(16, 12), samples=1, max_bounces=1)
    sphere_world(c, Linear(Vec3(-1.0, 0.4, 0.9), Vec3(4.0, 0.0, 1.0)), 0.35)
    cams = [c["camera"]] + list(moving_cameras(c, (16, 12)).values())
    for cam in cams:
        assert not c["world"].has_closures(cam)
        a, ka = c["world"].flatten(cam)
        b, kb = c["world"].flatten(cam, (0.25, 0.5))
        assert _bytes(a) == _bytes(b)
    h = a.hitables[a.n_hitables - 1]
    assert list(h.center) == [np.float32(-1.0), np.float32(0.4), np.float32(0.9)] and list(h.center_velocity) == [4.0, 0.0, 1.0]


def test_render_sequence_rules_for_closure_worlds():
    """a closure world goes through the same channel checks, before any device work"""
    from rayn_b200.film import Film
    c, cam = closure_world()
    args = (c["world"], cam, c["integrator"], None, (8, 8), range(1, 3), 24, 0.0, 1)
    with pytest.raises(ValueError):
        Film(["color", "alpha", "normal"], (16, 12)).render_sequence(*args)
    with pytest.raises(ValueError):
        Film(["color", "alpha", "background", "normal", "moments"], (16, 12)).render_sequence(*args)
    bad = lambda t: (1.0, 2.0)  # noqa: E731
    with pytest.raises(ValueError):
        Linear.chord(bad, 0.0, 1.0)

