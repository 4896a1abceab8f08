"""Reprojection of rendered frames through the temporal push, end to end on the CPU mirrors: the motion plane of frame k
(tests/render_mirror.cpp) must carry frame k-1's history to where frame k sees the same
surface point (tests/film_mirror.cpp).

Config 1's world with the camera 1.35 from the centre of its unit sphere, so the sphere fills the view and depth is smooth;
shutter 0, frames k-1 and k.  Frame k-1 is pushed into a new history with its per-pixel mean world-space hit point P as colour
and its view depth as background; frame k follows with colour 0, alpha_min 0.5, sigma_z 1e30 and normal_cos -1.  Every used
history tap then has n = 1, so n_h = 1 exactly, alpha = 0.5 and 2 * out is exactly the bilinearly reprojected history.  With a
static scene it must land on frame k's own mean hit point P; where a sphere moves it must land on P - v * frame_dt, and its
depth on frame k's z_prev.

The motion plane fed to the push is then edited into each wrong convention: negated motion, y flipped, half a pixel added in x
or in y, and zero motion.  P varies along both screen axes, so each of them moves the error.  Measured at 64x48 with 16
samples, i.e. 64 spp and 64 per-sample records per pixel (FrameInputs.spp = 4 x samples)
(median error of P in pixel footprints at the hit; the smallest wrong convention and its ratio to the correct one):

  | motion | median (dx, dy), px | correct | smallest wrong |
  |---|---|---|---|
  | diagonal pan (look-at velocity) | (3.6, -2.1) | 0.044 | y + 0.5: 0.53 (12x) |
  | dolly | radial, max abs(dy) 2.7 | 0.042 | y + 0.5: 0.58 (14x) |
  | vertical pan | (0.0, 4.7) | 0.043 | y + 0.5: 0.55 (13x) |
  | orthographic pan | (2.7, 1.7) | 0.039 | y + 0.5: 0.52 (13x) |
  | orbit (a closure camera, render_motion_prev) | (-5.0, 1.5) | 0.039 | y + 0.5: 0.53 (13x) |
  | sphere moving past a static camera | (-3.1, -1.6) | 0.039 | y + 0.5: 0.53 (14x) |

Negated, y-flipped and zero motion are 70x to 290x worse.  The median relative depth error against z_prev is 0.7e-4 to
2.2e-4.  At least 89 % of the pixels take history, and at least 96.9 % of those pass the default sigma_z = 0.1.  The
assertions: median P error under 0.1 footprints, every wrong convention at least 3x worse, median depth error under 1e-3,
more than 85 % of the pixels taking history and more than 95 % of those within sigma_z = 0.1."""
import math

import numpy as np
import pytest

from rayn_b200 import _lib as L
from rayn_b200 import configs
from rayn_b200.film import FrameInputs
from rayn_b200.scene import Linear, OrthographicCamera, PinholeCamera, Sphere, Vec3

import mirrors

f32 = np.float32
DT = 1.0 / 24.0
K = 3  # frame k; frame k - 1 is rendered at (k - 1) / 24
TILE = (8, 8)
DIST = 1.35  # camera distance from the centre of config 1's unit sphere
EYE = np.array([-0.45, 0.2, 2.0]) / np.linalg.norm([-0.45, 0.2, 2.0]) * DIST
MOTIONS = ["pan", "dolly", "vertical", "ortho", "orbit", "sphere"]
WRONG = {
    "negated": lambda m: m * f32([-1, -1, 1, 1]),
    "y flipped": lambda m: m * f32([1, -1, 1, 1]),
    "x + 0.5": lambda m: m + f32([0.5, 0, 0, 0]),
    "y + 0.5": lambda m: m + f32([0, 0.5, 0, 0]),
    "zero": lambda m: m * f32([0, 0, 1, 1]),
}


def shutter0(k):
    t = float(f32(k) * (f32(1.0) / f32(24.0)))  # frame_time_range's start, with no shutter
    return (t, t)


def orbit(t):
    """the camera origin on a tilted circle about the sphere's centre, 1.2 rad/s"""
    a = 1.2 * t
    u, v = EYE / DIST, np.cross(EYE / DIST, [0.3, 1.0, 0.0])
    v = v / np.linalg.norm(v)
    return Vec3(*(DIST * (math.cos(a) * u + math.sin(a) * v)))


def scene(motion, W, H, samples):
    """-> (config, camera, sphere velocity or None) for one of MOTIONS at W x H"""
    c = configs.baseline_config(1, res=(W, H), samples=samples, max_bounces=1)
    cams = c["world"].cameras
    v = None
    if motion == "pan":
        cam = PinholeCamera((W, H), 60.0, Vec3(*EYE), Linear(Vec3(0, 0, 0), Vec3(3.0, -2.0, 0.0)), Vec3(0, 1, 0))
    elif motion == "dolly":
        cam = PinholeCamera((W, H), 60.0, Linear(Vec3(*EYE), Vec3(*(-EYE * 0.6))), Vec3(0, 0, 0), Vec3(0, 1, 0))
    elif motion == "vertical":
        cam = PinholeCamera((W, H), 60.0, Vec3(*EYE), Linear(Vec3(0, 0, 0), Vec3(0.0, 3.5, 0.0)), Vec3(0, 1, 0))
    elif motion == "ortho":
        pan = Vec3(1.5, 0.75, -0.6)
        cam = OrthographicCamera((W, H), 1.0, Linear(Vec3(*(EYE * 2.2)), pan), Linear(Vec3(0, 0, 0), pan), Vec3(0, 1, 0))
    elif motion == "orbit":
        cam = PinholeCamera((W, H), 60.0, orbit, Vec3(0, 0, 0), Vec3(0, 1, 0))
    elif motion == "sphere":
        cam = PinholeCamera((W, H), 60.0, Vec3(*EYE), Vec3(0, 0, 0), Vec3(0, 1, 0))
        v = np.array([0.6, 0.35, 0.2])
        old = c["world"].hitables.items[1]
        c["world"].hitables.items[1] = Sphere(Linear(Vec3(0, 0, 0), Vec3(*v)), float(old.radius), old.material)
    else:
        raise ValueError(motion)
    return c, cams.add_camera(cam), v


def mean_hit(per, geo):
    """per-pixel mean of the valid samples' hit points (float64) and whether the pixel has any"""
    ok = ~np.isnan(per[..., 2])
    n = ok.sum(axis=2)
    P = np.where(ok[..., None], geo[..., :3], 0).astype(np.float64).sum(axis=2) / np.maximum(n, 1)[..., None]
    return P, n > 0


def render_pair(motion, W, H, samples, device=None):
    """Frames k-1 and k of one motion: {plane0, P0, has0, plane1, P1, has1, camera (frame k's RaynCamera), v}.  The hit
    points come from the CPU mirrors; with device (a Renderer) the two motion planes come from the device, and the mirror's are
    kept as mirror_plane0 and mirror_plane1."""
    c, cam, v = scene(motion, W, H, samples)
    inps = [FrameInputs(W, H, samples, c["integrator"], frame=k) for k in (K - 1, K)]
    d0, keep0 = c["world"].flatten(cam, shutter0(K - 1))
    d1, keep1 = c["world"].flatten(cam, shutter0(K))
    prev = motion == "orbit"  # a closure camera: motion against the previous frame's scene
    out = {"camera": d1.camera, "v": v}
    for i, (d, p, inp, tr) in enumerate(((d0, d0, inps[0], shutter0(K - 1)), (d1, d0, inps[1], shutter0(K)))):
        if prev:
            plane, per, geo = mirrors.render_motion(d, inp, TILE, c["integrator"], tr, DT, prev=p, geometry=True)
        else:
            plane, per, geo = mirrors.render_motion(c["world"].flatten(cam)[0], inp, TILE, c["integrator"], tr, DT, geometry=True)
        if device is not None:
            out[f"mirror_plane{i}"] = plane
            device.upload_scene(c["world"], cam, tr)
            plane = device.render_motion(inp, TILE, c["integrator"], tr, DT, prev=p if prev else None)
        out[f"P{i}"], out[f"has{i}"] = mean_hit(per, geo)
        out[f"plane{i}"] = plane
    del keep0, keep1
    return out


def footprint(cam, z, W):
    """the width of one pixel in scene units at view depth z"""
    if cam.kind == L.CAMERA_ORTHOGRAPHIC:
        return np.full(np.shape(z), cam.full_size[0] / W)
    return 2.0 * cam.half_size[0] * np.abs(z.astype(np.float64)) / W


def reproject(push, fr, motion):
    """push(planes, moments, motion, alpha_min, sigma_depth, normal_cos, reset) -> (out, moments, s), on a new history: frame
    k-1 with colour P0 and background (z0, 0, 0), then frame k with colour 0 and the given motion plane.
    -> (reprojected P [H, W, 3], reprojected z [H, W], took history [H, W])"""
    P0, has0, plane0 = fr["P0"], fr["has0"], fr["plane0"]
    H, W = has0.shape
    nrm = np.zeros((H, W, 3), f32)
    nrm[..., 2] = 1.0
    zero = np.zeros((H, W, 3), f32)
    bg = zero.copy()
    bg[..., 0] = np.where(has0, plane0[..., 2], 0.0)
    mom = np.zeros((H, W, 2), f32)
    push({"color": np.where(has0[..., None], P0, 0.0).astype(f32), "background": bg, "normal": nrm}, mom, plane0, 1.0, 0.1, -1.0, True)
    out, _, s = push({"color": zero, "background": zero, "normal": nrm}, mom, np.ascontiguousarray(motion, f32), 0.5, 1e30, -1.0, False)
    return 2.0 * out["color"].astype(np.float64), 2.0 * out["background"][..., 0].astype(np.float64), s == 0.5


def scores(push, fr):
    """{convention: (median error of P over the footprint, median relative error of z against z_prev, share of pixels that
    took history, share of those within the default sigma_z)} for the correct motion plane and each of WRONG"""
    p1, has1 = fr["plane1"], fr["has1"]
    target = fr["P1"] if fr["v"] is None else fr["P1"] - fr["v"] * DT
    foot = footprint(fr["camera"], p1[..., 2], has1.shape[1])
    res = {}
    for name, edit in [("correct", lambda m: m)] + list(WRONG.items()):
        P, z, took = reproject(push, fr, edit(p1))
        took &= has1
        e = np.linalg.norm(P - target, axis=2) / foot
        ez = np.abs(z - p1[..., 3]) / np.abs(p1[..., 3])
        res[name] = (float(np.median(e[took])), float(np.median(ez[took])), float(took.mean()), float((ez[took] <= 0.1).mean()))
    return res


def check(res, max_error):
    ok = res["correct"]
    assert ok[0] < max_error and ok[1] < 1e-3, res
    assert ok[2] > 0.85 and ok[3] > 0.95, res
    for name in WRONG:
        assert res[name][0] >= 3.0 * ok[0], (name, res)


def mirror_push(W, H):
    t = mirrors.TemporalMirror(W, H)

    def push(planes, moments, motion, alpha_min, sigma_depth, normal_cos, reset):
        rc, out, om, s = t.push(planes, moments, motion, alpha_min, sigma_depth, normal_cos, reset)
        assert rc == L.RAYN_OK
        return out, om, s
    return push


@pytest.mark.parametrize("motion", MOTIONS)
def test_history_lands_on_the_same_surface_point(motion):
    W, H = 64, 48
    fr = render_pair(motion, W, H, 16)
    p1 = fr["plane1"][fr["has1"]]
    assert np.median(np.hypot(p1[:, 0], p1[:, 1])) > 2.0 and np.abs(p1[:, 1]).max() > 1.5  # several pixels, dy != 0
    check(scores(mirror_push(W, H), fr), 0.1)
