"""CPU mirrors of the equirectangular camera and of the film filters that wrap round its seam.  TEST INFRASTRUCTURE ONLY.

tests/panorama_mirror.cpp (the render mirror and the oracle, included unchanged, with the panorama's camera branch and motion
projection): the oracle's film, the render mirror's film, albedo and motion planes, and the camera ray and projection KATs, for
every camera kind.  Built like tests/mirrors.py's libraries (the same flags, a temporary directory keyed by sources and flags).

The wrapped film filters, restated here:
  denoise_wrap  rayn_b200_film_denoise_wrap as the middle copy of the non-wrapped filter (tests/film_mirror.cpp) of the film tiled
                side by side often enough that no tap of the middle copy reaches an outer edge: each of its taps then reads the
                pixel at the floored-mod column, which is the statement, and every other rule is the non-wrapped entry point's;
  PushWrap      rayn_b200_temporal_push_wrap in numpy float32, one IEEE rounding per operation in the statement's order."""
import ctypes as C
import os

import numpy as np

from rayn_b200 import _lib as L

import mirrors

HERE = os.path.dirname(os.path.abspath(__file__))
PANO = ("panorama_mirror", [os.path.join(HERE, "panorama_mirror.cpp")] + mirrors.RENDER[1], mirrors.RENDER[2])
P = C.POINTER
fp = P(C.c_float)
_libs = {}


def lib():
    if "pano" not in _libs:
        l = mirrors._build(*PANO)
        l.rayn_oracle_render_frame.restype = C.c_int32
        l.rayn_oracle_render_frame.argtypes = [P(L.RaynSceneDesc), P(L.RaynFrameDesc), P(L.RaynFilmPlanes), C.c_int32, C.c_int32, P(C.c_int32),
                                               C.c_int64, P(C.c_int64), P(C.c_int64), P(C.c_int64)]
        l.rayn_mirror_render_frame.restype = C.c_int32
        l.rayn_mirror_render_frame.argtypes = [P(L.RaynSceneDesc), C.c_int32, P(L.RaynAlbedoTrap), P(L.RaynFrameDesc), P(L.RaynFilmPlanes),
                                               C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, P(C.c_int64), P(C.c_int64)]
        l.rayn_mirror_render_albedo.restype = C.c_int32
        l.rayn_mirror_render_albedo.argtypes = [P(L.RaynSceneDesc), C.c_int32, P(L.RaynAlbedoTrap), P(L.RaynFrameDesc), fp, fp, C.c_int32, C.c_int32]
        l.rayn_pano_render_motion.restype = C.c_int32
        l.rayn_pano_render_motion.argtypes = [P(L.RaynSceneDesc), P(L.RaynFrameDesc), C.c_float, P(L.RaynSceneDesc), fp, fp, C.c_int32, C.c_int32,
                                              C.c_void_p]
        l.rayn_pano_kat_camera_rays.argtypes = [P(L.RaynCamera), C.c_int64, fp, fp, C.c_float, fp, fp]
        l.rayn_pano_kat_project.argtypes = [P(L.RaynCamera), C.c_int32, C.c_int32, C.c_int64, fp, C.c_float, fp]
        _libs["pano"] = l
    return _libs["pano"]


def _f(a):
    return a.ctypes.data_as(fp)


def oracle_render(world, camera, inputs, tile_size, integrator, time_range):
    """the oracle's own render_frame (render_tile, film.rs:439-627) of the same FrameInputs -> planes dict"""
    from rayn_b200.film import host_planes
    desc, keep = world.flatten(camera, time_range)
    planes, p = host_planes(inputs.width, inputs.height)
    f = mirrors._frame(inputs, tile_size, integrator, time_range)
    qn, counters, tiles = C.c_int64(0), (C.c_int64 * 4)(), C.c_int64(0)
    rc = lib().rayn_oracle_render_frame(C.byref(desc), C.byref(f), C.byref(p), 0, 1, None, 0, C.byref(qn), counters, C.byref(tiles))
    if rc != 0:
        raise RuntimeError(f"oracle render failed: {rc}")
    return planes


def render(world, camera, inputs, tile_size, integrator, time_range, moments=False):
    """the render mirror's film (orbit traps, moments=True adds planes["moments"] [H, W, 2]) -> planes dict"""
    from rayn_b200.film import host_planes
    desc, keep = world.flatten(camera, time_range)
    w, h = inputs.width, inputs.height
    planes, p = host_planes(w, h)
    m = np.zeros((2, w * h), np.float32)
    f = mirrors._frame(inputs, tile_size, integrator, time_range)
    rc = lib().rayn_mirror_render_frame(C.byref(desc), *mirrors._traps(world, None), C.byref(f), C.byref(p), m[0].ctypes.data if moments else None,
                                        m[1].ctypes.data if moments else None, 0, 1, None, None)
    if rc != 0:
        raise RuntimeError(f"render mirror failed: {rc}")
    if moments:
        planes["moments"] = np.ascontiguousarray(m.reshape(2, h, w).transpose(1, 2, 0))
    return planes


def render_albedo(world, camera, inputs, tile_size, integrator, time_range):
    """the albedo plane [H, W, 3] of the same FrameInputs"""
    desc, keep = world.flatten(camera, time_range)
    w, h, spp = inputs.width, inputs.height, inputs.spp
    per, plane = np.zeros(w * h * spp * 3, np.float32), np.zeros(3 * w * h, np.float32)
    f = mirrors._frame(inputs, tile_size, integrator, time_range)
    rc = lib().rayn_mirror_render_albedo(C.byref(desc), *mirrors._traps(world, None), C.byref(f), _f(per), _f(plane), 0, 1)
    if rc != 0:
        raise RuntimeError(f"albedo mirror failed: {rc}")
    return plane.reshape(h, w, 3)


def render_motion(scene, inputs, tile_size, integrator, time_range, frame_dt, prev=None, geometry=False):
    """mirrors.render_motion for any camera kind, the equirectangular one included"""
    w, h, spp = inputs.width, inputs.height, inputs.spp
    per, plane = np.zeros(w * h * spp * 4, np.float32), np.zeros(4 * w * h, np.float32)
    f = mirrors._frame(inputs, tile_size, integrator, time_range)
    geo = np.zeros(w * h * spp * 6, np.float32) if geometry else None
    rc = lib().rayn_pano_render_motion(C.byref(scene), C.byref(f), float(frame_dt), None if prev is None else C.byref(prev), _f(per), _f(plane), 0, 1,
                                       None if geo is None else geo.ctypes.data)
    if rc != 0:
        raise RuntimeError(rc)
    out = (plane.reshape(h, w, 4), per.reshape(h, w, spp, 4))
    return out + (geo.reshape(h, w, spp, 6),) if geometry else out


def kat_camera_rays(camera, u, v, time=0.0):
    """(ro [n, 3], rd [n, 3]) of the camera packet (a RaynCamera) at film positions (u, v), lens centre, one time"""
    u, v = np.ascontiguousarray(u, np.float32).reshape(-1), np.ascontiguousarray(v, np.float32).reshape(-1)
    ro, rd = np.empty((len(u), 3), np.float32), np.empty((len(u), 3), np.float32)
    if lib().rayn_pano_kat_camera_rays(C.byref(camera), len(u), _f(u), _f(v), float(time), _f(ro), _f(rd)) != 0:
        raise ValueError("kat_camera_rays: bad argument")
    return ro, rd


def kat_project(camera, width, height, points, time=0.0):
    """proj(X, time) of the motion-plane statement per point -> float32 [n, 3] (px, py, z)"""
    p = np.ascontiguousarray(points, np.float32).reshape(-1, 3)
    out = np.empty((len(p), 3), np.float32)
    if lib().rayn_pano_kat_project(C.byref(camera), width, height, len(p), _f(p), float(time), _f(out)) != 0:
        raise ValueError("kat_project: bad argument")
    return out


def denoise_wrap(width, height, planes, desc, albedo=None, sigma_albedo=np.inf, moments=None, spp=None, sigma_luminance=np.inf, var_scale=None):
    """rayn_b200_film_denoise_wrap -> (status, {channel: float32 [H, W, 3]}); the guides as in mirrors.denoise (the variance term
    with moments and a finite sigma_luminance).  A level-i tap reaches 2^(i+1) pixels, so L levels reach 2^(L+1) - 2."""
    if moments is not None and not (sigma_luminance > 0):
        return L.RAYN_ERR_INVALID_ARG, {}
    if moments is not None and np.isinf(sigma_luminance):
        moments, var_scale = None, None
    reach = 2 ** (int(desc.iterations) + 1) - 2 if 1 <= desc.iterations <= 8 else 0
    n = 2 * -(-reach // width) + 1

    def tile(a, c):
        return None if a is None else np.concatenate([np.asarray(a, np.float32).reshape(height, width, c)] * n, axis=1)
    tiled = {k: tile(v, 1 if k == "alpha" else 3) for k, v in planes.items()}
    rc, out = mirrors.denoise(width * n, height, tiled, desc, albedo=tile(albedo, 3), sigma_albedo=sigma_albedo,
                              moments=tile(moments, 2), spp=spp, sigma_luminance=sigma_luminance, var_scale=tile(var_scale, 1))
    m = n // 2
    return rc, {k: np.ascontiguousarray(v.reshape(height, width * n, 3)[:, m * width:(m + 1) * width]) for k, v in out.items()}


F = np.float32
TC, TB, TM, TN, TZ, TLEN, TS = 0, 3, 6, 8, 11, 12, 13


class PushWrap:
    """The history of one panorama film, pushed like rayn_b200_temporal_push_wrap; mirrors.TemporalMirror's interface."""

    def __init__(self, width, height):
        self.width, self.height = width, height
        self.hist = np.zeros((mirrors.N_HIST, height, width), np.float32)

    def push(self, planes, moments, motion, alpha_min, sigma_depth, normal_cos, reset=False):
        """-> (status, planes {"color", "background"}, moments [H, W, 2], var_scale [H, W])"""
        W, H = self.width, self.height
        am, sd, nc = F(alpha_min), F(sigma_depth), F(normal_cos)
        if not (am > 0 and am <= 1) or not (sd > 0) or not (nc >= -1 and nc <= 1):
            return L.RAYN_ERR_INVALID_ARG, None, None, None
        c = np.asarray(planes["color"], F).reshape(H, W, 3)
        b = np.asarray(planes["background"], F).reshape(H, W, 3)
        nrm = np.asarray(planes["normal"], F).reshape(H, W, 3)
        mom = np.asarray(moments, F).reshape(H, W, 2)
        mv = np.asarray(motion, F).reshape(H, W, 4)
        cur = [c[..., 0], c[..., 1], c[..., 2], b[..., 0], b[..., 1], b[..., 2], mom[..., 0], mom[..., 1]]
        zp = mv[..., 3]
        h = self.hist
        hv = [np.zeros((H, W), F) for _ in range(10)]
        ws = np.zeros((H, W), F)
        y, x = np.mgrid[0:H, 0:W].astype(F)
        with np.errstate(all="ignore"):
            active = np.isfinite(zp) & (not reset)
            fx = ((x + F(0.5)) + mv[..., 0]) - F(0.5)
            fy = ((y + F(0.5)) + mv[..., 1]) - F(0.5)
            x0, y0 = np.floor(fx), np.floor(fy)
            ax, ay = fx - x0, fy - y0
            for j in (0, 1):
                for i in (0, 1):
                    w = (ax if i else F(1) - ax) * (ay if j else F(1) - ay)
                    qxf, qyf = x0 + F(i), y0 + F(j)
                    ok = active & (w != 0) & (np.abs(qxf) <= F(2.0 ** 24)) & (qyf >= 0) & (qyf <= F(H - 1))
                    qx = np.where(ok, qxf, 0).astype(np.int64) % W
                    qy = np.where(ok, qyf, 0).astype(np.int64)
                    tap = h[:, qy, qx]
                    ok &= tap[TLEN] > 0
                    ok &= np.isfinite(tap[TC:TC + 6]).all(axis=0)
                    ok &= np.isfinite(tap[TZ]) & (np.abs(tap[TZ] - zp) <= sd * np.abs(zp))
                    nd = (tap[TN] * nrm[..., 0] + tap[TN + 1] * nrm[..., 1]) + tap[TN + 2] * nrm[..., 2]
                    ok &= nd >= nc
                    ws = np.where(ok, ws + w, ws)
                    vals = [tap[TC + k] for k in range(8)] + [tap[TLEN], tap[TS]]
                    for k in range(10):
                        hv[k] = np.where(ok, hv[k] + w * vals[k], hv[k])
            some = ws != 0
            hv = [np.where(some, v / ws, F(0)) for v in hv]
            nh = np.where(some, hv[8], F(0))
            alpha = np.maximum(am, F(1) / (nh + F(1)))
            one = alpha == F(1)
            beta = F(1) - alpha
            out = [np.where(one, cur[k], beta * hv[k] + alpha * cur[k]) for k in range(8)]
            s = np.where(one, F(1), (beta * beta) * hv[9] + alpha * alpha)
        new = np.empty_like(h)
        for k in range(8):
            new[k] = out[k]
        new[TN:TN + 3] = nrm.transpose(2, 0, 1)
        new[TZ] = mv[..., 2]
        new[TLEN] = nh + F(1)
        new[TS] = s
        self.hist = new
        res = {"color": np.stack(out[0:3], axis=2).reshape(np.shape(planes["color"])),
               "background": np.stack(out[3:6], axis=2).reshape(np.shape(planes["background"]))}
        return L.RAYN_OK, res, np.stack(out[6:8], axis=2), s
