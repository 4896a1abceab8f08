"""ctypes bindings of the CPU mirrors of the motion plane (tests/motion_oracle.cpp, which includes tests/trap_oracle.cpp and
through it oracle/rayn_oracle.cpp unchanged), of the temporal push and of the scaled variance denoise
(tests/temporal_oracle.cpp, which includes tests/denoise_variance_oracle.cpp).  TEST INFRASTRUCTURE ONLY.

Each library is compiled on first use into a temporary directory keyed by its sources, in the mul_add variant of the
product library under test (rayn_b200/_lib.py), so the test tree itself is never written."""
import ctypes as C
import os

import numpy as np

from rayn_b200 import _lib as L

import denoise_oracle
import trap_oracle
from albedo_oracle import _build

HERE = os.path.dirname(os.path.abspath(__file__))
fp = C.POINTER(C.c_float)
N_HIST = 14  # history planes of a RaynTemporal


def motion_lib():
    l = _build("motion_oracle", os.path.join(HERE, "motion_oracle.cpp"), trap_oracle.SOURCES, trap_oracle.FLAGS)
    l.rayn_motion_oracle_render.restype = C.c_int32
    l.rayn_motion_oracle_render.argtypes = [C.POINTER(L.RaynSceneDesc), C.POINTER(L.RaynFrameDesc), C.c_float, fp, fp, C.c_int32, C.c_int32, C.c_void_p]
    return l


def temporal_lib():
    l = _build("temporal_oracle", os.path.join(HERE, "temporal_oracle.cpp"),
               [os.path.join(HERE, "denoise_variance_oracle.cpp")] + denoise_oracle.SOURCES[1:], denoise_oracle.FLAGS)
    l.rayn_oracle_temporal_push.restype = C.c_int32
    l.rayn_oracle_temporal_push.argtypes = [C.c_int32, C.c_int32, C.POINTER(L.RaynTemporalDesc)] + [C.c_void_p] * 13
    l.rayn_oracle_film_denoise_variance_scaled.restype = C.c_int32
    l.rayn_oracle_film_denoise_variance_scaled.argtypes = [C.POINTER(L.RaynDenoiseDesc), C.c_float, C.c_int32, C.POINTER(L.RaynMomentPlanes),
                                                           C.c_void_p, C.c_float, C.c_void_p, C.c_int32, C.c_int32, C.POINTER(L.RaynFilmPlanes),
                                                           C.POINTER(L.RaynFilmPlanes)]
    return l


def render_motion(world, camera, inputs, tile_size, integrator, time_range, frame_dt, n_threads=0, subsample_k=1, geometry=False):
    """CPU motion plane of the same FrameInputs -> (plane [H, W, 4], per-sample records [H, W, spp, 4]), float32; geometry=True
    adds per sample (hit point xyz, camera time, u, v) [H, W, spp, 6]."""
    from rayn_b200.film import make_frame_desc
    desc, keep = world.flatten(camera)
    w, h, spp = inputs.width, inputs.height, inputs.spp
    per = np.zeros(w * h * spp * 4, np.float32)
    plane = np.zeros(4 * w * h, np.float32)
    ptrs = tuple(a.ctypes.data for a in inputs.arrays())
    f = make_frame_desc(w, h, tile_size, inputs.samples, integrator, inputs.frame, time_range, ptrs, L.MEM_HOST,
                        sets=(inputs.sets_1d, inputs.sets_2d))
    geo = np.zeros(w * h * spp * 6, np.float32) if geometry else None
    rc = motion_lib().rayn_motion_oracle_render(C.byref(desc), C.byref(f), float(frame_dt), per.ctypes.data_as(fp), plane.ctypes.data_as(fp),
                                                n_threads, subsample_k, None if geo is None else geo.ctypes.data)
    if rc != 0:
        raise RuntimeError(f"motion oracle failed: {rc}")
    out = (plane.reshape(h, w, 4), per.reshape(h, w, spp, 4))
    return out + (geo.reshape(h, w, spp, 6),) if geometry else out


class TemporalMirror:
    """The CPU history of one film, pushed like rayn_b200_temporal_push (same ping-pong of two histories)."""

    def __init__(self, width, height):
        self.width, self.height = width, height
        self.hist = [np.zeros(N_HIST * width * height, np.float32) for _ in range(2)]
        self.cur = 0

    def push(self, planes, moments, motion, alpha_min, sigma_depth, normal_cos, reset=False):
        """-> (status, planes {"color", "background"}, moments [H, W, 2], var_scale [H, W]), like Renderer.temporal_push"""
        w, h = self.width, self.height
        c = np.ascontiguousarray(planes["color"], np.float32).reshape(-1)
        b = np.ascontiguousarray(planes["background"], np.float32).reshape(-1)
        n = np.ascontiguousarray(planes["normal"], np.float32).reshape(-1)
        m = np.ascontiguousarray(np.asarray(moments, np.float32).reshape(h, w, 2).transpose(2, 0, 1)).reshape(2, -1)
        mv = np.ascontiguousarray(motion, np.float32).reshape(-1)
        oc, ob, om, s = np.empty_like(c), np.empty_like(b), np.empty_like(m), np.empty(w * h, np.float32)
        d = L.RaynTemporalDesc(float(alpha_min), float(sigma_depth), float(normal_cos), 1 if reset else 0)
        hin, hout = self.hist[self.cur], self.hist[self.cur ^ 1]
        rc = temporal_lib().rayn_oracle_temporal_push(w, h, C.byref(d), hin.ctypes.data, hout.ctypes.data, c.ctypes.data, b.ctypes.data,
                                                      n.ctypes.data, m[0].ctypes.data, m[1].ctypes.data, mv.ctypes.data, oc.ctypes.data,
                                                      ob.ctypes.data, om[0].ctypes.data, om[1].ctypes.data, s.ctypes.data)
        if rc == 0:
            self.cur ^= 1
        out = {"color": oc.reshape(np.shape(planes["color"])), "background": ob.reshape(np.shape(planes["background"]))}
        return rc, out, np.ascontiguousarray(om.reshape(2, h, w).transpose(1, 2, 0)), s.reshape(h, w)


def denoise_scaled(width, height, planes, desc, sigma_luminance, spp, moments, var_scale, sigma_albedo=np.inf, albedo=None):
    """-> (status, {channel: new float32 array}), like moments_oracle.denoise with a per-pixel variance scale"""
    flat = {k: np.ascontiguousarray(v, np.float32).reshape(-1) for k, v in planes.items() if v is not None}
    outs = {k: np.empty_like(flat[k]) for k in ("color", "background") if k in flat}
    m = np.ascontiguousarray(np.asarray(moments, np.float32).reshape(height, width, 2).transpose(2, 0, 1)).reshape(2, -1)
    vs = np.ascontiguousarray(var_scale, np.float32).reshape(-1)
    alb = None if albedo is None else np.ascontiguousarray(albedo, np.float32).reshape(-1)

    def ptr(d, k):
        return d[k].ctypes.data if k in d else None
    pin = L.RaynFilmPlanes(ptr(flat, "color"), ptr(flat, "alpha"), ptr(flat, "background"), ptr(flat, "normal"), L.MEM_HOST)
    pout = L.RaynFilmPlanes(ptr(outs, "color"), None, ptr(outs, "background"), None, L.MEM_HOST)
    mp = L.RaynMomentPlanes(m[0].ctypes.data, m[1].ctypes.data, L.MEM_HOST)
    rc = temporal_lib().rayn_oracle_film_denoise_variance_scaled(C.byref(desc), float(sigma_luminance), int(spp), C.byref(mp), vs.ctypes.data,
                                                                 float(sigma_albedo), None if alb is None else alb.ctypes.data, width, height,
                                                                 C.byref(pin), C.byref(pout))
    return rc, outs
