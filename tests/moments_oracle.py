"""ctypes bindings of the CPU mirrors of the luminance-moment render (tests/moments_oracle.cpp, which includes
tests/trap_oracle.cpp and through it oracle/rayn_oracle.cpp unchanged) and of the variance-guided denoise
(tests/denoise_variance_oracle.cpp).  TEST INFRASTRUCTURE ONLY.

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


def moments_lib():
    l = _build("moments_oracle", os.path.join(HERE, "moments_oracle.cpp"), trap_oracle.SOURCES, trap_oracle.FLAGS)
    l.rayn_moments_oracle_render_frame.restype = C.c_int32
    l.rayn_moments_oracle_render_frame.argtypes = [C.POINTER(L.RaynSceneDesc), C.c_int32, C.POINTER(L.RaynAlbedoTrap), C.POINTER(L.RaynFrameDesc),
                                                   C.POINTER(L.RaynFilmPlanes), C.c_void_p, C.c_void_p, C.c_int32, C.c_int32]
    return l


def denoise_lib():
    l = _build("denoise_variance_oracle", os.path.join(HERE, "denoise_variance_oracle.cpp"), denoise_oracle.SOURCES[1:], denoise_oracle.FLAGS)
    l.rayn_oracle_film_denoise_variance.restype = C.c_int32
    l.rayn_oracle_film_denoise_variance.argtypes = [C.POINTER(L.RaynDenoiseDesc), C.c_float, C.c_int32, C.POINTER(L.RaynMomentPlanes), C.c_float,
                                                    C.c_void_p, C.c_int32, C.c_int32, C.POINTER(L.RaynFilmPlanes), C.POINTER(L.RaynFilmPlanes)]
    return l


def render(world, camera, inputs, tile_size, integrator, time_range, n_threads=0, subsample_k=1, tile_list=None, traps=None):
    """CPU render of the same FrameInputs with its moment planes -> (planes dict with flat film planes and "moments" float32
    [H, W, 2]).  subsample_k > 1: only tiles whose index is a multiple of k are computed, the others stay 0."""
    from rayn_b200.film import host_planes, make_frame_desc
    desc, keep = world.flatten(camera)
    traps = world.albedo_traps() if traps is None else traps
    w, h = inputs.width, inputs.height
    planes, p = host_planes(w, h)
    m = np.zeros((2, w * h), np.float32)
    ptrs = tuple(a.ctypes.data for a in inputs.arrays())
    f = make_frame_desc(w, h, tile_size, inputs.samples, integrator, inputs.frame, time_range, ptrs, L.MEM_HOST, 0, 1,
                        (inputs.sets_1d, inputs.sets_2d), tile_list)
    arr = (L.RaynAlbedoTrap * max(len(traps), 1))(*traps)
    rc = moments_lib().rayn_moments_oracle_render_frame(C.byref(desc), len(traps), arr, C.byref(f), C.byref(p), m[0].ctypes.data,
                                                        m[1].ctypes.data, n_threads, subsample_k)
    if rc != 0:
        raise RuntimeError(f"moments oracle render failed: {rc}")
    planes["moments"] = np.ascontiguousarray(m.reshape(2, h, w).transpose(1, 2, 0))
    return planes


def denoise(width, height, planes, desc, sigma_luminance, spp, moments, sigma_albedo=np.inf, albedo=None):
    """-> (status, {channel: new float32 array}) for the color / background planes given, like denoise_oracle.denoise.
    moments: float32 [H, W, 2] (color_lum2, background_lum2)."""
    flat = {k: np.ascontiguousarray(v, np.float32).reshape(-1) for k, v in planes.items() if v is not None}
    outs = {k: np.empty_like(flat[k]) for k in ("color", "background") if k in flat}
    m = np.ascontiguousarray(np.asarray(moments, np.float32).reshape(height, width, 2).transpose(2, 0, 1)).reshape(2, -1)
    alb = None if albedo is None else np.ascontiguousarray(albedo, np.float32).reshape(-1)

    def ptr(d, k):
        return d[k].ctypes.data if k in d else None
    pin = L.RaynFilmPlanes(ptr(flat, "color"), ptr(flat, "alpha"), ptr(flat, "background"), ptr(flat, "normal"), L.MEM_HOST)
    pout = L.RaynFilmPlanes(ptr(outs, "color"), None, ptr(outs, "background"), None, L.MEM_HOST)
    mp = L.RaynMomentPlanes(m[0].ctypes.data, m[1].ctypes.data, L.MEM_HOST)
    rc = denoise_lib().rayn_oracle_film_denoise_variance(C.byref(desc), float(sigma_luminance), int(spp), C.byref(mp), float(sigma_albedo),
                                                         None if alb is None else alb.ctypes.data, width, height, C.byref(pin), C.byref(pout))
    return rc, outs
