"""ctypes bindings of the CPU mirrors of the albedo plane (tests/albedo_oracle.cpp, which includes tests/trap_oracle.cpp and
through it oracle/rayn_oracle.cpp unchanged) and of the albedo-guided denoise (tests/denoise_albedo_oracle.cpp).  TEST
INFRASTRUCTURE ONLY.

Each library is compiled on first use into a temporary directory keyed by its sources, in the mul_add variant of the
product library under test (rayn_b200/_lib.py), so the test tree itself is never written."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from rayn_b200 import _lib as L

import denoise_oracle
import trap_oracle

HERE = os.path.dirname(os.path.abspath(__file__))
fp = C.POINTER(C.c_float)
_libs = {}


def _build(name, src, deps, flags):
    if name not in _libs:
        h = hashlib.sha256(" ".join(flags).encode())
        for s in [src] + deps:
            h.update(open(s, "rb").read())
        path = os.path.join(tempfile.gettempdir(), f"rayn_{name}_{os.getuid()}_{h.hexdigest()[:16]}.so")
        if not os.path.exists(path):
            tmp = f"{path}.{os.getpid()}.tmp"
            subprocess.run(["g++"] + flags + ["-o", tmp, src], check=True, capture_output=True)
            os.replace(tmp, path)
        l = C.CDLL(path)
        if l.rayn_oracle_muladd_fused() != (1 if L.MULADD_FUSED else 0):
            raise RuntimeError(f"{name} variant does not match RAYN_MULADD_FUSED")
        _libs[name] = l
    return _libs[name]


def albedo_lib():
    l = _build("albedo_oracle", os.path.join(HERE, "albedo_oracle.cpp"), [os.path.join(HERE, "trap_oracle.cpp")] + trap_oracle.SOURCES[1:],
               trap_oracle.FLAGS)
    l.rayn_albedo_oracle_render.restype = C.c_int32
    l.rayn_albedo_oracle_render.argtypes = [C.POINTER(L.RaynSceneDesc), C.c_int32, C.POINTER(L.RaynAlbedoTrap), C.POINTER(L.RaynFrameDesc),
                                            fp, fp, C.c_int32, C.c_int32]
    return l


def denoise_lib():
    l = _build("denoise_albedo_oracle", os.path.join(HERE, "denoise_albedo_oracle.cpp"), denoise_oracle.SOURCES[1:], denoise_oracle.FLAGS)
    l.rayn_oracle_film_denoise_albedo.restype = C.c_int32
    l.rayn_oracle_film_denoise_albedo.argtypes = [C.POINTER(L.RaynDenoiseDesc), C.c_float, fp, C.c_int32, C.c_int32,
                                                  C.POINTER(L.RaynFilmPlanes), C.POINTER(L.RaynFilmPlanes)]
    return l


def render_albedo(world, camera, inputs, tile_size, integrator, time_range, traps=None, n_threads=0, subsample_k=1):
    """CPU albedo plane of the same FrameInputs -> (plane [H, W, 3], per-sample albedos [H, W, spp, 3]), float32.
    subsample_k > 1: only tiles whose index is a multiple of k are computed, the others stay 0."""
    from rayn_b200.film import make_frame_desc
    desc, keep = world.flatten(camera)
    traps = world.albedo_traps() if traps is None else traps
    w, h, spp = inputs.width, inputs.height, inputs.spp
    per = np.zeros(w * h * spp * 3, np.float32)
    plane = np.zeros(3 * w * h, np.float32)
    ptrs = tuple(a.ctypes.data for a in inputs.arrays())
    f = make_frame_desc(w, h, tile_size, inputs.samples, integrator, inputs.frame, time_range, ptrs, L.MEM_HOST,
                        sets=(inputs.sets_1d, inputs.sets_2d))
    arr = (L.RaynAlbedoTrap * max(len(traps), 1))(*traps)
    rc = albedo_lib().rayn_albedo_oracle_render(C.byref(desc), len(traps), arr, C.byref(f), per.ctypes.data_as(fp), plane.ctypes.data_as(fp),
                                                n_threads, subsample_k)
    if rc != 0:
        raise RuntimeError(f"albedo oracle failed: {rc}")
    return plane.reshape(h, w, 3), per.reshape(h, w, spp, 3)


def denoise(width, height, planes, desc, albedo, sigma_albedo):
    """-> (status, {channel: new float32 array}) for the color / background planes given, like denoise_oracle.denoise"""
    flat = {k: np.ascontiguousarray(v, np.float32).reshape(-1) for k, v in planes.items() if v is not None}
    outs = {k: np.empty_like(flat[k]) for k in ("color", "background") if k in flat}
    alb = np.ascontiguousarray(albedo, np.float32).reshape(-1)

    def ptr(d, k):
        return d[k].ctypes.data if k in d else None
    pin = L.RaynFilmPlanes(ptr(flat, "color"), ptr(flat, "alpha"), ptr(flat, "background"), ptr(flat, "normal"), L.MEM_HOST)
    pout = L.RaynFilmPlanes(ptr(outs, "color"), None, ptr(outs, "background"), None, L.MEM_HOST)
    rc = denoise_lib().rayn_oracle_film_denoise_albedo(C.byref(desc), float(sigma_albedo), alb.ctypes.data_as(fp), width, height, C.byref(pin),
                                                       C.byref(pout))
    return rc, outs
