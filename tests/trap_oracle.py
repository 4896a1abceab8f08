"""ctypes binding of the CPU oracle of the orbit-trap albedo (tests/trap_oracle.cpp, which includes oracle/rayn_oracle.cpp
unchanged).  TEST INFRASTRUCTURE ONLY.

The library is compiled on first use into a temporary directory keyed by the sources, with the flags of oracle/Makefile, in
the mul_add variant of the product library under test (rayn_b200/_lib.py), so the test tree itself is never written."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from rayn_b200 import _lib as L

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SOURCES = [os.path.join(HERE, "trap_oracle.cpp"), os.path.join(ROOT, "oracle", "rayn_oracle.cpp"),
           os.path.join(ROOT, "include", "rayn_b200.h"), os.path.join(ROOT, "rayn_b200", "csrc", "detmath.h")]
FLAGS = ["-O3", "-std=c++17", "-msse4.1", "-mavx2", "-mfma", "-ffp-contract=off", "-fno-fast-math", "-fopenmp", "-fPIC", "-shared",
         f"-DRAYN_MULADD_FUSED={1 if L.MULADD_FUSED else 0}"]
fp = C.POINTER(C.c_float)
_lib = None


def lib():
    global _lib
    if _lib is None:
        h = hashlib.sha256(" ".join(FLAGS).encode())
        for s in SOURCES:
            h.update(open(s, "rb").read())
        path = os.path.join(tempfile.gettempdir(), f"rayn_trap_oracle_{os.getuid()}_{h.hexdigest()[:16]}.so")
        if not os.path.exists(path):
            tmp = f"{path}.{os.getpid()}.tmp"
            subprocess.run(["g++"] + FLAGS + ["-o", tmp, SOURCES[0]], check=True, capture_output=True)
            os.replace(tmp, path)
        l = C.CDLL(path)
        l.rayn_trap_oracle_render_frame.restype = C.c_int32
        l.rayn_trap_oracle_render_frame.argtypes = [C.POINTER(L.RaynSceneDesc), C.c_int32, C.POINTER(L.RaynAlbedoTrap),
                                                    C.POINTER(L.RaynFrameDesc), C.POINTER(L.RaynFilmPlanes), C.c_int32, C.c_int32,
                                                    C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
        l.rayn_trap_oracle_kat_sdf_trap.argtypes = [C.POINTER(L.RaynHitable), C.c_int64, fp, fp]
        l.rayn_trap_oracle_kat_trap_albedo.argtypes = [C.POINTER(L.RaynAlbedoTrap), C.c_int64, fp, fp, fp]
        if l.rayn_oracle_selfcheck() != 0:
            raise RuntimeError("trap oracle was built with FP contraction on")
        if l.rayn_oracle_muladd_fused() != (1 if L.MULADD_FUSED else 0):
            raise RuntimeError("trap oracle variant does not match RAYN_MULADD_FUSED")
        _lib = l
    return _lib


def _f(a):
    return a.ctypes.data_as(fp)


def render(world, camera, inputs, tile_size, integrator, time_range, n_threads=0, subsample_k=1, tile_list=None, traps=None):
    """CPU render of the same FrameInputs with the world's orbit-trap albedos (World.albedo_traps(), or `traps`: a list of
    RaynAlbedoTrap).  Returns (planes dict, info dict), like oracle.binding.render."""
    from rayn_b200.film import host_planes, make_frame_desc
    desc, keep = world.flatten(camera)
    traps = world.albedo_traps() if traps is None else traps
    w, h = inputs.width, inputs.height
    planes, p = host_planes(w, h)
    ptrs = tuple(a.ctypes.data for a in inputs.arrays())
    f = make_frame_desc(w, h, tile_size, inputs.samples, integrator, inputs.frame, time_range, ptrs, L.MEM_HOST, 0, 1,
                        (inputs.sets_1d, inputs.sets_2d), tile_list)
    arr = (L.RaynAlbedoTrap * max(len(traps), 1))(*traps)
    counters = (C.c_int64 * 4)()
    tiles = C.c_int64(0)
    rc = lib().rayn_trap_oracle_render_frame(C.byref(desc), len(traps), arr, C.byref(f), C.byref(p), n_threads, subsample_k, counters,
                                             C.byref(tiles))
    if rc != 0:
        raise RuntimeError(f"trap oracle render failed: {rc}")
    info = {"extend_rays": counters[0], "shade_lanes": counters[1], "shadow_rays": counters[2], "sdf_evals_extend": counters[3],
            "tiles": tiles.value}
    return planes, info


def kat_sdf_trap(hitable, points):
    """orbit trap per point (include/rayn_b200.h, RaynAlbedoTrap)"""
    p = np.ascontiguousarray(points, np.float32).reshape(-1, 3)
    out = np.empty(len(p), np.float32)
    lib().rayn_trap_oracle_kat_sdf_trap(C.byref(hitable), len(p), _f(p), _f(out))
    return out


def kat_trap_albedo(trap_desc, trap):
    """(s, albedo [n, 3]) of trap values for one RaynAlbedoTrap"""
    t = np.ascontiguousarray(trap, np.float32).reshape(-1)
    s, a = np.empty(len(t), np.float32), np.empty((len(t), 3), np.float32)
    lib().rayn_trap_oracle_kat_trap_albedo(C.byref(trap_desc), len(t), _f(t), _f(s), _f(a))
    return s, a
