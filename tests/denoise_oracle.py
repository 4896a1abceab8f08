"""ctypes binding of the CPU denoise mirror (tests/denoise_oracle.cpp).  TEST INFRASTRUCTURE ONLY.

The library is compiled on first use into a temporary directory keyed by the sources, in the mul_add variant of the
product library under test (rayn_b200/_lib.py), so the test tree itself is never written."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from rayn_b200 import _lib as L

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SOURCES = [os.path.join(HERE, "denoise_oracle.cpp"), os.path.join(ROOT, "include", "rayn_b200.h"),
           os.path.join(ROOT, "rayn_b200", "csrc", "detmath.h")]
FLAGS = ["-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math",
         f"-DRAYN_MULADD_FUSED={1 if L.MULADD_FUSED else 0}"]
_lib = None


def lib():
    global _lib
    if _lib is None:
        h = hashlib.sha256(" ".join(FLAGS).encode())
        for s in SOURCES:
            h.update(open(s, "rb").read())
        path = os.path.join(tempfile.gettempdir(), f"rayn_denoise_oracle_{os.getuid()}_{h.hexdigest()[:16]}.so")
        if not os.path.exists(path):
            tmp = f"{path}.{os.getpid()}.tmp"
            subprocess.run(["g++"] + FLAGS + ["-o", tmp, SOURCES[0]], check=True, capture_output=True)
            os.replace(tmp, path)
        l = C.CDLL(path)
        l.rayn_oracle_film_denoise.restype = C.c_int32
        l.rayn_oracle_film_denoise.argtypes = [C.POINTER(L.RaynDenoiseDesc), C.c_int32, C.c_int32, C.POINTER(L.RaynFilmPlanes),
                                               C.POINTER(L.RaynFilmPlanes)]
        l.rayn_oracle_exp.restype = C.c_float
        l.rayn_oracle_exp.argtypes = [C.c_float]
        if l.rayn_oracle_muladd_fused() != (1 if L.MULADD_FUSED else 0):
            raise RuntimeError("denoise oracle variant does not match RAYN_MULADD_FUSED")
        _lib = l
    return _lib


def denoise(width, height, planes, desc):
    """-> (status, {channel: new float32 array}) for the color / background planes given (flat or shaped)."""
    flat = {k: np.ascontiguousarray(v, np.float32).reshape(-1) for k, v in planes.items() if v is not None}
    outs = {k: np.empty_like(flat[k]) for k in ("color", "background") if k in flat}

    def ptr(d, k):
        return d[k].ctypes.data if k in d else None
    pin = L.RaynFilmPlanes(ptr(flat, "color"), ptr(flat, "alpha"), ptr(flat, "background"), ptr(flat, "normal"), L.MEM_HOST)
    pout = L.RaynFilmPlanes(ptr(outs, "color"), None, ptr(outs, "background"), None, L.MEM_HOST)
    rc = lib().rayn_oracle_film_denoise(C.byref(desc), width, height, C.byref(pin), C.byref(pout))
    return rc, outs


def exp(x):
    return np.float32(lib().rayn_oracle_exp(float(x)))
