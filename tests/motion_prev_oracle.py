"""ctypes binding of the CPU mirror of the motion plane against an explicit previous scene (tests/motion_prev_oracle.cpp, which
includes tests/motion_oracle.cpp and through it tests/trap_oracle.cpp and oracle/rayn_oracle.cpp unchanged).  TEST
INFRASTRUCTURE ONLY.

The library is compiled on first use into a temporary directory keyed by its sources, in the mul_add variant of the product
library under test (rayn_b200/_lib.py), so the test tree itself is never written."""
import ctypes as C
import os

import numpy as np

from rayn_b200 import _lib as L

import trap_oracle
from albedo_oracle import _build

HERE = os.path.dirname(os.path.abspath(__file__))
fp = C.POINTER(C.c_float)


def motion_prev_lib():
    l = _build("motion_prev_oracle", os.path.join(HERE, "motion_prev_oracle.cpp"), [os.path.join(HERE, "motion_oracle.cpp")] + trap_oracle.SOURCES,
               trap_oracle.FLAGS)
    l.rayn_motion_prev_oracle_render.restype = C.c_int32
    l.rayn_motion_prev_oracle_render.argtypes = [C.POINTER(L.RaynSceneDesc), C.POINTER(L.RaynFrameDesc), C.c_float, C.POINTER(L.RaynSceneDesc), fp, fp,
                                                 C.c_int32, C.c_int32, C.c_void_p]
    return l


def render_motion_prev(desc, prev, inputs, tile_size, integrator, time_range, frame_dt, n_threads=0, subsample_k=1, geometry=False):
    """CPU motion plane against an explicit previous scene (rayn_b200_render_motion_prev): desc is the uploaded scene and prev
    the previous frame's, both RaynSceneDesc (World.flatten's).  -> (plane [H, W, 4], per-sample records [H, W, spp, 4]),
    float32; geometry=True adds per sample (hit point xyz, camera time, u, v) [H, W, spp, 6].  A status other than RAYN_OK
    raises RuntimeError with the status as its argument."""
    from rayn_b200.film import make_frame_desc
    w, h, spp = inputs.width, inputs.height, inputs.spp
    per = np.zeros(w * h * spp * 4, np.float32)
    plane = np.zeros(4 * w * h, np.float32)
    ptrs = tuple(a.ctypes.data for a in inputs.arrays())
    f = make_frame_desc(w, h, tile_size, inputs.samples, integrator, inputs.frame, time_range, ptrs, L.MEM_HOST,
                        sets=(inputs.sets_1d, inputs.sets_2d))
    geo = np.zeros(w * h * spp * 6, np.float32) if geometry else None
    rc = motion_prev_lib().rayn_motion_prev_oracle_render(C.byref(desc), C.byref(f), float(frame_dt), None if prev is None else C.byref(prev),
                                                          per.ctypes.data_as(fp), plane.ctypes.data_as(fp), n_threads, subsample_k,
                                                          None if geo is None else geo.ctypes.data)
    if rc != 0:
        raise RuntimeError(rc)
    out = (plane.reshape(h, w, 4), per.reshape(h, w, spp, 4))
    return out + (geo.reshape(h, w, spp, 6),) if geometry else out
