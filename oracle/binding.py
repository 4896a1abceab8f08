"""ctypes binding of the CPU oracle (oracle/rayn_oracle.cpp).  TEST INFRASTRUCTURE ONLY.

Importable from tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
legs.  Nothing under rayn_b200/ may import this.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from rayn_b200 import _lib as L

HERE = os.path.dirname(os.path.abspath(__file__))
# the oracle variant always matches the product library's (rayn_b200/_lib.py): RAYN_MULADD_FUSED=1 -> `wide` mul_add fused (A6)
LIB_PATH = os.path.join(HERE, "_build", "librayn_oracle_fma.so" if L.MULADD_FUSED else "librayn_oracle.so")
fp = C.POINTER(C.c_float)
_lib = None


def build(force=False):
    src = os.path.join(HERE, "rayn_oracle.cpp")
    deps = [src, os.path.join(HERE, "..", "include", "rayn_b200.h"), os.path.join(HERE, "..", "rayn_b200", "csrc", "detmath.h")]
    outs = [os.path.join(HERE, "_build", n) for n in ("librayn_oracle.so", "librayn_oracle_fma.so")]
    if force or not all(os.path.exists(o) for o in outs) or any(os.path.getmtime(d) > min(os.path.getmtime(o) for o in outs) for d in deps):
        subprocess.run(["make", "-C", HERE, "-B"], check=True, capture_output=True)
    return LIB_PATH


def lib():
    global _lib
    if _lib is None:
        try:
            build()  # mtime check: do not test against an oracle that is older than its sources
        except Exception:
            if not os.path.exists(LIB_PATH):
                raise
        l = C.CDLL(LIB_PATH)
        l.rayn_oracle_selfcheck.restype = C.c_int32
        l.rayn_oracle_render_frame.restype = C.c_int32
        l.rayn_oracle_render_frame.argtypes = [C.POINTER(L.RaynSceneDesc), C.POINTER(L.RaynFrameDesc), C.POINTER(L.RaynFilmPlanes),
                                               C.c_int32, C.c_int32, C.POINTER(C.c_int32), C.c_int64, C.POINTER(C.c_int64),
                                               C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
        l.rayn_oracle_kat_detmath.argtypes = [C.c_int32, C.c_int64, fp, fp, fp]
        l.rayn_oracle_kat_sdf_dist.argtypes = [C.POINTER(L.RaynHitable), C.c_int64, fp, fp]
        l.rayn_oracle_kat_sdf_hit.argtypes = [C.POINTER(L.RaynHitable), C.POINTER(L.RaynRenderConsts), C.c_int64, fp, fp, fp,
                                              C.c_float, C.c_int32, fp]
        l.rayn_oracle_kat_occluded.argtypes = [C.POINTER(L.RaynSceneDesc), C.c_int64, fp, fp, fp]
        l.rayn_oracle_kat_closest_hit.argtypes = [C.POINTER(L.RaynSceneDesc), C.c_int32, C.c_int64, fp, fp, fp, C.POINTER(C.c_int32)]
        l.rayn_oracle_kat_light_sample.argtypes = [C.POINTER(L.RaynLight), C.c_int64, fp, fp, fp, fp, fp]
        l.rayn_oracle_kat_light_sample_volume.argtypes = [C.POINTER(L.RaynLight), C.c_int64, fp, fp, fp, fp, fp, fp]
        l.rayn_oracle_kat_bsdf.argtypes = [C.POINTER(L.RaynMaterial), C.c_int64, fp, fp, fp, fp, fp, fp, fp, fp]
        l.rayn_oracle_film_postprocess.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.POINTER(L.RaynFilmPlanes), C.c_void_p]
        if l.rayn_oracle_selfcheck() != 0:
            raise RuntimeError("oracle was built with FP contraction on: rebuild with -ffp-contract=off")
        if l.rayn_oracle_muladd_fused() != (1 if L.MULADD_FUSED else 0):
            raise RuntimeError("oracle library variant does not match RAYN_MULADD_FUSED")
        _lib = l
    return _lib


def _f(a):
    return a.ctypes.data_as(fp)


def render(world, camera, inputs, tile_size, integrator, time_range, n_threads=0, subsample_k=1, tile_offset=0, tile_stride=1,
           queue_log=False, tile_list=None):
    """CPU render of the same FrameInputs.  Returns (planes dict, info dict)."""
    from rayn_b200.film import host_planes, make_frame_desc
    desc, keep = world.flatten(camera)
    w, h = inputs.width, inputs.height
    planes, p = host_planes(w, h)
    ptrs = tuple(a.ctypes.data for a in inputs.arrays())
    f = make_frame_desc(w, h, tile_size, inputs.samples, integrator, inputs.frame, time_range, ptrs, L.MEM_HOST, tile_offset,
                        tile_stride, (inputs.sets_1d, inputs.sets_2d), tile_list)
    qbuf, qcap = None, 0
    if queue_log:
        qcap = 64 + 8 * (w * h * inputs.spp + 64 * 64) * (integrator.max_bounces + 1)
        qbuf = np.empty(qcap, np.int32)
    qn = C.c_int64(0)
    counters = (C.c_int64 * 4)()
    tiles = C.c_int64(0)
    rc = lib().rayn_oracle_render_frame(C.byref(desc), C.byref(f), C.byref(p), n_threads, subsample_k,
                                        qbuf.ctypes.data_as(C.POINTER(C.c_int32)) if queue_log else None, qcap, C.byref(qn),
                                        counters, C.byref(tiles))
    if rc != 0:
        raise RuntimeError(f"oracle render failed: {rc}")
    info = {"extend_rays": counters[0], "shade_lanes": counters[1], "shadow_rays": counters[2], "sdf_evals_extend": counters[3],
            "tiles": tiles.value}
    if queue_log:
        if qn.value > qcap:
            raise RuntimeError("oracle queue log overflow")
        info["queue_log"] = qbuf[:qn.value].copy()
    return planes, info


def kat_detmath(op, a, b=None):
    a = np.ascontiguousarray(a, np.float32)
    b = np.ascontiguousarray(b if b is not None else a, np.float32)
    out = np.empty_like(a)
    lib().rayn_oracle_kat_detmath(op, a.size, _f(a), _f(b), _f(out))
    return out


def kat_sdf_dist(hitable, points):
    p = np.ascontiguousarray(points, np.float32).reshape(-1, 3)
    out = np.empty(len(p), np.float32)
    lib().rayn_oracle_kat_sdf_dist(C.byref(hitable), len(p), _f(p), _f(out))
    return out


def kat_sdf_hit(hitable, consts, origins, dirs, t_max, thr_scale, thr_const=0):
    o = np.ascontiguousarray(origins, np.float32).reshape(-1, 3)
    d = np.ascontiguousarray(dirs, np.float32).reshape(-1, 3)
    tm = np.ascontiguousarray(t_max, np.float32)
    out = np.empty(len(o), np.float32)
    lib().rayn_oracle_kat_sdf_hit(C.byref(hitable), C.byref(consts), len(o), _f(o), _f(d), _f(tm), thr_scale, thr_const, _f(out))
    return out


def kat_occluded(scene_desc, start, end):
    s = np.ascontiguousarray(start, np.float32).reshape(-1, 3)
    e = np.ascontiguousarray(end, np.float32).reshape(-1, 3)
    out = np.empty(len(s), np.float32)
    lib().rayn_oracle_kat_occluded(C.byref(scene_desc), len(s), _f(s), _f(e), _f(out))
    return out


def kat_closest_hit(scene_desc, depth, origins, dirs):
    o = np.ascontiguousarray(origins, np.float32).reshape(-1, 3)
    d = np.ascontiguousarray(dirs, np.float32).reshape(-1, 3)
    t = np.empty(len(o), np.float32)
    obj = np.empty(len(o), np.int32)
    lib().rayn_oracle_kat_closest_hit(C.byref(scene_desc), depth, len(o), _f(o), _f(d), _f(t), obj.ctypes.data_as(C.POINTER(C.c_int32)))
    return t, obj


def film_postprocess(mode, width, height, planes):
    """CPU restatement of Film::save_to's pixel arithmetic (film.rs:205-377) -> uint8 array [H, W, bpp]."""
    p = L.RaynFilmPlanes(planes["color"].ctypes.data, planes["alpha"].ctypes.data, planes["background"].ctypes.data,
                         planes["normal"].ctypes.data, L.MEM_HOST)
    out = np.zeros((height, width, L.POST_BYTES[mode]), np.uint8)
    lib().rayn_oracle_film_postprocess(mode, width, height, C.byref(p), out.ctypes.data)
    return out


def kat_light_sample(light, s0, s1, p):
    s0, s1 = np.ascontiguousarray(s0, np.float32), np.ascontiguousarray(s1, np.float32)
    p = np.ascontiguousarray(p, np.float32).reshape(-1, 3)
    pt, pdf = np.empty_like(p), np.empty(len(p), np.float32)
    lib().rayn_oracle_kat_light_sample(C.byref(light), len(p), _f(s0), _f(s1), _f(p), _f(pt), _f(pdf))
    return pt, pdf


def kat_light_sample_volume(light, sample, o, d, t_max):
    sample, t_max = np.ascontiguousarray(sample, np.float32), np.ascontiguousarray(t_max, np.float32)
    o, d = np.ascontiguousarray(o, np.float32).reshape(-1, 3), np.ascontiguousarray(d, np.float32).reshape(-1, 3)
    t, pdf = np.empty(len(o), np.float32), np.empty(len(o), np.float32)
    lib().rayn_oracle_kat_light_sample_volume(C.byref(light), len(o), _f(sample), _f(o), _f(d), _f(t_max), _f(t), _f(pdf))
    return t, pdf


def kat_bsdf(mat, normals, wo, s1d, u4):
    n3, w3 = np.ascontiguousarray(normals, np.float32).reshape(-1, 3), np.ascontiguousarray(wo, np.float32).reshape(-1, 3)
    s1d, u4 = np.ascontiguousarray(s1d, np.float32), np.ascontiguousarray(u4, np.float32).reshape(-1, 4)
    wi, f, fe, pdf = np.empty_like(n3), np.empty_like(n3), np.empty_like(n3), np.empty(len(n3), np.float32)
    lib().rayn_oracle_kat_bsdf(C.byref(mat), len(n3), _f(n3), _f(w3), _f(s1d), _f(u4), _f(wi), _f(f), _f(pdf), _f(fe))
    return wi, f, pdf, fe


def set_decoupled_lights(on):
    """TEST-ONLY (SURVEY T5): per-lane instead of per-packet surface-NEE light choice.  Always reset to False."""
    lib().rayn_oracle_set_decoupled_lights(1 if on else 0)
