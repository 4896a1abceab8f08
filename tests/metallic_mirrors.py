"""CPU mirror of the Metallic material.  TEST INFRASTRUCTURE ONLY.

tests/metallic_mirror.cpp (the render mirror and the oracle, included unchanged, with the metal's f and scatter): the oracle's
film, the render mirror's film (orbit traps, moments), the first-hit albedo plane and the BSDF KAT, for every material kind.
Built like tests/mirrors.py's libraries (the same flags, a temporary directory keyed by sources and flags)."""
import ctypes as C
import os

import numpy as np

from rayn_b200 import _lib as L

import mirrors

HERE = os.path.dirname(os.path.abspath(__file__))
METAL = ("metallic_mirror", [os.path.join(HERE, "metallic_mirror.cpp")] + mirrors.RENDER[1], mirrors.RENDER[2])
P = C.POINTER
fp = P(C.c_float)
_libs = {}


def lib():
    if "metal" not in _libs:
        l = mirrors._build(*METAL)
        l.rayn_oracle_render_frame.restype = C.c_int32
        l.rayn_oracle_render_frame.argtypes = [P(L.RaynSceneDesc), P(L.RaynFrameDesc), P(L.RaynFilmPlanes), C.c_int32, C.c_int32, P(C.c_int32),
                                               C.c_int64, P(C.c_int64), P(C.c_int64), P(C.c_int64)]
        l.rayn_mirror_render_frame.restype = C.c_int32
        l.rayn_mirror_render_frame.argtypes = [P(L.RaynSceneDesc), C.c_int32, P(L.RaynAlbedoTrap), P(L.RaynFrameDesc), P(L.RaynFilmPlanes),
                                               C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, P(C.c_int64), P(C.c_int64)]
        l.rayn_metal_render_albedo.restype = C.c_int32
        l.rayn_metal_render_albedo.argtypes = [P(L.RaynSceneDesc), C.c_int32, P(L.RaynAlbedoTrap), P(L.RaynFrameDesc), fp, fp, C.c_int32, C.c_int32]
        l.rayn_metal_kat_bsdf.argtypes = [P(L.RaynMaterial), C.c_int64, fp, fp, fp, fp, fp, fp, fp, fp]
        _libs["metal"] = l
    return _libs["metal"]


def _f(a):
    return a.ctypes.data_as(fp)


def oracle_render(world, camera, inputs, tile_size, integrator, time_range, subsample_k=1, tile_list=None):
    """the oracle's own render_frame (render_tile, film.rs:439-627) of the same FrameInputs, metals included -> planes dict"""
    from rayn_b200.film import host_planes
    desc, keep = world.flatten(camera, time_range)
    planes, p = host_planes(inputs.width, inputs.height)
    f = mirrors._frame(inputs, tile_size, integrator, time_range, tile_list)
    qn, counters, tiles = C.c_int64(0), (C.c_int64 * 4)(), C.c_int64(0)
    rc = lib().rayn_oracle_render_frame(C.byref(desc), C.byref(f), C.byref(p), 0, subsample_k, None, 0, C.byref(qn), counters, C.byref(tiles))
    if rc != 0:
        raise RuntimeError(f"oracle render failed: {rc}")
    return planes


def render(world, camera, inputs, tile_size, integrator, time_range, moments=False, tile_list=None):
    """the render mirror's film (the world's orbit traps; moments=True adds planes["moments"] [H, W, 2]) -> planes dict"""
    from rayn_b200.film import host_planes
    desc, keep = world.flatten(camera, time_range)
    w, h = inputs.width, inputs.height
    planes, p = host_planes(w, h)
    m = np.zeros((2, w * h), np.float32)
    f = mirrors._frame(inputs, tile_size, integrator, time_range, tile_list)
    counters, tiles = (C.c_int64 * 4)(), C.c_int64(0)
    rc = lib().rayn_mirror_render_frame(C.byref(desc), *mirrors._traps(world, None), C.byref(f), C.byref(p), m[0].ctypes.data if moments else None,
                                        m[1].ctypes.data if moments else None, 0, 1, counters, C.byref(tiles))
    if rc != 0:
        raise RuntimeError(f"render mirror failed: {rc}")
    if moments:
        planes["moments"] = np.ascontiguousarray(m.reshape(2, h, w).transpose(1, 2, 0))
    return planes


def render_albedo(world, camera, inputs, tile_size, integrator, time_range):
    """the first-hit albedo plane [H, W, 3] of the same FrameInputs (F0 on a metal, or its trap palette)"""
    desc, keep = world.flatten(camera, time_range)
    w, h, spp = inputs.width, inputs.height, inputs.spp
    per, plane = np.zeros(w * h * spp * 3, np.float32), np.zeros(3 * w * h, np.float32)
    f = mirrors._frame(inputs, tile_size, integrator, time_range)
    rc = lib().rayn_metal_render_albedo(C.byref(desc), *mirrors._traps(world, None), C.byref(f), _f(per), _f(plane), 0, 1)
    if rc != 0:
        raise RuntimeError(f"albedo mirror failed: {rc}")
    return plane.reshape(h, w, 3)


def kat_bsdf(mat, normals, wo, s1d, u4):
    """oracle.binding.kat_bsdf for every kind, the metal included -> (wi, f, pdf, f(wo, wi, n))"""
    n3, w3 = np.ascontiguousarray(normals, np.float32).reshape(-1, 3), np.ascontiguousarray(wo, np.float32).reshape(-1, 3)
    s1d, u4 = np.ascontiguousarray(s1d, np.float32), np.ascontiguousarray(u4, np.float32).reshape(-1, 4)
    wi, f, fe, pdf = np.empty_like(n3), np.empty_like(n3), np.empty_like(n3), np.empty(len(n3), np.float32)
    lib().rayn_metal_kat_bsdf(C.byref(mat), len(n3), _f(n3), _f(w3), _f(s1d), _f(u4), _f(wi), _f(f), _f(pdf), _f(fe))
    return wi, f, pdf, fe
