"""ctypes bindings of the CPU mirrors the GPU passes are tested against bit for bit.  TEST INFRASTRUCTURE ONLY.

tests/render_mirror.cpp (which includes oracle/rayn_oracle.cpp unchanged): the film with orbit-trap albedos and luminance
moments, the first-hit albedo and motion planes and the trap KATs.  tests/film_mirror.cpp: the four denoise entry points and
the temporal push.  Each library is compiled on first use into a temporary directory keyed by its sources and flags, in the
mul_add variant of the product library under test (rayn_b200/_lib.py), so the test tree itself is never written."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from rayn_b200 import _lib as L

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
HEADERS = [os.path.join(ROOT, "include", "rayn_b200.h"), os.path.join(ROOT, "rayn_b200", "csrc", "detmath.h")]
COMMON = ["-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", f"-DRAYN_MULADD_FUSED={1 if L.MULADD_FUSED else 0}"]
RENDER = ("render_mirror", [os.path.join(HERE, "render_mirror.cpp"), os.path.join(ROOT, "oracle", "rayn_oracle.cpp")] + HEADERS,
          ["-O3", "-msse4.1", "-mavx2", "-mfma", "-fopenmp"] + COMMON)
FILM = ("film_mirror", [os.path.join(HERE, "film_mirror.cpp")] + HEADERS, ["-O2"] + COMMON)
SWEEP = ("detmath_sweep", [os.path.join(HERE, "detmath_sweep.cpp")] + HEADERS, RENDER[2])
N_HIST = 14  # history planes of a RaynTemporal
fp = C.POINTER(C.c_float)
P = C.POINTER
_libs = {}


def _build(name, sources, flags):
    """the library of sources[0] (its includes follow it), built once per key of sources and flags"""
    h = hashlib.sha256(" ".join(flags).encode())
    for s in sources:
        h.update(open(s, "rb").read())
    path = os.path.join(tempfile.gettempdir(), f"rayn_{name}_{os.getuid()}_{h.hexdigest()[:16]}.so")
    if not os.path.exists(path):
        tmp = f"{path}.{os.getpid()}.tmp"
        subprocess.run(["g++"] + flags + ["-o", tmp, sources[0]], check=True, capture_output=True)
        os.replace(tmp, path)
    l = C.CDLL(path)
    if l.rayn_oracle_selfcheck() != 0:
        raise RuntimeError(f"{name} was built with FP contraction on")
    if l.rayn_oracle_muladd_fused() != (1 if L.MULADD_FUSED else 0):
        raise RuntimeError(f"{name} variant does not match RAYN_MULADD_FUSED")
    return l


def render_lib():
    if "render" not in _libs:
        l = _build(*RENDER)
        l.rayn_mirror_render_frame.restype = C.c_int32
        l.rayn_mirror_render_frame.argtypes = [P(L.RaynSceneDesc), C.c_int32, P(L.RaynAlbedoTrap), P(L.RaynFrameDesc), P(L.RaynFilmPlanes),
                                               C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, P(C.c_int64), P(C.c_int64)]
        l.rayn_mirror_render_albedo.restype = C.c_int32
        l.rayn_mirror_render_albedo.argtypes = [P(L.RaynSceneDesc), C.c_int32, P(L.RaynAlbedoTrap), P(L.RaynFrameDesc), fp, fp, C.c_int32,
                                                C.c_int32]
        l.rayn_mirror_render_motion.restype = C.c_int32
        l.rayn_mirror_render_motion.argtypes = [P(L.RaynSceneDesc), P(L.RaynFrameDesc), C.c_float, P(L.RaynSceneDesc), fp, fp, C.c_int32,
                                                C.c_int32, C.c_void_p]
        l.rayn_mirror_kat_sdf_trap.argtypes = [P(L.RaynHitable), C.c_int64, fp, fp]
        l.rayn_mirror_kat_trap_albedo.argtypes = [P(L.RaynAlbedoTrap), C.c_int64, fp, fp, fp]
        _libs["render"] = l
    return _libs["render"]


def film_lib():
    if "film" not in _libs:
        l = _build(*FILM)
        planes = [C.c_int32, C.c_int32, P(L.RaynFilmPlanes), P(L.RaynFilmPlanes)]
        variance = [P(L.RaynDenoiseDesc), C.c_float, C.c_int32, P(L.RaynMomentPlanes)]
        for name, args in (("", [P(L.RaynDenoiseDesc)]), ("_albedo", [P(L.RaynDenoiseDesc), C.c_float, C.c_void_p]),
                           ("_variance", variance + [C.c_float, C.c_void_p]), ("_variance_scaled", variance + [C.c_void_p, C.c_float, C.c_void_p])):
            fn = getattr(l, "rayn_oracle_film_denoise" + name)
            fn.restype, fn.argtypes = C.c_int32, args + planes
        l.rayn_oracle_temporal_push.restype = C.c_int32
        l.rayn_oracle_temporal_push.argtypes = [C.c_int32, C.c_int32, P(L.RaynTemporalDesc)] + [C.c_void_p] * 13
        l.rayn_oracle_exp.restype = C.c_float
        l.rayn_oracle_exp.argtypes = [C.c_float]
        _libs["film"] = l
    return _libs["film"]


class SweepAcc(C.Structure):
    _fields_ = [("max_err", C.c_double), ("argmax", C.c_uint32), ("over", C.c_int64)]


def sweep_lib():
    if "sweep" not in _libs:
        l = _build(*SWEEP)
        l.detmath_sweep.restype = C.c_int32
        l.detmath_sweep.argtypes = [C.c_int32, C.c_float, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_double, P(C.c_uint64),
                                    P(SweepAcc)]
        l.detmath_error.restype = C.c_double
        l.detmath_error.argtypes = [C.c_int32, C.c_float, C.c_float, C.c_float]
        _libs["sweep"] = l
    return _libs["sweep"]


def detmath_sweep(op, fixed, swap, chunk0, n_chunks, accuracy, bound):
    """tests/detmath_sweep.cpp over chunks [chunk0, chunk0 + n_chunks) -> (hashes [n_chunks] uint64, None or
    ({"max", "argmax", "over"} over the contract domain, the same over the render-path domain))"""
    hashes = np.zeros(n_chunks, np.uint64)
    acc = (SweepAcc * 2)()
    rc = sweep_lib().detmath_sweep(op, float(fixed), 1 if swap else 0, chunk0, n_chunks, 1 if accuracy else 0, float(bound),
                                   hashes.ctypes.data_as(P(C.c_uint64)), acc)
    if rc != 0:
        raise ValueError(f"detmath_sweep: bad argument (op {op}, chunks {chunk0}+{n_chunks})")
    if not accuracy:
        return hashes, None
    return hashes, tuple({"max": a.max_err, "argmax": a.argmax, "over": a.over} for a in acc)


def detmath_error(op, a, b, got):
    """the sweep's error measure of one result against long-double libm (ulp; relative for ln_fast, op 8)"""
    return sweep_lib().detmath_error(op, float(a), float(b), float(got))


def _f(a):
    return a.ctypes.data_as(fp)


def _frame(inputs, tile_size, integrator, time_range, tile_list=None):
    from rayn_b200.film import make_frame_desc
    ptrs = tuple(a.ctypes.data for a in inputs.arrays())
    return make_frame_desc(inputs.width, inputs.height, tile_size, inputs.samples, integrator, inputs.frame, time_range, ptrs, L.MEM_HOST,
                           sets=(inputs.sets_1d, inputs.sets_2d), tile_list=tile_list)


def _traps(world, traps):
    traps = world.albedo_traps() if traps is None else traps
    return len(traps), (L.RaynAlbedoTrap * max(len(traps), 1))(*traps)


def _moment_planes(moments, width, height):
    """float32 [H, W, 2] (color_lum2, background_lum2) -> (the two planes [2, W*H], RaynMomentPlanes pointing at them)"""
    m = np.ascontiguousarray(np.asarray(moments, np.float32).reshape(height, width, 2).transpose(2, 0, 1)).reshape(2, -1)
    return m, L.RaynMomentPlanes(m[0].ctypes.data, m[1].ctypes.data, L.MEM_HOST)


def render(world, camera, inputs, tile_size, integrator, time_range, n_threads=0, subsample_k=1, tile_list=None, traps=None, moments=False):
    """CPU render of the same FrameInputs with the world's orbit-trap albedos (World.albedo_traps(), or `traps`: a list of
    RaynAlbedoTrap).  Returns (planes dict, info dict), like oracle.binding.render; moments=True adds planes["moments"],
    float32 [H, W, 2].  Tiles as rayn_b200_render_frame's, of which subsample_k > 1 computes every k-th; the others stay 0."""
    from rayn_b200.film import host_planes
    desc, keep = world.flatten(camera)
    w, h = inputs.width, inputs.height
    planes, p = host_planes(w, h)
    m = np.zeros((2, w * h), np.float32)
    f = _frame(inputs, tile_size, integrator, time_range, tile_list)
    counters, tiles = (C.c_int64 * 4)(), C.c_int64(0)
    rc = render_lib().rayn_mirror_render_frame(C.byref(desc), *_traps(world, traps), C.byref(f), C.byref(p), m[0].ctypes.data if moments else None,
                                               m[1].ctypes.data if moments else None, n_threads, subsample_k, counters, C.byref(tiles))
    if rc != 0:
        raise RuntimeError(f"render mirror failed: {rc}")
    if moments:
        planes["moments"] = np.ascontiguousarray(m.reshape(2, h, w).transpose(1, 2, 0))
    info = {"extend_rays": counters[0], "shade_lanes": counters[1], "shadow_rays": counters[2], "sdf_evals_extend": counters[3],
            "tiles": tiles.value}
    return planes, info


def render_albedo(world, camera, inputs, tile_size, integrator, time_range, traps=None, n_threads=0, subsample_k=1):
    """CPU albedo plane of the same FrameInputs -> (plane [H, W, 3], per-sample albedos [H, W, spp, 3]), float32.
    subsample_k > 1: only tiles whose index is a multiple of k are computed, the others stay 0."""
    desc, keep = world.flatten(camera)
    w, h, spp = inputs.width, inputs.height, inputs.spp
    per, plane = np.zeros(w * h * spp * 3, np.float32), np.zeros(3 * w * h, np.float32)
    f = _frame(inputs, tile_size, integrator, time_range)
    rc = render_lib().rayn_mirror_render_albedo(C.byref(desc), *_traps(world, traps), C.byref(f), _f(per), _f(plane), n_threads, subsample_k)
    if rc != 0:
        raise RuntimeError(f"albedo mirror failed: {rc}")
    return plane.reshape(h, w, 3), per.reshape(h, w, spp, 3)


def render_motion(scene, inputs, tile_size, integrator, time_range, frame_dt, prev=None, n_threads=0, subsample_k=1, geometry=False):
    """CPU motion plane of the same FrameInputs for the uploaded scene `scene` (a RaynSceneDesc, World.flatten's): against
    the previous frame's scene prev (rayn_b200_render_motion_prev), or with prev None against the scene run backwards
    (rayn_b200_render_motion).  -> (plane [H, W, 4], per-sample records [H, W, spp, 4]), float32; geometry=True adds per
    sample (hit point xyz, camera time, u, v) [H, W, spp, 6].  A status other than RAYN_OK raises RuntimeError with the status
    as its argument."""
    w, h, spp = inputs.width, inputs.height, inputs.spp
    per, plane = np.zeros(w * h * spp * 4, np.float32), np.zeros(4 * w * h, np.float32)
    f = _frame(inputs, tile_size, integrator, time_range)
    geo = np.zeros(w * h * spp * 6, np.float32) if geometry else None
    rc = render_lib().rayn_mirror_render_motion(C.byref(scene), C.byref(f), float(frame_dt), None if prev is None else C.byref(prev), _f(per),
                                                _f(plane), n_threads, subsample_k, None if geo is None else geo.ctypes.data)
    if rc != 0:
        raise RuntimeError(rc)
    out = (plane.reshape(h, w, 4), per.reshape(h, w, spp, 4))
    return out + (geo.reshape(h, w, spp, 6),) if geometry else out


def kat_sdf_trap(hitable, points):
    """orbit trap per point (include/rayn_b200.h, RaynAlbedoTrap)"""
    p = np.ascontiguousarray(points, np.float32).reshape(-1, 3)
    out = np.empty(len(p), np.float32)
    render_lib().rayn_mirror_kat_sdf_trap(C.byref(hitable), len(p), _f(p), _f(out))
    return out


def kat_trap_albedo(trap_desc, trap):
    """(s, albedo [n, 3]) of trap values for one RaynAlbedoTrap"""
    t = np.ascontiguousarray(trap, np.float32).reshape(-1)
    s, a = np.empty(len(t), np.float32), np.empty((len(t), 3), np.float32)
    render_lib().rayn_mirror_kat_trap_albedo(C.byref(trap_desc), len(t), _f(t), _f(s), _f(a))
    return s, a


def denoise(width, height, planes, desc, albedo=None, sigma_albedo=np.inf, moments=None, spp=None, sigma_luminance=np.inf, var_scale=None):
    """-> (status, {channel: new float32 array}) for the color / background planes given (flat or shaped).  The entry point
    is Renderer.denoise's: moments (float32 [H, W, 2]) with spp the variance filter, scaled by var_scale [H, W] if given;
    otherwise albedo [3*W*H] the albedo-guided filter; otherwise the plain filter."""
    flat = {k: np.ascontiguousarray(v, np.float32).reshape(-1) for k, v in planes.items() if v is not None}
    outs = {k: np.empty_like(flat[k]) for k in ("color", "background") if k in flat}

    def ptr(d, k):
        return d[k].ctypes.data if k in d else None
    pin = L.RaynFilmPlanes(ptr(flat, "color"), ptr(flat, "alpha"), ptr(flat, "background"), ptr(flat, "normal"), L.MEM_HOST)
    pout = L.RaynFilmPlanes(ptr(outs, "color"), None, ptr(outs, "background"), None, L.MEM_HOST)
    alb = None if albedo is None else np.ascontiguousarray(albedo, np.float32).reshape(-1)
    alb_p = None if alb is None else alb.ctypes.data
    tail = (width, height, C.byref(pin), C.byref(pout))
    l = film_lib()
    if moments is not None:
        m, mp = _moment_planes(moments, width, height)
        head = (C.byref(desc), float(sigma_luminance), int(spp), C.byref(mp))
        if var_scale is None:
            rc = l.rayn_oracle_film_denoise_variance(*head, float(sigma_albedo), alb_p, *tail)
        else:
            vs = np.ascontiguousarray(var_scale, np.float32).reshape(-1)
            rc = l.rayn_oracle_film_denoise_variance_scaled(*head, vs.ctypes.data, float(sigma_albedo), alb_p, *tail)
    elif var_scale is not None:
        raise ValueError("var_scale scales the variance of the moments: pass moments too")
    elif albedo is None:
        rc = l.rayn_oracle_film_denoise(C.byref(desc), *tail)
    else:
        rc = l.rayn_oracle_film_denoise_albedo(C.byref(desc), float(sigma_albedo), alb_p, *tail)
    return rc, outs


def exp(x):
    return np.float32(film_lib().rayn_oracle_exp(float(x)))


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
        m, _ = _moment_planes(moments, w, h)
        mv = np.ascontiguousarray(motion, np.float32).reshape(-1)
        oc, ob, om, s = np.empty_like(c), np.empty_like(b), np.empty_like(m), np.empty(w * h, np.float32)
        d = L.RaynTemporalDesc(float(alpha_min), float(sigma_depth), float(normal_cos), 1 if reset else 0)
        hin, hout = self.hist[self.cur], self.hist[self.cur ^ 1]
        rc = film_lib().rayn_oracle_temporal_push(w, h, C.byref(d), hin.ctypes.data, hout.ctypes.data, c.ctypes.data, b.ctypes.data,
                                                  n.ctypes.data, m[0].ctypes.data, m[1].ctypes.data, mv.ctypes.data, oc.ctypes.data,
                                                  ob.ctypes.data, om[0].ctypes.data, om[1].ctypes.data, s.ctypes.data)
        if rc == 0:
            self.cur ^= 1
        out = {"color": oc.reshape(np.shape(planes["color"])), "background": ob.reshape(np.shape(planes["background"]))}
        return rc, out, np.ascontiguousarray(om.reshape(2, h, w).transpose(1, 2, 0)), s.reshape(h, w)
