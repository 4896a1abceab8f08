"""Film + the render entry point: the host-side mirror of reference src/film.rs.

`Film.render_frame_into(world, camera, integrator, filter, tile_size, frame, time_range,
samples)` has the reference's signature (film.rs:382-395) and is the user-facing call; it
builds the host-owned sampler state exactly where the reference does (film.rs:429-434,
460-461), flattens the World and calls `rayn_b200_render_frame` through the C ABI.

`Renderer` is the thin handle on the C context for callers that keep buffers resident on the
device (bench, multi-GPU driver).  There is no CPU path: without the CUDA library or a GPU
these raise.
"""
import ctypes as C

import numpy as np

from . import _lib as L
from .scene import BlackmanHarrisFilter, PathTracingIntegrator

CHANNELS = ("color", "alpha", "background", "normal")  # ChannelKind, film.rs:103-120
# a Film may also hold the first-hit albedo plane (Renderer.render_albedo) and the luminance second moments of its colour
# and background planes (Renderer.render_host(moments=True)), which the reference has no channels for, and the first-hit
# motion plane (Renderer.render_motion, float32 [H, W, 4]), which Film.render_sequence fills
FILM_CHANNELS = CHANNELS + ("albedo", "moments", "motion")


def _fptr(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def host_planes(width, height):
    """Zeroed host planes of a width x height film (dict of flat float32 arrays, keyed by CHANNELS) and the host-space
    RaynFilmPlanes that points at them.  Keep the dict alive while the C side may write the planes."""
    planes = {k: np.zeros((1 if k == "alpha" else 3) * width * height, np.float32) for k in CHANNELS}
    return planes, L.RaynFilmPlanes(*(planes[k].ctypes.data for k in CHANNELS), L.MEM_HOST)


class FrameInputs:
    """Host-owned sampler state of one frame: `Samples::new_rd` tables (film.rs:434,
    sampler.rs:18-37), per-pixel SmallRng scramble (film.rs:460-461) and the
    FilterImportanceSampler table (film.rs:429).  Built by the pure-CPU helpers of the C ABI."""

    def __init__(self, width, height, samples, integrator, filt=None, frame=1, first_sample=0):
        lib = L.host_lib()  # pure CPU: building frame inputs must not need (or map) the CUDA library
        filt = filt or BlackmanHarrisFilter(1.5)
        self.width, self.height, self.samples, self.spp, self.frame = width, height, samples, 4 * samples, frame
        self.first_sample = first_sample  # > 0: samples [first_sample, first_sample + spp) of the frame, for a later sample round
        self.sets_1d = 1 + integrator.requested_1d_sample_sets()  # film.rs:431
        self.sets_2d = 2 + integrator.requested_2d_sample_sets()  # film.rs:432
        self.samples_1d = np.empty(self.spp * self.sets_1d, np.float32)
        self.samples_2d = np.empty(2 * self.spp * self.sets_2d, np.float32)
        self.scramble = np.empty(width * height, np.float32)
        self.fis = np.empty(L.RAYN_FIS_TABLE_SIZE, np.float32)
        L.check(lib.rayn_b200_host_rd_tables_at(self.spp, self.sets_1d, self.sets_2d, frame, first_sample, _fptr(self.samples_1d),
                                                _fptr(self.samples_2d)))
        L.check(lib.rayn_b200_host_scramble(width, height, _fptr(self.scramble)))
        L.check(lib.rayn_b200_host_fis_blackman_harris(filt.radius, _fptr(self.fis)))

    def arrays(self):
        return self.samples_1d, self.samples_2d, self.scramble, self.fis


def make_frame_desc(width, height, tile_size, samples, integrator, frame, time_range, ptrs, space, tile_offset=0,
                    tile_stride=1, sets=None, tile_list=None):
    f = L.RaynFrameDesc()
    f.width, f.height = width, height
    f.tile_w, f.tile_h = tile_size
    f.samples = samples
    f.max_bounces = integrator.max_bounces
    f.volume_marches = integrator.volume_marches
    f.frame = frame
    f.t0, f.t1 = float(np.float32(time_range[0])), float(np.float32(time_range[1]))
    f.sets_1d, f.sets_2d = sets if sets else (1 + integrator.requested_1d_sample_sets(), 2 + integrator.requested_2d_sample_sets())
    f.samples_1d, f.samples_2d, f.scramble, f.fis_inverse_cdf = ptrs
    f.input_space = space
    f.tile_offset, f.tile_stride = tile_offset, tile_stride
    if tile_list is not None:  # explicit shard (ascending tile indices); the array must outlive the render call
        arr = (C.c_int32 * len(tile_list))(*tile_list)
        f.tile_list, f.n_tile_list = C.cast(arr, C.POINTER(C.c_int32)), len(tile_list)
        f._keep_tile_list = arr
    return f


# Picked by `tools/bench_denoise.py --pick-sigmas` (DESIGN.md §4b): the lowest col+bg MSE against a 256 spp film of a
# 4 spp config 3 film at 96x96, 5 levels, over a grid of 9 x 6 x 4 sigmas.
DENOISE_DEFAULTS = dict(sigma_color=2.5, sigma_normal=0.4, sigma_alpha=0.5)


# The albedo-guided filter (rayn_b200_film_denoise_albedo) and the albedo plane of a Film: picked by `tools/bench_albedo.py`
# (DESIGN.md §4e) on config 3 with the README palette at 96x96.  ALBEDO_SAMPLES caps the plane's samples (4 * ALBEDO_SAMPLES
# spp, the first camera samples of the film's own sequences): first-hit albedo converges much faster than colour.
DENOISE_ALBEDO_SIGMA = 0.2
ALBEDO_SAMPLES = 16

# The variance-guided filter (rayn_b200_film_denoise_variance): sigma_luminance and the sigma_color it is paired with, picked
# by `tools/bench_variance.py` (DESIGN.md §4f) on config 3 at 96x96, grey and with the README palette: the lowest mean col+bg
# MSE over 4, 16 and 64 spp films (0.35 and 0.33 of the unguided defaults' MSE, with the albedo guide).  The luminance term
# replaces the global colour term, so sigma_color is +inf.
DENOISE_LUMINANCE_SIGMA = 4.0
DENOISE_VARIANCE_SIGMA_COLOR = float("inf")
# Temporal accumulation (Film.render_sequence, rayn_b200_temporal_push): picked by `tools/bench_temporal.py` (DESIGN.md §4g) by
# the rule "lowest mean col+bg MSE over frames 9-24 of a 24-frame config-3 sequence with a moving camera, averaged over 4 and
# 16 spp", over a grid of alpha_min, sigma_depth and normal_cos.
# On one H100 80GB HBM3 (700 W, 1980 MHz): alpha_min 0.2, sigma_depth 0.1, normal_cos 0.5 gives 0.87x (4 spp) and 0.98x (16 spp) of
# the spatial-only MSE, with 0.81x / 0.94x of its flicker.
TEMPORAL_DEFAULTS = dict(alpha_min=0.2, sigma_depth=0.1, normal_cos=0.5)


def denoise_desc(iterations=5, sigma_color=None, sigma_normal=None, sigma_alpha=None):
    """RaynDenoiseDesc; a sigma left None takes its DENOISE_DEFAULTS value."""
    given = dict(sigma_color=sigma_color, sigma_normal=sigma_normal, sigma_alpha=sigma_alpha)
    s = {k: float(DENOISE_DEFAULTS[k] if v is None else v) for k, v in given.items()}
    return L.RaynDenoiseDesc(int(iterations), s["sigma_color"], s["sigma_normal"], s["sigma_alpha"])


# Adaptive sampling (Film.render_adaptive, rayn_b200_accum_round): a tile stops once its error E <= threshold.  Picked by
# `tools/bench_adaptive.py` (DESIGN.md §4c): the largest speedup over uniform rounds at equal col+bg MSE on config 3
# (1.12 at 0.025; thresholds of 0.04 and above lose to uniform rendering there).
ADAPTIVE_THRESHOLD = 0.025
ADAPTIVE_MAX_ROUNDS = 32


def adaptive_desc(min_rounds=2, max_rounds=ADAPTIVE_MAX_ROUNDS, threshold=ADAPTIVE_THRESHOLD):
    return L.RaynAdaptiveDesc(int(min_rounds), int(max_rounds), float(threshold))


def tile_grid(width, height, tile_w, tile_h):
    nx, ny = C.c_int32(), C.c_int32()
    L.check(L.host_lib().rayn_b200_host_tile_grid(width, height, tile_w, tile_h, C.byref(nx), C.byref(ny)))
    return nx.value, ny.value


class Accum:
    """One device film accumulator (include/rayn_b200.h: rayn_b200_accum_*), made by Renderer.accum_create."""

    def __init__(self, renderer, width, height, tile_size):
        self._lib = renderer._lib
        self.width, self.height = width, height
        self.tile_size = tuple(tile_size)
        self.n_tiles_x, self.n_tiles_y = tile_grid(width, height, *self.tile_size)
        self.n_tiles = self.n_tiles_x * self.n_tiles_y
        self._h = C.c_void_p()
        L.check(self._lib.rayn_b200_accum_create(renderer.ctx, width, height, self.tile_size[0], self.tile_size[1], C.byref(self._h)),
                renderer.ctx)

    @property
    def handle(self):
        return self._h

    def close(self):
        if self._h:
            self._lib.rayn_b200_accum_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Temporal:
    """The reprojectable history of one film (include/rayn_b200.h: rayn_b200_temporal_*), made by Renderer.temporal_create."""

    def __init__(self, renderer, width, height):
        self._lib = renderer._lib
        self.width, self.height = width, height
        self._h = C.c_void_p()
        L.check(self._lib.rayn_b200_temporal_create(renderer.ctx, width, height, C.byref(self._h)), renderer.ctx)

    @property
    def handle(self):
        return self._h

    def close(self):
        if self._h:
            self._lib.rayn_b200_temporal_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Renderer:
    """Owns one RaynContext (one GPU)."""

    def __init__(self, device=0, max_paths_per_pass=0, flags=0):
        self._lib = L.lib()
        cfg = L.RaynConfig(device, max_paths_per_pass, flags)
        self._ctx = C.c_void_p()
        L.check(self._lib.rayn_b200_create(C.byref(cfg), C.byref(self._ctx)))
        self._keep = None
        self.device = device

    def close(self):
        if self._ctx:
            self._lib.rayn_b200_destroy(self._ctx)
            self._ctx = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def ctx(self):
        return self._ctx

    def upload_scene(self, world, camera, time_range=None):
        """Uploads the scene, then its orbit-trap albedos (OrbitTrapAlbedo materials), if it has any.  time_range: the (t0, t1)
        of the renders that follow, required if the scene has closure parameters (each is uploaded as its chord over it,
        Linear.chord).  Returns World.flatten's (RaynSceneDesc, keepalive), e.g. the `prev` of the next frame's
        render_motion."""
        desc, keep = world.flatten(camera, time_range)
        self._keep = (desc, keep)
        L.check(self._lib.rayn_b200_upload_scene(self._ctx, C.byref(desc)), self._ctx)
        traps = world.albedo_traps()
        if traps:
            self.set_albedo_traps(traps)
        return desc, keep

    def set_albedo_traps(self, traps):
        """Replaces the orbit-trap list of the uploaded scene (include/rayn_b200.h: rayn_b200_set_albedo_traps): a list of
        RaynAlbedoTrap, e.g. World.albedo_traps(); [] clears it."""
        arr = (L.RaynAlbedoTrap * max(len(traps), 1))(*traps)
        L.check(self._lib.rayn_b200_set_albedo_traps(self._ctx, len(traps), arr), self._ctx)

    def upload_scene_desc(self, desc):
        L.check(self._lib.rayn_b200_upload_scene(self._ctx, C.byref(desc)), self._ctx)

    def render(self, frame_desc, planes):
        L.check(self._lib.rayn_b200_render_frame(self._ctx, C.byref(frame_desc), C.byref(planes)), self._ctx)

    def stats(self):
        s = L.RaynStats()
        L.check(self._lib.rayn_b200_get_stats(self._ctx, C.byref(s)), self._ctx)
        return s

    def render_host(self, inputs, tile_size, integrator, time_range, tile_offset=0, tile_stride=1, tile_list=None, moments=False):
        """Host buffers in, host planes out (H2D + D2H inside the call).  Returns dict of numpy planes.  moments=True: the
        same render with its luminance second moments (include/rayn_b200.h: rayn_b200_render_frame_moments), returned as
        "moments", float32 [H, W, 2] (color_lum2, background_lum2)."""
        w, h = inputs.width, inputs.height
        planes, p = host_planes(w, h)
        ptrs = tuple(a.ctypes.data for a in inputs.arrays())
        f = make_frame_desc(w, h, tile_size, inputs.samples, integrator, inputs.frame, time_range, ptrs, L.MEM_HOST, tile_offset,
                            tile_stride, (inputs.sets_1d, inputs.sets_2d), tile_list)
        if not moments:
            self.render(f, p)
            return planes
        m = np.zeros((2, h * w), np.float32)
        mp = L.RaynMomentPlanes(m[0].ctypes.data, m[1].ctypes.data, L.MEM_HOST)
        L.check(self._lib.rayn_b200_render_frame_moments(self._ctx, C.byref(f), C.byref(p), C.byref(mp)), self._ctx)
        planes["moments"] = np.ascontiguousarray(m.reshape(2, h, w).transpose(1, 2, 0))
        return planes

    def render_albedo(self, inputs, tile_size, integrator, time_range):
        """First-hit albedo plane of the uploaded scene (include/rayn_b200.h: rayn_b200_render_albedo) for host FrameInputs:
        float32 [H, W, 3]."""
        return self._first_hit(inputs, tile_size, integrator, time_range, None, True, None)[1]

    def render_motion(self, inputs, tile_size, integrator, time_range, frame_dt, albedo=False, prev=None):
        """First-hit motion plane of the uploaded scene (include/rayn_b200.h: rayn_b200_render_motion) for host FrameInputs:
        float32 [H, W, 4] (dx, dy, z, z_prev); albedo=True: (motion, render_albedo's [H, W, 3] plane from the same pass).
        prev: the RaynSceneDesc the previous frame was rendered with (World.flatten's or upload_scene's, its keepalive still
        held): the motion against that scene instead of the uploaded one run backwards (rayn_b200_render_motion_prev)."""
        motion, alb = self._first_hit(inputs, tile_size, integrator, time_range, frame_dt, albedo, prev)
        return (motion, alb) if albedo else motion

    def _first_hit(self, inputs, tile_size, integrator, time_range, frame_dt, albedo, prev):
        """One first-hit pass: (motion [H, W, 4] or None, albedo [H, W, 3] or None).  frame_dt None: the albedo pass
        (rayn_b200_render_albedo); else render_motion, or render_motion_prev against prev."""
        w, h = inputs.width, inputs.height
        motion = None if frame_dt is None else np.zeros((h, w, 4), np.float32)
        alb = np.zeros((h, w, 3), np.float32) if albedo else None
        ptrs = tuple(a.ctypes.data for a in inputs.arrays())
        f = make_frame_desc(w, h, tile_size, inputs.samples, integrator, inputs.frame, time_range, ptrs, L.MEM_HOST,
                            sets=(inputs.sets_1d, inputs.sets_2d))
        m_ptr, a_ptr = (None if a is None else a.ctypes.data for a in (motion, alb))
        if frame_dt is None:
            rc = self._lib.rayn_b200_render_albedo(self._ctx, C.byref(f), a_ptr, L.MEM_HOST)
        elif prev is None:
            rc = self._lib.rayn_b200_render_motion(self._ctx, C.byref(f), float(frame_dt), m_ptr, a_ptr, L.MEM_HOST)
        else:
            rc = self._lib.rayn_b200_render_motion_prev(self._ctx, C.byref(f), float(frame_dt), C.byref(prev), m_ptr, a_ptr, L.MEM_HOST)
        L.check(rc, self._ctx)
        return motion, alb

    def temporal_create(self, width, height):
        return Temporal(self, width, height)

    def temporal_push(self, t, planes, moments, motion, alpha_min, sigma_depth, normal_cos, reset=False):
        """Blends one frame into the history t (include/rayn_b200.h: rayn_b200_temporal_push).  planes: numpy "color",
        "background" and "normal"; moments float32 [H, W, 2]; motion float32 [H, W, 4] (render_motion's).  Returns
        (planes with new "color" / "background", moments [H, W, 2], var_scale [H, W]) as float32 arrays."""
        w, h = t.width, t.height
        flat = {k: np.ascontiguousarray(planes[k], np.float32).reshape(-1) for k in ("color", "background", "normal")}
        m = np.ascontiguousarray(np.asarray(moments, np.float32).reshape(h, w, 2).transpose(2, 0, 1)).reshape(2, -1)
        mv = np.ascontiguousarray(motion, np.float32).reshape(-1)
        oc, ob = np.empty_like(flat["color"]), np.empty_like(flat["background"])
        om, scale = np.empty_like(m), np.empty(w * h, np.float32)
        pin = L.RaynFilmPlanes(flat["color"].ctypes.data, None, flat["background"].ctypes.data, flat["normal"].ctypes.data, L.MEM_HOST)
        pout = L.RaynFilmPlanes(oc.ctypes.data, None, ob.ctypes.data, None, L.MEM_HOST)
        mi = L.RaynMomentPlanes(m[0].ctypes.data, m[1].ctypes.data, L.MEM_HOST)
        mo = L.RaynMomentPlanes(om[0].ctypes.data, om[1].ctypes.data, L.MEM_HOST)
        d = L.RaynTemporalDesc(float(alpha_min), float(sigma_depth), float(normal_cos), 1 if reset else 0)
        L.check(self._lib.rayn_b200_temporal_push(self._ctx, t.handle, C.byref(d), C.byref(pin), C.byref(mi), mv.ctypes.data, C.byref(pout),
                                                  C.byref(mo), scale.ctypes.data), self._ctx)
        out = {"color": oc.reshape(np.shape(planes["color"])), "background": ob.reshape(np.shape(planes["background"]))}
        return out, np.ascontiguousarray(om.reshape(2, h, w).transpose(1, 2, 0)), scale.reshape(h, w)

    def postprocess(self, mode, width, height, planes):
        """Film::save_to pixel arithmetic on the device (film.rs:205-377): numpy planes in, uint8 [H, W, bpp] out (rows top to bottom)."""
        def ptr(k):
            return planes[k].ctypes.data if planes.get(k) is not None else None
        p = L.RaynFilmPlanes(ptr("color"), ptr("alpha"), ptr("background"), ptr("normal"), L.MEM_HOST)
        out = np.zeros((height, width, L.POST_BYTES[mode]), np.uint8)
        L.check(self._lib.rayn_b200_film_postprocess(self._ctx, mode, width, height, C.byref(p), out.ctypes.data, L.MEM_HOST), self._ctx)
        return out

    def denoise(self, width, height, planes, iterations=5, sigma_color=None, sigma_normal=None, sigma_alpha=None, albedo=None,
                sigma_albedo=None, moments=None, spp=None, sigma_luminance=None, var_scale=None):
        """Edge-avoiding a-trous filter of the color and background planes (include/rayn_b200.h: rayn_b200_film_denoise).
        numpy planes in ("normal" and "alpha" required, "color" / "background" optional); returns new arrays for the
        colour planes given, shaped like their inputs.  Sigmas default to DENOISE_DEFAULTS; +inf disables a term.
        albedo (a [3*W*H] plane, e.g. render_albedo's): the albedo-guided filter (rayn_b200_film_denoise_albedo) with
        sigma_albedo, default DENOISE_ALBEDO_SIGMA.  moments (float32 [H, W, 2], render_host(moments=True)'s) with the film's
        spp: the variance-guided filter (rayn_b200_film_denoise_variance) with sigma_luminance, default
        DENOISE_LUMINANCE_SIGMA, and sigma_color defaulting to DENOISE_VARIANCE_SIGMA_COLOR; combinable with albedo.
        var_scale (float32 [H, W], temporal_push's), with moments: rayn_b200_film_denoise_variance_scaled."""
        for k in ("normal", "alpha"):
            if planes.get(k) is None:
                raise ValueError(f"denoise needs the {k} guide plane")
        flat = {k: np.ascontiguousarray(v, np.float32).reshape(-1) for k, v in planes.items() if v is not None}
        outs = {k: np.empty_like(flat[k]) for k in ("color", "background") if k in flat}

        def ptr(d, k):
            return d[k].ctypes.data if k in d else None
        pin = L.RaynFilmPlanes(ptr(flat, "color"), ptr(flat, "alpha"), ptr(flat, "background"), ptr(flat, "normal"), L.MEM_HOST)
        pout = L.RaynFilmPlanes(ptr(outs, "color"), None, ptr(outs, "background"), None, L.MEM_HOST)
        if moments is not None and spp is None:
            raise ValueError("the variance-guided denoise needs the film's spp")
        if moments is not None and sigma_color is None:
            sigma_color = DENOISE_VARIANCE_SIGMA_COLOR
        desc = denoise_desc(iterations, sigma_color, sigma_normal, sigma_alpha)
        sa = float(DENOISE_ALBEDO_SIGMA if sigma_albedo is None else sigma_albedo)
        if moments is not None:
            m = np.ascontiguousarray(np.asarray(moments, np.float32).reshape(height, width, 2).transpose(2, 0, 1)).reshape(2, -1)
            mp = L.RaynMomentPlanes(m[0].ctypes.data, m[1].ctypes.data, L.MEM_HOST)
            sl = float(DENOISE_LUMINANCE_SIGMA if sigma_luminance is None else sigma_luminance)
            alb = None if albedo is None else np.ascontiguousarray(albedo, np.float32).reshape(-1)
            alb_p = None if alb is None else alb.ctypes.data
            if var_scale is None:
                L.check(self._lib.rayn_b200_film_denoise_variance(self._ctx, C.byref(desc), sl, int(spp), C.byref(mp), sa, alb_p, width, height,
                                                                  C.byref(pin), C.byref(pout)), self._ctx)
            else:
                vs = np.ascontiguousarray(var_scale, np.float32).reshape(-1)
                L.check(self._lib.rayn_b200_film_denoise_variance_scaled(self._ctx, C.byref(desc), sl, int(spp), C.byref(mp), vs.ctypes.data, sa,
                                                                         alb_p, width, height, C.byref(pin), C.byref(pout)), self._ctx)
        elif var_scale is not None:
            raise ValueError("var_scale scales the variance of the moments: pass moments too")
        elif albedo is None:
            L.check(self._lib.rayn_b200_film_denoise(self._ctx, C.byref(desc), width, height, C.byref(pin), C.byref(pout)), self._ctx)
        else:
            alb = np.ascontiguousarray(albedo, np.float32).reshape(-1)
            L.check(self._lib.rayn_b200_film_denoise_albedo(self._ctx, C.byref(desc), sa, alb.ctypes.data, width, height, C.byref(pin),
                                                            C.byref(pout)), self._ctx)
        return {k: v.reshape(np.shape(planes[k])) for k, v in outs.items()}

    # ---- progressive / adaptive rendering (rayn_b200_accum_*) ----
    def accum_create(self, width, height, tile_size):
        return Accum(self, width, height, tile_size)

    def accum_round(self, acc, frame_desc, min_rounds=2, max_rounds=ADAPTIVE_MAX_ROUNDS, threshold=ADAPTIVE_THRESHOLD):
        """Renders the active tiles of `acc` with `frame_desc` and folds them in; returns how many tiles rendered (0: all
        have stopped).  frame_desc's tables must hold the samples the active tiles have not seen: first_sample = their
        `samples` in accum_tiles."""
        d = adaptive_desc(min_rounds, max_rounds, threshold)
        n = C.c_int32(0)
        L.check(self._lib.rayn_b200_accum_round(self._ctx, acc.handle, C.byref(frame_desc), C.byref(d), C.byref(n)), self._ctx)
        return n.value

    def accum_tiles(self, acc):
        """(E float64, samples per pixel int64) per tile, indexed by tile_x * n_tiles_y + tile_y."""
        err, spp = np.empty(acc.n_tiles, np.float64), np.empty(acc.n_tiles, np.int64)
        L.check(self._lib.rayn_b200_accum_tiles(self._ctx, acc.handle, err.ctypes.data_as(C.POINTER(C.c_double)),
                                                spp.ctypes.data_as(C.POINTER(C.c_int64))), self._ctx)
        return err, spp

    def accum_resolve(self, acc, out=None):
        """The accumulated film.  out=None: returns new host planes (dict, like render_host); else `out` is a RaynFilmPlanes
        (host or device) written in place."""
        planes = None
        if out is None:
            planes, out = host_planes(acc.width, acc.height)
        L.check(self._lib.rayn_b200_accum_resolve(self._ctx, acc.handle, C.byref(out)), self._ctx)
        return planes

    # ---- known-answer entry points (tests) ----
    def kat_detmath(self, op, a, b=None):
        a = np.ascontiguousarray(a, np.float32)
        b = np.ascontiguousarray(b if b is not None else a, np.float32)
        out = np.empty_like(a)
        L.check(self._lib.rayn_b200_kat_detmath(self._ctx, op, a.size, _fptr(a), _fptr(b), _fptr(out)), self._ctx)
        return out

    def kat_sdf_dist(self, hitable, points):
        p = np.ascontiguousarray(points, np.float32).reshape(-1, 3)
        out = np.empty(len(p), np.float32)
        L.check(self._lib.rayn_b200_kat_sdf_dist(self._ctx, C.byref(hitable), len(p), _fptr(p), _fptr(out)), self._ctx)
        return out

    def kat_sdf_dist2(self, hitable, points, variant=-1):
        p = np.ascontiguousarray(points, np.float32).reshape(-1, 3)
        out = np.empty(len(p), np.float32)
        L.check(self._lib.rayn_b200_kat_sdf_dist2(self._ctx, C.byref(hitable), variant, len(p), _fptr(p), _fptr(out)), self._ctx)
        return out

    def kat_sdf_trap(self, hitable, points):
        """orbit trap per point on the device (the function k_normals evaluates for trap materials)"""
        p = np.ascontiguousarray(points, np.float32).reshape(-1, 3)
        out = np.empty(len(p), np.float32)
        L.check(self._lib.rayn_b200_kat_sdf_trap(self._ctx, C.byref(hitable), len(p), _fptr(p), _fptr(out)), self._ctx)
        return out

    def kat_fastdiv(self, num, first_bits, n):
        bad = C.c_int64(-1)
        L.check(self._lib.rayn_b200_kat_fastdiv(self._ctx, num, first_bits, n, C.byref(bad)), self._ctx)
        return bad.value

    def kat_sdf_hit(self, hitable, consts, origins, dirs, t_max, thr_scale, thr_const=0):
        o = np.ascontiguousarray(origins, np.float32).reshape(-1, 3)
        d = np.ascontiguousarray(dirs, np.float32).reshape(-1, 3)
        tm = np.ascontiguousarray(t_max, np.float32)
        out = np.empty(len(o), np.float32)
        L.check(self._lib.rayn_b200_kat_sdf_hit(self._ctx, C.byref(hitable), C.byref(consts), len(o), _fptr(o), _fptr(d), _fptr(tm),
                                                thr_scale, thr_const, _fptr(out)), self._ctx)
        return out

    def kat_occluded(self, start, end):
        s = np.ascontiguousarray(start, np.float32).reshape(-1, 3)
        e = np.ascontiguousarray(end, np.float32).reshape(-1, 3)
        out = np.empty(len(s), np.float32)
        L.check(self._lib.rayn_b200_kat_occluded(self._ctx, len(s), _fptr(s), _fptr(e), _fptr(out)), self._ctx)
        return out

    def kat_closest_hit(self, depth, origins, dirs):
        o = np.ascontiguousarray(origins, np.float32).reshape(-1, 3)
        d = np.ascontiguousarray(dirs, np.float32).reshape(-1, 3)
        t = np.empty(len(o), np.float32)
        obj = np.empty(len(o), np.int32)
        L.check(self._lib.rayn_b200_kat_closest_hit(self._ctx, depth, len(o), _fptr(o), _fptr(d), _fptr(t),
                                                    obj.ctypes.data_as(C.POINTER(C.c_int32))), self._ctx)
        return t, obj

    def kat_light_sample(self, light, s0, s1, p):
        s0, s1 = np.ascontiguousarray(s0, np.float32), np.ascontiguousarray(s1, np.float32)
        p = np.ascontiguousarray(p, np.float32).reshape(-1, 3)
        pt, pdf = np.empty_like(p), np.empty(len(p), np.float32)
        L.check(self._lib.rayn_b200_kat_light_sample(self._ctx, C.byref(light), len(p), _fptr(s0), _fptr(s1), _fptr(p), _fptr(pt), _fptr(pdf)), self._ctx)
        return pt, pdf

    def kat_light_sample_volume(self, light, sample, o, d, t_max):
        sample, t_max = np.ascontiguousarray(sample, np.float32), np.ascontiguousarray(t_max, np.float32)
        o, d = np.ascontiguousarray(o, np.float32).reshape(-1, 3), np.ascontiguousarray(d, np.float32).reshape(-1, 3)
        t, pdf = np.empty(len(o), np.float32), np.empty(len(o), np.float32)
        L.check(self._lib.rayn_b200_kat_light_sample_volume(self._ctx, C.byref(light), len(o), _fptr(sample), _fptr(o), _fptr(d), _fptr(t_max),
                                                            _fptr(t), _fptr(pdf)), self._ctx)
        return t, pdf

    def kat_bsdf(self, mat, normals, wo, s1d, u4):
        n3, w3 = np.ascontiguousarray(normals, np.float32).reshape(-1, 3), np.ascontiguousarray(wo, np.float32).reshape(-1, 3)
        s1d, u4 = np.ascontiguousarray(s1d, np.float32), np.ascontiguousarray(u4, np.float32).reshape(-1, 4)
        wi, f, fe, pdf = np.empty_like(n3), np.empty_like(n3), np.empty_like(n3), np.empty(len(n3), np.float32)
        L.check(self._lib.rayn_b200_kat_bsdf(self._ctx, C.byref(mat), len(n3), _fptr(n3), _fptr(w3), _fptr(s1d), _fptr(u4), _fptr(wi), _fptr(f),
                                             _fptr(pdf), _fptr(fe)), self._ctx)
        return wi, f, pdf, fe

    def sdf_variant(self, hitable_index):
        """march-kernel specialisation upload_scene selected for a hitable (include/rayn_b200.h: rayn_b200_debug_sdf_variant)"""
        return int(self._lib.rayn_b200_debug_sdf_variant(self._ctx, hitable_index))

    def enable_queue_log(self, on=True):
        L.check(self._lib.rayn_b200_debug_enable_queue_log(self._ctx, 1 if on else 0), self._ctx)

    def read_queue_log(self):
        n = self._lib.rayn_b200_debug_read_queue_log(self._ctx, None, 0)
        out = np.empty(max(n, 1), np.int32)
        self._lib.rayn_b200_debug_read_queue_log(self._ctx, out.ctypes.data_as(C.POINTER(C.c_int32)), n)
        return out[:n]


class Film:
    """film.rs:175-203.  Channel planes are numpy arrays, row-major, y up, already / spp."""

    def __init__(self, channels, res, device=0):
        if len(set(channels)) != len(channels):
            raise ValueError("Attempted to create multiple channels of one kind")  # film.rs:187-189
        for c in channels:
            if c not in FILM_CHANNELS:
                raise ValueError(f"unknown channel {c}")
        self.channel_kinds = tuple(channels)
        self.res = (int(res[0]), int(res[1]))
        self.channels = {}
        self.progressive_epoch = 0
        self._renderer = None
        self._device = device
        self.last_stats = None
        self.spp = None  # samples per pixel of the last render_frame_into (the "moments" channel's count)

    def render_frame_into(self, world, camera, integrator, filt, tile_size, frame, time_range, samples):
        """Drop-in for film.rs:382-395.  time_range = (start, end)."""
        if self._renderer is None:
            self._renderer = Renderer(self._device)
        w, h = self.res
        inputs = FrameInputs(w, h, samples, integrator, filt, frame)
        self._renderer.upload_scene(world, camera, time_range)
        planes = self._renderer.render_host(inputs, tile_size, integrator, time_range, moments="moments" in self.channel_kinds)
        self.last_stats = self._renderer.stats()
        self.spp = inputs.spp
        for k in self.channel_kinds:
            if k == "moments":
                self.channels[k] = planes[k]
            elif k not in ("albedo", "motion"):  # "motion" is filled by render_sequence
                self.channels[k] = planes[k].reshape((h, w, 3) if k != "alpha" else (h, w))
        self._render_albedo(integrator, filt, tile_size, frame, time_range, samples)
        self.progressive_epoch += 1  # film.rs:657

    def _render_albedo(self, integrator, filt, tile_size, frame, time_range, samples):
        """Fills the "albedo" channel, if the Film has one: one render_albedo call with the frame's seed and the first
        4 * min(samples, ALBEDO_SAMPLES) camera samples of its sequences."""
        if "albedo" not in self.channel_kinds:
            return
        w, h = self.res
        inputs = FrameInputs(w, h, min(samples, ALBEDO_SAMPLES), integrator, filt, frame)
        self.channels["albedo"] = self._renderer.render_albedo(inputs, tile_size, integrator, time_range)

    def render_adaptive(self, world, camera, integrator, filt, tile_size, frame, time_range, samples_per_round, min_rounds=2,
                        max_rounds=ADAPTIVE_MAX_ROUNDS, threshold=ADAPTIVE_THRESHOLD, on_round=None):
        """Progressive render in rounds of 4 * samples_per_round spp: every 16x16 (tile_size) tile keeps rendering until its
        error E <= threshold (after at least min_rounds, at most max_rounds rounds; include/rayn_b200.h: accum_round).
        A negative threshold renders every tile max_rounds times (uniform progressive rendering).  Fills self.channels
        like render_frame_into and sets self.tile_errors / self.tile_samples (per tile index tile_x * n_tiles_y + tile_y).
        on_round(film), if given, sees the film resolved after every round: a progressive preview.  Returns the number of
        rounds rendered."""
        if "moments" in self.channel_kinds:
            raise ValueError("render_adaptive does not fold luminance moments: use render_frame_into for a Film with \"moments\"")
        if "motion" in self.channel_kinds:
            raise ValueError("render_adaptive renders no motion plane: use render_sequence for a Film with \"motion\"")
        import torch  # device buffers for the sample tables and the scramble plane
        if self._renderer is None:
            self._renderer = Renderer(self._device)
        r, lib = self._renderer, self._renderer._lib
        w, h = self.res
        spp = 4 * samples_per_round
        sets = (1 + integrator.requested_1d_sample_sets(), 2 + integrator.requested_2d_sample_sets())  # film.rs:431-432
        r.upload_scene(world, camera, time_range)
        dev = torch.device("cuda", r.device)
        s1 = torch.empty(spp * sets[0], dtype=torch.float32, device=dev)
        s2 = torch.empty(2 * spp * sets[1], dtype=torch.float32, device=dev)
        scr = torch.empty(w * h, dtype=torch.float32, device=dev)
        fis_h = np.empty(L.RAYN_FIS_TABLE_SIZE, np.float32)
        L.check(L.host_lib().rayn_b200_host_fis_blackman_harris((filt or BlackmanHarrisFilter(1.5)).radius, _fptr(fis_h)))
        fis = torch.from_numpy(fis_h).to(dev)
        torch.cuda.synchronize(dev)
        L.check(lib.rayn_b200_device_frame_inputs(r.ctx, w, h, spp, 0, 0, frame, None, None, scr.data_ptr()), r.ctx)
        ptrs = (s1.data_ptr(), s2.data_ptr(), scr.data_ptr(), fis.data_ptr())
        f = make_frame_desc(w, h, tile_size, samples_per_round, integrator, frame, time_range, ptrs, L.MEM_DEVICE, sets=sets)
        acc = r.accum_create(w, h, tile_size)
        rounds, first = 0, 0
        try:
            while True:
                # every active tile has seen samples [0, first): this round renders the next spp of the same sequences
                L.check(lib.rayn_b200_device_rd_tables_at(r.ctx, spp, sets[0], sets[1], frame, first, s1.data_ptr(), s2.data_ptr()), r.ctx)
                if r.accum_round(acc, f, min_rounds, max_rounds, threshold) == 0:
                    break
                rounds += 1
                first += spp
                self.last_stats = r.stats()
                if on_round is not None:
                    self._take_accum(r, acc)
                    on_round(self)
            if on_round is None and rounds > 0:
                self._take_accum(r, acc)
        finally:
            acc.close()
        self._render_albedo(integrator, filt, tile_size, frame, time_range, samples_per_round * max_rounds)
        return rounds

    def _take_accum(self, r, acc):
        w, h = self.res
        planes = r.accum_resolve(acc)
        for k in self.channel_kinds:
            if k != "albedo":
                self.channels[k] = planes[k].reshape((h, w, 3) if k != "alpha" else (h, w))
        self.tile_errors, self.tile_samples = r.accum_tiles(acc)
        self.progressive_epoch += 1  # film.rs:657

    def render_sequence(self, world, camera, integrator, filt, tile_size, frames, frame_rate, shutter, samples, iterations=5, on_frame=None,
                        alpha_min=None, sigma_depth=None, normal_cos=None):
        """Renders and denoises a frame sequence with temporal accumulation, like main.rs:58-97's frame loop: frame k covers
        (k / frame_rate, k / frame_rate + shutter).  Per frame: a render with luminance moments; one motion pass (frame_dt =
        1 / frame_rate) whose depth-0 march also gives the albedo plane if the Film has "albedo" (the first
        4 * min(samples, ALBEDO_SAMPLES) samples, as render_frame_into's); the push into a film history (reset on the first
        frame); the variance-guided denoise of the blend with its per-pixel variance scale; then on_frame(film).  The
        temporal parameters default to TEMPORAL_DEFAULTS.  self.channels holds the denoised colour and background and the
        frame's alpha, normal, albedo and motion planes (the ones the Film has).  Returns the number of frames.

        A world with closure parameters (World.has_closures: a sphere on a curved path, an orbiting camera) is uploaded
        before every frame as its chord over that frame's time range, and every frame after the first measures its motion
        against the scene the previous frame was rendered with (Renderer.render_motion(prev=...)).  Any other world is
        uploaded once and its motion is the uploaded scene run backwards."""
        if "moments" in self.channel_kinds:
            raise ValueError("render_sequence consumes the moments of every frame: create the Film without \"moments\"")
        for k in ("color", "background", "alpha", "normal"):
            if k not in self.channel_kinds:
                raise ValueError(f"render_sequence needs the {k} channel")
        t_kw = {k: float(TEMPORAL_DEFAULTS[k] if v is None else v)
                for k, v in dict(alpha_min=alpha_min, sigma_depth=sigma_depth, normal_cos=normal_cos).items()}
        animated = world.has_closures(camera)
        if self._renderer is None:
            self._renderer = Renderer(self._device)
        r = self._renderer
        w, h = self.res
        frame_dt = float(np.float32(1.0) / np.float32(frame_rate))
        hist = r.temporal_create(w, h)
        n, prev, scene = 0, None, None
        try:
            if not animated:
                r.upload_scene(world, camera)
            for k in frames:
                start = np.float32(k) * np.float32(frame_dt)
                time_range = (float(start), float(start + np.float32(shutter)))
                if animated:
                    prev, scene = scene, r.upload_scene(world, camera, time_range)
                inputs = FrameInputs(w, h, samples, integrator, filt, k)
                planes = r.render_host(inputs, tile_size, integrator, time_range, moments=True)
                self.last_stats = r.stats()
                self.spp = inputs.spp
                g_inputs = FrameInputs(w, h, min(samples, ALBEDO_SAMPLES), integrator, filt, k)
                albedo = None
                p_desc = None if prev is None else prev[0]  # None on the first frame, which resets the history
                if "albedo" in self.channel_kinds:
                    motion, albedo = r.render_motion(g_inputs, tile_size, integrator, time_range, frame_dt, albedo=True, prev=p_desc)
                else:
                    motion = r.render_motion(g_inputs, tile_size, integrator, time_range, frame_dt, prev=p_desc)
                blend, moments, scale = r.temporal_push(hist, planes, planes["moments"], motion, reset=(n == 0), **t_kw)
                guides = {"color": blend["color"], "background": blend["background"], "alpha": planes["alpha"], "normal": planes["normal"]}
                out = r.denoise(w, h, guides, iterations, albedo=None if albedo is None else albedo.reshape(-1), moments=moments,
                                spp=inputs.spp, var_scale=scale)
                self.channels = {"color": out["color"].reshape(h, w, 3), "background": out["background"].reshape(h, w, 3),
                                 "alpha": planes["alpha"].reshape(h, w), "normal": planes["normal"].reshape(h, w, 3)}
                if albedo is not None:
                    self.channels["albedo"] = albedo
                if "motion" in self.channel_kinds:
                    self.channels["motion"] = motion
                self.progressive_epoch += 1
                n += 1
                if on_frame is not None:
                    on_frame(self)
        finally:
            hist.close()
        return n

    def save_to(self, write_channels, output_folder, base_name, transparent_background=False):
        """film.rs:205-377.  Same channel semantics and file names as the reference; the pixel arithmetic runs on the
        device (`rayn_b200_film_postprocess`), the PNG encoding stays host I/O (PIL)."""
        import os
        from PIL import Image
        os.makedirs(output_folder, exist_ok=True)
        w, h = self.res
        flat = {k: np.ascontiguousarray(v, np.float32).reshape(-1) for k, v in self.channels.items()}
        written = []
        for kind in write_channels:
            if kind in ("moments", "motion"):
                raise ValueError(f"the {kind} channel is not an image: read Film.channels[\"{kind}\"]")
            if kind == "color":
                if transparent_background and "color" in flat and "alpha" in flat:
                    mode, pil = L.POST_COLOR_ALPHA, "RGBA"
                elif not transparent_background and "color" in flat and "background" in flat:
                    mode, pil = L.POST_COLOR_PLUS_BACKGROUND, "RGB"
                elif not transparent_background and "color" in flat:
                    mode, pil = L.POST_COLOR_ONLY, "RGB"
                else:
                    raise ValueError("Attempted to write Color channel with insufficient channels")  # film.rs:294-298
            elif kind in ("background", "normal", "alpha", "albedo"):
                if kind not in flat:
                    raise ValueError(f"Attempted to write {kind} channel but it didn't exist")
                mode, pil = {"background": (L.POST_BACKGROUND, "RGB"), "normal": (L.POST_WORLD_NORMAL, "RGB"), "alpha": (L.POST_ALPHA, "L"),
                             "albedo": (L.POST_BACKGROUND, "RGB")}[kind]
            else:
                raise ValueError(kind)
            # the albedo plane is written with the background's arithmetic (saturate, gamma 2.2)
            px = self._renderer.postprocess(mode, w, h, {"background": flat["albedo"]} if kind == "albedo" else flat)
            path = os.path.join(output_folder, f"{base_name}_{kind}.png")
            Image.fromarray(px[:, :, 0] if pil == "L" else px, pil).save(path)
            written.append(path)
        return written

    def denoise(self, iterations=5, sigma_color=None, sigma_normal=None, sigma_alpha=None, sigma_albedo=None, sigma_luminance=None):
        """Filters the Film's color and background channels in place (Renderer.denoise), guided by its normal and alpha
        channels, by its albedo channel if it has one (sigma_albedo, default DENOISE_ALBEDO_SIGMA), and by each pixel's
        variance if it has the moments channel (sigma_luminance, default DENOISE_LUMINANCE_SIGMA).  Call it after
        render_frame_into and before save_to.  The moments describe the unfiltered render, so the variance-guided filter
        removes the "moments" channel from self.channels (a later call filters without it; render_frame_into fills it
        again)."""
        for k in ("normal", "alpha"):
            if k not in self.channels:
                raise ValueError(f"Film.denoise needs the {k} channel")
        if self._renderer is None:
            self._renderer = Renderer(self._device)
        w, h = self.res
        if "moments" in self.channels:
            self.channels.update(self._renderer.denoise(w, h, {k: self.channels.get(k) for k in CHANNELS}, iterations, sigma_color,
                                                        sigma_normal, sigma_alpha, albedo=self.channels.get("albedo"),
                                                        sigma_albedo=sigma_albedo, moments=self.channels["moments"], spp=self.spp,
                                                        sigma_luminance=sigma_luminance))
            del self.channels["moments"]  # M - lum(c)^2 of filtered colour is not the variance of anything
        elif "albedo" in self.channels:
            self.channels.update(self._renderer.denoise(w, h, self.channels, iterations, sigma_color, sigma_normal, sigma_alpha,
                                                        albedo=self.channels["albedo"], sigma_albedo=sigma_albedo))
        else:
            self.channels.update(self._renderer.denoise(w, h, self.channels, iterations, sigma_color, sigma_normal, sigma_alpha))

    def tonemapped_rgb8(self):
        """The display formula of save_to (film.rs:253-267): (color + background).saturated().gamma(2.2), y flipped."""
        col = self.channels["color"] + self.channels.get("background", 0.0)
        rgb = np.clip(col, 0.0, 1.0) ** (1.0 / 2.2)
        return (np.clip(rgb * 255.0, 0, 255).astype(np.uint8))[::-1]
