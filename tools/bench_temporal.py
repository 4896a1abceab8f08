"""Measures the temporal accumulation of DESIGN.md §4g on one GPU: the quality study TEMPORAL_DEFAULTS was picked from, and the
cost of the motion pass, k_temporal and the scaled variance denoise.

    python tools/bench_temporal.py [--quality] [--cost] [--reps 3]

Quality: a 24-frame config-3 sequence at 96x96 (frames 1..24, frame k over (k/24, k/24 + 1/24) as main.rs) with a moving
camera: the origin moves at 0.6 units/s along the camera's right axis and the look-at point pans at 0.3 units/s the same way.
At 4 and 16 spp every frame is filtered (5 levels, no albedo guide) by the spatial variance denoise alone (the §4f defaults) and
by temporal push + scaled variance denoise over alpha_min in {0.1, 0.2, 0.4} x sigma_depth in {0.02, 0.1} x normal_cos in
{0.5, 0.9}.  Each frame's reference is a 1024 spp render of the same time range with the tables of frame k + 1000.  Reported per
setting: the col+bg MSE of every frame, the mean over frames 9-24, and the flicker mean |(d_k - d_{k-1}) - (ref_k - ref_{k-1})|
over frames 2-24.  TEMPORAL_DEFAULTS is the setting with the lowest mean MSE over frames 9-24, averaged over both spp.
Cost (config 3 at 1920x1080): render_motion with and without the albedo plane against render_albedo at 4 * ALBEDO_SAMPLES spp
(device ms of the call, RaynStats.total_ms); k_temporal (device planes) at 1080p, 4K and 8K with an HBM byte model; the scaled
against the unscaled variance denoise (5 levels, device planes).  Prints JSON lines, with the card's name and power limit read
in the same run.  Needs a GPU; writes nothing."""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_denoise import HBM_PEAK_GBS, gpu_info  # noqa: E402
from rayn_b200 import _lib as L  # noqa: E402
from rayn_b200 import configs  # noqa: E402
from rayn_b200.film import ALBEDO_SAMPLES, FrameInputs, Renderer, denoise_desc  # noqa: E402
from rayn_b200.scene import Linear, PinholeCamera, Vec3  # noqa: E402

ORIGIN = np.array([-0.45, 0.2, 2.0]) * 2.25
FRAMES = range(1, 25)
DT = float(np.float32(1.0) / np.float32(24.0))
GRID = [(a, s, n) for a in (0.1, 0.2, 0.4) for s in (0.02, 0.1) for n in (0.5, 0.9)]
# k_temporal's HBM bytes per pixel: the frame (colour 3, background 3, normal 3, moments 2, motion 4), the outputs (colour 3,
# background 3, moments 2, scale 1) and the two histories (14 floats read at the pixel's own reprojected taps, which neighbouring
# threads share, so counted once; 14 written)
TEMPORAL_FLOATS = 15 + 9 + 14 + 14


def time_range(k):
    s = np.float32(k) * np.float32(DT)
    return float(s), float(s + np.float32(1.0) / np.float32(24.0))


def moving_config(w, h, samples):
    c = configs.baseline_config(3, res=(w, h), samples=samples, max_bounces=None)
    back = ORIGIN / np.linalg.norm(ORIGIN)
    right = np.cross([0.0, 1.0, 0.0], back)
    right /= np.linalg.norm(right)
    cam = c["world"].cameras.add_camera(PinholeCamera((w, h), 60.0, Linear(Vec3(*ORIGIN), Vec3(*(0.6 * right))),
                                                      Linear(Vec3(0, 0, 0), Vec3(*(0.3 * right))), Vec3(0, 1, 0)))
    return c, cam


def cb(p, w, h):
    return (np.asarray(p["color"], np.float64) + np.asarray(p["background"], np.float64)).reshape(h, w, 3)


def quality(r):
    w = h = 96
    c, cam = moving_config(w, h, 1)
    integ = c["integrator"]
    r.upload_scene(c["world"], cam)
    refs = [cb(r.render_host(FrameInputs(w, h, 256, integ, frame=k + 1000), (16, 16), integ, time_range(k)), w, h) for k in FRAMES]
    result = {}
    for samples in (1, 4):
        spp = 4 * samples
        frames = []
        for k in FRAMES:
            inp = FrameInputs(w, h, samples, integ, frame=k)
            p = r.render_host(inp, (16, 16), integ, time_range(k), moments=True)
            mv = r.render_motion(FrameInputs(w, h, min(samples, ALBEDO_SAMPLES), integ, frame=k), (16, 16), integ, time_range(k), DT)
            frames.append((p, mv))

        def score(outs):
            mse = [float(np.mean((o - ref) ** 2)) for o, ref in zip(outs, refs)]
            flick = [float(np.mean(np.abs((outs[i] - outs[i - 1]) - (refs[i] - refs[i - 1])))) for i in range(1, len(outs))]
            return dict(mse=mse, mse_9_24=float(np.mean(mse[8:])), flicker=float(np.mean(flick)))

        settings = {"raw": [cb(p, w, h) for p, _ in frames],
                    "spatial": [cb(r.denoise(w, h, p, 5, moments=p["moments"], spp=spp), w, h) for p, _ in frames]}
        for (a, s, n) in GRID:
            hist = r.temporal_create(w, h)
            outs = []
            try:
                for i, (p, mv) in enumerate(frames):
                    blend, m, scale = r.temporal_push(hist, p, p["moments"], mv, a, s, n, reset=(i == 0))
                    guides = dict(p, color=blend["color"], background=blend["background"])
                    outs.append(cb(r.denoise(w, h, guides, 5, moments=m, spp=spp, var_scale=scale), w, h))
            finally:
                hist.close()
            settings[f"temporal a={a} sd={s} nc={n}"] = outs
        for name, outs in settings.items():
            sc = score(outs)
            result.setdefault(name, {})[spp] = sc
            print(json.dumps(dict(kind="temporal_quality", setting=name, spp=spp, **sc)), flush=True)
    temporal = [k for k in result if k.startswith("temporal")]
    pick = min(temporal, key=lambda k: np.mean([result[k][s]["mse_9_24"] for s in (4, 16)]))
    summary = {k: dict(mse_9_24={s: result[k][s]["mse_9_24"] for s in (4, 16)}, flicker={s: result[k][s]["flicker"] for s in (4, 16)})
               for k in ("raw", "spatial", pick)}
    print(json.dumps(dict(kind="temporal_pick", pick=pick, summary=summary)), flush=True)


def cost_motion(reps):
    c, cam = moving_config(1920, 1080, 128)
    r = Renderer(0)
    try:
        r.upload_scene(c["world"], cam)
        inp = FrameInputs(1920, 1080, ALBEDO_SAMPLES, c["integrator"])
        calls = {"render_albedo": lambda: r.render_albedo(inp, (16, 16), c["integrator"], time_range(1)),
                 "render_motion": lambda: r.render_motion(inp, (16, 16), c["integrator"], time_range(1), DT),
                 "render_motion+albedo": lambda: r.render_motion(inp, (16, 16), c["integrator"], time_range(1), DT, albedo=True)}
        for f in calls.values():
            f()
        t = {k: [] for k in calls}
        for _ in range(reps):
            for k, f in calls.items():
                f()
                t[k].append(r.stats().total_ms)
        for k in calls:
            print(json.dumps(dict(kind="motion_cost", call=k, spp=inp.spp, ms=float(np.median(t[k])), runs=t[k])), flush=True)
    finally:
        r.close()


def cost_temporal_and_denoise(reps):
    import torch
    lib = L.lib()
    for (w, h) in ((1920, 1080), (3840, 2160), (7680, 4320)):
        r = Renderer(0)
        try:
            npx = w * h
            g = torch.Generator(device="cuda").manual_seed(0)
            rnd = lambda n: torch.rand(n, device="cuda", generator=g)  # noqa: E731
            c, b, n = rnd(3 * npx), rnd(3 * npx), rnd(3 * npx) * 0.1 + 0.5
            m = rnd(2 * npx)
            mv = torch.zeros(npx, 4, device="cuda")
            mv[:, 0:2] = rnd(2 * npx).view(npx, 2) * 2 - 1
            mv[:, 2:] = 3.0
            oc, ob, om, s = torch.empty_like(c), torch.empty_like(b), torch.empty_like(m), torch.ones(npx, device="cuda")
            alpha = torch.ones(npx, device="cuda")
            pin = L.RaynFilmPlanes(c.data_ptr(), alpha.data_ptr(), b.data_ptr(), n.data_ptr(), L.MEM_DEVICE)
            pout = L.RaynFilmPlanes(oc.data_ptr(), None, ob.data_ptr(), None, L.MEM_DEVICE)
            pm = L.RaynMomentPlanes(m.data_ptr(), m.data_ptr() + 4 * npx, L.MEM_DEVICE)
            pmo = L.RaynMomentPlanes(om.data_ptr(), om.data_ptr() + 4 * npx, L.MEM_DEVICE)
            t = r.temporal_create(w, h)
            td = L.RaynTemporalDesc(0.2, 0.05, 0.5, 0)
            d = denoise_desc(5)
            calls = {"k_temporal": lambda: lib.rayn_b200_temporal_push(r.ctx, t.handle, C.byref(td), C.byref(pin), C.byref(pm), mv.data_ptr(),
                                                                       C.byref(pout), C.byref(pmo), s.data_ptr()),
                     "denoise_variance": lambda: lib.rayn_b200_film_denoise_variance(r.ctx, C.byref(d), 4.0, 16, C.byref(pm), 1.0, None, w, h,
                                                                                     C.byref(pin), C.byref(pout)),
                     "denoise_variance_scaled": lambda: lib.rayn_b200_film_denoise_variance_scaled(r.ctx, C.byref(d), 4.0, 16, C.byref(pm),
                                                                                                   s.data_ptr(), 1.0, None, w, h, C.byref(pin),
                                                                                                   C.byref(pout))}
            torch.cuda.synchronize()
            for f in calls.values():
                L.check(f(), r.ctx)
            torch.cuda.synchronize()
            times = {k: [] for k in calls}
            for _ in range(reps):
                for k, f in calls.items():
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    t0 = time.perf_counter()
                    for _ in range(10):
                        L.check(f(), r.ctx)
                    L.check(lib.rayn_b200_sync(r.ctx), r.ctx)
                    times[k].append((time.perf_counter() - t0) / 10 * 1e3)
            for k in calls:
                ms = float(np.median(times[k]))
                line = dict(kind="temporal_cost", call=k, res=f"{w}x{h}", ms=ms, runs=times[k])
                if k == "k_temporal":
                    by = TEMPORAL_FLOATS * 4 * npx
                    line.update(model_bytes=by, hbm_gbs=by / ms / 1e6, hbm_frac=by / ms / 1e6 / HBM_PEAK_GBS)
                print(json.dumps(line), flush=True)
            t.close()
        finally:
            r.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quality", action="store_true")
    ap.add_argument("--cost", action="store_true")
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    print(json.dumps(dict(kind="gpu", info=gpu_info())), flush=True)
    if a.quality or not a.cost:
        r = Renderer(0)
        try:
            quality(r)
        finally:
            r.close()
    if a.cost or not a.quality:
        cost_motion(a.reps)
        cost_temporal_and_denoise(a.reps)


if __name__ == "__main__":
    main()
