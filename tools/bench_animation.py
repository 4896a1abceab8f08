"""Measures temporal denoising of an animated scene (DESIGN.md §4h) on one GPU: how much motion against the previous frame's
scene (rayn_b200_render_motion_prev) helps over motion from the per-frame scene alone, and what it costs.

    python tools/bench_animation.py [--quality] [--cost] [--reps 5]

Quality: config 3 at 96x96, frames 1..24 at 24 fps, the camera origin orbiting the Mandelbox about the y axis at 30 degrees/s
(a closure, uploaded per frame as its chord over the frame's time range) and looking at the centre.  Shutter 0 and 1/24, at 4
and 16 spp.  Arms: the raw film; the spatial variance denoise (§4f defaults); temporal push + scaled denoise (TEMPORAL_DEFAULTS)
with render_motion on the per-frame chord scene, the best a caller could do without the previous scene; the same with
render_motion_prev against the previous frame's scene.  Each frame's reference is a 1024 spp render of the same scene and time
range with the tables of frame k + 1000.  Reported as in §4g: the col+bg MSE of every frame, its mean over frames 9-24, and the
flicker mean |(d_k - d_{k-1}) - (ref_k - ref_{k-1})| over frames 2-24.
Cost (1920x1080, 64 spp, the orbit at frame 2 against frame 1): render_motion against render_motion_prev (device ms of the
call, RaynStats.total_ms), and the host time of one upload_scene of the closure world (flatten with chords + upload).  Prints
JSON lines, with the card's name, power limit and SM clock read in the same run.  Needs a GPU; writes nothing."""
import argparse
import json
import math
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_denoise import gpu_info  # noqa: E402
from rayn_b200 import configs  # noqa: E402
from rayn_b200.film import ALBEDO_SAMPLES, TEMPORAL_DEFAULTS, FrameInputs, Renderer  # noqa: E402
from rayn_b200.scene import PinholeCamera, Vec3  # noqa: E402

ORIGIN = np.array([-0.45, 0.2, 2.0]) * 2.25
FRAMES = range(1, 25)
DT = float(np.float32(1.0) / np.float32(24.0))
DEG_PER_S = 30.0


def time_range(k, shutter):
    s = np.float32(k) * np.float32(DT)
    return float(s), float(s + np.float32(shutter))


def orbit_config(w, h, samples):
    c = configs.baseline_config(3, res=(w, h), samples=samples, max_bounces=None)
    r0, a0 = float(np.hypot(ORIGIN[0], ORIGIN[2])), math.atan2(ORIGIN[2], ORIGIN[0])

    def origin(t):
        a = a0 + math.radians(DEG_PER_S) * t
        return (r0 * math.cos(a), float(ORIGIN[1]), r0 * math.sin(a))
    cam = c["world"].cameras.add_camera(PinholeCamera((w, h), 60.0, origin, Vec3(0, 0, 0), Vec3(0, 1, 0)))
    return c, cam


def cb(p, w, h):
    return (np.asarray(p["color"], np.float64) + np.asarray(p["background"], np.float64)).reshape(h, w, 3)


def score(outs, refs):
    mse = [float(np.mean((o - ref) ** 2)) for o, ref in zip(outs, refs)]
    flick = [float(np.mean(np.abs((outs[i] - outs[i - 1]) - (refs[i] - refs[i - 1])))) for i in range(1, len(outs))]
    return dict(mse=mse, mse_9_24=float(np.mean(mse[8:])), flicker=float(np.mean(flick)))


def temporal(r, w, h, spp, frames, which):
    hist = r.temporal_create(w, h)
    outs = []
    try:
        for i, f in enumerate(frames):
            p = f["planes"]
            blend, m, scale = r.temporal_push(hist, p, p["moments"], f[which], reset=(i == 0), **TEMPORAL_DEFAULTS)
            outs.append(cb(r.denoise(w, h, dict(p, color=blend["color"], background=blend["background"]), 5, moments=m, spp=spp,
                                     var_scale=scale), w, h))
    finally:
        hist.close()
    return outs


def quality(r):
    w = h = 96
    c, cam = orbit_config(w, h, 1)
    integ = c["integrator"]
    for shutter in (0.0, 1.0 / 24.0):
        refs = []
        for k in FRAMES:
            r.upload_scene(c["world"], cam, time_range(k, shutter))
            refs.append(cb(r.render_host(FrameInputs(w, h, 256, integ, frame=k + 1000), (16, 16), integ, time_range(k, shutter)), w, h))
        for samples in (1, 4):
            spp = 4 * samples
            frames, prev = [], None
            for k in FRAMES:
                tr = time_range(k, shutter)
                scene = r.upload_scene(c["world"], cam, tr)
                p = r.render_host(FrameInputs(w, h, samples, integ, frame=k), (16, 16), integ, tr, moments=True)
                g = FrameInputs(w, h, min(samples, ALBEDO_SAMPLES), integ, frame=k)
                chord = r.render_motion(g, (16, 16), integ, tr, DT)
                frames.append(dict(planes=p, chord=chord, prev=chord if prev is None else r.render_motion(g, (16, 16), integ, tr, DT, prev=prev[0])))
                prev = scene
            arms = {"raw": [cb(f["planes"], w, h) for f in frames],
                    "spatial": [cb(r.denoise(w, h, f["planes"], 5, moments=f["planes"]["moments"], spp=spp), w, h) for f in frames],
                    "temporal_chord_motion": temporal(r, w, h, spp, frames, "chord"),
                    "temporal_prev_motion": temporal(r, w, h, spp, frames, "prev")}
            for name, outs in arms.items():
                print(json.dumps(dict(kind="animation_quality", shutter=shutter, spp=spp, arm=name, **score(outs, refs))), flush=True)


def cost(reps):
    c, cam = orbit_config(1920, 1080, 16)
    integ = c["integrator"]
    r = Renderer(0)
    try:
        prev = r.upload_scene(c["world"], cam, time_range(1, 0.0))
        inp = FrameInputs(1920, 1080, 16, integ, frame=2)
        tr = time_range(2, 0.0)
        host = []
        for _ in range(reps + 1):
            t0 = time.perf_counter()
            r.upload_scene(c["world"], cam, tr)
            host.append((time.perf_counter() - t0) * 1e3)
        calls = {"render_motion": lambda: r.render_motion(inp, (16, 16), integ, tr, DT),
                 "render_motion_prev": lambda: r.render_motion(inp, (16, 16), integ, tr, DT, prev=prev[0])}
        for f in calls.values():
            f()
        t = {k: [] for k in calls}
        for _ in range(reps):
            for k, f in calls.items():
                f()
                t[k].append(r.stats().total_ms)
        for k in calls:
            print(json.dumps(dict(kind="animation_cost", call=k, res="1920x1080", spp=inp.spp, ms=float(np.median(t[k])), runs=t[k])), flush=True)
        print(json.dumps(dict(kind="animation_cost", call="upload_scene (host)", ms=float(np.median(host[1:])), runs=host[1:])), flush=True)
    finally:
        r.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quality", action="store_true")
    ap.add_argument("--cost", action="store_true")
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    print(json.dumps(dict(kind="gpu", info=gpu_info())), flush=True)
    if a.quality or not a.cost:
        r = Renderer(0)
        try:
            quality(r)
        finally:
            r.close()
    if a.cost or not a.quality:
        cost(a.reps)
    print(json.dumps(dict(kind="gpu_after", info=gpu_info())), flush=True)


if __name__ == "__main__":
    main()
