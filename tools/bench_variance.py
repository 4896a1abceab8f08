"""Measures the luminance-moment render (rayn_b200_render_frame_moments) and the variance-guided denoise
(rayn_b200_film_denoise_variance) on one GPU: the quality sweep DENOISE_LUMINANCE_SIGMA and DENOISE_VARIANCE_SIGMA_COLOR were
picked from, and the cost of both calls.

    python tools/bench_variance.py [--quality] [--cost] [--reps 3]

Quality: config 3 at 96x96, grey and with the README palette (trap 0.6676 .. 1.45, (0.9, 0.35, 0.1) -> (0.1, 0.3, 0.8)).
Films of 4, 16 and 64 spp (frame 1) are filtered with 5 levels; the col+bg MSE is taken against a 1024 spp film whose tables
use frame 2.  Compared: raw, the unguided defaults, the albedo-guided defaults (albedo plane of 4 * min(samples,
ALBEDO_SAMPLES) spp), and the variance-guided filter over sigma_luminance in {1, 2, 4, 8, 16, inf} x sigma_color in {2.5, inf},
with and without the albedo guide.  The default is the setting with the lowest mean MSE ratio to the unguided defaults over the
three sample counts.
Cost: render_frame against render_frame_moments on config 3 at 1920x1080, 512 spp, 8 bounces (frame ms and k_resolve ms of
RAYN_FLAG_TIMING, medians of `reps` runs alternated in one process); and the variance-guided against the unguided denoise
(color + background, 5 levels, device planes) at 1080p, 4K and 8K, with the HBM model of tools/bench_denoise.py extended by the
moment-plane reads.  Prints JSON lines, with the card's name and power limit read in the same run.  Needs a GPU; writes nothing."""
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

from bench_denoise import HBM_PEAK_GBS, gpu_info, model  # noqa: E402
from rayn_b200 import _lib as L  # noqa: E402
from rayn_b200 import configs  # noqa: E402
from rayn_b200.film import ALBEDO_SAMPLES, FrameInputs, Renderer, denoise_desc  # noqa: E402
from rayn_b200.scene import Dielectric, OrbitTrapAlbedo  # noqa: E402

TR = configs.frame_time_range(1)
SIGMA_L = (1.0, 2.0, 4.0, 8.0, 16.0, float("inf"))
SIGMA_C = (2.5, float("inf"))
CH = ("color", "alpha", "background", "normal")


def config(trap, w, h, samples, mb=None):
    c = configs.baseline_config(3, res=(w, h), samples=samples, **({} if mb is None else {"max_bounces": mb}))
    if trap:  # the README example
        c["world"].materials.items[1] = Dielectric.new_remap(OrbitTrapAlbedo(0.6676, 1.45, (0.9, 0.35, 0.1), (0.1, 0.3, 0.8)), 0.6)
    return c


def quality(r):
    w = h = 96
    table = {}
    for trap in (True, False):
        c = config(trap, w, h, 1)
        r.upload_scene(c["world"], c["camera"])
        hi = r.render_host(FrameInputs(w, h, 256, c["integrator"], frame=2), (16, 16), c["integrator"], TR)
        target = (hi["color"] + hi["background"]).astype(np.float64)

        def mse(d):
            return float(np.mean((d["color"].reshape(-1) + d["background"].reshape(-1) - target) ** 2))
        for samples in (1, 4, 16):
            inp = FrameInputs(w, h, samples, c["integrator"])
            lo = r.render_host(inp, (16, 16), c["integrator"], TR, moments=True)
            alb = r.render_albedo(FrameInputs(w, h, min(samples, ALBEDO_SAMPLES), c["integrator"]), (16, 16), c["integrator"], TR)
            planes = {k: lo[k].reshape((h, w, 3) if k != "alpha" else (h, w)) for k in CH}
            raw, unguided, albedo = mse(lo), mse(r.denoise(w, h, planes, 5)), mse(r.denoise(w, h, planes, 5, albedo=alb))
            rows = []
            for with_alb in (False, True):
                for sc in SIGMA_C:
                    for sl in SIGMA_L:
                        e = mse(r.denoise(w, h, planes, 5, sigma_color=sc, albedo=alb if with_alb else None, moments=lo["moments"],
                                          spp=inp.spp, sigma_luminance=sl))
                        rows.append(dict(albedo=with_alb, sigma_color=sc, sigma_luminance=sl, vs_raw=e / raw, vs_unguided=e / unguided,
                                         vs_albedo=e / albedo))
                        table.setdefault((trap, with_alb, sc, sl), []).append(e / unguided)
            print(json.dumps(dict(kind="quality", trap=trap, spp=inp.spp, raw=raw, unguided_vs_raw=unguided / raw,
                                  albedo_vs_raw=albedo / raw, rows=rows)), flush=True)
    for trap in (True, False):
        best = min(((k, float(np.mean(v))) for k, v in table.items() if k[0] == trap), key=lambda kv: kv[1])
        wins = [k for k, v in table.items() if k[0] == trap and not np.isinf(k[3]) and v[1] < 1.0 and v[2] < 1.0]
        print(json.dumps(dict(kind="pick", trap=trap, best=dict(albedo=best[0][1], sigma_color=best[0][2], sigma_luminance=best[0][3]),
                              mean_vs_unguided=best[1], n_settings_beating_unguided_at_16_and_64_spp=len(wins))), flush=True)


def cost_render(reps):
    c = config(False, 1920, 1080, 128, 8)
    r = Renderer(0, flags=L.FLAG_TIMING)
    try:
        r.upload_scene(c["world"], c["camera"])
        inp = FrameInputs(1920, 1080, 128, c["integrator"])
        r.render_host(inp, (16, 16), c["integrator"], TR)  # warm-up of both paths
        r.render_host(inp, (16, 16), c["integrator"], TR, moments=True)
        t = {False: [], True: []}
        for _ in range(reps):
            for mom in (False, True):
                r.render_host(inp, (16, 16), c["integrator"], TR, moments=mom)
                s = r.stats()
                t[mom].append((s.total_ms, s.kernel_ms[L.KERNEL_NAMES.index("resolve")]))
        for mom in (False, True):
            a = np.array(t[mom])
            print(json.dumps(dict(kind="render_cost", moments=mom, spp=inp.spp, frame_ms=float(np.median(a[:, 0])),
                                  resolve_ms=float(np.median(a[:, 1])), runs=t[mom])), flush=True)
    finally:
        r.close()


def cost_denoise(reps):
    import torch
    for (w, h) in ((1920, 1080), (3840, 2160), (7680, 4320)):
        c = config(False, w, h, 1)
        r = Renderer(0)
        try:
            r.upload_scene(c["world"], c["camera"])
            inp = FrameInputs(w, h, 1, c["integrator"])
            film = r.render_host(inp, (16, 16), c["integrator"], TR, moments=True)
            dev = {k: torch.from_numpy(film[k]).cuda() for k in CH}
            m = torch.from_numpy(np.ascontiguousarray(film["moments"].transpose(2, 0, 1))).cuda()
            out = {k: torch.empty_like(dev[k]) for k in ("color", "background")}
            pin = L.RaynFilmPlanes(*(dev[k].data_ptr() for k in CH), L.MEM_DEVICE)
            pout = L.RaynFilmPlanes(out["color"].data_ptr(), None, out["background"].data_ptr(), None, L.MEM_DEVICE)
            pm = L.RaynMomentPlanes(m[0].data_ptr(), m[1].data_ptr(), L.MEM_DEVICE)
            d = denoise_desc(5)
            lib = L.lib()
            calls = {"unguided": lambda: lib.rayn_b200_film_denoise(r.ctx, C.byref(d), w, h, C.byref(pin), C.byref(pout)),
                     "variance": lambda: lib.rayn_b200_film_denoise_variance(r.ctx, C.byref(d), 4.0, inp.spp, C.byref(pm), 1.0, None, w, h,
                                                                            C.byref(pin), C.byref(pout))}
            torch.cuda.synchronize()
            times = {k: [] for k in calls}
            for k, f in calls.items():  # warm-up
                L.check(f(), r.ctx)
            torch.cuda.synchronize()
            for _ in range(reps):
                for k, f in calls.items():
                    t0 = time.perf_counter()
                    for _ in range(5):
                        L.check(f(), r.ctx)
                    torch.cuda.synchronize()
                    times[k].append((time.perf_counter() - t0) / 5 * 1e3)
            base_bytes, _ = model(w, h, 5, 2)
            for k in calls:
                ms = float(np.median(times[k]))
                bytes_ = base_bytes + (2 * w * h * 4 if k == "variance" else 0)  # the two moment planes, read once by the pack
                print(json.dumps(dict(kind="denoise_cost", call=k, res=f"{w}x{h}", ms=ms, model_bytes=bytes_,
                                      hbm_gbs=bytes_ / ms / 1e6, hbm_frac=bytes_ / ms / 1e6 / HBM_PEAK_GBS, runs=times[k])), flush=True)
        finally:
            r.close()


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--quality", action="store_true")
    ap.add_argument("--cost", action="store_true")
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    both = not (a.quality or a.cost)
    print(json.dumps(dict(kind="gpu", info=gpu_info())), flush=True)
    if a.quality or both:
        r = Renderer(0)
        try:
            quality(r)
        finally:
            r.close()
    if a.cost or both:
        cost_render(a.reps)
        cost_denoise(a.reps)
    print(json.dumps(dict(kind="gpu", info=gpu_info())), flush=True)
