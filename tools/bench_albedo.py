"""Measures the first-hit albedo plane (rayn_b200_render_albedo) and the albedo-guided denoise (rayn_b200_film_denoise_albedo)
on one GPU: the quality sweep DENOISE_ALBEDO_SIGMA and ALBEDO_SAMPLES were picked from, and the cost of both calls.

    python tools/bench_albedo.py [--quality] [--cost] [--reps 5]

Quality: config 3 at 96x96 with the README palette (trap 0.6676 .. 1.45, (0.9, 0.35, 0.1) -> (0.1, 0.3, 0.8)) and, as a
control, the grey config 3.  The 4 spp film (frame 1) is filtered with 5 levels; the col+bg MSE is taken against a 256 spp
film whose tables use frame 2.  Compared: raw, the unguided defaults, and the guided filter with sigma_albedo in {0.02, 0.05,
0.1, 0.2, 0.5, inf}, for albedo planes of 4, 16 and 64 spp (the film's own frame seed).
Cost: render_albedo at 1920x1080 (ALBEDO_SAMPLES and 512 spp) against one 512 spp render_frame of the trap scene, with the
per-kernel device times of RAYN_FLAG_TIMING; and the guided against the unguided denoise (color + background, 5 levels) at
1080p, 4K and 8K, with the HBM / FP64 model of tools/bench_denoise.py extended by the albedo guide.  Times are host clocks
around synchronous calls (median of `reps`).  Prints JSON lines, with the card's name and power limit read in the same run.
Needs a GPU; writes nothing."""
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

from bench_denoise import FP64_PEAK_TFLOPS, HBM_PEAK_GBS, gpu_info, model  # noqa: E402
from rayn_b200 import _lib as L  # noqa: E402
from rayn_b200 import configs  # noqa: E402
from rayn_b200.film import ALBEDO_SAMPLES, FrameInputs, Renderer, denoise_desc  # noqa: E402
from rayn_b200.scene import Dielectric, OrbitTrapAlbedo  # noqa: E402

TR = configs.frame_time_range(1)
SIGMAS = (0.02, 0.05, 0.1, 0.2, 0.5, float("inf"))


def config(trap, w, h, samples):
    c = configs.baseline_config(3, res=(w, h), samples=samples)
    if trap:  # the README example
        c["world"].materials.items[1] = Dielectric.new_remap(OrbitTrapAlbedo(0.6676, 1.45, (0.9, 0.35, 0.1), (0.1, 0.3, 0.8)), 0.6)
    return c


def render(r, c, w, h, samples, frame=1):
    inp = FrameInputs(w, h, samples, c["integrator"], frame=frame)
    r.upload_scene(c["world"], c["camera"])
    return r.render_host(inp, (16, 16), c["integrator"], TR)


def albedo(r, c, w, h, samples, frame=1):
    inp = FrameInputs(w, h, samples, c["integrator"], frame=frame)
    r.upload_scene(c["world"], c["camera"])
    return r.render_albedo(inp, (16, 16), c["integrator"], TR)


def quality(r):
    w = h = 96
    for trap in (True, False):
        c = config(trap, w, h, 1)
        lo, hi = render(r, c, w, h, 1), render(r, c, w, h, 64, frame=2)
        target = (hi["color"] + hi["background"]).astype(np.float64)
        planes = {k: lo[k].reshape((h, w, 3) if k != "alpha" else (h, w)) for k in lo}

        def mse(d):
            return float(np.mean((d["color"].reshape(-1) + d["background"].reshape(-1) - target) ** 2))
        raw = mse(lo)
        unguided = mse(r.denoise(w, h, planes, 5))
        rows = []
        for a_samples in (1, 4, 16):
            alb = albedo(r, c, w, h, a_samples)
            for s in SIGMAS:
                m = mse(r.denoise(w, h, planes, 5, albedo=alb, sigma_albedo=s))
                rows.append(dict(scene="cfg3 trap" if trap else "cfg3 grey", albedo_spp=4 * a_samples, sigma_albedo=s, mse=m,
                                 ratio_raw=m / raw, ratio_unguided=m / unguided))
        print(json.dumps(dict(scene="cfg3 trap" if trap else "cfg3 grey", mse_raw=raw, mse_unguided=unguided)))
        for row in rows:
            print(json.dumps(row))
        best = min(rows, key=lambda x: x["mse"])
        print(json.dumps(dict(scene=best["scene"], best=best)))


def timed(fn, reps):
    fn()  # warm-up
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    ts.sort()
    return ts[len(ts) // 2], ts[0], ts[-1]


def cost(reps):
    w, h = 1920, 1080
    c = config(True, w, h, 1)
    r = Renderer(0, flags=L.FLAG_TIMING)
    try:
        r.upload_scene(c["world"], c["camera"])
        names = L.KERNEL_NAMES
        for label, samples in ((f"albedo {4 * ALBEDO_SAMPLES} spp", ALBEDO_SAMPLES), ("albedo 512 spp", 128)):
            inp = FrameInputs(w, h, samples, c["integrator"])
            med, lo, hi = timed(lambda: r.render_albedo(inp, (16, 16), c["integrator"], TR), reps)
            st = r.stats()
            km = {names[i]: float(st.kernel_ms[i]) for i in range(L.STAT_KERNELS) if st.kernel_ms[i] > 0}
            print(json.dumps(dict(call=label, size="1920x1080", median_ms=med, min_ms=lo, max_ms=hi, device_ms=float(st.total_ms), kernel_ms=km,
                                  march_share=(km.get("extend", 0.0) + km.get("extend_spheres", 0.0)) / float(st.total_ms))), flush=True)
        inp = FrameInputs(w, h, 128, c["integrator"])
        med, lo, hi = timed(lambda: r.render_host(inp, (16, 16), c["integrator"], TR), max(1, reps // 2))
        st = r.stats()
        km = {names[i]: float(st.kernel_ms[i]) for i in range(L.STAT_KERNELS) if st.kernel_ms[i] > 0}
        print(json.dumps(dict(call="render_frame 512 spp", size="1920x1080", median_ms=med, min_ms=lo, max_ms=hi, device_ms=float(st.total_ms),
                              kernel_ms=km, depth0_and_later_march_share=km.get("extend", 0.0) / float(st.total_ms))), flush=True)
    finally:
        r.close()
    import torch
    lib = L.lib()
    for w, h in ((1920, 1080), (3840, 2160), (7680, 4320)):
        r = Renderer(0)
        try:
            c = config(True, w, h, 1)
            film = render(r, c, w, h, 1)
            alb = albedo(r, c, w, h, ALBEDO_SAMPLES).reshape(-1)
        finally:
            r.close()
        r = Renderer(0)
        try:
            dev = {k: torch.from_numpy(v).cuda() for k, v in film.items()}
            dalb = torch.from_numpy(alb).cuda()
            out = {k: torch.empty_like(dev[k]) for k in ("color", "background")}
            pin = L.RaynFilmPlanes(dev["color"].data_ptr(), dev["alpha"].data_ptr(), dev["background"].data_ptr(), dev["normal"].data_ptr(),
                                   L.MEM_DEVICE)
            pout = L.RaynFilmPlanes(out["color"].data_ptr(), None, out["background"].data_ptr(), None, L.MEM_DEVICE)
            d = denoise_desc(5)
            torch.cuda.synchronize()

            def unguided():
                for _ in range(5):
                    L.check(lib.rayn_b200_film_denoise(r.ctx, C.byref(d), w, h, C.byref(pin), C.byref(pout)), r.ctx)
                L.check(lib.rayn_b200_sync(r.ctx), r.ctx)

            def guided():
                for _ in range(5):
                    L.check(lib.rayn_b200_film_denoise_albedo(r.ctx, C.byref(d), 0.1, dalb.data_ptr(), w, h, C.byref(pin), C.byref(pout)), r.ctx)
                L.check(lib.rayn_b200_sync(r.ctx), r.ctx)
            b0, f0 = model(w, h, 5, 2)
            # the albedo guide: its pack (read 12, write 16 B per pixel) and, per channel and level, one more 16 B read;
            # about 10 FP32 operations per tap, no FP64
            b1 = b0 + w * h * (28 + 2 * 5 * 16)
            res = {}
            for name, fn, b in (("unguided", unguided, b0), ("guided", guided, b1)):
                med, lo, hi = timed(fn, reps)
                med, lo, hi = med / 5, lo / 5, hi / 5
                res[name] = med
                print(json.dumps(dict(call=f"denoise {name}", size=f"{w}x{h}", median_ms=med, min_ms=lo, max_ms=hi, model_bytes=b, model_fp64_flop=f0,
                                      hbm_frac=b / med / 1e6 / HBM_PEAK_GBS, fp64_frac_upper=f0 / med / 1e9 / FP64_PEAK_TFLOPS)), flush=True)
            print(json.dumps(dict(size=f"{w}x{h}", guided_over_unguided=res["guided"] / res["unguided"])))
        finally:
            r.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quality", action="store_true")
    ap.add_argument("--cost", action="store_true")
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    print(json.dumps(dict(gpu=gpu_info())))
    if a.quality:
        r = Renderer(0)
        try:
            quality(r)
        finally:
            r.close()
    if a.cost:
        cost(a.reps)
    print(json.dumps(dict(gpu_after=gpu_info())))


if __name__ == "__main__":
    main()
