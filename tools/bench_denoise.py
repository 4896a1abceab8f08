"""Times the film denoiser (rayn_b200_film_denoise) on config 3 films and reports its share of the H100 SXM data-sheet
HBM bandwidth and FP64 rate; with --pick-sigmas, also the sweep the default sigmas were picked from.

    python tools/bench_denoise.py [--sizes 1920x1080,3840x2160,7680x4320] [--iterations 5] [--reps 7] [--pick-sigmas]

Each film is config 3 rendered on the GPU at 4 spp (so the filter sees real noise and edges).  Both the color and the
background plane are filtered, device planes in and out.  A call's time is the host clock around `calls` back-to-back
calls that ends in a stream synchronise, divided by `calls`; the median of `reps` such windows is reported.  Prints one
JSON line per size.  Needs a GPU; writes nothing."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from rayn_b200 import _lib as L  # noqa: E402
from rayn_b200 import configs  # noqa: E402
from rayn_b200.film import FrameInputs, Renderer, denoise_desc  # noqa: E402

HBM_PEAK_GBS = 3350.0    # H100 SXM data sheet (700 W card)
FP64_PEAK_TFLOPS = 34.0  # H100 SXM data sheet, FP64 without tensor cores (700 W card)
# FP64 operations of one dm::exp (detmath.h): x*log2e + 0.5, two reduction DFMAs, 13 Horner DFMAs, the final scale;
# a DFMA counts 2
EXP_FP64_FLOP = 2 + 2 * 2 + 13 * 2 + 1


def render(w, h, samples):
    """On a context of its own, so that its pass buffers are released before anything is timed."""
    c = configs.baseline_config(3, res=(w, h), samples=samples)
    inp = FrameInputs(w, h, c["samples"], c["integrator"])
    r = Renderer(0)
    try:
        r.upload_scene(c["world"], c["camera"])
        return r.render_host(inp, (16, 16), c["integrator"], configs.frame_time_range(1))
    finally:
        r.close()


def model(w, h, iterations, n_channels):
    """Bytes and FP64 operations the filter needs, from the shapes.  Bytes: the guide pack (read 16, write 16 B per pixel),
    per channel the colour pack (read 12, write 16), and per level one read of the colour and guide planes and one write
    (16 + 16 + 16 B, 12 for the last level's rgb output).  FP64: one dm::exp per in-image tap (an upper bound: taps with
    e = 0 or a weight of exactly +0 skip it)."""
    npx = w * h
    bytes_ = npx * (32 + n_channels * (28 + iterations * 48 - 4))
    taps = 0
    for i in range(iterations):
        s = 2 ** i
        tx = sum(max(0, w - abs(s * d)) for d in range(-2, 3))
        ty = sum(max(0, h - abs(s * d)) for d in range(-2, 3))
        taps += tx * ty
    return bytes_, n_channels * taps * EXP_FP64_FLOP


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except Exception as e:  # the timing itself does not depend on it
        return f"unavailable: {e}"


def bench(r, w, h, iterations, reps, calls):
    import torch
    film = render(w, h, 1)
    dev = {k: torch.from_numpy(v).cuda() for k, v in film.items()}
    out = {k: torch.empty_like(dev[k]) for k in ("color", "background")}
    pin = L.RaynFilmPlanes(dev["color"].data_ptr(), dev["alpha"].data_ptr(), dev["background"].data_ptr(), dev["normal"].data_ptr(), L.MEM_DEVICE)
    pout = L.RaynFilmPlanes(out["color"].data_ptr(), None, out["background"].data_ptr(), None, L.MEM_DEVICE)
    d = denoise_desc(iterations)
    lib = L.lib()
    torch.cuda.synchronize()

    def window(n):
        t0 = time.perf_counter()
        for _ in range(n):
            L.check(lib.rayn_b200_film_denoise(r.ctx, C.byref(d), w, h, C.byref(pin), C.byref(pout)), r.ctx)
        L.check(lib.rayn_b200_sync(r.ctx), r.ctx)
        return (time.perf_counter() - t0) / n * 1e3
    window(2)  # warm-up: module load, pool growth
    ms = sorted(window(calls) for _ in range(reps))
    med = ms[len(ms) // 2]
    bytes_, flop = model(w, h, iterations, 2)
    return dict(size=f"{w}x{h}", iterations=iterations, channels=2, median_ms=med, min_ms=ms[0], max_ms=ms[-1],
                hbm_gbs=bytes_ / med / 1e6, hbm_frac=bytes_ / med / 1e6 / HBM_PEAK_GBS,
                fp64_tflops_upper=flop / med / 1e9, fp64_frac_upper=flop / med / 1e9 / FP64_PEAK_TFLOPS,
                model_bytes=bytes_, model_fp64_flop=flop)


def pick_sigmas(r, iterations):
    """Config 3 at 96x96: col+bg MSE against a 256 spp film of the 4 spp film denoised with every sigma combination."""
    lo, hi = render(96, 96, 1), render(96, 96, 64)
    target = (hi["color"] + hi["background"]).astype(np.float64)
    raw = float(np.mean((lo["color"] + lo["background"] - target) ** 2))
    res = []
    for sc in (0.1, 0.2, 0.35, 0.5, 0.75, 1.0, 1.5, 2.5, np.inf):
        for sn in (0.05, 0.1, 0.2, 0.4, 0.8, np.inf):
            for sa in (0.05, 0.2, 0.5, np.inf):
                den = r.denoise(96, 96, lo, iterations, sc, sn, sa)
                mse = float(np.mean((den["color"] + den["background"] - target) ** 2))
                res.append((mse, sc, sn, sa))
    res.sort()
    for mse, sc, sn, sa in res[:10]:
        print(json.dumps(dict(sigma_color=sc, sigma_normal=sn, sigma_alpha=sa, mse=mse, mse_raw=raw, ratio=mse / raw)))
    dflt = r.denoise(96, 96, lo, iterations)
    mse = float(np.mean((dflt["color"] + dflt["background"] - target) ** 2))
    print(json.dumps(dict(defaults=True, mse=mse, mse_raw=raw, ratio=mse / raw)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1920x1080,3840x2160,7680x4320")
    ap.add_argument("--iterations", type=int, default=5)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--pick-sigmas", action="store_true")
    a = ap.parse_args()
    print(json.dumps(dict(gpu=gpu_info())))
    r = Renderer(0)
    try:
        if a.pick_sigmas:
            pick_sigmas(r, a.iterations)
        for s in a.sizes.split(","):
            w, h = (int(v) for v in s.split("x"))
            print(json.dumps(bench(r, w, h, a.iterations, a.reps, a.calls)), flush=True)
        print(json.dumps(dict(gpu_after=gpu_info())))
    finally:
        r.close()


if __name__ == "__main__":
    main()
