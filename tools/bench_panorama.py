"""Measures the equirectangular camera of DESIGN.md §4i on one GPU: what a 360-degree panorama costs against the pinhole
headline, and what the wrapped film filter costs against the unwrapped one.

    python tools/bench_panorama.py [--samples 16] [--reps 3]

Render: config 3 (the Mandelbox scene, 8 bounces) as a 3840x1920 panorama from the config's camera position, against the
1920x1080 pinhole view of bench.py's headline, both at 4 * samples spp with device frame inputs and device planes, alternated
rep by rep.  Reported per view: Msamples/s (camera paths over the host wall time of a synchronous render) and, from a second
context with RAYN_FLAG_TIMING, the device ms of k_raygen and of the whole render (RaynStats).  The panorama's extra raygen
work is two sincos per sample.
Denoise: the variance-guided filter (5 levels, device planes, the §4f sigmas) at 3840x2160 through
rayn_b200_film_denoise_variance against rayn_b200_film_denoise_wrap with the same guides.
Prints JSON lines, with the card's name and power limit read in the same run.  Needs a GPU; writes nothing."""
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

from bench_denoise import gpu_info  # noqa: E402
from rayn_b200 import _lib as L  # noqa: E402
from rayn_b200 import configs  # noqa: E402
from rayn_b200.film import Renderer, denoise_desc, make_frame_desc  # noqa: E402
from rayn_b200.scene import EquirectangularCamera, Linear  # noqa: E402

TILE = (16, 16)


def views(samples):
    c = configs.baseline_config(3, res=(1920, 1080), samples=samples)
    src = c["world"].cameras.get(c["camera"])
    pano = c["world"].cameras.add_camera(EquirectangularCamera((3840, 1920), *(Linear(*p) for p in (src.origin, src.at, src.up))))
    return c, {"pinhole_1920x1080": (c["camera"], 1920, 1080), "panorama_3840x1920": (pano, 3840, 1920)}


def device_frame(r, c, w, h, samples):
    """device tables, scramble and planes for one view (kept alive by the returned tuple)"""
    import torch
    integ = c["integrator"]
    spp, sets = 4 * samples, (1 + integ.requested_1d_sample_sets(), 2 + integ.requested_2d_sample_sets())
    s1 = torch.empty(spp * sets[0], device="cuda")
    s2 = torch.empty(2 * spp * sets[1], device="cuda")
    scr = torch.empty(w * h, device="cuda")
    fis_h = np.empty(L.RAYN_FIS_TABLE_SIZE, np.float32)
    L.check(L.host_lib().rayn_b200_host_fis_blackman_harris(1.5, fis_h.ctypes.data_as(C.POINTER(C.c_float))))
    fis = torch.from_numpy(fis_h).cuda()
    torch.cuda.synchronize()
    L.check(r._lib.rayn_b200_device_frame_inputs(r.ctx, w, h, spp, sets[0], sets[1], 1, s1.data_ptr(), s2.data_ptr(), scr.data_ptr()), r.ctx)
    planes = {k: torch.zeros((1 if k == "alpha" else 3) * w * h, device="cuda") for k in ("color", "alpha", "background", "normal")}
    f = make_frame_desc(w, h, TILE, samples, integ, 1, configs.frame_time_range(1), (s1.data_ptr(), s2.data_ptr(), scr.data_ptr(), fis.data_ptr()),
                        L.MEM_DEVICE, sets=sets)
    p = L.RaynFilmPlanes(*(planes[k].data_ptr() for k in ("color", "alpha", "background", "normal")), L.MEM_DEVICE)
    return f, p, (s1, s2, scr, fis, planes)


def bench_render(samples, reps):
    c, vs = views(samples)
    out = {}
    for flags, key in ((0, "wall"), (L.FLAG_TIMING, "timing")):
        rs = {}
        try:
            for name, (cam, w, h) in vs.items():
                r = Renderer(0, flags=flags)
                r.upload_scene(c["world"], cam)
                rs[name] = (r, *device_frame(r, c, w, h, samples))
                r.render(rs[name][1], rs[name][2])  # warm-up
                L.check(r._lib.rayn_b200_sync(r.ctx), r.ctx)
            for _ in range(reps):
                for name, (r, f, p, _) in rs.items():
                    t0 = time.perf_counter()
                    r.render(f, p)
                    L.check(r._lib.rayn_b200_sync(r.ctx), r.ctx)
                    dt = time.perf_counter() - t0
                    s = r.stats()
                    out.setdefault((name, key), []).append((dt, s.paths, s.kernel_ms[L.KERNEL_NAMES.index("raygen")], s.total_ms))
        finally:
            for r, *_ in rs.values():
                r.close()
    for name in vs:
        wall = out[(name, "wall")]
        timing = out[(name, "timing")]
        msps = [p / dt / 1e6 for dt, p, _, _ in wall]
        print(json.dumps(dict(kind="panorama_render", view=name, spp=4 * samples, msamples_s=float(np.median(msps)), runs=msps,
                              raygen_ms=float(np.median([t[2] for t in timing])), device_ms=float(np.median([t[3] for t in timing])))),
              flush=True)


def bench_denoise(reps):
    import torch
    lib = L.lib()
    w, h = 3840, 2160
    npx = w * h
    r = Renderer(0)
    try:
        g = torch.Generator(device="cuda").manual_seed(0)
        c, b, n, a = (torch.rand(k * npx, device="cuda", generator=g) for k in (3, 3, 3, 1))
        m = torch.rand(2 * npx, device="cuda", generator=g)
        oc, ob = torch.empty_like(c), torch.empty_like(b)
        pin = L.RaynFilmPlanes(c.data_ptr(), a.data_ptr(), b.data_ptr(), n.data_ptr(), L.MEM_DEVICE)
        pout = L.RaynFilmPlanes(oc.data_ptr(), None, ob.data_ptr(), None, L.MEM_DEVICE)
        pm = L.RaynMomentPlanes(m.data_ptr(), m.data_ptr() + 4 * npx, L.MEM_DEVICE)
        d = denoise_desc(5, sigma_color=float("inf"))
        calls = {"denoise_variance": lambda: lib.rayn_b200_film_denoise_variance(r.ctx, C.byref(d), 4.0, 16, C.byref(pm), 1.0, None, w, h,
                                                                                 C.byref(pin), C.byref(pout)),
                 "denoise_wrap": lambda: lib.rayn_b200_film_denoise_wrap(r.ctx, C.byref(d), 4.0, 16, C.byref(pm), None, 1.0, None, w, h,
                                                                         C.byref(pin), C.byref(pout))}
        for f in calls.values():
            L.check(f(), r.ctx)
        L.check(lib.rayn_b200_sync(r.ctx), r.ctx)
        times = {k: [] for k in calls}
        for _ in range(reps):
            for k, f in calls.items():
                t0 = time.perf_counter()
                for _ in range(10):
                    L.check(f(), r.ctx)
                L.check(lib.rayn_b200_sync(r.ctx), r.ctx)
                times[k].append((time.perf_counter() - t0) / 10 * 1e3)
        for k in calls:
            print(json.dumps(dict(kind="panorama_denoise", call=k, res=f"{w}x{h}", levels=5, ms=float(np.median(times[k])), runs=times[k])),
                  flush=True)
    finally:
        r.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=16)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    print(json.dumps(dict(kind="gpu", info=gpu_info())), flush=True)
    bench_render(a.samples, a.reps)
    bench_denoise(a.reps)
    print(json.dumps(dict(kind="gpu", info=gpu_info())), flush=True)


if __name__ == "__main__":
    main()
