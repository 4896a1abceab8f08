"""Cost of the Metallic material (include/rayn_b200.h, RAYN_MATERIAL_METALLIC) on config 3: the same frame with the Mandelbox as
the reference's Dielectric.new_remap(0.2 grey, 0.6), and as a copper metal at roughness 0.6 and 0.2, each plain and with an
orbit-trap palette in place of F0 (the example range of tools/trap_range.py).

    python tools/bench_metallic.py [--res 1920x1080] [--samples 16] [--bounces 8] [--reps 3] [--json out.json]

--samples is rayn's packet count: 16 packets are 64 spp.  Each arm is warmed up once, then the arms alternate `reps` times.
Msamples/s is camera samples over the host time of the render call (which ends in a device synchronise) on a context without
timing; k_shade_pre / k_shade_post are the summed per-launch CUDA-event times of a second context with RAYN_FLAG_TIMING.  Mean
path length is RaynStats.extend_rays / paths (traced segments per camera sample).  Medians are reported.  Card, power limit
and SM clocks are read in the same call.  Needs a GPU; writes nothing unless --json is given."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from rayn_b200 import _lib as L  # noqa: E402
from rayn_b200 import configs  # noqa: E402
from rayn_b200.film import FrameInputs, Renderer  # noqa: E402
from rayn_b200.scene import Metallic, OrbitTrapAlbedo  # noqa: E402
from bench_trap import gpu_info  # noqa: E402
from trap_range import TRAP_HI, TRAP_LO  # noqa: E402

TR = configs.frame_time_range(1)
COPPER = (0.95, 0.64, 0.54)
ALBEDO_LO, ALBEDO_HI = (0.9, 0.35, 0.1), (0.1, 0.3, 0.8)
KERNELS = ("shade_pre", "shade_post", "normals", "extend", "shadow")


def arms(w, h, samples, bounces):
    out = {}
    for name, mat in (("dielectric", None), ("metal_r0.6", Metallic.new_remap(COPPER, 0.6)), ("metal_r0.2", Metallic.new_remap(COPPER, 0.2)),
                      ("metal_r0.6_trap", Metallic.new_remap(OrbitTrapAlbedo(TRAP_LO, TRAP_HI, ALBEDO_LO, ALBEDO_HI), 0.6)),
                      ("metal_r0.2_trap", Metallic.new_remap(OrbitTrapAlbedo(TRAP_LO, TRAP_HI, ALBEDO_LO, ALBEDO_HI), 0.2))):
        c = configs.baseline_config(3, res=(w, h), samples=samples, max_bounces=bounces)
        if mat is not None:
            c["world"].materials.items[1] = mat  # configs.setup(): sky, then the fractal's Dielectric.new_remap(0.2 grey, 0.6)
        out[name] = c
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", default="1920x1080")
    ap.add_argument("--samples", type=int, default=16)
    ap.add_argument("--bounces", type=int, default=8)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    w, h = (int(v) for v in a.res.split("x"))
    cs = arms(w, h, a.samples, a.bounces)
    inp = FrameInputs(w, h, a.samples, cs["dielectric"]["integrator"])
    fast, timed = Renderer(0), Renderer(0, flags=L.FLAG_TIMING)
    res = {n: [] for n in cs}
    try:
        for rep in range(a.reps + 1):
            for name, c in cs.items():
                fast.upload_scene(c["world"], c["camera"])
                t0 = time.perf_counter()
                fast.render_host(inp, (16, 16), c["integrator"], TR)
                wall = time.perf_counter() - t0
                st = fast.stats()
                timed.upload_scene(c["world"], c["camera"])
                timed.render_host(inp, (16, 16), c["integrator"], TR)
                tst = timed.stats()
                if rep == 0:
                    continue  # warm-up
                ms = {k: float(tst.kernel_ms[L.KERNEL_NAMES.index(k)]) for k in KERNELS}
                res[name].append(dict(msamples_s=st.paths / wall / 1e6, wall_ms=1e3 * wall, path_len=st.extend_rays / st.paths, **ms))
    finally:
        fast.close()
        timed.close()
    med = {n: {k: float(np.median([x[k] for x in v])) for k in v[0]} for n, v in res.items()}
    out = dict(gpu=gpu_info(), res=[w, h], spp=4 * a.samples, bounces=a.bounces, median=med, runs=res)
    print(f"config 3 {w}x{h}, {4 * a.samples} spp, {a.bounces} bounces; {out['gpu']}")
    cols = ("msamples_s", "wall_ms", "path_len") + KERNELS
    print(f"{'arm (median of ' + str(a.reps) + ')':22s}" + "".join(f"{k:>12s}" for k in cols))
    for n, m in med.items():
        print(f"{n:22s}" + "".join(f"{m[k]:12.3f}" for k in cols))
    print(json.dumps(dict(gpu=out["gpu"], median=med)))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
