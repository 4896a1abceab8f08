"""Cost of an orbit-trap albedo (rayn_b200_set_albedo_traps) on config 3: the same frame rendered with the reference's
constant grey and with an orbit trap on the Mandelbox's material (the example range of tools/trap_range.py).

    python tools/bench_trap.py [--res 1920x1080] [--samples 128] [--bounces 8] [--reps 3] [--json out.json]

Each arm is warmed up once, then the arms alternate `reps` times on one context with RAYN_FLAG_TIMING: frame time is the
device time of the render call (RaynStats.total_ms, CUDA events around the whole frame), and k_normals / k_shade_pre /
k_shade_post are the summed per-launch CUDA-event times.  The host tables are built before the timed window.  Medians are
reported.  Card, power limit and SM clocks are read in the same call.  Needs a GPU; writes nothing unless --json is given."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from rayn_b200 import _lib as L  # noqa: E402
from rayn_b200 import configs  # noqa: E402
from rayn_b200.film import FrameInputs, Renderer  # noqa: E402
from rayn_b200.scene import Dielectric, OrbitTrapAlbedo  # noqa: E402
from trap_range import TRAP_HI, TRAP_LO  # noqa: E402

TR = configs.frame_time_range(1)
ALBEDO_LO, ALBEDO_HI = (0.9, 0.35, 0.1), (0.1, 0.3, 0.8)
KERNELS = ("normals", "shade_pre", "shade_post", "extend", "shadow")


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except Exception as e:
        return f"unavailable: {e}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", default="1920x1080")
    ap.add_argument("--samples", type=int, default=128)
    ap.add_argument("--bounces", type=int, default=8)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    w, h = (int(v) for v in a.res.split("x"))
    plain = configs.baseline_config(3, res=(w, h), samples=a.samples, max_bounces=a.bounces)
    trap = configs.baseline_config(3, res=(w, h), samples=a.samples, max_bounces=a.bounces)
    mats = trap["world"].materials.items
    mats[1] = Dielectric(OrbitTrapAlbedo(TRAP_LO, TRAP_HI, ALBEDO_LO, ALBEDO_HI), mats[1].roughness)
    inp = FrameInputs(w, h, a.samples, plain["integrator"])
    r = Renderer(0, flags=L.FLAG_TIMING)
    res = {"plain": [], "trap": []}
    try:
        for rep in range(a.reps + 1):
            for name, c in (("plain", plain), ("trap", trap)):
                r.upload_scene(c["world"], c["camera"])
                r.render_host(inp, (16, 16), c["integrator"], TR)
                st = r.stats()
                if rep == 0:
                    continue  # warm-up
                ms = {k: float(st.kernel_ms[L.KERNEL_NAMES.index(k)]) for k in KERNELS}
                res[name].append(dict(frame_ms=float(st.total_ms), evals_normals=int(st.sdf_evals_normals), **ms))
    finally:
        r.close()
    med = {n: {k: float(np.median([x[k] for x in v])) for k in v[0]} for n, v in res.items()}
    out = dict(gpu=gpu_info(), res=[w, h], spp=4 * a.samples, bounces=a.bounces, trap=[TRAP_LO, TRAP_HI], median=med, runs=res)
    print(f"config 3 {w}x{h}, {4 * a.samples} spp, {a.bounces} bounces; {out['gpu']}")
    print(f"{'ms (median of ' + str(a.reps) + ')':24s}{'plain':>10s}{'trap':>10s}{'delta':>10s}")
    for k in ("frame_ms",) + KERNELS:
        p, t = med["plain"][k], med["trap"][k]
        print(f"{k:24s}{p:10.1f}{t:10.1f}{100 * (t / p - 1):+9.1f}%")
    print(f"frame share of k_normals (plain): {100 * med['plain']['normals'] / med['plain']['frame_ms']:.1f} %")
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
