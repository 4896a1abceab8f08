"""Orbit-trap distribution of config 3's first hits, on the CPU: pinhole camera rays through pixel centres, the render
oracle's closest hit, then the trap oracle's trap (tests/trap_oracle.py) at every hit on the Mandelbox.  Its 5th and 95th
percentiles are the example trap range documented in the README and DESIGN.md §4d (TRAP_LO / TRAP_HI below, used by
tools/bench_trap.py and the trap golden fixture).  Needs no GPU.

    python tools/trap_range.py [--res 480x270] [--config 3]
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))  # the trap oracle (tests/trap_oracle.py) is test infrastructure

# printed by this script for config 3 at 480x270, rounded (5th percentile 0.66756, 95th 1.45031; the fused mul_add oracle
# agrees to 5 digits)
TRAP_LO, TRAP_HI = 0.6676, 1.45


def camera_rays(cam, w, h):
    """camera.rs:81-114 at the pixel centres (float64: the rays only sample the distribution)"""
    o, at, up = (np.array(v, np.float64) for v in (cam.origin, cam.at, cam.up))
    n = lambda v: v / np.linalg.norm(v, axis=-1, keepdims=True)
    bw = n(o - at)
    bu = n(np.cross(up, bw))
    bv = np.cross(bw, bu)
    hx, hy = cam.half_size
    u, v = np.meshgrid((np.arange(w) + 0.5) / w, (np.arange(h) + 0.5) / h)
    ll = o - bu * hx - bv * hy - bw
    d = ll + bu * (hx * 2.0) * u.reshape(-1, 1) + bv * (hy * 2.0) * v.reshape(-1, 1) - o
    return np.broadcast_to(o, d.shape).astype(np.float32), n(d).astype(np.float32)


def first_hit_traps(config=3, res=(480, 270)):
    import trap_oracle
    from oracle import binding as ob
    from rayn_b200 import _lib as L
    from rayn_b200 import configs
    c = configs.baseline_config(config, res=res)
    desc, keep = c["world"].flatten(c["camera"])
    o, d = camera_rays(desc.camera, *res)
    t, obj = ob.kat_closest_hit(desc, 0, o, d)
    sdf = [i for i in range(desc.n_hitables) if desc.hitables[i].kind != L.HITABLE_SPHERE][0]
    hit = obj == sdf
    p = (d[hit] * t[hit, None] + o[hit]).astype(np.float32)
    return trap_oracle.kat_sdf_trap(desc.hitables[sdf], p), hit.mean()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", type=int, default=3)
    ap.add_argument("--res", default="480x270")
    a = ap.parse_args()
    res = tuple(int(v) for v in a.res.split("x"))
    traps, frac = first_hit_traps(a.config, res)
    p5, p50, p95 = (np.float32(np.percentile(traps, q)) for q in (5, 50, 95))
    print(f"config {a.config} at {res[0]}x{res[1]}: {traps.size} camera rays hit the fractal ({100 * frac:.1f} %)")
    print(f"trap percentiles: 5th {p5!r}  50th {p50!r}  95th {p95!r}  (min {traps.min()!r}, max {traps.max()!r})")
    print(f"TRAP_LO, TRAP_HI = {float(p5):.4g}, {float(p95):.4g}")


if __name__ == "__main__":
    main()
