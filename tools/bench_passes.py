"""Measures the fixed cost of a render pass: config 3 rendered with several pass sizes, and a least-squares fit of
time = passes * a + samples * b.

    python tools/bench_passes.py [--res 1920x1080] [--samples 128] [--frames 3] [--max-paths 16,32,64,96,max] [--json out.json]

Every frame is the bench.py headline (config 3, 16x16 tiles, device-resident inputs and film) rendered with
max_paths_per_pass set to each value of --max-paths, in Mi paths; "max" asks for 2^27 - 1, the most a pass of an SDF scene
may hold, and the driver then sizes the pass from free device memory.  Per setting: one warm-up frame, then the median of
--frames frames of device time (RaynStats.total_ms) and the passes per frame.  All settings render the same samples, so
the fit's samples * b is one constant and a is the slope of time over passes: what each pass costs beyond its share of
the work (kernel tails, march drains, single-CTA scans, underfilled deep depths).  Card, power limit and SM clock are
read in the same call.  Needs a GPU; prints one JSON line and writes nothing unless --json is given."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from rayn_b200 import _lib as L  # noqa: E402
from rayn_b200 import configs  # noqa: E402
from rayn_b200.dist import device_frame_desc  # noqa: E402
from rayn_b200.film import FrameInputs, Renderer  # noqa: E402

TILE = (16, 16)
MAX_SDF_PATHS = (1 << 27) - 1


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except Exception as e:  # the timing itself does not depend on it
        return f"unavailable: {e}"


def parse_caps(s):
    return [MAX_SDF_PATHS if v == "max" else int(v) << 20 for v in s.split(",")]


def fit(passes, ms, samples):
    """Least squares of ms = passes * a + c; b = c / samples (every point renders the same samples)."""
    A = np.stack([np.asarray(passes, dtype=np.float64), np.ones(len(passes))], axis=1)
    (a, c), *_ = np.linalg.lstsq(A, np.asarray(ms, dtype=np.float64), rcond=None)
    return float(a), float(c) / samples


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--res", default="1920x1080")
    ap.add_argument("--samples", type=int, default=None, help="4 * samples spp (default: config 3's own)")
    ap.add_argument("--frames", type=int, default=3)
    ap.add_argument("--max-paths", default="16,32,64,96,max", help="pass sizes in Mi paths; 'max' = 2^27 - 1")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    w, h = (int(v) for v in args.res.split("x"))
    c = configs.baseline_config(3, res=(w, h), samples=args.samples)
    tr = configs.frame_time_range(1)
    inputs = FrameInputs(w, h, c["samples"], c["integrator"])
    dev = torch.device("cuda:0")
    inputs_dev = [torch.from_numpy(a).to(dev) for a in inputs.arrays()]
    fdesc = device_frame_desc(inputs_dev, w, h, TILE, c["samples"], c["integrator"], 1, tr, (inputs.sets_1d, inputs.sets_2d))
    film = torch.zeros(10 * w * h, dtype=torch.float32, device=dev)
    npx = w * h
    planes = L.RaynFilmPlanes(film[:3 * npx].data_ptr(), film[3 * npx:4 * npx].data_ptr(), film[4 * npx:7 * npx].data_ptr(),
                              film[7 * npx:].data_ptr(), L.MEM_DEVICE)
    torch.cuda.synchronize()
    info_before = gpu_info()
    rows, ref_film, samples = [], None, None
    for cap in parse_caps(args.max_paths):
        r = Renderer(0, max_paths_per_pass=cap)
        try:
            r.upload_scene(c["world"], c["camera"])
            r.render(fdesc, planes)  # warm-up: module load, pass buffers
            ms, passes = [], set()
            for _ in range(args.frames):
                r.render(fdesc, planes)
                st = r.stats()
                ms.append(st.total_ms)
                passes.add(int(st.passes))
                samples = int(st.paths)
            torch.cuda.synchronize()
        finally:
            r.close()
        if ref_film is None:
            ref_film = film.clone()
        same = bool(torch.equal(film.view(torch.int32), ref_film.view(torch.int32)))  # passes never change the film
        rows.append({"max_paths": cap, "passes": passes.pop() if len(passes) == 1 else sorted(passes), "ms_median": statistics.median(ms),
                     "ms": ms, "film_equal": same})
        print(json.dumps(rows[-1]), file=sys.stderr, flush=True)
    a, b = fit([r["passes"] for r in rows], [r["ms_median"] for r in rows], samples)
    frame_ms = rows[-1]["ms_median"]
    res = {"tool": "bench_passes", "config": 3, "res": f"{w}x{h}", "spp": 4 * c["samples"], "samples": samples, "frames": args.frames,
           "rows": rows, "fit": {"a_ms_per_pass": a, "b_ns_per_sample": b * 1e6,
                                 "a_share_of_frame_at_largest_pass": a * rows[-1]["passes"] / frame_ms if isinstance(rows[-1]["passes"], int) else None},
           "gpu_before": info_before, "gpu_after": gpu_info()}
    line = json.dumps(res)
    print(line)
    if args.json:
        with open(args.json, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
