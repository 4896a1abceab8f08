"""Measures adaptive sampling (rayn_b200_accum_round) against uniform progressive rendering on config 3, and the cost of
the accumulator's own kernels.

    python tools/bench_adaptive.py [--res 1920x1080] [--samples 4] [--rounds 32] [--thresholds 0.3,0.2,...] [--ref-samples 512]
                                   [--json out.json]

Every film is config 3 (setup.rs, 8 bounces, time range of frame 1) in rounds of 4 * samples spp on 16x16 tiles.
  reference  one render_frame of 4 * ref_samples spp whose sample tables use `frame` 1000, so the measured films (frame
             1) share none of its samples and their error is not read too low
  uniform    threshold -1: every tile renders every round; time and col+bg MSE against the reference after every round
  adaptive   one run per threshold, max_rounds = rounds: final time, samples spent, MSE, active tiles and ms per round
Each threshold's time is compared with the uniform arm's time to the same MSE, interpolated log-log between rounds.
A round's time is the host clock around accum_round, which ends in a stream synchronise; resolving the film and the MSE
happen outside the timed window.  Every shape is warmed up first.  The fold + error kernel (k_accum_fold) is timed with
torch.profiler (CUPTI kernel records) in a run of its own.  Card, power limit and SM clocks are read in the same call.
Needs a GPU; writes nothing unless --json is given."""
import argparse
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
from rayn_b200.film import FrameInputs, Renderer, make_frame_desc  # noqa: E402

TILE = (16, 16)
TR = configs.frame_time_range(1)


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except Exception as e:  # the timing itself does not depend on it
        return f"unavailable: {e}"


class Driver:
    """One config-3 scene on one context, rendering into accumulators with host tables (FrameInputs first_sample)."""

    def __init__(self, r, w, h, samples):
        self.r, self.w, self.h, self.samples = r, w, h, samples
        self.c = configs.baseline_config(3, res=(w, h), samples=samples)
        r.upload_scene(self.c["world"], self.c["camera"])
        self.tables = {}

    def frame(self, first):
        if first not in self.tables:  # built before any timed window
            inp = FrameInputs(self.w, self.h, self.samples, self.c["integrator"], frame=1, first_sample=first)
            ptrs = tuple(a.ctypes.data for a in inp.arrays())
            f = make_frame_desc(self.w, self.h, TILE, self.samples, self.c["integrator"], 1, TR, ptrs, L.MEM_HOST,
                                sets=(inp.sets_1d, inp.sets_2d))
            self.tables[first] = (inp, f)
        return self.tables[first][1]

    def run(self, rounds, threshold, ref_img=None, per_round_mse=False):
        spp = 4 * self.samples
        for k in range(rounds):
            self.frame(k * spp)
        acc = self.r.accum_create(self.w, self.h, TILE)
        out = dict(threshold=threshold, ms=[], active=[], mse=[], cum_ms=[])
        total = 0.0
        try:
            for k in range(rounds + 1):
                f = self.frame(k * spp) if k < rounds else self.frame(0)
                t0 = time.perf_counter()
                n = self.r.accum_round(acc, f, 2, rounds, threshold)
                ms = (time.perf_counter() - t0) * 1e3
                if n == 0:
                    break
                total += ms
                out["ms"].append(ms)
                out["active"].append(n)
                out["cum_ms"].append(total)
                if per_round_mse and ref_img is not None:
                    out["mse"].append(mse(self.r.accum_resolve(acc), ref_img))
                    out.setdefault("err_p75", []).append(float(np.quantile(self.r.accum_tiles(acc)[0], 0.75)))
            err, k = self.r.accum_tiles(acc)
            film = self.r.accum_resolve(acc)
        finally:
            acc.close()
        out["time_ms"] = total
        out["n_rounds"] = len(out["ms"])
        out["mean_spp"] = float(k.mean())
        out["final_mse"] = mse(film, ref_img) if ref_img is not None else None
        out["err_quantiles"] = {q: float(np.quantile(err, q)) for q in (0.1, 0.25, 0.5, 0.75, 0.9)}
        return out


def mse(planes, ref_img):
    img = planes["color"].astype(np.float64) + planes["background"]
    return float(np.mean((img - ref_img) ** 2))


def reference(w, h, samples):
    c = configs.baseline_config(3, res=(w, h), samples=samples)
    inp = FrameInputs(w, h, samples, c["integrator"], frame=1000)
    r = Renderer(0)  # a context of its own: its large pass buffers are released before anything is timed
    try:
        r.upload_scene(c["world"], c["camera"])
        t0 = time.perf_counter()
        p = r.render_host(inp, TILE, c["integrator"], TR)
        return p["color"].astype(np.float64) + p["background"], (time.perf_counter() - t0) * 1e3
    finally:
        r.close()


def time_to_mse(uniform, target):
    """Uniform time at which its MSE reaches `target`, interpolated linearly in log(time), log(MSE) between rounds; None if
    the target lies beyond the uniform arm's rounds."""
    t, m = np.log(uniform["cum_ms"]), np.log(uniform["mse"])
    if target >= uniform["mse"][0]:
        return float(uniform["cum_ms"][0]) if target == uniform["mse"][0] else None
    for i in range(1, len(m)):
        if np.log(target) >= m[i]:
            a = (np.log(target) - m[i - 1]) / (m[i] - m[i - 1])
            return float(np.exp(t[i - 1] + a * (t[i] - t[i - 1])))
    return None


def fold_kernel_time(d):
    """Round 2 of a fresh accumulator (every tile active, with the error) under torch.profiler: k_accum_fold's device time
    and the round's."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    acc = d.r.accum_create(d.w, d.h, TILE)
    try:
        d.r.accum_round(acc, d.frame(0), 2, 4, -1.0)
        f = d.frame(4 * d.samples)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            t0 = time.perf_counter()
            n = d.r.accum_round(acc, f, 2, 4, -1.0)
            round_ms = (time.perf_counter() - t0) * 1e3
    finally:
        acc.close()
    fold_us, all_us, n_fold = 0.0, 0.0, 0
    for e in prof.events():
        dt = e.device_time
        if e.device_type == torch.autograd.DeviceType.CUDA:
            all_us += dt
            if "k_accum_fold" in e.name:
                fold_us += dt
                n_fold += 1
    return dict(tiles=n, round_ms=round_ms, fold_ms=fold_us / 1e3, fold_launches=n_fold, device_ms_all_kernels=all_us / 1e3,
                fold_share_of_round=fold_us / 1e3 / round_ms)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", default="1920x1080")
    ap.add_argument("--samples", type=int, default=4, help="4 * samples spp per round")
    ap.add_argument("--rounds", type=int, default=32)
    ap.add_argument("--thresholds", default="0.2,0.1,0.05,0.04,0.03,0.025,0.02,0.015,0.01,0.007,0.005,0.003,0.002,0.001")
    ap.add_argument("--ref-samples", type=int, default=512, help="4 * ref_samples spp for the reference film")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    w, h = (int(v) for v in a.res.split("x"))
    res = dict(gpu_before=gpu_info(), res=a.res, spp_per_round=4 * a.samples, rounds=a.rounds)
    print(json.dumps(dict(gpu=res["gpu_before"])), flush=True)
    ref_img, ref_ms = reference(w, h, a.ref_samples)
    res["reference"] = dict(spp=4 * a.ref_samples, frame=1000, ms=ref_ms)
    print(json.dumps(res["reference"]), flush=True)
    r = Renderer(0)
    try:
        d = Driver(r, w, h, a.samples)
        d.run(2, -1.0)  # warm-up: module load, pass buffers, the accumulator's kernels
        uni = d.run(a.rounds, -1.0, ref_img, per_round_mse=True)
        res["uniform"] = uni
        print(json.dumps(dict(arm="uniform", time_ms=uni["time_ms"], final_mse=uni["final_mse"], mse=uni["mse"], cum_ms=uni["cum_ms"],
                              err_p75=uni["err_p75"], err_quantiles=uni["err_quantiles"])), flush=True)
        res["adaptive"] = []
        for thr in (float(t) for t in a.thresholds.split(",")):
            ad = d.run(a.rounds, thr, ref_img)
            ad["uniform_ms_same_mse"] = time_to_mse(uni, ad["final_mse"])
            ad["speedup"] = ad["uniform_ms_same_mse"] / ad["time_ms"] if ad["uniform_ms_same_mse"] else None
            res["adaptive"].append(ad)
            print(json.dumps(dict(arm="adaptive", **{k: ad[k] for k in ("threshold", "time_ms", "n_rounds", "mean_spp", "final_mse",
                                                                      "uniform_ms_same_mse", "speedup", "active", "ms")})), flush=True)
        res["fold"] = fold_kernel_time(d)
        print(json.dumps(res["fold"]), flush=True)
    finally:
        r.close()
    res["gpu_after"] = gpu_info()
    print(json.dumps(dict(gpu_after=res["gpu_after"])), flush=True)
    print("\n| threshold | rounds | mean spp | time ms | col+bg MSE | uniform ms to same MSE | speedup |")
    print("|---|---|---|---|---|---|---|")
    u = res["uniform"]
    print(f"| uniform | {u['n_rounds']} | {u['mean_spp']:.0f} | {u['time_ms']:.0f} | {u['final_mse']:.4g} | | |")
    for ad in res["adaptive"]:
        same = f"{ad['uniform_ms_same_mse']:.0f}" if ad["uniform_ms_same_mse"] else "beyond uniform"
        sp = f"{ad['speedup']:.2f}" if ad["speedup"] else "-"
        print(f"| {ad['threshold']:g} | {ad['n_rounds']} | {ad['mean_spp']:.1f} | {ad['time_ms']:.0f} | {ad['final_mse']:.4g} | {same} | {sp} |")
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
