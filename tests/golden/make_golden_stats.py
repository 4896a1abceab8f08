"""Regenerates tests/golden/host_driver_stats.json: the RaynStats of the host-driver cases of tests/test_gpu_host_driver.py, per
library variant.  Needs a GPU.  Run once per mul_add variant from the repo root:
    python tests/golden/make_golden_stats.py;  RAYN_MULADD_FUSED=1 python tests/golden/make_golden_stats.py
Every case runs twice.  The pass and launch counts, paths and reserved_ must agree between the runs; a ray or evaluation
counter is recorded only where they agree.
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from rayn_b200 import _lib as L  # noqa: E402
from test_gpu_host_driver import CASES, COUNTERS, GOLDEN, STRUCTURE  # noqa: E402

if __name__ == "__main__":
    runs = [{case: f() for case, f in CASES.items()} for _ in range(2)]
    stats = {}
    for case in CASES:
        calls = []
        for a, b in zip(runs[0][case], runs[1][case]):
            for k in STRUCTURE:
                if a[k] != b[k]:
                    raise SystemExit(f"{case}: {k} differs between two runs: {a[k]} vs {b[k]}")
            calls.append({k: v for k, v in a.items() if k not in COUNTERS or v == b[k]})
        stats[case] = calls
    data = {}
    if os.path.exists(GOLDEN):
        with open(GOLDEN) as fh:
            data = json.load(fh)
    data[L.LIB_NAME] = stats
    with open(GOLDEN, "w") as fh:
        json.dump(data, fh, indent=1, sort_keys=True)
        fh.write("\n")
    dropped = sorted({k for calls in stats.values() for c in calls for k in COUNTERS if k not in c})
    print(L.LIB_NAME, "cases:", len(stats), "counters not recorded (they differ between runs):", dropped or "none")
