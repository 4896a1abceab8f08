"""Regenerates tests/golden/cfg3_trap_albedo_32x32_8spp{,_fma}.npz: the first-hit albedo plane of the config-3 trap scene of
cfg3_trap_32x32_8spp_3b (tests/golden/make_golden_trap.py), computed by the CPU albedo mirror (tests/albedo_oracle.py).  Run
once per mul_add variant from the repo root:
    python tests/golden/make_golden_albedo.py;  RAYN_MULADD_FUSED=1 python tests/golden/make_golden_albedo.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import albedo_oracle  # noqa: E402
from rayn_b200 import configs  # noqa: E402
from test_cpu_trap import trap_golden_config  # noqa: E402
from test_cpu_oracle import GOLD_SUFFIX  # noqa: E402

ALBEDO_GOLDEN = "cfg3_trap_albedo_32x32_8spp"

if __name__ == "__main__":
    c, inp = trap_golden_config()
    plane, _ = albedo_oracle.render_albedo(c["world"], c["camera"], inp, (16, 16), c["integrator"], configs.frame_time_range(1))
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", ALBEDO_GOLDEN + GOLD_SUFFIX + ".npz"), albedo=plane)
    print(ALBEDO_GOLDEN + GOLD_SUFFIX, float(plane.mean()))
