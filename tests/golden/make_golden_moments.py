"""Regenerates tests/golden/cfg3_moments_32x32_8spp{,_fma}.npz: the film and moment planes of the config-3 trap scene of
cfg3_trap_32x32_8spp_3b (tests/golden/make_golden_trap.py), computed by the CPU moments mirror (tests/moments_oracle.py).  Run
once per mul_add variant from the repo root:
    python tests/golden/make_golden_moments.py;  RAYN_MULADD_FUSED=1 python tests/golden/make_golden_moments.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import moments_oracle  # noqa: E402
from rayn_b200 import configs  # noqa: E402
from test_cpu_trap import trap_golden_config  # noqa: E402
from test_cpu_oracle import GOLD_SUFFIX  # noqa: E402

MOMENTS_GOLDEN = "cfg3_moments_32x32_8spp"

if __name__ == "__main__":
    c, inp = trap_golden_config()
    planes = moments_oracle.render(c["world"], c["camera"], inp, (16, 16), c["integrator"], configs.frame_time_range(1))
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", MOMENTS_GOLDEN + GOLD_SUFFIX + ".npz"), **planes)
    print(MOMENTS_GOLDEN + GOLD_SUFFIX, float(planes["moments"].mean()))
