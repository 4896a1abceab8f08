"""Regenerates tests/golden/cfg3_trap_32x32_8spp_3b{,_fma}.npz: the config-3 film with an orbit-trap albedo on the Mandelbox
(the example range of tools/trap_range.py), rendered by the CPU trap oracle (tests/trap_oracle.py).  Run once per mul_add variant from the repo root:
    python tests/golden/make_golden_trap.py;  RAYN_MULADD_FUSED=1 python tests/golden/make_golden_trap.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import trap_oracle  # noqa: E402
from rayn_b200 import configs  # noqa: E402
from test_cpu_trap import TRAP_GOLDEN, trap_golden_config  # noqa: E402
from test_cpu_oracle import GOLD_SUFFIX  # noqa: E402

if __name__ == "__main__":
    c, inp = trap_golden_config()
    o, info = trap_oracle.render(c["world"], c["camera"], inp, (16, 16), c["integrator"], configs.frame_time_range(1))
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", TRAP_GOLDEN + GOLD_SUFFIX + ".npz"), **o)
    print(TRAP_GOLDEN + GOLD_SUFFIX, info)
