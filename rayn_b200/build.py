"""In-tree build of the native libraries for sm_90a (H100) (nvcc cross-compiles without a GPU).

  librayn_b200.so         the product: wavefront kernels + C ABI, `wide` mul_add UNFUSED (stock `cargo run --release` rayn)
  librayn_b200_fma.so     same with -DRAYN_MULADD_FUSED=1 (a `-C target-feature=+fma` rayn); selected by RAYN_MULADD_FUSED=1
  librayn_b200_legacy.so  TEST BUILD: additionally carries the round-1 one-thread-per-ray kernels (-DRAYN_LEGACY_KERNELS)
  librayn_hostinputs.so   pure-CPU builders of the host-owned frame inputs (sampler tables, scramble, filter table, tile
                          grid) for consumers that must not map the CUDA library (bench.py --impl reference)
  rayn_host               C++ stand-in for rayn's main.rs on top of the C ABI

The arithmetic flags are part of the parity contract (csrc/detmath.h): no implicit FMA
contraction, IEEE division and square root, no flush-to-zero.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT_DIR = os.path.join(HERE, "_build")
OUT = os.path.join(OUT_DIR, "librayn_b200.so")
SOURCES = [os.path.join(CSRC, "api.cu"), os.path.join(CSRC, "host_inputs.cpp")]
DEPS = SOURCES + [os.path.join(CSRC, f) for f in ("rt_kernels.cuh", "rt_device.cuh", "rt_sdf2.cuh", "rt_legacy.cuh", "rt_denoise.cuh", "rt_accum.cuh", "rt_first_hit.cuh", "rt_temporal.cuh", "detmath.h")] + [
    os.path.join(HERE, "..", "include", "rayn_b200.h")]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo",
    "--fmad=false", "-prec-div=true", "-prec-sqrt=true", "-ftz=false",
    "-Xcompiler", "-fPIC,-ffp-contract=off,-fno-fast-math", "-shared", "-ldl",
]
VARIANTS = {  # file name -> extra defines
    "librayn_b200.so": ["-DRAYN_MULADD_FUSED=0"],
    "librayn_b200_fma.so": ["-DRAYN_MULADD_FUSED=1"],
    "librayn_b200_legacy.so": ["-DRAYN_MULADD_FUSED=0", "-DRAYN_LEGACY_KERNELS"],
}
if os.environ.get("RAYN_BUILD_EXPERIMENTS"):  # tuning experiments only (selected with RAYN_B200_LIB=<file name>)
    for occ in os.environ["RAYN_BUILD_EXPERIMENTS"].split(","):
        if occ.startswith("p"):  # "p7": k_shade_pre at 7 CTAs per SM
            VARIANTS[f"librayn_b200_occ{occ}.so"] = ["-DRAYN_MULADD_FUSED=0", f"-DRAYN_SHADE_PRE_OCC={occ[1:]}"]
        elif occ.startswith("b"):  # "b6": only the Mandelbulb march kernels at 6 CTAs per SM
            VARIANTS[f"librayn_b200_occ{occ}.so"] = ["-DRAYN_MULADD_FUSED=0", f"-DRAYN_MARCH_OCC_BULB={occ[1:]}"]
        else:
            VARIANTS[f"librayn_b200_occ{occ}.so"] = ["-DRAYN_MULADD_FUSED=0", f"-DRAYN_MARCH_OCC={occ}"]
HOSTINPUTS = os.path.join(OUT_DIR, "librayn_hostinputs.so")


def _outputs():
    return [os.path.join(OUT_DIR, n) for n in VARIANTS] + [HOSTINPUTS]


def needs_build():
    t = None
    for o in _outputs():
        if not os.path.exists(o):
            return True
        t = os.path.getmtime(o) if t is None else min(t, os.path.getmtime(o))
    return any(os.path.getmtime(d) > t for d in DEPS if os.path.exists(d))


def build(force=False, verbose=False):
    if not force and not needs_build():
        if not os.path.exists(os.path.join(OUT_DIR, "rayn_host")):
            build_host()
        return OUT
    os.makedirs(OUT_DIR, exist_ok=True)
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    procs = []
    for name, defs in VARIANTS.items():
        cmd = [nvcc] + NVCC_FLAGS + defs + (["-Xptxas", "-v"] if verbose else []) + ["-o", os.path.join(OUT_DIR, name)] + SOURCES
        procs.append((name, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    cmd = ["g++", "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-shared", "-o", HOSTINPUTS, os.path.join(CSRC, "host_inputs.cpp")]
    procs.append(("librayn_hostinputs.so", subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = []
    for name, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            failed.append(name)
            sys.stderr.write(out)
        elif verbose:
            sys.stderr.write(f"==== {name}\n{out}")
    if failed:
        raise RuntimeError("building failed: " + ", ".join(failed))
    build_host()
    return OUT


def build_host():
    """C++ host stand-in (rayn_b200/host): links against the C ABI only."""
    r = subprocess.run(["make", "-C", os.path.join(HERE, "host"), "-B"], capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("building rayn_host failed")
    return os.path.join(OUT_DIR, "rayn_host")


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(OUT)
