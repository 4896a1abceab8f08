"""Regenerates tests/golden/detmath_sweep.json: exhaustive sweeps of rayn_b200/csrc/detmath.h over 32-bit input patterns
(tests/detmath_sweep.cpp).  CPU only; about half an hour on 8 threads.  Run from the repo root:
    python tests/golden/make_golden_detmath.py
Per sweep it records the 256 chunk hashes of every output bit pattern and the worst error against long-double libm over
the sweep's accuracy chunks: all 2^32 inputs for every unary function and post_gamma's pow(x, 1/2.2); every x in [0, 1]
(chunks 0x00-0x3f) and the check chunks for the pow exponents of the configs' Dielectric; otherwise CHECK_CHUNKS (the
chunks tests/test_cpu_shared_numerics.py recomputes).  powi5 is checked bit for bit against its
definition x * ((x * x) * (x * x)) restated in numpy float32, over every input, before anything is written.
"""
import hashlib
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import mirrors as M  # noqa: E402
from rayn_b200.scene import Dielectric, Srgb  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "detmath_sweep.json")
DETMATH = os.path.join(ROOT, "rayn_b200", "csrc", "detmath.h")
ULP_BOUND = 0.5 + 2.0 ** -20   # correctly rounded but for the reference's own last bits
LN_FAST_BOUND = 2.0 ** -22     # relative (absolute where |ln x| < 1)
# +0 and the subnormals, 1/2.2, [0.5, 2) (pi/2), [2, 8) (2 pi), +inf and NaN, -0, -pi/2, exp's subnormal outputs, -inf
CHECK_CHUNKS = [0x00, 0x3e, 0x3f, 0x40, 0x7f, 0x80, 0xbf, 0xc2, 0xff]
OPS = {"exp": 0, "ln": 1, "pow": 2, "sin": 3, "cos": 4, "tan": 5, "atan2": 6, "powi5": 7, "ln_fast": 8}
f32 = np.float32


def render_exponents():
    """the pow exponents of the configs' Dielectric (rayn_b200/configs.py): its roughness (the specular lobe) and
    1 / (roughness + 1) (cosine_power)"""
    r = f32(Dielectric.new_remap(Srgb(0.2, 0.2, 0.2), 0.6).roughness)
    return [r, f32(1) / (r + f32(1))]


ALL, UNIT = list(range(256)), sorted(set(range(0x40)) | set(CHECK_CHUNKS))  # UNIT: x in [0, 1] (u0, cos) and the check chunks


def sweeps():
    """(name, op, fixed operand float32, swap: the second operand is swept, the chunks whose error is measured)"""
    out = [(n, OPS[n], f32(0), False, [] if n == "powi5" else ALL) for n in ("exp", "ln", "sin", "cos", "tan", "powi5", "ln_fast")]
    out.append(("pow(x, 1/2.2)", 2, f32(1) / f32(2.2), False, ALL))  # post_gamma
    out += [(f"pow(x, {float(y)!r})", 2, y, False, UNIT) for y in render_exponents()]
    out += [(f"pow(x, {float(y)!r})", 2, f32(y), False, CHECK_CHUNKS) for y in (0.5, 1, 3, 12, 1000)]
    out += [(f"atan2(y, {float(x)!r})", 6, f32(x), False, CHECK_CHUNKS) for x in (0.0, -0.0, 1e-30, 1, -1, 1e30, np.inf)]
    out += [(f"pow({float(x)!r}, y)", 2, f32(x), True, CHECK_CHUNKS) for x in (0.5, 0.999, 2)]
    out += [(f"atan2({float(y)!r}, x)", 6, f32(y), True, CHECK_CHUNKS) for y in (0.0, -0.0, 1, -1, np.inf)]
    return out


def bits(x):
    return int(np.asarray(x, np.float32).view(np.uint32))


def splitmix64(z):
    z = z + np.uint64(0x9E3779B97F4A7C15)
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def powi5_chunk_hash(chunk):
    """the chunk hash of x * ((x * x) * (x * x)) in numpy float32"""
    x_bits = np.arange(chunk << 24, (chunk + 1) << 24, dtype=np.uint64)
    x = x_bits.astype(np.uint32).view(np.float32)
    with np.errstate(all="ignore"):
        x2 = x * x
        y = x * (x2 * x2)
    y_bits = np.where(np.isnan(y), np.uint32(0x7FC00000), y.view(np.uint32))  # the sweep's NaN of powi5
    h = splitmix64((x_bits << np.uint64(32)) | y_bits.astype(np.uint64))
    return int(h.sum(dtype=np.uint64))


def acc_json(a):
    return {"max": a["max"], "argmax": f"0x{a['argmax']:08x}", "over": a["over"]}


def run(name, op, fixed, swap, acc_chunks):
    bound = LN_FAST_BOUND if op == OPS["ln_fast"] else ULP_BOUND
    rec = {"name": name, "op": op, "fixed": f"0x{bits(fixed):08x}", "swap": swap, "bound": bound, "accuracy_chunks": acc_chunks}
    accurate = bool(acc_chunks)
    hashes, acc = M.detmath_sweep(op, fixed, swap, 0, 256, acc_chunks == ALL, bound)
    if accurate and acc_chunks != ALL:
        parts = [M.detmath_sweep(op, fixed, swap, c, 1, True, bound) for c in acc_chunks]
        for c, (h, _) in zip(acc_chunks, parts):
            assert h[0] == hashes[c], (name, c)
        acc = tuple(max((p[1][k] for p in parts), key=lambda a: (a["max"], -a["argmax"])) | {"over": sum(p[1][k]["over"] for p in parts)}
                    for k in range(2))
    if op == OPS["powi5"]:
        for c in range(256):
            if powi5_chunk_hash(c) != int(hashes[c]):
                raise SystemExit(f"powi5 differs from x * ((x * x) * (x * x)) in chunk 0x{c:02x}")
    rec["hashes"] = [f"0x{int(h):016x}" for h in hashes]
    if accurate:
        rec["contract"], rec["render"] = acc_json(acc[0]), acc_json(acc[1])
    return rec


if __name__ == "__main__":
    out = {"detmath_sha256": hashlib.sha256(open(DETMATH, "rb").read()).hexdigest(), "check_chunks": CHECK_CHUNKS, "sweeps": []}
    if len(sys.argv) > 1:  # a quick look at some sweeps: python tests/golden/make_golden_detmath.py <name>...; writes nothing
        for s in sweeps():
            if s[0] in sys.argv[1:]:
                print(s[0], {k: v for k, v in run(*s).items() if k not in ("hashes", "accuracy_chunks")}, flush=True)
        sys.exit(0)
    for s in sweeps():
        t = time.time()
        out["sweeps"].append(run(*s))
        r = out["sweeps"][-1]
        print(f"{s[0]:24s} {time.time() - t:7.1f} s", r.get("contract"), r.get("render"), flush=True)
    with open(GOLDEN, "w") as fh:
        json.dump(out, fh, indent=1)
        fh.write("\n")
