"""The numerics the oracle shares with the kernels, against statements that share nothing with them.

rayn_b200/csrc/detmath.h is compiled into the kernels and the oracle alike, and both consume the same R_d tables and scramble
plane, so a defect there passes every parity test.  Here:
- detmath against the exhaustive sweeps of tests/golden/detmath_sweep.json (tests/detmath_sweep.cpp; regenerate with
  tests/golden/make_golden_detmath.py): output hashes and accuracy of a fixed set of chunks recomputed, each recorded worst
  case recomputed with mpmath, and the bounds asserted;
- detmath at every combination of special operands against C99 Annex F (glibc), except the deviations detmath.h lists;
- the R_d tables and the scramble plane against Python-int statements of quasi-rd and rand_core / rand_pcg.
tests/test_gpu_shared_numerics.py holds the device against the same data."""
import ctypes as C
import hashlib
import json
import os

import mpmath as mp
import numpy as np
import pytest

import mirrors as M
from rayn_b200 import _lib as L

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = os.path.join(HERE, "golden", "detmath_sweep.json")
DETMATH = os.path.join(ROOT, "rayn_b200", "csrc", "detmath.h")
ULP_BOUND = 0.5 + 2.0 ** -20  # correctly rounded, up to the reference's own last bits
CONTRACT_ULP = 1.0            # the stated contract of detmath.h
LN_FAST_BOUND = 2.0 ** -22    # ln_fast: relative (absolute where |ln x| < 1)
OP = {"exp": 0, "ln": 1, "pow": 2, "sin": 3, "cos": 4, "tan": 5, "atan2": 6, "powi5": 7, "ln_fast": 8}
f32, u32 = np.float32, np.uint32


def golden():
    with open(GOLDEN) as fh:
        return json.load(fh)


def u2f(bits):
    return float(np.array([bits], np.uint32).view(np.float32)[0])


def f2u(x):
    return int(np.array([x], np.float32).view(np.uint32)[0])


def sweep_ids():
    return [s["name"] for s in golden()["sweeps"]]


def sweep_by_name(name):
    return next(s for s in golden()["sweeps"] if s["name"] == name)


def test_golden_matches_detmath_h():
    h = hashlib.sha256(open(DETMATH, "rb").read()).hexdigest()
    assert h == golden()["detmath_sha256"], "rayn_b200/csrc/detmath.h changed: regenerate tests/golden/detmath_sweep.json with " \
                                            "tests/golden/make_golden_detmath.py (and check what moved)"


# ---- exhaustive sweeps ------------------------------------------------------------------------------------------------
ZEROS_AND_INFINITIES = [0x00, 0x7f, 0x80, 0xff]  # +0 and the subnormals, +inf and NaN, -0 and the negative subnormals, -inf
# per op, the chunks of the swept operand where it is easiest to get wrong: exp's subnormal outputs (0xc2), ln around 1,
# sin / cos / tan around +-pi/2 (0x3f, 0xbf), pow around 1/2.2 and below 1 (0x3e), atan2 around |y| = |x| = 1
HARD_CHUNKS = {0: [0xc2], 1: [0x3f], 2: [0x3e], 3: [0x3f, 0xbf], 4: [0x3f, 0xbf], 5: [0x3f, 0xbf], 6: [0x3f], 7: [0x3f], 8: [0x3f]}


def recheck_chunks(s):
    return ZEROS_AND_INFINITIES + HARD_CHUNKS[s["op"]]


@pytest.mark.parametrize("name", sweep_ids())
def test_sweep_chunks_recomputed(name):
    """the output hashes of the zeros-and-infinities chunks and of the op's hard chunks equal the golden's, and the error
    over the hard chunks is no worse than recorded"""
    s = sweep_by_name(name)
    fixed = u2f(int(s["fixed"], 16))
    for c in recheck_chunks(s):
        accurate = "contract" in s and c in HARD_CHUNKS[s["op"]]
        assert not accurate or c in s["accuracy_chunks"]
        h, acc = M.detmath_sweep(s["op"], fixed, s["swap"], c, 1, accurate, s["bound"])
        assert f"0x{int(h[0]):016x}" == s["hashes"][c], f"{name}: chunk 0x{c:02x} output bits differ from the golden"
        if accurate:
            for dom in (0, 1):
                rec = s[("contract", "render")[dom]]
                assert acc[dom]["max"] <= rec["max"] * (1 + 1e-12), f"{name} chunk 0x{c:02x}: {acc[dom]} worse than recorded {rec}"
                assert acc[dom]["over"] <= rec["over"]


def _mp_ref(op, a, b):
    x, y = mp.mpf(a), mp.mpf(b)
    if op == 0:
        return mp.exp(x)
    if op in (1, 8):
        return mp.log(x)
    if op == 2:
        return mp.power(x, y)
    if op == 3:
        return mp.sin(x)
    if op == 4:
        return mp.cos(x)
    if op == 5:
        return mp.tan(x)
    return mp.atan2(x, y)


def mp_error(op, a, b, got):
    """the sweep's error measure, in mpmath at 40 digits (which has no signed zero: atan2 at a zero y or two infinite
    operands is C99's exact multiple of pi/4)"""
    with mp.workdps(40):
        ref = _mp_ref(op, a, b)
        if op == OP["atan2"] and (a == 0 or (np.isinf(a) and np.isinf(b))):
            ref = (mp.pi if b < 0 or (b == 0 and np.signbit(b)) else 0) if a == 0 else (3 * mp.pi / 4 if b < 0 else mp.pi / 4)
            ref = -ref if np.signbit(a) else ref
        if op == 8:
            return float(abs(mp.mpf(got) - ref) / max(abs(ref), 1))
        if abs(ref) >= mp.mpf(2) ** 128 - mp.mpf(2) ** 103:
            return 0.0 if np.isinf(got) and (got < 0) == (ref < 0) else 1e300
        e = -149 if ref == 0 else max(int(mp.floor(mp.log(abs(ref), 2))) - 23, -149)
        if ref != 0 and abs(ref) >= mp.mpf(2) ** (e + 24):  # log2 rounded up across a power of two
            e += 1
        return float(abs(mp.mpf(got) - ref) / mp.mpf(2) ** e)


@pytest.mark.parametrize("name", [n for n in sweep_ids() if "contract" in sweep_by_name(n)])
def test_sweep_worst_case_in_mpmath(oracle, name):
    """each recorded maximum error, recomputed at its argument with mpmath at 40 digits (which also checks the long-double
    libm reference the sweep used)"""
    s = sweep_by_name(name)
    fixed = u2f(int(s["fixed"], 16))
    for dom in ("contract", "render"):
        v = u2f(int(s[dom]["argmax"], 16))
        a, b = (fixed, v) if s["swap"] else (v, fixed)
        got = float(oracle.kat_detmath(s["op"], np.array([a], f32), np.array([b], f32))[0])
        err = mp_error(s["op"], a, b, got)
        tol = 1e-6 * (2.0 ** -24 if s["op"] == 8 else 1.0)
        assert abs(err - s[dom]["max"]) <= tol, f"{name} {dom} at {a!r}, {b!r}: mpmath {err} vs recorded {s[dom]['max']}"
        assert abs(M.detmath_error(s["op"], a, b, got) - err) <= tol


@pytest.mark.parametrize("name", [n for n in sweep_ids() if "contract" in sweep_by_name(n)])
def test_sweep_bounds(name):
    """correctly rounded on the render-path domains (exp on x <= 0, ln on x > 0, sin / cos on [0, 2 pi], tan on
    (-pi/2, pi/2), every pow and atan2 sweep), within the 1-ulp contract elsewhere (sin / cos / tan on |x| <= 1e5);
    ln_fast within 2^-22 on every positive finite float"""
    s = sweep_by_name(name)
    if s["op"] == OP["ln_fast"]:
        assert s["contract"]["max"] <= LN_FAST_BOUND and s["contract"]["over"] == 0
        return
    assert s["render"]["max"] <= ULP_BOUND and s["render"]["over"] == 0, s["render"]
    assert s["contract"]["max"] <= CONTRACT_ULP, s["contract"]


def test_sweeps_cover_the_render_path():
    """every function hashed over all inputs; the error of every unary function and of post_gamma measured over all
    inputs, of the config Dielectric's pow exponents over every x in [0, 1]; atan2 at the signed zeros and infinities the
    equi-angular sampler can pass"""
    from rayn_b200.scene import Dielectric, Srgb
    g = golden()
    by = {(s["op"], s["fixed"], s["swap"]): s for s in g["sweeps"]}
    for s in g["sweeps"]:
        assert len(s["hashes"]) == 256
        if s["op"] != OP["powi5"]:
            assert set(g["check_chunks"]) <= set(s["accuracy_chunks"]), s["name"]
    for op in range(9):
        if op not in (OP["pow"], OP["atan2"], OP["powi5"]):
            assert by[(op, "0x00000000", False)]["accuracy_chunks"] == list(range(256))
    assert by[(OP["pow"], f"0x{f2u(f32(1) / f32(2.2)):08x}", False)]["accuracy_chunks"] == list(range(256))
    r = f32(Dielectric.new_remap(Srgb(0.2, 0.2, 0.2), 0.6).roughness)
    for y in (r, f32(1) / (r + f32(1))):
        assert set(range(0x40)) <= set(by[(OP["pow"], f"0x{f2u(y):08x}", False)]["accuracy_chunks"])
    for x in (0.0, -0.0, np.inf):
        assert (OP["atan2"], f"0x{f2u(x):08x}", False) in by
    for y in (0.0, -0.0, np.inf):
        assert (OP["atan2"], f"0x{f2u(y):08x}", True) in by


def test_powi5_is_its_definition():
    """powi5(x) = x * ((x * x) * (x * x)) in float32, bit for bit on the check chunks (the golden checked every input)"""
    s = sweep_by_name("powi5")
    for c in recheck_chunks(s):
        x = np.arange(c << 24, (c + 1) << 24, dtype=np.uint64).astype(np.uint32).view(np.float32)
        with np.errstate(all="ignore"):
            x2 = x * x
            y = x * (x2 * x2)
        h = chunk_hash(np.arange(c << 24, (c + 1) << 24, dtype=np.uint64), y)
        assert f"0x{h:016x}" == s["hashes"][c], f"chunk 0x{c:02x}"


def chunk_hash(in_bits, out):
    out_bits = np.where(np.isnan(out), np.uint32(0x7FC00000), out.view(np.uint32))  # the sweep's NaN of powi5
    z = (in_bits << np.uint64(32)) | out_bits.astype(np.uint64)
    z = z + np.uint64(0x9E3779B97F4A7C15)
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return int((z ^ (z >> np.uint64(31))).sum(dtype=np.uint64))


# ---- special operands against C99 Annex F ------------------------------------------------------------------------------
FMIN_SUB, FMIN_NORM, FMAX = u2f(1), u2f(0x00800000), u2f(0x7f7fffff)
SPECIAL = np.array([0.0, -0.0, FMIN_SUB, -FMIN_SUB, FMIN_NORM, -FMIN_NORM, 1.0, -1.0, FMAX, -FMAX, np.inf, -np.inf, np.nan], f32)
UNARY = {"exp": "expf", "ln": "logf", "sin": "sinf", "cos": "cosf", "tan": "tanf", "ln_fast": "logf"}
BINARY = {"pow": "powf", "atan2": "atan2f"}
NAN = float("nan")


def deviation(name, a, b=None):
    """the value detmath.h documents where it departs from C99 Annex F (its comment block 'documented domain
    restrictions'), else None"""
    if name == "pow" and b != 0 and not np.isnan(b):
        if a < 0 or (a == 0 and np.signbit(a) and np.isfinite(b) and b == int(b) and int(b) % 2 == 1):
            return NAN if a < 0 else (0.0 if b > 0 else np.inf)
    if name == "pow" and a == 1 and np.isnan(b):
        return NAN
    if name in ("sin", "cos", "tan") and np.isfinite(a) and abs(a) > 1e5:
        return NAN
    return None


def libm():
    l = C.CDLL("libm.so.6")
    for n in set(UNARY.values()):
        getattr(l, n).restype, getattr(l, n).argtypes = C.c_float, [C.c_float]
    for n in BINARY.values():
        getattr(l, n).restype, getattr(l, n).argtypes = C.c_float, [C.c_float, C.c_float]
    return l


def special_cases():
    """[(name, op, a, b)] over the special operands (pairs for pow and atan2)"""
    out = [(n, OP[n], float(a), 0.0) for n in UNARY for a in SPECIAL]
    out += [(n, OP[n], float(a), float(b)) for n in BINARY for a in SPECIAL for b in SPECIAL]
    return out + [("powi5", OP["powi5"], float(a), 0.0) for a in SPECIAL]


def same_class(got, want):
    """NaN for NaN; +-0 and +-inf with their sign; finite non-zero within 1 ulp of the C99 value"""
    if np.isnan(want) or np.isnan(got):
        return np.isnan(want) and np.isnan(got)
    if want == 0 or np.isinf(want) or got == 0 or np.isinf(got):
        return got == want and np.signbit(got) == np.signbit(want)
    with np.errstate(over="ignore"):  # the spacing above FLT_MAX is inf, which is what 1 ulp means there
        return abs(f32(got) - f32(want)) <= np.spacing(abs(f32(want)))


def test_special_values_match_c99(oracle):
    l = libm()
    bad = []
    pinned = 0
    for name, op, a, b in special_cases():
        got = float(oracle.kat_detmath(op, np.array([a], f32), np.array([b], f32))[0])
        if name == "powi5":
            x = f32(a)
            with np.errstate(all="ignore"):
                want = float(x * ((x * x) * (x * x)))
        elif name in UNARY:
            want = getattr(l, UNARY[name])(a)
        else:
            want = getattr(l, BINARY[name])(a, b)
        dev = deviation(name, a, b)
        if dev is not None:
            pinned += 1
            if not (same_class(got, dev) and (not np.isnan(dev) or np.isnan(got))):
                bad.append((name, a, b, got, "documented", dev))
            continue
        if name == "ln_fast" and np.isfinite(want) and want != 0:
            ok = abs(got - float(mp.log(mp.mpf(a)))) <= LN_FAST_BOUND * max(abs(want), 1.0)
        else:
            ok = same_class(got, want)
        if not ok:
            bad.append((name, a, b, got, "C99", want))
    assert not bad, bad
    assert pinned > 0


def test_documented_deviations_are_listed_in_detmath_h():
    """every deviation the table above allows is written down in detmath.h, and what detmath.h writes down is pinned"""
    src = open(DETMATH).read()
    block = src[src.index("documented domain restrictions"):src.index("DM_HD float pow(")]
    for line in ("pow(x, y), x < 0 (-inf included), y != 0:   NaN", "pow(-0, y), y an odd integer:                +0 for y > 0, +inf for y < 0",
                 "pow(1, NaN):                                 NaN", "sin, cos, tan of |x| > 1e5:                  NaN"):
        assert line in block, line
    assert np.isnan(deviation("pow", -2.0, 2.0)) and np.isnan(deviation("pow", -np.inf, 3.0))
    assert deviation("pow", -0.0, 3.0) == 0.0 and deviation("pow", -0.0, -1.0) == np.inf
    assert np.isnan(deviation("pow", 1.0, NAN)) and np.isnan(deviation("tan", 1e6))


def test_edges_the_render_path_reaches(oracle):
    """atan2 at the signed zeros and infinities equi-angular sampling can pass (C99), ln_fast on subnormals (the
    Mandelbulb estimator at tiny radii), exp into and below the subnormal range"""
    pi = float(f32(np.pi))
    a = oracle.kat_detmath(OP["atan2"], np.array([0.0, -0.0, 0.0, -0.0, -0.0, np.inf, -np.inf, np.inf, -np.inf], f32),
                           np.array([0.0, 0.0, -0.0, -0.0, 1.0, np.inf, np.inf, -np.inf, -np.inf], f32))
    want = [0.0, -0.0, pi, -pi, -0.0, float(f32(np.pi / 4)), -float(f32(np.pi / 4)), float(f32(3 * np.pi / 4)), -float(f32(3 * np.pi / 4))]
    assert [f2u(v) for v in a] == [f2u(v) for v in want]
    sub = np.array([FMIN_SUB, 1e-40, 1e-45 * 3, u2f(0x007fffff)], f32)
    got = oracle.kat_detmath(OP["ln_fast"], sub)
    for x, g in zip(sub, got):
        ref = float(mp.log(mp.mpf(float(x))))
        assert abs(float(g) - ref) <= LN_FAST_BOUND * abs(ref), (x, g, ref)
    e = oracle.kat_detmath(OP["exp"], np.array([-87.33654, -100.0, -103.27893, -103.9721, -104.0], f32))
    assert e[0] > 0 and 0 < e[1] < FMIN_NORM and f2u(e[2]) == 1 and e[3] == 0 and e[4] == 0


# ---- R_d tables: quasi-rd restated in Python integers ------------------------------------------------------------------
def rd_alphas():
    """floor(2^64 alpha) for alpha = 1/phi_1 and 1/phi_2, 1/phi_2^2 (phi_d: x^(d+1) = x + 1)"""
    with mp.workdps(60):
        phi1 = mp.findroot(lambda x: x ** 2 - x - 1, 1.6)
        phi2 = mp.findroot(lambda x: x ** 3 - x - 1, 1.3)
        return tuple(int(mp.floor(mp.mpf(2) ** 64 / p)) for p in (phi1, phi2, phi2 ** 2))


def rd_value(alpha, n):
    return ((alpha * n + (1 << 63)) % (1 << 64) >> 40) / float(1 << 24)


def rd_statement(spp, sets_1d, sets_2d, offset, first):
    """(1d [sets_1d * spp], 2d [sets_2d * spp * 2]) float32: element n of set i at index ((offset + i) << 32) + first + n + 1
    mod 2^64, the 2D sets after the 1D ones"""
    a1, a2x, a2y = rd_alphas()
    m = 1 << 64

    def idx(i, n):
        return ((((offset + i) % m) << 32) % m + first + n + 1) % m
    s1 = [rd_value(a1, idx(i, n)) for i in range(sets_1d) for n in range(spp)]
    s2 = [rd_value(a, idx(sets_1d + i, n)) for i in range(sets_2d) for n in range(spp) for a in (a2x, a2y)]
    return np.array(s1, f32), np.array(s2, f32)


def config_set_counts():
    from rayn_b200 import configs
    from rayn_b200.film import FrameInputs
    out = []
    for k in range(1, 6):
        c = configs.baseline_config(k, res=(8, 8), samples=1)
        i = FrameInputs(8, 8, c["samples"], c["integrator"])
        out.append((i.sets_1d, i.sets_2d))
    return sorted(set(out))


RD_OFFSETS = (0, 3, 2 ** 32 - 1, 2 ** 63 + 5, 2 ** 64 - 1)
RD_SPP = (1, 4, 12, 256)


def rd_cases():
    """(spp, sets_1d, sets_2d, offset, first) at every offset, first sample and spp above and the set counts of configs 1-5"""
    return [(spp, s1, s2, off, first) for s1, s2 in config_set_counts() for spp in RD_SPP for off in RD_OFFSETS
            for first in (0, 1, 2 ** 32 - spp)]


def test_rd_alphas_are_the_floor():
    assert rd_alphas() == (0x9E3779B97F4A7C15, 0xC13FA9A902A6328F, 0x91E10DA5C79E7B1C)


def host_rd(spp, s1, s2, off, first):
    a, b = np.zeros(max(s1 * spp, 1), f32), np.zeros(max(2 * s2 * spp, 1), f32)
    fp = C.POINTER(C.c_float)
    assert L.host_lib().rayn_b200_host_rd_tables_at(spp, s1, s2, off, first, a.ctypes.data_as(fp), b.ctypes.data_as(fp)) == L.RAYN_OK
    return a[:s1 * spp], b[:2 * s2 * spp]


def test_host_rd_tables_match_the_statement():
    for case in rd_cases():
        want = rd_statement(*case)
        got = host_rd(*case)
        for g, w, k in zip(got, want, ("1d", "2d")):
            assert np.array_equal(g.view(u32), w.view(u32)), f"{k} tables at (spp, sets_1d, sets_2d, offset, first) = {case}"


# ---- scramble plane: rand_core 0.5.1 seed_from_u64 + rand_pcg Mcg128Xsl64, restated in Python integers --------------------
M64, M128 = (1 << 64) - 1, (1 << 128) - 1
PCG_MUL, PCG_INC = 6364136223846793005, 11634580027462260723
MCG_MUL = (2549297995355413924 << 64) | 4865540595714422341


def scramble_statement(seed):
    """first f32 of SmallRng::seed_from_u64(seed): PCG32 fills the 16-byte seed as four little-endian u32; Mcg128Xsl64 takes
    it as a little-endian u128, forced odd; one step, XSL-RR output; (low u32 >> 8) * 2^-24"""
    state, seed_bytes = seed, b""
    for _ in range(4):
        state = (state * PCG_MUL + PCG_INC) & M64
        xorshifted = (((state >> 18) ^ state) >> 27) & 0xFFFFFFFF
        rot = state >> 59
        seed_bytes += (((xorshifted >> rot) | (xorshifted << ((32 - rot) & 31))) & 0xFFFFFFFF).to_bytes(4, "little")
    s = (int.from_bytes(seed_bytes, "little") | 1) * MCG_MUL & M128
    rot = s >> 122
    xsl = ((s >> 64) ^ s) & M64
    out = ((xsl >> rot) | (xsl << ((64 - rot) & 63))) & M64
    return ((out & 0xFFFFFFFF) >> 8) / float(1 << 24)


SCRAMBLE_SHAPES = [(1, 1), (7, 3), (33, 17), (301, 77)]  # every pixel
BIG = (16384, 8192)                                     # sampled pixels, first and last included


def big_sample_pixels():
    w, h = BIG
    rng = np.random.default_rng(11)
    idx = np.concatenate([[0, 1, w - 1, w, w * h // 2, w * h - w, w * h - 1], rng.integers(0, w * h, 2000)])
    return idx.astype(np.int64)


def test_host_scramble_matches_the_statement():
    fp = C.POINTER(C.c_float)
    for w, h in SCRAMBLE_SHAPES:
        out = np.zeros(w * h, f32)
        assert L.host_lib().rayn_b200_host_scramble(w, h, out.ctypes.data_as(fp)) == L.RAYN_OK
        want = np.array([scramble_statement(i) for i in range(w * h)], f32)
        assert np.array_equal(out.view(u32), want.view(u32)), (w, h)
    w, h = BIG
    out = np.zeros(w * h, f32)
    assert L.host_lib().rayn_b200_host_scramble(w, h, out.ctypes.data_as(fp)) == L.RAYN_OK
    idx = big_sample_pixels()
    want = np.array([scramble_statement(int(i)) for i in idx], f32)
    assert np.array_equal(out[idx].view(u32), want.view(u32))
