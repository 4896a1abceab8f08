"""The numpy statement of the sphere marches (tests/march_ref.py) against the oracle, without a GPU.

The statement is what tests/test_gpu_march.py holds the persistent march kernels to, so it is checked here first: its t
equals oracle.kat_sdf_hit and its verdicts oracle.kat_occluded bit for bit on the whole case list, its fused mul_add equals
exact rational arithmetic, the case list reaches every end kind and tie, and deliberately wrong statements fail on it."""
import copy
import os
import subprocess
import sys

import numpy as np
import pytest

from rayn_b200 import _lib as L
from rayn_b200 import configs

import march_ref as mr
from helpers import assert_bit_equal

THRS = [(np.float32(0.000563), False), (np.float32(0.0002), False), (np.float32(0.001), True)]


def scene(kind, **consts):
    cam, world = configs.setup((64, 64), volume=False, fractal=kind)
    for k, v in consts.items():
        setattr(world.consts, k, v)
    desc, keep = world.flatten(cam)
    return desc, keep, desc.hitables[1]


def dist_of(oracle, h):
    return lambda p: oracle.kat_sdf_dist(h, np.asarray(p, np.float32).reshape(-1, 3))


def consts_with(desc, **kw):
    c = copy.copy(desc.consts)
    for k, v in kw.items():
        setattr(c, k, v)
    return c


@pytest.mark.parametrize("kind", ["mandelbox", "mandelbulb"])
@pytest.mark.parametrize("max_marches", [1, 2, 3, 256])
def test_hit_statement_equals_the_oracle(oracle, kind, max_marches):
    desc, keep, h = scene(kind)
    dist = dist_of(oracle, h)
    S = desc.consts.sdf_detail_scale
    kinds = set()
    for thr in THRS:
        c = mr.extend_cases(dist, S, thr, seed=max_marches)
        got = mr.march_hit(dist, S, max_marches, c["o"], c["d"], c["t_max"], thr)
        want = oracle.kat_sdf_hit(h, consts_with(desc, max_marches=max_marches), c["o"], c["d"], c["t_max"], float(thr[0]), int(thr[1]))
        assert_bit_equal(got["t"], want, f"{kind} max_marches={max_marches} thr={thr}")
        kinds |= set(got["kind"].tolist())
        # every march ends once: the kernel's count is the reference's less its dead evaluations, never more than it
        assert (got["dead"] <= got["evals"] - 1).all() and (got["evals"] <= max_marches + 1).all()
        past = got["kind"] == mr.END_PAST
        if max_marches > 1:
            assert (got["dead"][past & (got["evals"] <= max_marches)] == 1).all()
    want_kinds = {mr.END_HIT, mr.END_PAST, mr.END_NAN} | ({mr.END_EXHAUSTED} if max_marches < 256 else set())
    assert want_kinds <= kinds, (kind, max_marches, kinds)


def test_hit_case_list_covers_every_rule(oracle):
    desc, keep, h = scene("mandelbox")
    dist = dist_of(oracle, h)
    S = desc.consts.sdf_detail_scale
    thr = THRS[0]
    c = mr.extend_cases(dist, S, thr, seed=3)
    r = mr.march_hit(dist, S, 256, c["o"], c["d"], c["t_max"], thr)
    g = c["groups"]
    counts = {mr.END_NAMES[k]: int((r["kind"] == k).sum()) for k in range(4)}
    assert counts["hit"] >= 100 and counts["past"] >= 50 and counts["nan"] >= 30, counts
    # past t_max on the first evaluation (t_max = +-0) and after several steps
    assert ((r["kind"] == mr.END_PAST) & (r["evals"] == 2)).sum() >= 10
    assert ((r["kind"] == mr.END_PAST) & (r["evals"] > 3)).sum() >= 10
    # t == t_max after k steps: the march goes on, one more update (which passes t_max, or hits)
    st = g["step_tie"]
    assert (r["t"][st] != c["t_max"][st]).mean() > 0.9
    # final t == t_max: the fold's tie, which a key on either side of hk decides with spheres_first, and never without it
    ft = g["fold_tie"]
    assert (r["t"][ft] == c["t_max"][ft]).sum() >= 40
    for sf in (False, True):
        w_lo = mr.write_rule(r["t"][ft], c["t_max"][ft], np.full(ft.size, 0), 1, sf)
        w_hi = mr.write_rule(r["t"][ft], c["t_max"][ft], np.full(ft.size, 5), 1, sf)
        assert not w_lo.any() and w_hi.any() == sf
    # dead evaluations: one per march ending past t_max with marches left, and those at a NaN t
    assert (r["dead"] > 0).sum() >= 50 and mr.kernel_evals(r) < r["evals"].sum()


@pytest.mark.parametrize("alter", ["first_hit", "ge", "early"])
def test_altered_hit_statements_fail_the_cases(oracle, alter):
    desc, keep, h = scene("mandelbox")
    dist = dist_of(oracle, h)
    S = desc.consts.sdf_detail_scale
    bad = 0
    for mm in (1, 256):
        thr = THRS[0]
        c = mr.extend_cases(dist, S, thr, seed=mm)
        want = oracle.kat_sdf_hit(h, consts_with(desc, max_marches=mm), c["o"], c["d"], c["t_max"], float(thr[0]), int(thr[1]))
        got = mr.march_hit(dist, S, mm, c["o"], c["d"], c["t_max"], thr, alter=alter)
        bad += int((~((got["t"].view(np.uint32) == want.view(np.uint32)) | (np.isnan(got["t"]) & np.isnan(want)))).sum())
    assert bad > 0, alter


def _occluded_scene(kind):
    """a scene of the SDF alone, so that oracle.kat_occluded is that SDF's TracedSDF::occluded"""
    from rayn_b200 import HitableStore
    cam, world = configs.setup((64, 64), volume=False, fractal=kind)
    hs = HitableStore()
    hs.push(world.hitables.items[1])
    world.hitables = hs
    desc, keep = world.flatten(cam)
    return desc, keep, desc.hitables[0]


@pytest.mark.parametrize("kind", ["mandelbox", "mandelbulb"])
@pytest.mark.parametrize("max_vis", [1, 2, 100])
def test_occluded_statement_equals_the_oracle(oracle, kind, max_vis):
    desc, keep, h = _occluded_scene(kind)
    desc.consts.max_vis_marches = max_vis
    dist = dist_of(oracle, h)
    S = desc.consts.sdf_detail_scale
    c = mr.shadow_cases(dist, S, seed=7)
    # the oracle takes (start, end); the statement the segment it builds from them (sdf.rs:26-28)
    end = (c["start"] + c["dir"] * c["max_dist"][:, None]).astype(np.float32)
    dirn, md = mr.segments(c["start"], end)
    got = mr.march_occluded(dist, S, max_vis, c["start"], dirn, md)
    want = oracle.kat_occluded(desc, c["start"], end)
    assert ((want == 0.0) == got["occluded"]).all(), (kind, max_vis, np.flatnonzero((want == 0.0) != got["occluded"])[:10])
    kinds = set(got["kind"].tolist())
    assert {mr.END_HIT, mr.END_NAN} <= kinds and (mr.END_PAST if max_vis == 100 else mr.END_EXHAUSTED) in kinds, kinds


def test_altered_occluded_statement_fails_the_cases(oracle):
    desc, keep, h = _occluded_scene("mandelbox")
    dist = dist_of(oracle, h)
    S = desc.consts.sdf_detail_scale
    c = mr.shadow_cases(dist, S, seed=7)
    end = (c["start"] + c["dir"] * c["max_dist"][:, None]).astype(np.float32)
    dirn, md = mr.segments(c["start"], end)
    want = oracle.kat_occluded(desc, c["start"], end) == 0.0
    got = mr.march_occluded(dist, S, 100, c["start"], dirn, md, alter="first_occ")["occluded"]
    assert (got != want).any()


def test_fused_mul_add_equals_rational_arithmetic():
    rng = np.random.default_rng(11)
    a = (rng.standard_normal(3000) * np.exp2(rng.integers(-20, 20, 3000))).astype(np.float32)
    b = (rng.standard_normal(3000) * np.exp2(rng.integers(-20, 20, 3000))).astype(np.float32)
    c = (rng.standard_normal(3000) * np.exp2(rng.integers(-40, 40, 3000))).astype(np.float32)
    # triples whose exact value lies next to a float32 midpoint: c = -(a*b rounded) + half an ulp of it, nudged by a*b's tail
    m = 1000
    a2 = (1.0 + rng.integers(1, 1 << 12, m) * 2.0 ** -12).astype(np.float32)
    b2 = (1.0 + rng.integers(1, 1 << 12, m) * 2.0 ** -12).astype(np.float32)
    c2 = (np.ldexp(rng.integers(1, 1 << 23, m).astype(np.float64), -23 - rng.integers(0, 3, m)) + 2.0 ** -24).astype(np.float32)
    A, B, Cc = np.concatenate([a, a2]), np.concatenate([b, b2]), np.concatenate([c, c2])
    got = mr.mul_add_fused(A, B, Cc)
    n_mid = 0
    for i in range(len(A)):
        w = mr.mul_add_fraction(A[i], B[i], Cc[i])
        if w is None:
            continue
        assert got[i].view(np.uint32) == np.float32(w).view(np.uint32), (A[i], B[i], Cc[i], got[i], w)
        s = float(A[i]) * float(B[i]) + float(Cc[i])
        r = np.float32(s)
        n_mid += abs(s - float(r)) * 2 == abs(float(np.nextafter(r, np.float32(np.inf if s > float(r) else -np.inf))) - float(r))
    assert n_mid >= 100  # the float64 sum sat exactly on a float32 midpoint this often


def test_shading_normal_statement_is_the_tetrahedral_estimator(oracle):
    """the statement's normal at hit points against the same formula in float64 where it is well conditioned"""
    desc, keep, h = scene("mandelbox")
    dist = dist_of(oracle, h)
    S = desc.consts.sdf_detail_scale
    o, d = mr.random_rays(400, 2)
    thr = THRS[0]
    r = mr.march_hit(dist, S, 256, o, d, np.full(len(o), np.float32(200.0)), thr)
    k = r["kind"] == mr.END_HIT
    p, eps, n = mr.shading_normal(dist, S, o[k], d[k], r["t"][k], thr)
    n64 = sum(mr.TETRA[i].astype(np.float64)[None, :] * dist(p + mr.TETRA[i][None, :] * eps[:, None]).astype(np.float64)[:, None] for i in range(4))
    mag = np.linalg.norm(n64, axis=1)
    good = mag > 64 * eps * 1e-5
    assert good.sum() > 50
    assert np.abs(n[good] - n64[good] / mag[good, None]).max() < 1e-4


@pytest.mark.skipif(L.MULADD_FUSED, reason="already inside the fused run")
def test_fused_mul_add_variant_passes_this_file():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "pytest", "-x", "-q", "-m", "not gpu", "-p", "no:cacheprovider", "tests/test_cpu_march.py"],
                       cwd=root, env=dict(os.environ, RAYN_MULADD_FUSED="1"), capture_output=True, text=True)
    assert r.returncode == 0 and " passed" in r.stdout, r.stdout[-3000:] + r.stderr[-1500:]
