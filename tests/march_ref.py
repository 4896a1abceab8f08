"""numpy statement of the reference's sphere marches, per ray, written from the reference source (src/sdf.rs):

  march_hit       TracedSDF::hit (sdf.rs:59-83), with its frozen-t merge and the evaluation it runs after t passed t_max;
  march_occluded  TracedSDF::occluded (sdf.rs:25-57);
  shading_normal  get_shading_info (sdf.rs:85-101): sdfu's tetrahedral normals_fast (oracle/README.md A8) with
                  eps = max(1e-4, S * threshold(t)).

Every operation is one float32 rounding; max(a, b) is maxps, `a > b ? a : b`; mul_add follows the library variant (unfused
(a * b) + c, or fused: one rounding of the exact a * b + c, mul_add_fused).  Distances come from the oracle's estimator
(oracle.kat_sdf_dist, proven equal to every packed estimator of the kernels by test_gpu_parity.py): this module owns the
march logic only.  The reference marches four lanes at once; a lane's result does not depend on its neighbours (a finished
lane is frozen by the merge), so each ray is stated alone, and its evaluation count is the lane's own: evaluations up to and
including the one whose mask ended it.

Evaluation counts.  The kernels stop a march at the update that decides its result and run no evaluation after it
(rt_kernels.cuh, extend_step / shadow_step).  The reference runs some evaluations whose result cannot change anything:
those at a t that is NaN, and, in hit, the one at a t already past t_max.  So

    kernel evaluations = reference evaluations - dead evaluations,

where `dead` counts the reference's evaluations at a NaN t or at a t > t_max (hit) - one for a march that ends past t_max
with marches left, one for a NaN first distance, and all those after a NaN update.  occluded tests t > max_dist before it
evaluates, so it has no dead evaluation past max_dist.
"""
import fractions

import numpy as np

from rayn_b200 import _lib as L

f32 = np.float32
END_HIT, END_PAST, END_NAN, END_EXHAUSTED = 0, 1, 2, 3  # march_hit; march_occluded uses END_HIT for "occluded"
END_NAMES = ("hit", "past", "nan", "exhausted")


# ---- float32 arithmetic ------------------------------------------------------------------------------------------------
def fmax(a, b):
    """wide's f32x4::max, SSE maxps: a > b ? a : b, so b when either is NaN.  `a < b ? b : a` differs from it only for a NaN
    b, which a NaN detail scale reaches in get_shading_info's eps (NaN there, as in the oracle and the kernel)."""
    return np.where(a > b, a, b).astype(np.float32)


def mul_add_fused(a, b, c):
    """a * b + c rounded once to float32 (nearest, ties to even).  a * b is exact in float64; a TwoSum adds c, s + err being the
    exact sum; s rounds to the float32 of the exact sum unless s lies exactly on a float32 midpoint and err != 0, where the
    sign of err decides."""
    a, b, c = (np.asarray(v, np.float32).astype(np.float64) for v in (a, b, c))
    with np.errstate(all="ignore"):
        p = a * b
        s = p + c
        bp = s - c
        err = (p - bp) + (c - (s - bp))
        r = s.astype(np.float32)
        other = np.nextafter(r, np.where(s > r.astype(np.float64), f32(np.inf), f32(-np.inf)).astype(np.float32))
        mid = (r.astype(np.float64) + other.astype(np.float64)) * 0.5
        tie = np.isfinite(s) & np.isfinite(other) & (s != r.astype(np.float64)) & (s == mid) & (err != 0)
        up = err > 0  # the exact sum lies above s
        pick_other = tie & ((other.astype(np.float64) > r.astype(np.float64)) == up)
    return np.where(pick_other, other, r).astype(np.float32)


def mul_add_fraction(a, b, c):
    """the same, one triple at a time, through exact rational arithmetic (the check of mul_add_fused)"""
    q = fractions.Fraction(float(f32(a))) * fractions.Fraction(float(f32(b))) + fractions.Fraction(float(f32(c)))
    if q == 0:
        return None  # the sign of an exact zero is not what this helper is checked on
    sign = -1 if q < 0 else 1
    q = abs(q)
    e = q.numerator.bit_length() - q.denominator.bit_length()
    if fractions.Fraction(2) ** e > q:
        e -= 1  # 2^e <= q < 2^(e+1)
    ulp = fractions.Fraction(2) ** (max(e, -126) - 23)
    n, rem = divmod(q, ulp)
    n = int(n)
    if rem * 2 > ulp or (rem * 2 == ulp and n % 2 == 1):
        n += 1
    v = n * ulp
    if v >= fractions.Fraction(2) ** 128:
        return f32(sign * np.inf)
    return f32(sign * float(v))


def mul_add(a, b, c):
    """wide's f32x4::mul_add in this library variant (oracle/README.md A6)"""
    if L.MULADD_FUSED:
        return mul_add_fused(a, b, c)
    a, b, c = (np.asarray(v, np.float32) for v in (a, b, c))
    with np.errstate(all="ignore"):
        return ((a * b).astype(np.float32) + c).astype(np.float32)


def point_at(o, d, t):
    """ray.point_at (ray.rs:22-24): dir.mul_add(t, origin), per component"""
    return np.stack([mul_add(d[:, k], t, o[:, k]) for k in range(3)], axis=1)


def thr_at(scale, is_const, t):
    """the hit_threshold_at closure (film.rs:540-551): scale, or scale * t"""
    t = np.asarray(t, np.float32)
    with np.errstate(all="ignore"):
        return np.full_like(t, f32(scale)) if is_const else (f32(scale) * t).astype(np.float32)


def make_thr(camera, depth):
    """(scale, is_const) of make_thr (rt_device.cuh) for a RaynCamera"""
    if depth == 0:
        return f32(camera.half_pixel_size), camera.kind == L.CAMERA_ORTHOGRAPHIC
    return f32(f32(0.0001) * f32(2.0)) * f32(depth), False


# ---- the marches ----------------------------------------------------------------------------------------------------
def march_hit(dist, S, max_marches, o, d, t_max, thr, alter=None):
    """TracedSDF::hit per ray.  dist(points [n, 3]) -> float32 [n]; thr = (scale, is_const).  Returns dict of float32 t,
    int end kind, int evals (the reference's) and int dead (see the module docstring).  alter names a deliberately wrong
    statement the CPU tests use to show that the cases can tell: "first_hit" (a hit test on the first evaluation), "ge"
    (t >= t_max ends the march), "early" (max_marches - 1 marches)."""
    o, d = np.asarray(o, np.float32).reshape(-1, 3), np.asarray(d, np.float32).reshape(-1, 3)
    t_max = np.asarray(t_max, np.float32).reshape(-1)
    n = len(o)
    S = f32(S)
    c0, c1 = f32(f32(0.00005) * S), f32(f32(0.05) * S)
    t = dist(o).astype(np.float32)
    nan = np.isnan(t)
    evals = np.ones(n, np.int64)
    dead = np.zeros(n, np.int64)
    kind = np.full(n, END_EXHAUSTED, np.int64)
    live = np.ones(n, bool)
    if alter == "first_hit":  # as if the first evaluation had the hit test of the loop at t = -0
        h0 = np.abs(t) < fmax(np.full(n, c0), (c1 * thr_at(thr[0], thr[1], np.full(n, f32(-0.0)))).astype(np.float32))
        t = np.where(h0, f32(-0.0), t).astype(np.float32)
        kind[h0] = END_HIT
        live &= ~h0
    marches = max_marches - 1 if alter == "early" else max_marches
    with np.errstate(all="ignore"):
        for _ in range(marches):
            idx = np.flatnonzero(live)
            if idx.size == 0:
                break
            ti = t[idx]
            dd = dist(point_at(o[idx], d[idx], ti)).astype(np.float32)
            evals[idx] += 1
            dead[idx] += (np.isnan(ti) | (ti > t_max[idx])).astype(np.int64)
            hit = np.abs(dd) < fmax(np.full(idx.size, c0), (c1 * thr_at(thr[0], thr[1], ti)).astype(np.float32))
            gt = (ti >= t_max[idx]) if alter == "ge" else (ti > t_max[idx])
            stop = hit | nan[idx] | gt
            k = np.where(nan[idx], END_NAN, np.where(gt, END_PAST, END_HIT))
            kind[idx[stop]] = k[stop]
            live[idx[stop]] = False
            t[idx] = np.where(stop, ti, (ti + dd).astype(np.float32))
    kind[live & np.isnan(t)] = END_NAN  # a NaN update: the reference marches on to exhaustion and returns the NaN
    return dict(t=t, kind=kind, evals=evals, dead=dead)


def march_occluded(dist, S, max_vis_marches, start, dirn, max_dist, alter=None):
    """TracedSDF::occluded per segment (start, unit dir, max_dist).  Returns dict of bool occluded, int end kind (END_HIT =
    occluded), int evals and int dead.  alter="first_occ": an occlusion test on the first evaluation (at t = -0)."""
    s, dv = np.asarray(start, np.float32).reshape(-1, 3), np.asarray(dirn, np.float32).reshape(-1, 3)
    md = np.asarray(max_dist, np.float32).reshape(-1)
    n = len(s)
    S = f32(S)
    oc0, oc1 = f32(f32(0.0001) * S), f32(f32(0.00001) * S)
    d0 = dist(s).astype(np.float32)
    nan = np.isnan(d0)
    with np.errstate(all="ignore"):
        gtn = (d0 > md) | nan
        hit = d0 < f32(0.0001)
    t = d0.copy()
    evals = np.ones(n, np.int64)
    dead = np.zeros(n, np.int64)
    live = np.ones(n, bool)
    if alter == "first_occ":
        h0 = np.abs(d0) < fmax(np.full(n, oc0), (oc1 * f32(-0.0)) * np.ones(n, np.float32))
        hit = np.where(h0, True, hit)
        gtn = np.where(h0, False, gtn)
        live &= ~h0
    with np.errstate(all="ignore"):
        for _ in range(max_vis_marches):
            gtn = np.where(live, (t > md) | nan, gtn)
            live &= ~gtn
            idx = np.flatnonzero(live)
            if idx.size == 0:
                break
            ti = t[idx]
            dd = dist(point_at(s[idx], dv[idx], ti)).astype(np.float32)
            evals[idx] += 1
            dead[idx] += np.isnan(ti).astype(np.int64)
            h = np.abs(dd) < fmax(np.full(idx.size, oc0), (oc1 * ti).astype(np.float32))
            hit[idx] = h
            live[idx[h]] = False
            t[idx] = np.where(h, ti, (ti + dd).astype(np.float32))
    occ = hit & ~gtn
    kind = np.where(occ, END_HIT, np.where(nan | np.isnan(t), END_NAN, np.where(gtn, END_PAST, END_EXHAUSTED)))
    return dict(occluded=occ, kind=kind, evals=evals, dead=dead, t=t)


def segments(start, end):
    """a shadow segment as TracedSDF::occluded builds it (sdf.rs:26-28): dir = end - start, max_dist = |dir| (mag = sqrt of
    the mul_add dot, A1), dir / max_dist"""
    s, e = np.asarray(start, np.float32).reshape(-1, 3), np.asarray(end, np.float32).reshape(-1, 3)
    with np.errstate(all="ignore"):
        v = (e - s).astype(np.float32)
        md = np.sqrt(mul_add(v[:, 0], v[:, 0], mul_add(v[:, 1], v[:, 1], (v[:, 2] * v[:, 2]).astype(np.float32)))).astype(np.float32)
        return (v / md[:, None]).astype(np.float32), md


def normalized(n):
    """ultraviolet normalized (A1, A2): n * (1 / sqrt(mul_add dot))"""
    with np.errstate(all="ignore"):
        m = np.sqrt(mul_add(n[:, 0], n[:, 0], mul_add(n[:, 1], n[:, 1], (n[:, 2] * n[:, 2]).astype(np.float32)))).astype(np.float32)
        inv = (f32(1.0) / m).astype(np.float32)
        return (n * inv[:, None]).astype(np.float32)


TETRA = np.array([[1, -1, -1], [-1, -1, 1], [-1, 1, -1], [1, 1, 1]], np.float32)  # normals_fast's k0..k3, in that order


def shading_normal(dist, S, o, d, t, thr):
    """get_shading_info at t along (o, d): (point, eps, normal).  n = ((k0 d0 + k1 d1) + k2 d2) + k3 d3, di = dist(p + ki eps)."""
    o, d = np.asarray(o, np.float32).reshape(-1, 3), np.asarray(d, np.float32).reshape(-1, 3)
    t = np.asarray(t, np.float32).reshape(-1)
    p = point_at(o, d, t)
    with np.errstate(all="ignore"):
        eps = fmax(np.full(len(t), f32(0.0001)), (f32(S) * thr_at(thr[0], thr[1], t)).astype(np.float32))
        n = None
        for k in TETRA:
            q = (p + (k[None, :] * eps[:, None]).astype(np.float32)).astype(np.float32)
            term = (k[None, :] * dist(q)[:, None]).astype(np.float32)
            n = term if n is None else (n + term).astype(np.float32)
    return p, eps, normalized(n)


def kernel_evals(res):
    """the evaluations the kernel runs for these marches (module docstring)"""
    return int((res["evals"] - res["dead"]).sum())


def write_rule(t, t_max, key_in, hk, spheres_first):
    """hitable.rs:190-193 and the sphere-first tie rule (rt_kernels.cuh at k_extend_march): whether a march's t replaces the
    closest hit so far"""
    w = t < t_max
    if spheres_first:
        w = w | ((t == t_max) & (np.asarray(key_in) > hk))
    return w


# ---- the case list -------------------------------------------------------------------------------------------------
def random_rays(n, seed, radius=4.5, spread=0.5):
    """rays from a shell around the fractal aimed near its centre"""
    rng = np.random.default_rng(seed)
    o = rng.normal(size=(n, 3))
    o = o / np.linalg.norm(o, axis=1, keepdims=True) * radius
    d = rng.uniform(-spread, spread, size=(n, 3)) * 2.0 - o
    return o.astype(np.float32), (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)


def extend_cases(dist, S, thr, seed, n=600):
    """rays (o, d, t_max) that reach every end kind of march_hit: hits, t_max past on the first evaluation and after k steps,
    t_max equal to the march's t after k steps (the march goes on) and to its final hit t (a tie for the fold), t_max of
    +inf, +0 and -0, NaN origins and directions, and starts within the hit threshold of the surface.  Returns a dict of the
    arrays and the index groups."""
    o, d = random_rays(n, seed)
    t_max = np.full(n, f32(200.0), np.float32)
    t_max[1::7] = f32(4.0)
    t_max[2::11] = f32(np.inf)
    t_max[3::13] = f32(0.0)
    t_max[4::17] = f32(-0.0)
    o[5::19] = np.nan
    d[6::23, 1] = np.nan
    groups = dict(base=np.arange(n))
    base = march_hit(dist, S, 256, o, d, np.full(n, f32(np.inf), np.float32), thr)
    hits = np.flatnonzero(base["kind"] == END_HIT)
    # t_max = t after k steps (k = 1..3): t == t_max continues
    stepped = hits[: 60]
    ks = 1 + np.arange(stepped.size) % 3
    tk = np.empty(stepped.size, np.float32)
    for k in (1, 2, 3):
        sel = ks == k
        tk[sel] = march_hit(dist, S, k, o[stepped[sel]], d[stepped[sel]], np.full(sel.sum(), f32(np.inf), np.float32), thr)["t"]
    # t_max = the final hit t: the fold tie
    tie = hits[60:120]
    # starts on the surface: the hit point, marched again along the same direction
    surf = hits[120:180]
    p = point_at(o[surf], d[surf], base["t"][surf])
    O = np.concatenate([o, o[stepped], o[tie], p])
    D = np.concatenate([d, d[stepped], d[tie], d[surf]])
    T = np.concatenate([t_max, tk, base["t"][tie], np.full(surf.size, f32(200.0), np.float32)])
    groups["step_tie"] = n + np.arange(stepped.size)
    groups["fold_tie"] = n + stepped.size + np.arange(tie.size)
    groups["surface"] = n + stepped.size + tie.size + np.arange(surf.size)
    return dict(o=O, d=D, t_max=T, groups=groups)


def shadow_cases(dist, S, seed, n=600):
    """segments (start, dir, max_dist) that reach every end kind of march_occluded: occluded at the first tested step and later,
    unoccluded past max_dist, by NaN and by exhaustion, max_dist equal to the march's t after k steps, and starts within the
    occlusion threshold of the surface, leaving it."""
    o, d = random_rays(n, seed + 1)
    hit = march_hit(dist, S, 256, o, d, np.full(n, f32(np.inf), np.float32), (f32(0.0002), False))
    h = np.flatnonzero(hit["kind"] == END_HIT)
    P = point_at(o[h], d[h], hit["t"][h])
    rng = np.random.default_rng(seed)
    # from the shell to near the hit point: occluded or not depending on the end
    ends = P + d[h] * rng.uniform(-0.05, 0.05, size=(h.size, 1)).astype(np.float32)
    dir1, md1 = segments(o[h], ends)
    # leaving the surface back along the ray, from points just off it (a start within the occlusion threshold)
    off = (f32(S) * f32(0.0001) * rng.uniform(0.0, 2.0, size=h.size).astype(np.float32)).astype(np.float32)
    starts = (P - d[h] * off[:, None]).astype(np.float32)
    dir2, md2 = segments(starts, o[h])
    # max_dist = t after k steps
    ks = 1 + np.arange(h.size) % 3
    tk = np.empty(h.size, np.float32)
    for k in (1, 2, 3):
        sel = ks == k
        tk[sel] = march_occluded(dist, S, k, o[h[sel]], dir1[sel], np.full(sel.sum(), f32(np.inf), np.float32))["t"]
    S0 = np.concatenate([o[h], starts, o[h], o[:40]])
    D0 = np.concatenate([dir1, dir2, dir1, d[:40]])
    M0 = np.concatenate([md1, md2, tk, np.full(40, f32(500.0), np.float32)])
    S0[5::31] = np.nan
    D0[7::37, 0] = np.nan
    return dict(start=S0, dir=D0, max_dist=M0, groups=dict(to_surface=np.arange(h.size), leaving=h.size + np.arange(h.size),
                                                           step_tie=2 * h.size + np.arange(h.size)))
