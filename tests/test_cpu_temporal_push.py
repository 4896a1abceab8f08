"""The temporal push (rayn_b200_temporal_push) restated from the header in numpy, against the CPU mirror
(tests/film_mirror.cpp, TemporalMirror) bit for bit, and against a float64 statement of its intent: bilinear history at
(x + dx, y + dy) in exact arithmetic.

The numpy statement is written from include/rayn_b200.h, not from the mirror: taps j outer and i inner, every product and sum
rounded on its own, the tap rules in the header's order, alpha, the alpha == 1 copy, n' and s', and both histories in the
14-plane layout.  The inputs are chosen where a restatement and the mirror could part: integer, signed-zero, half-pixel, tiny,
huge, infinite and NaN motion; positions landing exactly on the first and last column / row or just outside; a tap factor
1 - ax that rounds to 0 (fx = -2^-25, where ax rounds to 1); history taps that are empty, fractional, non-finite, or at depth
0 or +-infinity; z_prev negative, zero, huge and infinite; sigma_depth at +inf and at 3e38, where sigma_depth * |z_prev|
overflows and only the finite-z_h rule keeps a history without a hit out; normal_cos at -1 and 1; alpha_min at 1 and 1e-6;
random resets and outputs that alias the inputs.  Every other zero weight comes from an integer position: a non-zero ax or
ay is at least 2^-24, so 1 - ax is exact and no product of two non-zero factors underflows (tested).

The float64 intent agrees with the float statement on well-conditioned inputs.  They part at x >= 2^23, where x + 0.5f is no
longer exact: the film-width limit of rayn_b200_temporal_create (W, H <= 2^23) keeps every pixel centre below that."""
import ctypes as C

import numpy as np
import pytest

from rayn_b200 import _lib as L

import mirrors
from helpers import assert_bit_equal

f32 = np.float32
# history plane indices (include/rayn_b200.h: colour 3, background 3, moments 2, normal 3, z, n, s)
HC, HB, HM, HN, HZ, HLEN, HS = 0, 3, 6, 8, 11, 12, 13
BLEND = list(range(8)) + [HLEN, HS]  # the history values a push interpolates, in the order of hv
MAX_SIDE = 1 << 23


def np_push(W, H, hin, cur, nrm, motion, alpha_min, sigma_depth, normal_cos, reset, counts=None):
    """The header's statement of one push in numpy float32.  hin [14 * W * H] is the history read; cur [8, W * H] the current
    colour, background and moments; nrm [3, W * H]; motion [4, W * H].  -> (hout [14 * W * H], out [8, W * H], s [W * H]).
    counts: a dict that gains, per tap rule, the taps of active pixels that rule rejects first, and the taps used."""
    npx = W * H
    hp = np.asarray(hin, f32).reshape(14, npx)
    nx, ny, nz = nrm
    z, zp = motion[2], motion[3]
    y, x = np.divmod(np.arange(npx, dtype=np.int64), W)
    sd, nc = f32(sigma_depth), f32(normal_cos)
    hv = np.zeros((10, npx), f32)
    ws = np.zeros(npx, f32)
    nh = np.zeros(npx, f32)
    with np.errstate(all="ignore"):
        active = np.isfinite(zp) & (not reset)
        fx = ((x.astype(f32) + f32(0.5)) + motion[0]) - f32(0.5)
        fy = ((y.astype(f32) + f32(0.5)) + motion[1]) - f32(0.5)
        x0, y0 = np.floor(fx), np.floor(fy)
        ax, ay = fx - x0, fy - y0
        for j in (0, 1):
            for i in (0, 1):
                w = (ax if i else f32(1) - ax) * (ay if j else f32(1) - ay)
                qx, qy = x0 + f32(i), y0 + f32(j)
                inside = (qx >= f32(0)) & (qx <= f32(W - 1)) & (qy >= f32(0)) & (qy <= f32(H - 1))
                q = np.where(inside, qy, f32(0)).astype(np.int64) * W + np.where(inside, qx, f32(0)).astype(np.int64)
                t = hp[:, q]
                near = np.abs(t[HZ] - zp) <= sd * np.abs(zp)
                rules = (("weight", w != f32(0)), ("inside", inside), ("n", t[HLEN] > f32(0)),
                         ("finite", np.isfinite(t[HC:HC + 6]).all(axis=0)), ("z_h finite", np.isfinite(t[HZ])), ("depth", near),
                         ("normal", ((t[HN] * nx + t[HN + 1] * ny) + t[HN + 2] * nz) >= nc))
                used = active.copy()
                for name, ok in rules:
                    if counts is not None:
                        counts[name] = counts.get(name, 0) + int((used & ~ok).sum())
                        if name == "z_h finite":  # taps that only this rule rejects: sigma_depth * |z_prev| is +inf
                            counts["z_h finite only"] = counts.get("z_h finite only", 0) + int((used & ~ok & near).sum())
                    used &= ok
                if counts is not None:
                    counts["used"] = counts.get("used", 0) + int(used.sum())
                ws = np.where(used, ws + w, ws)
                hv = np.where(used, hv + w * t[BLEND], hv)
        some = ws != f32(0)
        hv = np.where(some, hv / ws, hv)
        nh = np.where(some, hv[8], nh)
        alpha = np.fmax(f32(alpha_min), f32(1) / (nh + f32(1)))
        copy = alpha == f32(1)
        beta = f32(1) - alpha
        out = np.where(copy, cur, beta * hv[:8] + alpha * cur)
        s = np.where(copy, f32(1), (beta * beta) * hv[9] + alpha * alpha)
        hout = np.concatenate([out, nrm, z[None], (nh + f32(1))[None], s[None]]).astype(f32)
    return hout.reshape(-1), out, s


def np_push64(W, H, hin, cur, nrm, motion, alpha_min, sigma_depth, normal_cos):
    """The intent of one push in float64: bilinear history at (x + dx, y + dy), the same tap rules, the same blend.
    -> (out [8, W * H], s [W * H], n' [W * H])."""
    npx = W * H
    hp = np.asarray(hin, np.float64).reshape(14, npx)
    cur, nrm, motion = (np.asarray(a, np.float64) for a in (cur, nrm, motion))
    zp = motion[3]
    y, x = np.divmod(np.arange(npx, dtype=np.int64), W)
    fx, fy = x + motion[0], y + motion[1]
    x0, y0 = np.floor(fx), np.floor(fy)
    ax, ay = fx - x0, fy - y0
    hv, ws = np.zeros((10, npx)), np.zeros(npx)
    for j in (0, 1):
        for i in (0, 1):
            w = (ax if i else 1 - ax) * (ay if j else 1 - ay)
            qx, qy = x0 + i, y0 + j
            inside = (qx >= 0) & (qx <= W - 1) & (qy >= 0) & (qy <= H - 1)
            q = np.where(inside, qy, 0).astype(np.int64) * W + np.where(inside, qx, 0).astype(np.int64)
            t = hp[:, q]
            used = np.isfinite(zp) & (w != 0) & inside & (t[HLEN] > 0) & np.isfinite(t[HC:HC + 6]).all(axis=0) & np.isfinite(t[HZ])
            used &= (np.abs(t[HZ] - zp) <= sigma_depth * np.abs(zp)) & ((nrm * t[HN:HN + 3]).sum(axis=0) >= normal_cos)
            ws += np.where(used, w, 0)
            hv += np.where(used, w * t[BLEND], 0)
    some = ws != 0
    hv = np.where(some, hv / np.where(some, ws, 1), 0)
    alpha = np.maximum(alpha_min, 1 / (hv[8] + 1))
    out = (1 - alpha) * hv[:8] + alpha * cur
    s = (1 - alpha) ** 2 * hv[9] + alpha ** 2
    return out, s, hv[8] + 1


# ---- inputs -------------------------------------------------------------------------------------------------------------
TINY = 2.0 ** -25
MOTION_VALUES = [0.0, -0.0, 1.0, -2.0, 3.0, 0.5, -0.5, TINY, -TINY, 1e30, -1e30, np.inf, -np.inf, np.nan, -2.0 ** -26,
                 0.25, -0.75]


def edge_motion(W, H, rng):
    """motion [4, W * H]: a random mix of MOTION_VALUES, uniform fractions, landings on the first / last column and row or
    just outside them, and depths with z_prev negative, zero, huge, infinite or NaN (z = z_prev = +inf is a pixel without
    a hit, which leaves z_h = +inf in the history)"""
    npx = W * H
    y, x = np.divmod(np.arange(npx), W)
    m = np.empty((4, npx), f32)
    for a, (pos, n) in enumerate(((x, W), (y, H))):
        v = rng.choice(np.array(MOTION_VALUES, f32), npx)
        v = np.where(rng.uniform(size=npx) < 0.3, rng.uniform(-2.5, 2.5, npx).astype(f32), v)
        land = {0: -pos, 1: (n - 1) - pos, 2: -pos - 2.0 ** -20, 3: (n - 1) - pos + 2.0 ** -20, 4: -pos - 1, 5: n - pos}
        pick = rng.integers(0, 12, npx)
        for k, d in land.items():
            v = np.where(pick == k, np.asarray(d, np.float64).astype(f32), v)
        m[a] = v
    z = rng.choice(np.array([3.0, 3.0, 3.0, -2.0, 0.0, 1e-3, 1e38, np.inf], f32), npx)  # +inf: a pixel without a hit
    m[2] = z
    zp = z * np.where(rng.uniform(size=npx) < 0.5, f32(1), rng.uniform(0.9, 1.1, npx).astype(f32))
    m[3] = np.where(rng.uniform(size=npx) < 0.06, rng.choice(np.array([np.inf, -np.inf, np.nan, 0.0, -0.0], f32), npx), zp)
    return m


def edge_frame(W, H, rng):
    """(cur [8, npx], normal [3, npx], motion [4, npx]); normals from a small set so exact +-1 dot products occur"""
    npx = W * H
    cur = rng.uniform(0.0, 2.0, (8, npx)).astype(f32)
    cur[:, rng.uniform(size=npx) < 0.03] = f32(1e-40)  # subnormal values: w * x may underflow
    axes = np.array([[0, 0, 1], [0, 0, -1], [0, 1, 0], [0.6, 0.8, 0], [0, 0, 0]], f32)
    nrm = axes[rng.choice(len(axes), npx, p=[0.5, 0.15, 0.15, 0.15, 0.05])].T.copy()
    return cur, nrm, edge_motion(W, H, rng)


def spoil_history(hist, npx, rng):
    """History taps the rules must skip or carry: n = 0, fractional or infinite n, non-finite colour or background, and z_h
    non-finite or zero.  Writes hist in place."""
    hp = hist.reshape(14, npx)
    pick = rng.integers(0, 24, npx)
    hp[HLEN, pick == 0] = 0.0
    hp[HLEN, pick == 1] = 0.375
    hp[HLEN, pick == 2] = 2.5
    hp[HLEN, pick == 3] = np.inf
    hp[HC + 1, pick == 4] = np.nan
    hp[HC, pick == 5] = np.inf
    hp[HB + 2, pick == 6] = -np.inf
    hp[HB, pick == 7] = np.nan
    hp[HZ, pick == 8] = np.inf
    hp[HZ, pick == 9] = np.nan
    hp[HZ, pick == 10] = 0.0
    hp[HZ, pick == 11] = -0.0
    hp[HZ, pick == 14] = -np.inf
    hp[HM, pick == 12] = np.inf  # moments are not tested: they carry through
    hp[HS, pick == 13] = 0.0


# sigma_depth = +inf switches the depth test off, and 3e38 * |z_prev| overflows for a huge z_prev: only the finite-z_h rule
# then keeps a history without a hit (z_h = +inf) out
DESCS = [(0.2, 0.1, 0.5), (1e-6, 0.05, -1.0), (1.0, 0.1, 0.5), (0.5, 1e30, 1.0), (1e-6, 2.0, -1.0), (0.3, 0.01, 0.9),
         (0.2, np.inf, -1.0), (0.5, 3e38, 0.5)]


def mirror_push(t, cur, nrm, motion, desc, reset, alias):
    """One TemporalMirror push of flat planes; alias: out and out_moments are the input planes themselves.
    -> (status, out [8, npx], s [npx])"""
    W, H = t.width, t.height
    npx = W * H
    if not alias:
        planes = {"color": cur[0:3].T.copy(), "background": cur[3:6].T.copy(), "normal": nrm.T.copy()}
        rc, out, om, s = t.push(planes, cur[6:8].T.reshape(H, W, 2), motion.T.copy(), *desc, reset=reset)
        return rc, np.concatenate([out["color"].T, out["background"].T, om.reshape(npx, 2).T]), s.reshape(-1)
    c, b, n = cur[0:3].T.copy(), cur[3:6].T.copy(), nrm.T.copy()
    mc, mb, mv = cur[6].copy(), cur[7].copy(), motion.T.copy()
    s = np.empty(npx, f32)
    d = L.RaynTemporalDesc(*(float(v) for v in desc), 1 if reset else 0)
    hin, hout = t.hist[t.cur], t.hist[t.cur ^ 1]
    rc = mirrors.film_lib().rayn_oracle_temporal_push(W, H, C.byref(d), hin.ctypes.data, hout.ctypes.data, c.ctypes.data, b.ctypes.data,
                                                     n.ctypes.data, mc.ctypes.data, mb.ctypes.data, mv.ctypes.data, c.ctypes.data,
                                                     b.ctypes.data, mc.ctypes.data, mb.ctypes.data, s.ctypes.data)
    if rc == L.RAYN_OK:
        t.cur ^= 1
    return rc, np.concatenate([c.T, b.T, mc[None], mb[None]]), s


@pytest.mark.parametrize("W,H", [(1, 1), (1, 13), (17, 1), (257, 3), (9, 9), (31, 31)])
def test_numpy_statement_equals_the_mirror(W, H):
    """16 pushes with edge-case motion, spoiled histories, every descriptor of DESCS, random resets and aliased outputs: the
    numpy statement and the mirror agree on every output and on the history they write, bit for bit"""
    rng = np.random.default_rng(1000 * W + H)
    t = mirrors.TemporalMirror(W, H)
    npx = W * H
    for k in range(2 * len(DESCS)):
        cur, nrm, motion = edge_frame(W, H, rng)
        desc = DESCS[k % len(DESCS)]
        reset = k > 0 and rng.uniform() < 0.15
        if k > 1:
            spoil_history(t.hist[t.cur], npx, rng)
        hin = t.hist[t.cur].copy()
        hout, out, s = np_push(W, H, hin, cur, nrm, motion, *desc, reset)
        rc, got, gs = mirror_push(t, cur, nrm, motion, desc, reset, alias=k % 3 == 2)
        assert rc == L.RAYN_OK
        what = f"{W}x{H} push {k} desc {desc} reset {reset}"
        assert_bit_equal(got, out, what + " outputs")
        assert_bit_equal(gs, s, what + " var_scale")
        assert_bit_equal(t.hist[t.cur], hout, what + " history")
        assert_bit_equal(t.hist[t.cur ^ 1], hin, what + " history read")  # a push never writes the history it reads


def test_the_edge_inputs_reach_every_rule():
    """the inputs above exercise what they claim: fractional and non-finite positions, taps skipped by each rule, weights of
    exactly 1 and 0, the copy path and the blend"""
    W, H = 31, 31
    rng = np.random.default_rng(5)
    t = mirrors.TemporalMirror(W, H)
    counts = {}
    # 16 pushes: every descriptor of DESCS twice
    seen = dict(copy=0, blend=0, n_frac=0, half=0, nonfinite=0, weight_rounds_to_zero=0)
    with np.errstate(all="ignore"):
        for k in range(2 * len(DESCS)):
            cur, nrm, motion = edge_frame(W, H, rng)
            if k > 1:
                spoil_history(t.hist[t.cur], W * H, rng)
            desc = DESCS[k % len(DESCS)]
            hout, _, _ = np_push(W, H, t.hist[t.cur], cur, nrm, motion, *desc, False, counts)
            mirror_push(t, cur, nrm, motion, desc, False, False)
            n_new = hout.reshape(14, -1)[HLEN]
            seen["copy"] += int((n_new == 1).sum())
            seen["blend"] += int((n_new > 1).sum())
            seen["n_frac"] += int(((n_new % 1) != 0).sum())
            fx = pixel_centre(np.arange(W * H) % W, motion[0])
            ax = fx - np.floor(fx)
            seen["half"] += int((ax == 0.5).sum())
            seen["nonfinite"] += int((~np.isfinite(motion[:2])).sum())
            small = np.isfinite(ax) & (ax != 0) & (ax != 1)
            assert (ax[small] >= f32(2.0 ** -24)).all() and (f32(1) - ax[small] != 1).all()
            seen["weight_rounds_to_zero"] += int((ax == 1).sum())  # fx = -2^-25: ax rounds to 1, so 1 - ax is 0
    assert set(counts) == {"weight", "inside", "n", "finite", "z_h finite", "z_h finite only", "depth", "normal", "used"}
    assert min(counts.values()) > 0 and min(seen.values()) > 0, (counts, seen)


def test_float64_intent_on_well_conditioned_inputs():
    """fractional motion within the image, finite history of random length, matching depths and normals: the float statement
    is the float64 bilinear reprojection at (x + dx, y + dy) within 1e-5 relative, over 8 pushes"""
    W, H = 41, 29
    rng = np.random.default_rng(11)
    t = mirrors.TemporalMirror(W, H)
    npx = W * H
    nrm = np.tile(np.array([[0.0], [0.6], [0.8]], f32), npx)
    for k in range(8):
        cur = rng.uniform(0.5, 1.5, (8, npx)).astype(f32)
        motion = np.empty((4, npx), f32)
        motion[0] = rng.uniform(-3, 3, npx)
        motion[1] = rng.uniform(-3, 3, npx)
        motion[2] = rng.uniform(2.0, 2.2, npx)
        motion[3] = rng.uniform(2.0, 2.2, npx)
        desc = DESCS[k % 2]
        hin = t.hist[t.cur].copy()
        rc, out, s = mirror_push(t, cur, nrm, motion, desc, False, False)
        assert rc == L.RAYN_OK
        ref, s64, n64 = np_push64(W, H, hin, cur, nrm, motion, *desc)
        np.testing.assert_allclose(out, ref, rtol=1e-5, atol=0)
        np.testing.assert_allclose(s, s64, rtol=1e-5, atol=0)
        np.testing.assert_allclose(t.hist[t.cur].reshape(14, npx)[HLEN], n64, rtol=1e-5, atol=0)
        if k > 0:
            assert (n64 > 1).mean() > 0.5  # most pixels took history


def pixel_centre(x, d=0.0):
    """the statement's fx for pixel x and motion d, in float32"""
    return ((np.asarray(x).astype(f32) + f32(0.5)) + np.asarray(d, f32)) - f32(0.5)


def test_pixel_centre_is_exact_below_two_to_the_23():
    """with motion 0 the float32 pixel centre fx is x itself for every x < 2^23 (the widest film temporal_create accepts),
    and it is not at 2^23 and 2^23 + 1, where x + 0.5f rounds"""
    x = np.arange(MAX_SIDE, dtype=np.int64)
    assert (pixel_centre(x).astype(np.int64) == x).all()
    assert pixel_centre(MAX_SIDE - 1) == MAX_SIDE - 1
    assert pixel_centre(MAX_SIDE) == MAX_SIDE - 0.5  # x + 0.5f rounds to even: x; then - 0.5f is exact
    assert pixel_centre(MAX_SIDE + 1) == MAX_SIDE + 2  # x + 0.5f rounds to x + 1 (even)


@pytest.mark.parametrize("x", [MAX_SIDE - 1, MAX_SIDE, MAX_SIDE + 1])
def test_pixel_centre_against_the_intent(x):
    """a static pixel should read its own history: the float statement's taps against the intent's (x, weight 1)"""
    fx = pixel_centre(x)
    x0 = np.floor(fx)
    ax = fx - x0
    taps = {int(x0): float(f32(1) - ax), int(x0) + 1: float(ax)}
    used = {q: w for q, w in taps.items() if w != 0}
    if x < MAX_SIDE:
        assert used == {x: 1.0}
    else:
        assert used != {x: 1.0}  # beyond the film-width limit the statement reads another pixel


def test_mirror_rejects_films_wider_or_taller_than_two_to_the_23():
    d = L.RaynTemporalDesc(0.2, 0.1, 0.5, 0)
    z = np.zeros(14, np.float32)
    for W, H in ((MAX_SIDE + 1, 1), (1, MAX_SIDE + 1)):
        rc = mirrors.film_lib().rayn_oracle_temporal_push(W, H, C.byref(d), *([z.ctypes.data] * 13))
        assert rc == L.RAYN_ERR_INVALID_ARG, (W, H)


# ---- what var_scale means -------------------------------------------------------------------------------------------
STAT_N, STAT_FRAMES, SIGMA, MU = 192, 40, 1.0, 0.5


def smooth_field(rng, amplitude=0.6):
    """a smooth random motion field [2, N, N]: a few low-frequency waves with random phases, scaled to +-amplitude px"""
    y, x = np.mgrid[0:STAT_N, 0:STAT_N] / STAT_N
    out = []
    for _ in range(2):
        f = sum(rng.normal() * np.cos(2 * np.pi * (kx * x + ky * y) + rng.uniform(0, 2 * np.pi))
                for kx, ky in ((1, 0), (0, 1), (1, 1), (2, 1), (1, 2)))
        out.append((amplitude * f / np.abs(f).max()).astype(f32))
    return out


def variance_ratio(dx, dy, seed):
    """Pushes STAT_FRAMES frames of iid N(MU, SIGMA^2) colour and background with constant depth and normal along the motion
    (dx, dy) (scalars or [N, N] fields), alpha_min 0.2.  -> r = mean of (c' - MU)^2 / (s' SIGMA^2) over the six channels of
    the last frame, on the pixels whose history chain stays inside the image"""
    N = STAT_N
    rng = np.random.default_rng(seed)
    t = mirrors.TemporalMirror(N, N)
    nrm = np.zeros((N, N, 3), f32)
    nrm[..., 2] = 1.0
    mv = np.zeros((N, N, 4), f32)
    mv[..., 0], mv[..., 1], mv[..., 2], mv[..., 3] = dx, dy, 2.0, 2.0
    mom = np.zeros((N, N, 2), f32)
    for k in range(STAT_FRAMES):
        planes = {"color": (MU + SIGMA * rng.standard_normal((N, N, 3))).astype(f32),
                  "background": (MU + SIGMA * rng.standard_normal((N, N, 3))).astype(f32), "normal": nrm}
        rc, out, _, s = t.push(planes, mom, mv, 0.2, 0.1, 0.5, reset=k == 0)
        assert rc == L.RAYN_OK
    reach = [STAT_FRAMES * np.asarray(d, np.float64) for d in (dx, dy)]  # how far a chain can travel along each axis
    lo = [int(np.ceil(max(0.0, -np.min(r)))) + 1 for r in reach]
    hi = [N - 2 - int(np.ceil(max(0.0, np.max(r)))) for r in reach]
    keep = (slice(lo[1], hi[1]), slice(lo[0], hi[0]))
    e = np.concatenate([out["color"], out["background"]], axis=2)[keep].astype(np.float64) - MU
    assert e.shape[0] * e.shape[1] > 2000
    return float((e * e / (s[keep][..., None] * SIGMA ** 2)).mean())


@pytest.mark.parametrize("dx,dy,expect", [(0.0, 0.0, 1.0), (1.0, -2.0, 1.0), (0.1, 0.0, 0.78), (0.5, 0.0, 0.60), (0.25, 0.75, 0.51),
                                          (0.5, 0.5, 0.46)])
def test_var_scale_bounds_the_variance_of_the_blend(dx, dy, expect):
    """s' SIGMA^2 is the variance of the blended pixel when no tap resamples (integer motion: r = 1 within 5 %, with about 17k
    independent pixels) and an upper bound under sub-pixel motion, where bilinear resampling averages the independent noise of
    neighbouring history pixels while s_h is interpolated linearly.  Then r is 0.46 to 0.78; over four seeds r at (0.5, 0)
    spans 0.598 to 0.601 and at (1, -2) 0.998 to 1.006."""
    r = variance_ratio(dx, dy, seed=int(100 * dx + 10 * dy) + 7)
    assert r <= 1.03
    assert abs(r - expect) <= 0.05, r


def test_var_scale_bounds_the_variance_under_a_smooth_motion_field():
    r = variance_ratio(*smooth_field(np.random.default_rng(3)), seed=3)
    assert r <= 1.03 and r < 0.9, r  # fractional almost everywhere: well below 1


def sky_then_hit(W, H, rng):
    """two frames (planes, moments, motion) [H, W, ...]: frame 1 has no hit anywhere (motion (0, 0, +inf, +inf), normal 0),
    frame 2 hits everything at z = z_prev = 2 with zero motion"""
    frames = []
    for z, n in ((np.inf, 0.0), (2.0, 1.0)):
        p = {k: rng.uniform(0.1, 1.0, (H, W, 3)).astype(f32) for k in ("color", "background")}
        p["normal"] = np.zeros((H, W, 3), f32)
        p["normal"][..., 2] = n
        mv = np.zeros((H, W, 4), f32)
        mv[..., 2:] = z
        frames.append((p, rng.uniform(0.1, 1.0, (H, W, 2)).astype(f32), mv))
    return frames


@pytest.mark.parametrize("sigma_depth", [0.1, 3e38, np.inf])
def test_history_without_a_hit_is_never_used(sigma_depth):
    """a sky history (z_h = +inf) is rejected even where sigma_depth * |z_prev| is +inf: frame 2 comes back unchanged, in the
    mirror and in the numpy statement"""
    W, H = 4, 3
    (p0, m0, mv0), (p1, m1, mv1) = sky_then_hit(W, H, np.random.default_rng(4))
    t = mirrors.TemporalMirror(W, H)
    t.push(p0, m0, mv0, 0.2, sigma_depth, -1.0)
    hin = t.hist[t.cur].copy()
    rc, out, om, s = t.push(p1, m1, mv1, 0.2, sigma_depth, -1.0)
    assert rc == L.RAYN_OK
    assert_bit_equal(out["color"], p1["color"]), assert_bit_equal(out["background"], p1["background"]), assert_bit_equal(om, m1)
    assert (s == 1).all()
    cur = np.concatenate([p1["color"].reshape(-1, 3).T, p1["background"].reshape(-1, 3).T, m1.reshape(-1, 2).T])
    _, ref, rs = np_push(W, H, hin, cur, p1["normal"].reshape(-1, 3).T, mv1.reshape(-1, 4).T, 0.2, sigma_depth, -1.0, False)
    assert_bit_equal(ref, cur), assert_bit_equal(rs, np.ones(W * H, f32))
