"""numpy float32 restatement of the orbit-trap albedo (include/rayn_b200.h, RaynAlbedoTrap) for the unfused `mul_add`
build.  Every float32 operation below is one IEEE rounding, like the oracle's SSE operations compiled without contraction.
The Mandelbulb's Horner forms are fused by definition; fma32 rounds them exactly (round-to-odd in float64, then one rounding
to float32)."""
import numpy as np

f32 = np.float32
INF = f32(np.inf)


def fma32(a, b, c):
    """correctly rounded float32 a * b + c"""
    a, b, c = (np.asarray(v, np.float32).astype(np.float64) for v in (a, b, c))
    p = a * b  # exact: 24 + 24 significant bits
    s = p + c
    bp = s - c
    err = (p - bp) + (c - (s - bp))  # two-sum: s + err == p + c exactly
    odd = (s.view(np.uint64) & 1) == 1
    fix = (err != 0) & ~odd & np.isfinite(s)
    s = np.where(fix, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)  # round to odd: 53 >= 24 + 2 bits
    return s.astype(np.float32)


def _min_fold(x, trap):
    return np.where(x < trap, x, trap)  # (x < trap) ? x : trap - NaN never replaces


def mandelbox_trap(h, p):
    p = np.asarray(p, np.float32).reshape(-1, 3)
    trap = np.full(len(p), INF, np.float32)
    if h.iterations <= 0:
        return trap
    x, y, z = (p[:, k].copy() for k in range(3))
    cx, cy, cz = x.copy(), y.copy(), z.copy()
    dr = np.ones(len(p), np.float32)
    l, nl = f32(h.box_l), -f32(h.box_l)
    mn, fx, sc, one = f32(h.min_rad_sq), f32(h.fixed_rad_sq), f32(h.scale), f32(1.0)

    def clamp(v):  # clamped(neg_l, l) = maxps then minps: the constant wins when unordered
        m = np.where(v > nl, v, nl)
        return np.where(m < l, m, l)
    with np.errstate(all="ignore"):
        for _ in range(h.iterations):
            x, y, z = clamp(x) * f32(2.0) + (-x), clamp(y) * f32(2.0) + (-y), clamp(z) * f32(2.0) + (-z)
            r2 = x * x + (y * y + z * z)  # mag_sq: mul_add(x, x, mul_add(y, y, z * z)), unfused
            trap = _min_fold(r2, trap)
            den = np.where(mn > r2, mn, r2)
            q = fx / den
            mul = np.where(one > q, one, q)
            x, y, z, dr = x * mul, y * mul, z * mul, dr * mul
            x, y, z = x * sc + cx, y * sc + cy, z * sc + cz
            dr = (-dr) * sc + one
    return trap


def mandelbulb_trap(h, p):
    p = np.asarray(p, np.float32).reshape(-1, 3)
    trap = np.full(len(p), INF, np.float32)
    if h.iterations <= 0:
        return trap
    cx, cy, cz = (p[:, k].copy() for k in range(3))
    wx, wy, wz = cx.copy(), cy.copy(), cz.copy()
    bail2 = f32(h.bulb_bailout) * f32(h.bulb_bailout)
    with np.errstate(all="ignore"):
        m = wx * wx + (wy * wy + wz * wz)
        trap = _min_fold(m, trap)
        for _ in range(h.iterations):
            go = ~(m > bail2)
            if not go.any():
                break
            a, b = wz * wz, m
            b2 = b * b
            b3, b4 = b2 * b, b2 * b2
            P = fma32(fma32(fma32(fma32(f32(128), a, f32(-256) * b), a, f32(160) * b2), a, f32(-32) * b3), a, b4)
            A = fma32(fma32(fma32(f32(128), a, f32(-192) * b), a, f32(80) * b2), a, f32(-8) * b3)
            ax = wx * wx
            q = fma32(wx, wx, wy * wy)
            q2 = q * q
            q3, q4 = q2 * q, q2 * q2
            C = fma32(fma32(fma32(fma32(f32(128), ax, f32(-256) * q), ax, f32(160) * q2), ax, f32(-32) * q3), ax, q4)
            B = fma32(fma32(fma32(f32(128), ax, f32(-192) * q), ax, f32(80) * q2), ax, f32(-8) * q3)
            k = (wz * A) / (q3 * np.sqrt(q))
            k = np.where(q > f32(0), k, f32(0))
            nx, ny, nz = fma32(k, C, cx), fma32(k, (wx * wy) * B, cy), P + cz
            nm = nx * nx + (ny * ny + nz * nz)
            wx, wy, wz = np.where(go, nx, wx), np.where(go, ny, wy), np.where(go, nz, wz)
            m = np.where(go, nm, m)
            trap = np.where(go, _min_fold(nm, trap), trap)
    return trap


def sdf_trap(h, p):
    from rayn_b200 import _lib as L
    return mandelbulb_trap(h, p) if h.kind == L.HITABLE_MANDELBULB else mandelbox_trap(h, p)


def palette(trap_lo, trap_hi, albedo_lo, albedo_hi, trap):
    """-> (s, albedo [n, 3])"""
    t = np.asarray(trap, np.float32).reshape(-1)
    lo, hi = f32(trap_lo), f32(trap_hi)
    with np.errstate(all="ignore"):
        s = np.where(~(t > lo), f32(0), np.where(t >= hi, f32(1), (t - lo) / (hi - lo))).astype(np.float32)
        r = f32(1) - s
        a = np.stack([f32(albedo_lo[c]) * r + f32(albedo_hi[c]) * s for c in range(3)], axis=1)
    return s, a.astype(np.float32)
