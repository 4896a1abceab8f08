// detmath.h — deterministic numeric primitives shared by host and device code.
//
// Why this exists: the render path thresholds a chaotic fractal distance field at ~1e-5
// (reference src/sdf.rs:48,69-71), so a 1-ulp difference between two implementations can
// change a march count and hence a path.  Parity between the CUDA kernels and the CPU
// oracle is therefore demanded BIT-exact, which needs every arithmetic step to be an IEEE
// correctly-rounded operation on both sides.  + - * / sqrt and explicit fma are; libm's
// exp/pow/sin/cos/tan/atan2/log are not (glibc and CUDA differ).  The functions below
// rebuild those from + - * / sqrt, floor and bit operations only, evaluated in double and
// rounded once to float, so `g++ -ffp-contract=off` and `nvcc --fmad=false -prec-div=true
// -prec-sqrt=true -ftz=false` produce identical bits.
//
// These stand in for the lane-wise `f32x4::{exp, powf, powi, sin_cos, tan, atan2}` of the
// `wide` 0.4.6 crate (reference call sites: src/integrator.rs:65,123,234,272;
// src/material.rs:199,236; src/math.rs:108,111,123,217; src/light.rs:61,93-97).  That crate
// is not on disk (SURVEY F4), so agreement with real rayn is to within the accuracy of a
// good libm (< 1 ulp here), not bitwise.
//
// This header is numeric plumbing, not the render algorithm: the algorithm is written
// twice (CUDA kernels in this directory; SSE-packet oracle under oracle/).
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#if defined(__CUDACC__)
#define DM_HD __host__ __device__ __forceinline__
#else
#define DM_HD inline
#endif

namespace dm {

// ---- bit casts ---------------------------------------------------------------------
DM_HD uint32_t f2u(float x) {
#ifdef __CUDA_ARCH__
  return __float_as_uint(x);
#else
  uint32_t u;
  memcpy(&u, &x, 4);
  return u;
#endif
}
DM_HD float u2f(uint32_t u) {
#ifdef __CUDA_ARCH__
  return __uint_as_float(u);
#else
  float x;
  memcpy(&x, &u, 4);
  return x;
#endif
}
DM_HD int64_t d2i(double x) {
#ifdef __CUDA_ARCH__
  return __double_as_longlong(x);
#else
  int64_t u;
  memcpy(&u, &x, 8);
  return u;
#endif
}
DM_HD double i2d(int64_t u) {
#ifdef __CUDA_ARCH__
  return __longlong_as_double(u);
#else
  double x;
  memcpy(&x, &u, 8);
  return x;
#endif
}

// ---- exactly-defined float helpers -------------------------------------------------
// Explicit single-rounding fused multiply-add.  Used directly only where the arithmetic is OURS to
// define (the authored Mandelbulb, the float-only transcendental cores below).
DM_HD float fma(float a, float b, float c) {
#ifdef __CUDA_ARCH__
  return __fmaf_rn(a, b, c);
#else
  return __builtin_fmaf(a, b, c);
#endif
}
// `wide` 0.4.6 `f32x4::mul_add` — what the reference writes at src/sdf.rs:45,134-135,161; src/ray.rs:23;
// src/math.rs:203-204,210; src/light.rs:99 and what ultraviolet's dot / cross / mag_sq are built from.
// That crate fuses only under `cfg(target_feature = "fma")`; the reference builds with a plain
// `cargo run --release` (README.md:42-44, Cargo.toml:10-14: no RUSTFLAGS, no .cargo/config), so the x86-64
// baseline target has no `fma` feature and mul_add is `(a * b) + c` with TWO roundings.  That is the default here
// (RAYN_MULADD_FUSED = 0).  RAYN_MULADD_FUSED = 1 builds the variant a `-C target-feature=+fma` rayn would give;
// kernels, oracle and golden fixtures exist for both (oracle/README.md A6).
#ifndef RAYN_MULADD_FUSED
#define RAYN_MULADD_FUSED 0
#endif
DM_HD float mul_add(float a, float b, float c) {
#if RAYN_MULADD_FUSED
  return dm::fma(a, b, c);
#else
#ifdef __CUDA_ARCH__
  return __fadd_rn(__fmul_rn(a, b), c);  // never contracted, whatever --fmad says
#else
  return a * b + c;  // host TUs are compiled with -ffp-contract=off
#endif
#endif
}
// SSE minps/maxps semantics (`wide` f32x4::min/max): second operand on NaN.
DM_HD float min(float a, float b) { return a < b ? a : b; }
DM_HD float max(float a, float b) { return a > b ? a : b; }
DM_HD float abs(float a) { return u2f(f2u(a) & 0x7fffffffu); }
DM_HD bool is_nan(float a) { return a != a; }
// Rust f32::signum: NaN -> NaN, otherwise copysign(1, x) (so signum(-0.0) = -1).
DM_HD float signum(float a) {
  if (a != a) return a;
  return u2f((f2u(a) & 0x80000000u) | 0x3f800000u);
}
// Rust f32::fract = x - trunc(x)
DM_HD float fract(float a) { return a - truncf(a); }
// compiler-rt __powisf2(x, 5): r = x; x2 = x*x; x4 = x2*x2; r *= x4
DM_HD float powi5(float x) {
  float x2 = x * x;
  float x4 = x2 * x2;
  return x * x4;
}

// ---- double-precision cores --------------------------------------------------------
// Horner steps and argument reductions use an explicit double fma (one DFMA instead of DMUL + DADD under --fmad=false /
// -ffp-contract=off; also one rounding less).  Same operation on host and device, so the bits stay identical.
DM_HD double dfma(double a, double b, double c) {
#ifdef __CUDA_ARCH__
  return __fma_rn(a, b, c);
#else
  return __builtin_fma(a, b, c);
#endif
}

#define DM_LN2_HI 6.93147180369123816490e-01
#define DM_LN2_LO 1.90821492927058770002e-10
#define DM_LOG2E 1.4426950408889634
#define DM_PIO2_HI 1.57079632673412561417e+00
#define DM_PIO2_LO 6.07710050650619224932e-11
#define DM_2OPI 0.6366197723675814
#define DM_PI 3.141592653589793
#define DM_PIO2 1.5707963267948966

// exp for |x| <= ~700; Taylor degree 13 on |r| <= ln2/2
DM_HD double exp_core(double x) {
  double kf = floor(x * DM_LOG2E + 0.5);
  double r = dfma(-kf, DM_LN2_LO, dfma(-kf, DM_LN2_HI, x));
  double p = 1.0 / 6227020800.0;
  p = dfma(p, r, 1.0 / 479001600.0);
  p = dfma(p, r, 1.0 / 39916800.0);
  p = dfma(p, r, 1.0 / 3628800.0);
  p = dfma(p, r, 1.0 / 362880.0);
  p = dfma(p, r, 1.0 / 40320.0);
  p = dfma(p, r, 1.0 / 5040.0);
  p = dfma(p, r, 1.0 / 720.0);
  p = dfma(p, r, 1.0 / 120.0);
  p = dfma(p, r, 1.0 / 24.0);
  p = dfma(p, r, 1.0 / 6.0);
  p = dfma(p, r, 0.5);
  p = dfma(p, r, 1.0);
  p = dfma(p, r, 1.0);
  int64_t k = (int64_t)kf;
  return p * i2d((k + 1023) << 52);
}

// natural log of a positive, finite, normal double
DM_HD double ln_core(double x) {
  int64_t bits = d2i(x);
  int64_t e = ((bits >> 52) & 0x7ff) - 1023;
  double m = i2d((bits & 0x000fffffffffffffLL) | 0x3ff0000000000000LL);
  if (m > 1.4142135623730951) {
    m = m * 0.5;
    e = e + 1;
  }
  double s = (m - 1.0) / (m + 1.0);
  double z = s * s;
  double p = 1.0 / 19.0;
  p = dfma(p, z, 1.0 / 17.0);
  p = dfma(p, z, 1.0 / 15.0);
  p = dfma(p, z, 1.0 / 13.0);
  p = dfma(p, z, 1.0 / 11.0);
  p = dfma(p, z, 1.0 / 9.0);
  p = dfma(p, z, 1.0 / 7.0);
  p = dfma(p, z, 1.0 / 5.0);
  p = dfma(p, z, 1.0 / 3.0);
  p = dfma(p, z, 1.0);
  double ef = (double)e;
  return dfma(ef, DM_LN2_HI, dfma(2.0 * s, p, ef * DM_LN2_LO));
}

// sin and cos of a finite double with |x| < 2^20
DM_HD void sincos_core(double x, double* sn, double* cs) {
  double kf = floor(x * DM_2OPI + 0.5);
  double r = dfma(-kf, DM_PIO2_LO, dfma(-kf, DM_PIO2_HI, x));
  double z = r * r;
  double ps = -1.0 / 1307674368000.0;
  ps = dfma(ps, z, 1.0 / 6227020800.0);
  ps = dfma(ps, z, -(1.0 / 39916800.0));
  ps = dfma(ps, z, 1.0 / 362880.0);
  ps = dfma(ps, z, -(1.0 / 5040.0));
  ps = dfma(ps, z, 1.0 / 120.0);
  ps = dfma(ps, z, -(1.0 / 6.0));
  ps = dfma(ps, z, 1.0);
  double sr = ps * r;
  double pc = 1.0 / 20922789888000.0;
  pc = dfma(pc, z, -(1.0 / 87178291200.0));
  pc = dfma(pc, z, 1.0 / 479001600.0);
  pc = dfma(pc, z, -(1.0 / 3628800.0));
  pc = dfma(pc, z, 1.0 / 40320.0);
  pc = dfma(pc, z, -(1.0 / 720.0));
  pc = dfma(pc, z, 1.0 / 24.0);
  pc = dfma(pc, z, -(0.5));
  double cr = dfma(pc, z, 1.0);
  int q = (int)(((int64_t)kf) & 3);
  if (q == 0) {
    *sn = sr;
    *cs = cr;
  } else if (q == 1) {
    *sn = cr;
    *cs = -sr;
  } else if (q == 2) {
    *sn = -sr;
    *cs = -cr;
  } else {
    *sn = -cr;
    *cs = sr;
  }
}

// atan of z in [0, 1]
DM_HD double atan01_core(double z) {
  // two half-angle reductions: atan(z) = 2 atan(z / (1 + sqrt(1 + z^2)))
  z = z / (1.0 + sqrt(1.0 + z * z));
  z = z / (1.0 + sqrt(1.0 + z * z));
  double w = z * z;
  double p = -1.0 / 19.0;
  p = dfma(p, w, 1.0 / 17.0);
  p = dfma(p, w, -(1.0 / 15.0));
  p = dfma(p, w, 1.0 / 13.0);
  p = dfma(p, w, -(1.0 / 11.0));
  p = dfma(p, w, 1.0 / 9.0);
  p = dfma(p, w, -(1.0 / 7.0));
  p = dfma(p, w, 1.0 / 5.0);
  p = dfma(p, w, -(1.0 / 3.0));
  p = dfma(p, w, 1.0);
  return 4.0 * (z * p);
}

// ---- float API ---------------------------------------------------------------------
DM_HD float exp(float x) {
  if (x != x) return x;
  double xd = (double)x;
  if (xd > 100.0) xd = 100.0;    // e^100 overflows float -> +inf after the final rounding
  if (xd < -110.0) xd = -110.0;  // e^-110 underflows float -> 0
  return (float)exp_core(xd);
}

DM_HD float ln(float x) {
  if (x != x) return x;
  if (x < 0.0f) return u2f(0x7fc00000u);
  if (x == 0.0f) return u2f(0xff800000u);
  if (f2u(x) == 0x7f800000u) return x;
  return (float)ln_core((double)x);
}

// ln of 2^((b >> 23) - 127) * 1.m, m the low 23 bits of b: a positive normal float's bit pattern, or a subnormal's
// normalised one (exponent field below 1, so b >> 23 is negative)
DM_HD float ln_fast_bits(int32_t b) {
  int e = (b >> 23) - 127;
  float m = u2f(((uint32_t)b & 0x007fffffu) | 0x3f800000u);  // [1, 2)
  if (m > 1.41421356f) {
    m = m * 0.5f;
    e = e + 1;
  }
  const float s = (m - 1.0f) / (m + 1.0f);
  const float z = s * s;
  float p = 1.0f / 9.0f;
  p = dfma(p, z, 1.0f / 7.0f);
  p = dfma(p, z, 0.2f);
  p = dfma(p, z, 1.0f / 3.0f);
  p = dfma(p, z, 1.0f);
  return (float)e * 0.693147180559945f + 2.0f * s * p;
}
// Float-only natural log (no double pipe): ~2e-7 relative accuracy.  Used by the AUTHORED
// Mandelbulb distance estimator, whose definition is ours to make; bit-identical host/device
// because it is built from IEEE float + - * / and integer bit operations only.
DM_HD float ln_fast(float x) {
  if (x != x) return x;
  if (x < 0.0f) return u2f(0x7fc00000u);
  const int32_t b = (int32_t)f2u(x);
  if (b < 0x00800000) {  // +-0 (-0 has the sign bit) or subnormal: an early return, so the march loop's path is unchanged
    if (x == 0.0f) return u2f(0xff800000u);
    return ln_fast_bits((int32_t)f2u(x * 0x1p23f) - (23 << 23));  // x * 2^23 is exact and normal
  }
  if (b == 0x7f800000) return x;
  return ln_fast_bits(b);
}

// ---- documented domain restrictions: where the functions below differ from C99 Annex F --------------------------
// Everything else matches Annex F for zeros, subnormals, infinities and NaN (tests/test_cpu_shared_numerics.py
// checks the full table of special operands on host and device and pins each value listed here).  These stay
// because pow and sincos/tan sit on the shading path and no render reaches these operands:
//   pow(x, y), x < 0 (-inf included), y != 0:   NaN     (C99: x^y for integer y, e.g. pow(-2, 2) = 4)
//   pow(-0, y), y an odd integer:                +0 for y > 0, +inf for y < 0   (C99: -0, -inf)
//   pow(1, NaN):                                 NaN     (C99: 1)
//   sin, cos, tan of |x| > 1e5:                  NaN     (C99: finite)
// NaN payloads: exp, ln and ln_fast return a NaN input as it is; pow, sin, cos, tan and atan2 return 0x7fc00000.
// powi5 is plain float multiplies, so its NaN is the hardware's: the input's, quieted, on x86; 0x7fffffff on the GPU.
// The measured accuracy over every float is in oracle/README.md (A9).

// powf for the domain the render path uses (x >= 0).
DM_HD float pow(float x, float y) {
  if (y == 0.0f) return 1.0f;
  if (x != x || y != y) return u2f(0x7fc00000u);
  if (x < 0.0f) return u2f(0x7fc00000u);
  if (x == 0.0f) return y > 0.0f ? 0.0f : u2f(0x7f800000u);
  if (f2u(x) == 0x7f800000u) return y > 0.0f ? x : 0.0f;
  if (x == 1.0f) return 1.0f;
  double e = (double)y * ln_core((double)x);
  if (e != e) return u2f(0x7fc00000u);
  if (e > 100.0) e = 100.0;
  if (e < -110.0) e = -110.0;
  return (float)exp_core(e);
}

DM_HD void sincos(float x, float* s, float* c) {
  if (x != x || dm::abs(x) > 1.0e5f) {
    *s = u2f(0x7fc00000u);
    *c = u2f(0x7fc00000u);
    return;
  }
  double sd, cd;
  sincos_core((double)x, &sd, &cd);
  *s = (float)sd;
  *c = (float)cd;
}

DM_HD float tan(float x) {
  if (x != x || dm::abs(x) > 1.0e5f) return u2f(0x7fc00000u);
  double sd, cd;
  sincos_core((double)x, &sd, &cd);
  return (float)(sd / cd);
}

// C99 Annex F atan2, signed zeros and infinite operands included: the quadrant follows the SIGN BITS, so
// atan2(+-0, -0) = +-pi and atan2(-0, x > 0) = -0; |y| = |x| = inf gives +-pi/4 or +-3pi/4.
DM_HD float atan2(float y, float x) {
  if (x != x || y != y) return u2f(0x7fc00000u);
  double ax = (double)dm::abs(x), ay = (double)dm::abs(y);
  double a;
  if (ay > ax) {
    a = DM_PIO2 - atan01_core(ax / ay);
  } else if (ay == 0.0) {
    a = 0.0;
  } else {
    a = atan01_core(ay == ax ? 1.0 : ay / ax);  // ay / ax = 1 for finite ties; inf / inf would be NaN
  }
  if (f2u(x) >> 31) a = DM_PI - a;
  if (f2u(y) >> 31) a = -a;
  return (float)a;
}

}  // namespace dm
