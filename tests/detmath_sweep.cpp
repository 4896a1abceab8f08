// detmath_sweep.cpp — exhaustive sweeps of rayn_b200/csrc/detmath.h over 32-bit input patterns.  TEST INFRASTRUCTURE ONLY.
//
// A sweep is one function (op, numbered as rayn_b200_kat_detmath's) with an optional fixed second operand, evaluated at
// every pattern of a contiguous range of 2^24-pattern chunks.  Per chunk it returns the order-free hash
//   sum over the chunk of splitmix64((in_bits << 32) | out_bits)  mod 2^64
// (the device computes the same sum with atomics), and over the range the worst error against long-double libm.
// Built by tests/mirrors.py with the render mirror's flags; includes detmath.h and nothing of the oracle.
#include <math.h>
#include <stdint.h>

#include "../rayn_b200/csrc/detmath.h"

namespace {

enum { OP_EXP, OP_LN, OP_POW, OP_SIN, OP_COS, OP_TAN, OP_ATAN2, OP_POWI5, OP_LN_FAST };

inline uint64_t splitmix64(uint64_t z) {
  z += 0x9e3779b97f4a7c15ull;
  z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
  z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
  return z ^ (z >> 31);
}

inline float eval(int op, float a, float b) {
  float s, c;
  switch (op) {
    case OP_EXP: return dm::exp(a);
    case OP_LN: return dm::ln(a);
    case OP_POW: return dm::pow(a, b);
    case OP_SIN: dm::sincos(a, &s, &c); return s;
    case OP_COS: dm::sincos(a, &s, &c); return c;
    case OP_TAN: return dm::tan(a);
    case OP_ATAN2: return dm::atan2(a, b);
    case OP_POWI5: return dm::powi5(a);
    default: return dm::ln_fast(a);
  }
}

// The hashed result bits: exact, NaN payloads included, except powi5's NaN, whose payload is the hardware's (detmath.h)
inline uint32_t out_bits(int op, float out) { return op == OP_POWI5 && out != out ? 0x7fc00000u : dm::f2u(out); }

// Where the error is measured (the function's contract; elsewhere the result is a documented NaN or, for powi5, checked
// bit for bit against its definition) and where the render path needs it correctly rounded.
inline bool in_contract(int op, float a, float b) {
  if (a != a || b != b) return false;
  switch (op) {
    case OP_POW: return !(a < 0.0f);
    case OP_SIN: case OP_COS: case OP_TAN: return fabsf(a) <= 1.0e5f;
    case OP_POWI5: return false;
    case OP_LN_FAST: return a > 0.0f && a < INFINITY;
    default: return true;
  }
}
inline bool in_render(int op, float a) {
  switch (op) {
    case OP_EXP: return a <= 0.0f;
    case OP_LN: return a > 0.0f;
    case OP_SIN: case OP_COS: return a >= 0.0f && a <= 6.28318548f;  // [0, 2 pi]
    case OP_TAN: return fabsf(a) <= 1.57079625f;                     // (-pi/2, pi/2): the last float below pi/2
    default: return true;
  }
}

inline long double reference(int op, float a, float b) {
  const long double x = a, y = b;
  switch (op) {
    case OP_EXP: return expl(x);
    case OP_LN: case OP_LN_FAST: return logl(x);
    case OP_POW: return powl(x, y);
    case OP_SIN: return sinl(x);
    case OP_COS: return cosl(x);
    case OP_TAN: return tanl(x);
    default: return atan2l(x, y);
  }
}

const double kHuge = 1e300;  // a wrong class of result (NaN, inf or finite where the other is not)

// ulp error of float `got` against the exact `ref`: one ulp is the spacing of the float binade holding ref (2^-149 for
// subnormals); a ref at or past the overflow threshold 2^128 - 2^103 must give the infinity of its sign.
inline double ulp_error(float got, long double ref) {
  if (ref != ref) return got != got ? 0.0 : kHuge;
  if (got != got) return kHuge;
  const long double aref = fabsl(ref);
  if (aref >= 0x1.ffffffp127L) return (isinf(got) && (got < 0) == (ref < 0)) ? 0.0 : kHuge;
  if (isinf(got)) return kHuge;
  int ex = 0;
  if (aref != 0) frexpl(aref, &ex);
  const long double ulp = ldexpl(1.0L, ex - 24 > -149 ? ex - 24 : -149);
  return (double)(fabsl((long double)got - ref) / ulp);
}
// ln_fast: relative error, absolute where |ln x| < 1
inline double rel_error(float got, long double ref) {
  if (got != got || isinf(got)) return kHuge;
  const long double aref = fabsl(ref);
  return (double)(fabsl((long double)got - ref) / (aref > 1.0L ? aref : 1.0L));
}

struct Acc {
  double max_err;
  uint32_t argmax;  // input pattern of max_err (the smallest one on ties)
  int64_t over;     // errors above the bound
};
inline void acc_add(Acc& a, double e, uint32_t in, double bound) {
  if (e > a.max_err || (e == a.max_err && in < a.argmax)) {
    a.max_err = e;
    a.argmax = in;
  }
  a.over += e > bound;
}
inline void acc_merge(Acc& a, const Acc& b) {
  if (b.max_err > a.max_err || (b.max_err == a.max_err && b.argmax < a.argmax)) {
    a.max_err = b.max_err;
    a.argmax = b.argmax;
  }
  a.over += b.over;
}

}  // namespace

extern "C" {

// the two checks tests/mirrors.py makes of every library it builds
int32_t rayn_oracle_selfcheck(void) {
  volatile float a = 1.0f + 0x1p-12f, c = -(1.0f + 0x1p-11f);
  float x = a, z = c;
  return (x * x + z == 0.0f && dm::fma(x, x, z) == 0x1p-24f) ? 0 : 1;
}
int32_t rayn_oracle_muladd_fused(void) { return RAYN_MULADD_FUSED; }

// op 0..8 as rayn_b200_kat_detmath; the swept operand runs over patterns [chunk0 << 24, (chunk0 + n_chunks) << 24) and
// is the first operand, or the second (swap != 0) with `fixed` the first.  hashes[n_chunks]; with accuracy != 0,
// acc[0] is the error over the contract domain and acc[1] over the render-path domain (in_contract / in_render), each
// {max, argmax pattern, count above `bound`}: ulp error, or relative error for ln_fast.
int32_t detmath_sweep(int32_t op, float fixed, int32_t swap, int32_t chunk0, int32_t n_chunks, int32_t accuracy, double bound,
                      uint64_t* hashes, Acc* acc) {
  if (op < OP_EXP || op > OP_LN_FAST || chunk0 < 0 || n_chunks < 0 || chunk0 + n_chunks > 256 || !hashes || (accuracy && !acc))
    return 1;
  Acc total[2] = {{0.0, 0xffffffffu, 0}, {0.0, 0xffffffffu, 0}};
  for (int32_t k = 0; k < n_chunks; ++k) {
    const uint64_t base = (uint64_t)(chunk0 + k) << 24;
    uint64_t h = 0;
#pragma omp parallel reduction(+ : h)
    {
      Acc local[2] = {{0.0, 0xffffffffu, 0}, {0.0, 0xffffffffu, 0}};
#pragma omp for schedule(static, 4096)
      for (int64_t i = 0; i < (1 << 24); ++i) {
        const uint32_t in = (uint32_t)(base + (uint64_t)i);
        const float v = dm::u2f(in);
        const float a = swap ? fixed : v, b = swap ? v : fixed;
        const float out = eval(op, a, b);
        h += splitmix64(((uint64_t)in << 32) | out_bits(op, out));
        if (accuracy && in_contract(op, a, b)) {
          const long double ref = reference(op, a, b);
          const double e = op == OP_LN_FAST ? rel_error(out, ref) : ulp_error(out, ref);
          acc_add(local[0], e, in, bound);
          if (swap || in_render(op, a)) acc_add(local[1], e, in, bound);
        }
      }
#pragma omp critical
      {
        acc_merge(total[0], local[0]);
        acc_merge(total[1], local[1]);
      }
    }
    hashes[k] = h;
  }
  if (accuracy) acc[0] = total[0], acc[1] = total[1];
  return 0;
}

// the error measure of one result (tests recompute recorded maxima with mpmath against it)
double detmath_error(int32_t op, float a, float b, float got) {
  const long double ref = reference(op, a, b);
  return op == OP_LN_FAST ? rel_error(got, ref) : ulp_error(got, ref);
}

}  // extern "C"
