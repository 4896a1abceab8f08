// rayn_oracle.cpp — CPU ORACLE.  TEST INFRASTRUCTURE ONLY: nothing under rayn_b200/ may
// include, link, import or execute this.  Only tests/, __graft_entry__.smoke() and the
// cpu_baseline / --impl reference legs of bench.py use it, and only as the checker.
//
// PARITY UNPINNED: the reference (fu5ha/rayn @ 6486a86) has no tests, golden vectors or
// fixtures for this path (SURVEY F2), and cannot be compiled here (no rustc/cargo; its
// arithmetic crates ultraviolet/wide/sdfu/quasi-rd/rand are not on disk, SURVEY F4).  This
// file is a restatement of the reference's algorithm written from its source; where the
// behaviour lives in an absent crate the assumption is listed in oracle/README.md.
//
// What is restated (reference file:line):
//   film.rs:439-627   per-tile wavefront closure: raygen, depth loop, extend, bin, shade,
//                     splat, compact            -> render_tile()
//   film.rs:695-709   sample_uv                 -> sample_uv()
//   filter.rs:222-235 FilterImportanceSampler::sample -> fis_sample()
//   sampler.rs:62-126 Samples::sample_{1d,2d}   -> Tables::s1 / s2
//   camera.rs:81-118,168-212,249-284            -> camera_get_rays(), half_pixel_size_at()
//   hitable.rs:30-48,94-133,164-210             -> ShadingPoint, process_hits(), test_occluded(),
//                                                  add_hits()
//   sdf.rs:25-101,125-188                       -> sdf_occluded(), sdf_hit(), sdf_shading_info(),
//                                                  mandelbox_dist()
//   sphere.rs:24-86                             -> sphere_*()
//   integrator.rs:47-281                        -> integrate(), surface_sample_one_light(),
//                                                  volume_sample_one_light()
//   material.rs:117-142,195-256,425-449,495-520 -> bsdf_*()
//   light.rs:38-107                             -> light_sample(), light_sample_volume()
//   math.rs:49-59,99-113,122-124,201-219        -> onb(), cosine_weighted(), cosine_power(),
//                                                  f_schlick(), concentric()
//   ray.rs:54-66                                -> Ray::invalid()
//
// Structure: rayn computes on 4-lane SSE packets (`wide::f32x4`), and lanes of a packet are
// coupled through next-event light selection (integrator.rs:76-93).  The oracle keeps that
// structure literally: F4 wraps __m128 with the SSE semantics `wide` 0.4.6 exposes
// (minps/maxps NaN behaviour, all-ones compare masks, merge, move_mask), V3 is `Wec3`.
// The CUDA path is organised completely differently (one thread per lane, wavefront
// kernels, index queues), which is what makes a bit-exact comparison meaningful.
//
// Build: see oracle/Makefile.  MUST be compiled with -ffp-contract=off (GCC implements the
// SSE intrinsics as plain vector operators and would otherwise fuse a*b+c).

#include <immintrin.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "../include/rayn_b200.h"
#include "../rayn_b200/csrc/detmath.h"

#ifdef _OPENMP
#include <omp.h>
#endif

namespace {

// ------------------------------------------------------------------------------------------
// f32x4 with `wide` 0.4.6 / SSE semantics
// ------------------------------------------------------------------------------------------
struct F4 {
  __m128 v;
  float operator[](int i) const {
    alignas(16) float t[4];
    _mm_store_ps(t, v);
    return t[i];
  }
};
inline F4 splat(float x) { return {_mm_set1_ps(x)}; }
inline F4 make4(float a, float b, float c, float d) { return {_mm_setr_ps(a, b, c, d)}; }
inline F4 load4(const float* p) { return {_mm_loadu_ps(p)}; }
inline void store4(float* p, F4 a) { _mm_storeu_ps(p, a.v); }
inline F4 operator+(F4 a, F4 b) { return {_mm_add_ps(a.v, b.v)}; }
inline F4 operator-(F4 a, F4 b) { return {_mm_sub_ps(a.v, b.v)}; }
inline F4 operator*(F4 a, F4 b) { return {_mm_mul_ps(a.v, b.v)}; }
inline F4 operator/(F4 a, F4 b) { return {_mm_div_ps(a.v, b.v)}; }
inline F4 operator-(F4 a) { return {_mm_xor_ps(a.v, _mm_set1_ps(-0.0f))}; }
inline F4 operator|(F4 a, F4 b) { return {_mm_or_ps(a.v, b.v)}; }
inline F4 operator&(F4 a, F4 b) { return {_mm_and_ps(a.v, b.v)}; }
inline F4 f4not(F4 a) { return {_mm_xor_ps(a.v, _mm_castsi128_ps(_mm_set1_epi32(-1)))}; }
inline F4 f4abs(F4 a) { return {_mm_andnot_ps(_mm_set1_ps(-0.0f), a.v)}; }
inline F4 f4sqrt(F4 a) { return {_mm_sqrt_ps(a.v)}; }
inline F4 f4min(F4 a, F4 b) { return {_mm_min_ps(a.v, b.v)}; }  // a.min(b): b if unordered
inline F4 f4max(F4 a, F4 b) { return {_mm_max_ps(a.v, b.v)}; }  // a.max(b): b if unordered
inline F4 fma4(F4 a, F4 b, F4 c) { return {_mm_fmadd_ps(a.v, b.v, c.v)}; }  // a*b+c fused: only where the arithmetic is ours (authored Mandelbulb)
// wide 0.4.6 f32x4::mul_add (A6): `(self * b) + c` unless the crate is built with target_feature = "fma".
// RAYN_MULADD_FUSED (detmath.h) selects; default 0 = what a stock `cargo run --release` of rayn produces.
#if RAYN_MULADD_FUSED
inline F4 mul_add(F4 a, F4 b, F4 c) { return {_mm_fmadd_ps(a.v, b.v, c.v)}; }
#else
inline F4 mul_add(F4 a, F4 b, F4 c) { return {_mm_add_ps(_mm_mul_ps(a.v, b.v), c.v)}; }
#endif
inline F4 cmp_lt(F4 a, F4 b) { return {_mm_cmplt_ps(a.v, b.v)}; }
inline F4 cmp_le(F4 a, F4 b) { return {_mm_cmple_ps(a.v, b.v)}; }
inline F4 cmp_gt(F4 a, F4 b) { return {_mm_cmpgt_ps(a.v, b.v)}; }
inline F4 cmp_eq(F4 a, F4 b) { return {_mm_cmpeq_ps(a.v, b.v)}; }
inline F4 cmp_nan(F4 a, F4 b) { return {_mm_cmpunord_ps(a.v, b.v)}; }
inline F4 merge(F4 m, F4 t, F4 f) { return {_mm_or_ps(_mm_and_ps(m.v, t.v), _mm_andnot_ps(m.v, f.v))}; }
inline int move_mask(F4 a) { return _mm_movemask_ps(a.v); }

template <class Fn>
inline F4 map4(F4 a, Fn fn) {
  alignas(16) float t[4];
  _mm_store_ps(t, a.v);
  for (int i = 0; i < 4; ++i) t[i] = fn(t[i]);
  return {_mm_load_ps(t)};
}
template <class Fn>
inline F4 map4(F4 a, F4 b, Fn fn) {
  alignas(16) float t[4], u[4];
  _mm_store_ps(t, a.v);
  _mm_store_ps(u, b.v);
  for (int i = 0; i < 4; ++i) t[i] = fn(t[i], u[i]);
  return {_mm_load_ps(t)};
}
inline F4 f4floor(F4 a) { return map4(a, [](float x) { return floorf(x); }); }
inline F4 f4signum(F4 a) { return map4(a, [](float x) { return dm::signum(x); }); }
inline F4 f4exp(F4 a) { return map4(a, [](float x) { return dm::exp(x); }); }
inline F4 f4powf(F4 a, F4 b) { return map4(a, b, [](float x, float y) { return dm::pow(x, y); }); }
inline F4 f4powi5(F4 a) { return map4(a, [](float x) { return dm::powi5(x); }); }
inline F4 f4tan(F4 a) { return map4(a, [](float x) { return dm::tan(x); }); }
inline F4 f4atan2(F4 y, F4 x) { return map4(y, x, [](float a, float b) { return dm::atan2(a, b); }); }
inline void f4sincos(F4 a, F4* s, F4* c) {
  alignas(16) float t[4], ss[4], cc[4];
  _mm_store_ps(t, a.v);
  for (int i = 0; i < 4; ++i) dm::sincos(t[i], &ss[i], &cc[i]);
  s->v = _mm_load_ps(ss);
  c->v = _mm_load_ps(cc);
}
// sdfu::mathtypes::Lerp: a*(1-t) + b*t   (assumption A7)
inline F4 f4lerp(F4 a, F4 b, F4 t) { return a * (splat(1.0f) - t) + b * t; }
inline float lerpf(float a, float b, float t) { return a * (1.0f - t) + b * t; }

const float kPI = 3.14159265358979323846f;
const float kTWO_PI = 6.28318530717958647692f;
const float kFRAC_PI_2 = 1.57079632679489661923f;
const float kFRAC_PI_4 = 0.78539816339744830962f;
const float kEPSILON = 1.1920929e-7f;

// ------------------------------------------------------------------------------------------
// Wec3 (ultraviolet 0.4.6; assumptions A1-A6)
// ------------------------------------------------------------------------------------------
struct V3 {
  F4 x, y, z;
};
inline V3 v3splat(float x, float y, float z) { return {splat(x), splat(y), splat(z)}; }
inline V3 v3broadcast(F4 a) { return {a, a, a}; }
inline V3 operator+(V3 a, V3 b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
inline V3 operator-(V3 a, V3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
inline V3 operator*(V3 a, V3 b) { return {a.x * b.x, a.y * b.y, a.z * b.z}; }
inline V3 operator*(V3 a, F4 s) { return {a.x * s, a.y * s, a.z * s}; }
inline V3 operator/(V3 a, F4 s) { return {a.x / s, a.y / s, a.z / s}; }
inline V3 operator-(V3 a) { return {-a.x, -a.y, -a.z}; }
inline V3 v3mul_add(V3 a, V3 b, V3 c) {
  return {mul_add(a.x, b.x, c.x), mul_add(a.y, b.y, c.y), mul_add(a.z, b.z, c.z)};
}
inline F4 dot(V3 a, V3 b) { return mul_add(a.x, b.x, mul_add(a.y, b.y, a.z * b.z)); }
inline F4 mag_sq(V3 a) { return dot(a, a); }
inline F4 mag(V3 a) { return f4sqrt(mag_sq(a)); }
inline V3 normalized(V3 a) {
  F4 r = splat(1.0f) / mag(a);
  return a * r;
}
inline V3 cross(V3 a, V3 b) {
  return {mul_add(a.y, b.z, -(a.z * b.y)), mul_add(a.z, b.x, -(a.x * b.z)),
          mul_add(a.x, b.y, -(a.y * b.x))};
}
inline V3 v3merge(F4 m, V3 t, V3 f) { return {merge(m, t.x, f.x), merge(m, t.y, f.y), merge(m, t.z, f.z)}; }
inline V3 v3clamped(V3 a, V3 lo, V3 hi) {
  return {f4min(f4max(a.x, lo.x), hi.x), f4min(f4max(a.y, lo.y), hi.y), f4min(f4max(a.z, lo.z), hi.z)};
}
inline V3 reflected(V3 v, V3 n) { return v - n * (splat(2.0f) * dot(v, n)); }
inline F4 component_max(V3 a) { return f4max(f4max(a.x, a.y), a.z); }

struct M3 {
  V3 c0, c1, c2;
};  // Wat3, column major
inline V3 operator*(M3 m, V3 v) { return m.c0 * v.x + m.c1 * v.y + m.c2 * v.z; }

// math.rs:49-59
inline M3 onb(V3 nor) {
  F4 one = splat(1.0f);
  F4 ks = f4signum(nor.z);
  F4 ka = one / (one + f4abs(nor.z));
  F4 kb = -ks * nor.x * nor.y * ka;
  V3 uu = {one - nor.x * nor.x * ka, ks * kb, -ks * nor.x};
  V3 vv = {kb, ks - nor.y * nor.y * ka * ks, -nor.y};
  return {uu, vv, nor};
}

// math.rs:201-219
inline void concentric(F4 u0, F4 u1, F4* ox, F4* oy) {
  F4 two = splat(2.0f), one = splat(1.0f);
  F4 a = mul_add(u0, two, -one);
  F4 b = mul_add(u1, two, -one);
  F4 zero_mask = cmp_eq(a, splat(0.0f)) & cmp_eq(b, splat(0.0f));
  b = merge(zero_mask, splat(0.0001f), b);
  F4 phi1 = splat(kFRAC_PI_4) * b / a;
  F4 phi2 = mul_add(-splat(kFRAC_PI_4) / b, a, splat(kFRAC_PI_2));
  F4 mask = cmp_gt(a * a, b * b);
  F4 r = merge(mask, a, b);
  F4 phi = merge(mask, phi1, phi2);
  F4 s, c;
  f4sincos(phi, &s, &c);
  *ox = r * c;
  *oy = r * s;
}
// math.rs:99-103
inline V3 cosine_weighted(F4 u0, F4 u1) {
  F4 x, y;
  concentric(u0, u1, &x, &y);
  F4 msq = mul_add(x, x, y * y);  // Wec2::mag_sq (A1: dot uses mul_add)
  F4 z = f4sqrt(splat(1.0f) - f4min(msq, splat(1.0f)));
  return {x, y, z};
}
// math.rs:106-113 (note 2*u, not 2*pi*u: SURVEY F8)
inline V3 cosine_power(F4 u0, F4 u1, F4 power) {
  F4 one = splat(1.0f);
  F4 a = f4powf(u0, one / (power + one));
  F4 a2 = a * a;
  F4 b = f4sqrt(one - a2);
  F4 s, c;
  f4sincos(splat(2.0f) * u1, &s, &c);
  return {b * c, b * s, a};
}
// math.rs:122-124
inline F4 f_schlick(F4 cosv, F4 f0) { return f0 + (splat(1.0f) - f0) * f4powi5(splat(1.0f) - cosv); }

// ------------------------------------------------------------------------------------------
// Ray / WRay (ray.rs)
// ------------------------------------------------------------------------------------------
struct Ray {
  float time;
  float o[3], d[3], radiance[3], throughput[3];
  uint32_t tx, ty;  // tile_coord
  bool valid;
  float scramble;
  uint32_t sample;
  static Ray invalid() {  // ray.rs:54-66
    Ray r;
    float nanv = dm::u2f(0x7fc00000u);
    r.time = nanv;
    for (int i = 0; i < 3; ++i) {
      r.o[i] = nanv;
      r.d[i] = nanv;
      r.radiance[i] = 0.0f;
      r.throughput[i] = 0.0f;
    }
    r.tx = r.ty = 0;
    r.valid = false;
    r.scramble = 0.0f;
    r.sample = 0;
    return r;
  }
};

struct WRay {
  F4 time;
  V3 origin, dir, radiance, throughput;
  uint32_t tx[4], ty[4];
  bool valid[4];
  float scramble[4];
  uint32_t sample[4];
};

inline WRay wray_from(const Ray* r4) {  // ray.rs:114-160
  WRay w;
  w.time = make4(r4[0].time, r4[1].time, r4[2].time, r4[3].time);
#define PACK(field, k) make4(r4[0].field[k], r4[1].field[k], r4[2].field[k], r4[3].field[k])
  w.origin = {PACK(o, 0), PACK(o, 1), PACK(o, 2)};
  w.dir = {PACK(d, 0), PACK(d, 1), PACK(d, 2)};
  w.radiance = {PACK(radiance, 0), PACK(radiance, 1), PACK(radiance, 2)};
  w.throughput = {PACK(throughput, 0), PACK(throughput, 1), PACK(throughput, 2)};
#undef PACK
  for (int i = 0; i < 4; ++i) {
    w.tx[i] = r4[i].tx;
    w.ty[i] = r4[i].ty;
    w.valid[i] = r4[i].valid;
    w.scramble[i] = r4[i].scramble;
    w.sample[i] = r4[i].sample;
  }
  return w;
}
inline void wray_into(const WRay& w, Ray* r4) {  // ray.rs:162-214
  for (int i = 0; i < 4; ++i) {
    Ray& r = r4[i];
    r.time = w.time[i];
    r.o[0] = w.origin.x[i], r.o[1] = w.origin.y[i], r.o[2] = w.origin.z[i];
    r.d[0] = w.dir.x[i], r.d[1] = w.dir.y[i], r.d[2] = w.dir.z[i];
    r.radiance[0] = w.radiance.x[i], r.radiance[1] = w.radiance.y[i], r.radiance[2] = w.radiance.z[i];
    r.throughput[0] = w.throughput.x[i], r.throughput[1] = w.throughput.y[i],
    r.throughput[2] = w.throughput.z[i];
    r.tx = w.tx[i], r.ty = w.ty[i];
    r.valid = w.valid[i];
    r.scramble = w.scramble[i];
    r.sample = w.sample[i];
  }
}
inline V3 point_at(const WRay& r, F4 t) { return v3mul_add(r.dir, v3broadcast(t), r.origin); }  // ray.rs:22-24

// ------------------------------------------------------------------------------------------
// Sample tables (sampler.rs:62-126)
// ------------------------------------------------------------------------------------------
struct Tables {
  int n;  // spp
  const float* t1;
  const float* t2;
  float s1(uint32_t sample, float scramble, int set) const {
    return dm::fract(t1[sample + (size_t)n * set] + scramble);
  }
  float s2(int dim, uint32_t sample, float scramble, int set) const {
    return dm::fract(t2[dim + (size_t)sample * 2 + (size_t)n * 2 * set] + scramble);
  }
  F4 w1(const uint32_t* s, const float* sc, int set) const {
    return make4(s1(s[0], sc[0], set), s1(s[1], sc[1], set), s1(s[2], sc[2], set), s1(s[3], sc[3], set));
  }
  F4 w2(int dim, const uint32_t* s, const float* sc, int set) const {
    return make4(s2(dim, s[0], sc[0], set), s2(dim, s[1], sc[1], set), s2(dim, s[2], sc[2], set),
                 s2(dim, s[3], sc[3], set));
  }
};

// filter.rs:222-235
inline float fis_sample(const float* inv, float u) {
  u = 2.0f * (u - 0.5f);
  float mult = u < 0.0f ? -1.0f : 1.0f;
  u = fminf(fmaxf(fabsf(u), 0.0f), 0.99999f);
  float idx_full = u * (float)(RAYN_FIS_TABLE_SIZE - 1);
  int idx = (int)floorf(idx_full);
  float t = dm::fract(idx_full);
  return mult * lerpf(inv[idx], inv[idx + 1], t);
}
// film.rs:695-709
inline void sample_uv(uint32_t x, uint32_t y, float ndc_x, float ndc_y, const float* fis, float u0,
                      float u1, float* ox, float* oy) {
  float fx = fis_sample(fis, u0), fy = fis_sample(fis, u1);
  float sx = ((float)x + 0.5f) + fx;
  float sy = ((float)y + 0.5f) + fy;
  *ox = ndc_x * sx;
  *oy = ndc_y * sy;
}

// ------------------------------------------------------------------------------------------
// World
// ------------------------------------------------------------------------------------------
struct World {
  const RaynSceneDesc* s;
  int n_hit() const { return s->n_hitables; }
  int n_lights() const { return s->n_lights; }
};

typedef F4 (*ThrFn)(const void* ctx, F4 t);
struct Thr {  // the Box<dyn Fn(f32x4)->f32x4> of film.rs:540-551
  int depth;
  const RaynCamera* cam;
  F4 at(F4 t) const {
    if (depth == 0) {
      if (cam->kind == RAYN_CAMERA_ORTHOGRAPHIC) return splat(cam->half_pixel_size);  // camera.rs:282-284
      return splat(cam->half_pixel_size) * t;                                        // camera.rs:116-118
    }
    return splat(0.0001f * 2.0f * (float)depth) * t;  // film.rs:549
  }
};
// KAT variant: thr(t) = scale*t or scale
struct ThrKat {
  float scale;
  int is_const;
};

// ---- SDFs --------------------------------------------------------------------------------
// sdf.rs:125-141 with BoxFold :160-162 and SphereFold :181-187
inline F4 mandelbox_dist(const RaynHitable& h, V3 p) {
  V3 offset = p;
  F4 one = splat(1.0f);
  F4 dr = one;
  V3 l = v3broadcast(splat(h.box_l));
  V3 neg_l = -l;
  V3 two = v3broadcast(splat(2.0f));
  F4 scale = splat(h.scale);
  V3 scale_vec = v3broadcast(scale);
  F4 min_rad_sq = splat(h.min_rad_sq), fixed_rad_sq = splat(h.fixed_rad_sq);
  for (int i = 0; i < h.iterations; ++i) {
    p = v3mul_add(v3clamped(p, neg_l, l), two, -p);
    F4 r2 = mag_sq(p);
    F4 mul = f4max(one, fixed_rad_sq / f4max(min_rad_sq, r2));
    p = p * mul;
    dr = dr * mul;
    p = v3mul_add(p, scale_vec, offset);
    dr = mul_add(-dr, scale, one);
  }
  return mag(p) / f4abs(dr);
}

// AUTHORED (no reference counterpart, SURVEY F1): power-8 Mandelbulb distance estimator,
// White/Nylander triplex power with the z axis as pole, written without trigonometry via
// Chebyshev polynomials: cos(8a) = T8(cos a), sin(8a) = sin a * U7(cos a).
//   w' = r^8 (sin 8th cos 8ph, sin 8th sin 8ph, cos 8th) + c,   th = acos(z/r), ph = atan2(y,x)
//   dr' = 8 r^7 dr + 1,   DE = 0.5 ln(r) r / dr
// Lanes that have escaped (|w|^2 > bailout^2) stop iterating; the SIMD form keeps their values
// with a merge.  The definition is per lane.
inline F4 mandelbulb_dist(const RaynHitable& h, V3 p) {
  V3 w = p;
  F4 dr = splat(1.0f);
  F4 m = dot(w, w);
  F4 bail2 = splat(h.bulb_bailout * h.bulb_bailout);
  F4 one = splat(1.0f);
  for (int i = 0; i < h.iterations; ++i) {
    F4 esc = cmp_gt(m, bail2);
    if (move_mask(esc) == 0xf) break;
    F4 m2 = m * m, m3 = m2 * m;
    F4 r = f4sqrt(m);
    F4 r7 = m3 * r;
    F4 ndr = fma4(splat(8.0f) * r7, dr, one);
    // polar part: a = z^2, b = r^2
    F4 a = w.z * w.z, b = m;
    F4 b2 = b * b, b3 = b2 * b, b4 = b2 * b2;
    // Horner forms with explicit fused multiply-adds (the definition is ours: DESIGN.md §7)
    F4 P = fma4(fma4(fma4(fma4(splat(128.0f), a, splat(-256.0f) * b), a, splat(160.0f) * b2), a, splat(-32.0f) * b3), a, b4);
    F4 A = fma4(fma4(fma4(splat(128.0f), a, splat(-192.0f) * b), a, splat(80.0f) * b2), a, splat(-8.0f) * b3);
    // azimuth part: a' = x^2, b' = rho^2
    F4 ax = w.x * w.x;
    F4 q = fma4(w.x, w.x, w.y * w.y);
    F4 q2 = q * q, q3 = q2 * q, q4 = q2 * q2;
    F4 C = fma4(fma4(fma4(fma4(splat(128.0f), ax, splat(-256.0f) * q), ax, splat(160.0f) * q2), ax, splat(-32.0f) * q3), ax, q4);
    F4 B = fma4(fma4(fma4(splat(128.0f), ax, splat(-192.0f) * q), ax, splat(80.0f) * q2), ax, splat(-8.0f) * q3);
    F4 k = (w.z * A) / (q3 * f4sqrt(q));
    k = merge(cmp_gt(q, splat(0.0f)), k, splat(0.0f));
    V3 nw = {fma4(k, C, p.x), fma4(k, w.x * w.y * B, p.y), P + p.z};
    F4 nm = dot(nw, nw);
    w = v3merge(esc, w, nw);
    dr = merge(esc, dr, ndr);
    m = merge(esc, m, nm);
  }
  F4 r = f4sqrt(m);
  F4 lnr = map4(r, [](float x) { return dm::ln_fast(x); });
  return splat(0.5f) * lnr * r / dr;
}

inline F4 sdf_dist(const RaynHitable& h, V3 p) {
  if (h.kind == RAYN_HITABLE_MANDELBULB) return mandelbulb_dist(h, p);
  return mandelbox_dist(h, p);
}

// sdf.rs:25-57
inline F4 sdf_occluded(const RaynHitable& h, const RaynRenderConsts& rc, V3 start, V3 end) {
  V3 dir = end - start;
  F4 max_dist = mag(dir);
  dir = dir / max_dist;
  F4 dist = sdf_dist(h, start);
  F4 nan_mask = cmp_nan(dist, dist);
  F4 gt_mask = cmp_gt(dist, max_dist);
  F4 gt_nan_mask = gt_mask | nan_mask;
  F4 hit_mask = cmp_lt(dist, splat(0.0001f));
  F4 t = dist;
  const float S = rc.sdf_detail_scale;
  for (int march = 0; march < rc.max_vis_marches; ++march) {
    gt_mask = cmp_gt(t, max_dist);
    gt_nan_mask = gt_mask | nan_mask;
    if (move_mask(gt_nan_mask) == 0xf) break;
    V3 point = v3mul_add(dir, v3broadcast(t), start);
    F4 d = sdf_dist(h, point);
    hit_mask = cmp_lt(f4abs(d), f4max(splat(0.0001f * S), splat(0.00001f * S) * t));
    F4 hit_gt_nan_mask = hit_mask | gt_nan_mask;
    if (move_mask(hit_gt_nan_mask) == 0xf) break;
    t = merge(hit_gt_nan_mask, t, t + d);
  }
  return merge(hit_mask & f4not(gt_nan_mask), splat(0.0f), splat(1.0f));
}

// sdf.rs:59-83
template <class ThrT>
inline F4 sdf_hit(const RaynHitable& h, const RaynRenderConsts& rc, V3 origin, V3 dirv, F4 t_max,
                  const ThrT& thr, int64_t* evals) {
  F4 dist = sdf_dist(h, origin);
  F4 t = dist;
  F4 nan_mask = cmp_nan(t, t);
  const float S = rc.sdf_detail_scale;
  if (evals) *evals += 1;
  for (int march = 0; march < rc.max_marches; ++march) {
    V3 point = v3mul_add(dirv, v3broadcast(t), origin);
    F4 d = sdf_dist(h, point);
    if (evals) *evals += 1;
    F4 hit_mask = cmp_lt(f4abs(d), f4max(splat(0.00005f * S), splat(0.05f * S) * thr.at(t)));
    F4 gt_mask = cmp_gt(t, t_max);
    F4 hit_gt_nan_mask = hit_mask | nan_mask | gt_mask;
    t = merge(hit_gt_nan_mask, t, t + d);
    if (move_mask(hit_gt_nan_mask) == 0xf) break;
  }
  return t;
}

// WSequenced<Wec3>::sample_at (animation.rs).  Constants: impl_inherent_wsequenced (:52).  A parameter with a
// non-zero velocity stands for the closure `|t| base + velocity * t`, whose impl (:62-67) evaluates the closure at
// LANE 0's time and broadcasts it to all four lanes.
inline V3 seq_v3(const float* base, const float* vel, F4 time) {
  if (vel[0] == 0.0f && vel[1] == 0.0f && vel[2] == 0.0f) return v3splat(base[0], base[1], base[2]);
  const float t0 = time[0];
  return v3splat(base[0] + vel[0] * t0, base[1] + vel[1] * t0, base[2] + vel[2] * t0);
}
inline F4 seq_f(float base, float rate, F4 time) { return rate == 0.0f ? splat(base) : splat(base + rate * time[0]); }

// ---- Sphere (sphere.rs) --------------------------------------------------------------------
inline F4 sphere_occluded(const RaynHitable& h, V3 start, V3 end, F4 time) {  // :24-46
  V3 dir = end - start;
  F4 dist = mag(dir);
  dir = dir / dist;
  V3 origin = seq_v3(h.center, h.center_velocity, time);
  V3 oc = start - origin;
  F4 b = dot(oc, dir);
  F4 c = mag_sq(oc) - splat(h.radius * h.radius);
  F4 descrim = b * b - c;
  F4 desc_pos = cmp_gt(descrim, splat(0.0f));
  F4 desc_sqrt = f4sqrt(descrim);
  F4 t1 = -b - desc_sqrt;
  F4 t2 = -b + desc_sqrt;
  F4 mn = f4min(t1, t2);
  F4 valid = cmp_gt(mn, splat(0.001f)) & cmp_le(t1, dist) & desc_pos;
  return merge(valid, splat(0.0f), splat(1.0f));
}
inline F4 sphere_hit(const RaynHitable& h, V3 ro, V3 rd, F4 t_max, F4 time) {  // :48-72
  V3 origin = seq_v3(h.center, h.center_velocity, time);
  V3 oc = ro - origin;
  F4 b = dot(oc, rd);
  F4 c = mag_sq(oc) - splat(h.radius * h.radius);
  F4 descrim = b * b - c;
  F4 desc_pos = cmp_gt(descrim, splat(0.0f));
  F4 miss = splat(3.40282347e+38f);
  F4 desc_sqrt = f4sqrt(descrim);
  F4 t1 = -b - desc_sqrt;
  F4 t1_valid = cmp_gt(t1, splat(0.0001f)) & cmp_le(t1, t_max) & desc_pos;
  F4 t2 = -b + desc_sqrt;
  F4 t2_valid = cmp_gt(t2, splat(0.0001f)) & cmp_le(t2, t_max) & desc_pos;
  F4 take_t1 = cmp_lt(t1, t2) & t1_valid;
  F4 t = merge(take_t1, t1, t2);
  return merge(t1_valid | t2_valid, t, miss);
}

// ---- Hitable dispatch ------------------------------------------------------------------------
struct WHit {
  WRay ray;
  F4 t;
};
struct ShadingPoint {  // hitable.rs:21-48
  WRay ray;
  F4 t;
  V3 point;
  F4 offset_by;
  V3 normal;
  M3 basis;
};
inline ShadingPoint make_sp(const WHit& hit, V3 point, F4 offset_by, V3 normal) {
  return {hit.ray, hit.t, point, offset_by, normal, onb(normal)};
}
inline WRay create_rays(const ShadingPoint& sp, V3 dir) {  // hitable.rs:42-47
  WRay r = sp.ray;
  r.origin = sp.point + sp.normal * f4signum(dot(sp.normal, dir)) * sp.offset_by;
  r.dir = dir;
  return r;
}

// sdf.rs:85-101 + sdfu normals_fast (tetrahedral estimator; assumption A8)
inline ShadingPoint sdf_shading_info(const RaynHitable& h, const RaynRenderConsts& rc, const WHit& hit,
                                     const Thr& thr) {
  V3 point = point_at(hit.ray, hit.t);
  F4 eps = f4max(splat(0.0001f), splat(rc.sdf_detail_scale) * thr.at(hit.t));
  F4 one = splat(1.0f), neg = splat(-1.0f);
  V3 xyy = {one, neg, neg}, yyx = {neg, neg, one}, yxy = {neg, one, neg}, xxx = {one, one, one};
  V3 n = xyy * sdf_dist(h, point + xyy * eps) + yyx * sdf_dist(h, point + yyx * eps) +
         yxy * sdf_dist(h, point + yxy * eps) + xxx * sdf_dist(h, point + xxx * eps);
  return make_sp(hit, point, eps, normalized(n));
}
inline ShadingPoint sphere_shading_info(const RaynHitable& h, const WHit& hit) {  // sphere.rs:74-86
  V3 point = point_at(hit.ray, hit.t);
  V3 origin = seq_v3(h.center, h.center_velocity, hit.ray.time);
  V3 normal = normalized(point - origin);
  return make_sp(hit, point, splat(0.0f), normal);
}

inline F4 hitable_hit(const World& w, int id, const WRay& ray, F4 t_max, const Thr& thr, int64_t* evals) {
  const RaynHitable& h = w.s->hitables[id];
  if (h.kind == RAYN_HITABLE_SPHERE) return sphere_hit(h, ray.origin, ray.dir, t_max, ray.time);
  return sdf_hit(h, w.s->consts, ray.origin, ray.dir, t_max, thr, evals);
}
inline F4 hitable_occluded(const World& w, int id, V3 start, V3 end, F4 time) {
  const RaynHitable& h = w.s->hitables[id];
  if (h.kind == RAYN_HITABLE_SPHERE) return sphere_occluded(h, start, end, time);
  return sdf_occluded(h, w.s->consts, start, end);
}
// hitable.rs:164-168: product over ALL hitables, no early out
inline F4 test_occluded(const World& w, V3 start, V3 end, F4 time) {
  F4 acc = splat(1.0f);
  for (int i = 0; i < w.n_hit(); ++i) acc = acc * hitable_occluded(w, i, start, end, time);
  return acc;
}

// ---- Lights (light.rs) -------------------------------------------------------------------------
inline F4 uniform_cone_pdf(F4 cos_theta_max) {  // :105-107
  return splat(1.0f) / (splat(kTWO_PI) * (splat(1.0f) - cos_theta_max));
}
inline void light_sample(const RaynLight& L, F4 s0, F4 s1, V3 p, V3* out_point, V3* out_li, F4* out_pdf) {  // :38-72
  F4 zero = splat(0.0f), one = splat(1.0f);
  V3 pos = v3splat(L.pos[0], L.pos[1], L.pos[2]);
  F4 rad = splat(L.rad);
  V3 dir_to_light = pos - p;
  F4 dist_sq = mag_sq(dir_to_light);
  F4 dist = f4sqrt(dist_sq);
  dir_to_light = dir_to_light / dist;
  M3 basis = onb(-dir_to_light);
  F4 r2 = rad * rad;
  F4 sin_theta_max_2 = r2 / dist_sq;
  F4 cos_theta_max = f4sqrt(f4max(zero, one - sin_theta_max_2));
  F4 cos_theta = (one - s0) + s0 * cos_theta_max;
  F4 sin_theta = f4sqrt(f4max(zero, one - cos_theta * cos_theta));
  F4 phi = s1 * splat(kTWO_PI);
  F4 ds = dist * cos_theta - f4sqrt(f4max(zero, r2 - dist_sq * sin_theta * sin_theta));
  F4 cos_alpha = (dist_sq + r2 - ds * ds) / (splat(2.0f) * dist * rad);
  F4 sin_alpha = f4sqrt(f4max(zero, one - cos_alpha * cos_alpha));
  F4 sin_phi, cos_phi;
  f4sincos(phi, &sin_phi, &cos_phi);
  V3 offset = basis.c0 * sin_alpha * cos_phi + basis.c1 * sin_alpha * sin_phi + basis.c2 * cos_alpha;
  *out_point = pos + offset * rad;
  *out_li = v3splat(L.emission[0], L.emission[1], L.emission[2]);
  *out_pdf = uniform_cone_pdf(cos_theta_max);
}
inline void light_sample_volume(const RaynLight& L, F4 sample, V3 ray_o, V3 ray_d, F4 max_distance, F4* out_dist,
                                F4* out_pdf) {  // :75-102
  V3 pos = v3splat(L.pos[0], L.pos[1], L.pos[2]);
  F4 delta = dot(pos - ray_o, ray_d);
  V3 closest_point = ray_o + ray_d * delta;  // `delta * ray_d`
  F4 d = mag(closest_point - pos);
  F4 theta_a = f4atan2(-delta, d);
  F4 theta_b = f4atan2(max_distance - delta, d);
  F4 t = d * f4tan(f4lerp(theta_a, theta_b, sample));
  *out_dist = delta + t;
  *out_pdf = d / ((theta_b - theta_a) * mul_add(d, d, t * t));
}

// ---- BSDFs (material.rs) ------------------------------------------------------------------------
struct Scatter {
  V3 wi, f;
  F4 pdf;
};
inline bool receives_light(const RaynMaterial& m) {
  return m.kind == RAYN_MATERIAL_LAMBERTIAN || m.kind == RAYN_MATERIAL_DIELECTRIC;
}
inline V3 bsdf_le(const RaynMaterial& m, V3 wo) {
  if (m.kind == RAYN_MATERIAL_SKY) {  // :444-448
    F4 t = splat(0.5f) * (wo.y + splat(1.0f));
    V3 top = v3splat(m.sky_top[0], m.sky_top[1], m.sky_top[2]);
    V3 bottom = v3splat(m.sky_bottom[0], m.sky_bottom[1], m.sky_bottom[2]);
    return top * (splat(1.0f) - t) + bottom * t;
  }
  if (m.kind == RAYN_MATERIAL_EMISSIVE) return v3splat(m.emission[0], m.emission[1], m.emission[2]);  // :517-519
  return v3splat(0, 0, 0);
}
// BSDF::f called as bsdf.f(wo, wi, n) (integrator.rs:230); the Dielectric impl names its
// parameters (wi, wo, n) (material.rs:195) - the first argument is what it calls `wi`.
inline V3 bsdf_f(const RaynMaterial& m, V3 first, V3 second, V3 n) {
  V3 albedo = v3splat(m.albedo[0], m.albedo[1], m.albedo[2]);
  if (m.kind == RAYN_MATERIAL_LAMBERTIAN) return albedo / splat(kPI);  // :139-141
  // Dielectric :195-205
  F4 one = splat(1.0f), zero = splat(0.0f), two = splat(2.0f);
  F4 rough = splat(m.roughness);
  F4 dotv = f4max(zero, dot(first, n));
  F4 fresnel = f_schlick(dotv, splat(0.04f));
  V3 half = normalized(second + first);  // (wo + wi) in the callee's names
  F4 cos_alpha = f4powf(f4max(zero, dot(half, n)), rough);
  F4 spec_factor = cos_alpha * (rough + two) / (two * splat(kPI));
  V3 spec_f = v3splat(1, 1, 1) * spec_factor * fresnel;
  V3 diffuse_f = albedo / splat(kPI) * (one - fresnel);
  return spec_f + diffuse_f;
}
inline Scatter lambert_scatter(V3 albedo, const ShadingPoint& sp, F4 u0, F4 u1, bool dielectric_floor) {
  V3 ds = cosine_weighted(u0, u1);
  V3 bounce = normalized(sp.basis * ds);
  (void)dielectric_floor;
  return {bounce, albedo / splat(kPI), ds.z / splat(kPI)};  // :125-136
}
inline Scatter bsdf_scatter(const RaynMaterial& m, V3 wo, const ShadingPoint& sp, F4 s1d, const F4* s2d) {
  if (m.kind == RAYN_MATERIAL_LAMBERTIAN)
    return lambert_scatter(v3splat(m.albedo[0], m.albedo[1], m.albedo[2]), sp, s2d[0], s2d[1], false);
  if (m.kind == RAYN_MATERIAL_EMISSIVE) return lambert_scatter(v3splat(0.5f, 0.5f, 0.5f), sp, s2d[0], s2d[1], false);
  if (m.kind == RAYN_MATERIAL_SKY) return {v3splat(0, 0, 0), v3splat(0, 0, 0), splat(0.0f)};
  // Dielectric :207-256
  F4 one = splat(1.0f), two = splat(2.0f);
  V3 albedo = v3splat(m.albedo[0], m.albedo[1], m.albedo[2]);
  F4 rough = splat(m.roughness);
  V3 norm = sp.normal;
  F4 cosv = f4abs(dot(norm, wo));
  V3 diffuse_sample = cosine_weighted(s2d[0], s2d[1]);
  V3 diffuse_bounce = normalized(sp.basis * diffuse_sample);
  F4 diffuse_pdf = f4max(splat(0.00001f), diffuse_sample.z / splat(kPI));
  V3 diffuse_f = albedo / splat(kPI);
  V3 spec_sample = cosine_power(s2d[2], s2d[3], rough);
  V3 reflection = reflected(wo, norm);
  M3 basis = onb(reflection);
  V3 spec_bounce = normalized(basis * spec_sample);
  F4 cos_alpha_pow = f4max(f4powf(spec_sample.z, rough), splat(kEPSILON));
  F4 spec_pdf = (rough + one) / splat(kTWO_PI) * cos_alpha_pow;
  F4 spec_coeff = (rough + two) / splat(kTWO_PI) * cos_alpha_pow;
  F4 below_horizon = cmp_lt(dot(norm, spec_bounce), splat(0.0f));
  spec_coeff = merge(below_horizon, splat(0.0f), spec_coeff);
  V3 spec_f = v3splat(1, 1, 1) * spec_coeff;
  F4 fresnel = f_schlick(cosv, splat(0.04f));
  F4 fresnel_mask = cmp_lt(s1d, fresnel);
  Scatter se;
  se.wi = v3merge(fresnel_mask, spec_bounce, diffuse_bounce);
  se.f = v3merge(fresnel_mask, spec_f, diffuse_f);
  se.pdf = fresnel * spec_pdf + (one - fresnel) * diffuse_pdf;
  return se;
}

// ---- integrator.rs ----------------------------------------------------------------------------------
struct Counters {
  int64_t extend_rays = 0, shade_lanes = 0, shadow_rays = 0, sdf_evals_extend = 0;
};

inline V3 surface_sample_one_light(const World& w, int light_idx, F4 s0, F4 s1, const ShadingPoint& sp,
                                   const RaynMaterial& mat) {  // :207-240
  V3 end_point, li;
  F4 pdf;
  light_sample(w.s->lights[light_idx], s0, s1, sp.point, &end_point, &li, &pdf);
  V3 wo = -sp.ray.dir;
  V3 wi = end_point - sp.point;
  F4 dist = mag(wi);
  wi = wi / dist;
  V3 occlude_point = sp.point + sp.normal * f4signum(dot(sp.normal, wi)) * sp.offset_by;
  F4 occluded = test_occluded(w, occlude_point, end_point, sp.ray.time);
  V3 f = bsdf_f(mat, wo, wi, sp.normal) * f4max(dot(sp.normal, wi), splat(0.0f));
  F4 transmission = w.s->volume.has_extinction ? f4exp(splat(-w.s->volume.coeff_extinction) * dist) : splat(1.0f);
  return li * f * transmission * occluded / pdf;
}
inline V3 volume_sample_one_light(const World& w, int light_idx, F4 ls0, F4 ls1, F4 volume_sample, V3 ray_o,
                                  V3 ray_d, F4 max_distance, F4 time, F4* out_t) {  // :242-281
  const RaynLight& L = w.s->lights[light_idx];
  F4 vol_dist, vol_pdf;
  light_sample_volume(L, volume_sample, ray_o, ray_d, max_distance, &vol_dist, &vol_pdf);
  V3 sampled_point = ray_o + ray_d * vol_dist;
  V3 end_point, li;
  F4 light_pdf;
  light_sample(L, ls0, ls1, sampled_point, &end_point, &li, &light_pdf);
  V3 wi = end_point - sampled_point;
  F4 dist_point_to_light = mag(wi);
  F4 occluded = test_occluded(w, sampled_point, end_point, time);
  F4 f = splat(1.0f) / (splat(4.0f) * splat(kPI));
  F4 transmission =
      w.s->volume.has_extinction ? f4exp(splat(-w.s->volume.coeff_extinction) * dist_point_to_light) : splat(1.0f);
  *out_t = vol_dist;
  return li * f * transmission * occluded / (vol_pdf * light_pdf);
}

// TEST-ONLY switch (SURVEY T5): when set, every lane draws its four surface-NEE lights from its OWN sample
// (index_i = floor(fract(s + i/4) * L)) instead of taking one index from each packet lane.  Both estimators are unbiased
// with the same L/4 weight, so their high-spp means must agree; this guards the correction factor independently of the
// bit-parity tests (which compare two statements of the same formula).  Never set on a parity or timing path.
static int g_decoupled_lights = 0;

enum Channel { CH_COLOR = 0, CH_ALPHA = 1, CH_BACKGROUND = 2, CH_NORMAL = 3 };
struct OutSample {
  uint32_t tx, ty;
  int channel;
  float v[3];
};

inline int light_index(float s, int n_lights) {
  // `(sample * L).floor() as usize` (integrator.rs:76-77).  The reference would index out of
  // bounds if rounding produced L; clamp instead (assumption A10).
  int i = (int)floorf(s * (float)n_lights);
  if (i < 0) i = 0;
  if (i > n_lights - 1) i = n_lights - 1;
  return i;
}

void integrate(const World& w, int max_bounces, int volume_marches, const F4* s1d, const F4* s2d, int depth,
               int material, ShadingPoint sp, std::vector<Ray>& spawned_rays, std::vector<OutSample>& out,
               Counters& cnt) {  // :47-205
  V3 wo = -sp.ray.dir;
  const RaynMaterial& mat = w.s->materials[material];
  const RaynVolume& vol = w.s->volume;
  const int nl = w.n_lights();
  F4 volume_transmission = vol.has_extinction ? f4exp(splat(-vol.coeff_extinction) * sp.t) : splat(1.0f);
  sp.ray.radiance = sp.ray.radiance + bsdf_le(mat, wo) * sp.ray.throughput * volume_transmission;
  for (int i = 0; i < 4; ++i) cnt.shade_lanes += sp.ray.valid[i] ? 1 : 0;

  if (receives_light(mat) && nl > 0) {
    F4 correction = splat((float)nl / 4.0f);
    for (int i = 0; i < 4; ++i) {
      V3 li;
      if (!g_decoupled_lights) {
        int li_idx = light_index(s1d[0][i], nl);
        li = surface_sample_one_light(w, li_idx, s2d[0 + i * 2], s2d[1 + i * 2], sp, mat);
      } else {  // per-lane light choice: evaluate the packet once per lane and keep that lane's result
        float lx[4], ly[4], lz[4];
        for (int lane = 0; lane < 4; ++lane) {
          float u = s1d[0][lane] + 0.25f * (float)i;
          u = u - floorf(u);
          V3 one = surface_sample_one_light(w, light_index(u, nl), s2d[0 + i * 2], s2d[1 + i * 2], sp, mat);
          lx[lane] = one.x[lane], ly[lane] = one.y[lane], lz[lane] = one.z[lane];
        }
        li = {load4(lx), load4(ly), load4(lz)};
      }
      sp.ray.radiance = sp.ray.radiance + li * sp.ray.throughput * correction * volume_transmission;
      cnt.shadow_rays += 4;
    }
  }
  if (vol.has_scattering && nl > 0) {  // nl == 0 would panic in the reference
    F4 rho_s = splat(vol.coeff_scattering);
    for (int march = 0; march < volume_marches; ++march) {
      F4 correction = splat((float)nl / 4.0f / (float)volume_marches);
      for (int i = 0; i < 4; ++i) {
        int li_idx = light_index(s1d[march + 1][i], nl);
        F4 t;
        V3 li = volume_sample_one_light(w, li_idx, s2d[8 + 8 * march + i * 2], s2d[8 + 8 * march + i * 2 + 1],
                                        s1d[1], sp.ray.origin, sp.ray.dir, sp.t, sp.ray.time, &t);
        F4 transmission = vol.has_extinction ? f4exp(splat(-vol.coeff_extinction) * t) : splat(1.0f);
        sp.ray.radiance = sp.ray.radiance + li * sp.ray.throughput * correction * rho_s * transmission;
        cnt.shadow_rays += 4;
      }
    }
  }

  if (receives_light(mat)) {
    Scatter se = bsdf_scatter(mat, wo, sp, s1d[3], s2d + 8 + 8 * volume_marches);
    F4 ndl = f4abs(dot(se.wi, sp.normal));
    V3 new_throughput = sp.ray.throughput * volume_transmission * se.f * ndl / se.pdf;
    F4 roulette_factor;
    if (depth > 2) {
      roulette_factor = f4max(splat(1.0f) - component_max(sp.ray.throughput), splat(0.05f));
      new_throughput = new_throughput / (splat(1.0f) - roulette_factor);
    } else {
      roulette_factor = splat(0.0f);
    }
    WRay nr = create_rays(sp, se.wi);
    Ray new_rays[4];
    wray_into(nr, new_rays);
    if (depth == 0) {
      for (int i = 0; i < 4; ++i)
        if (new_rays[i].valid) {
          out.push_back({new_rays[i].tx, new_rays[i].ty, CH_ALPHA, {1.0f, 0, 0}});
          out.push_back({new_rays[i].tx, new_rays[i].ty, CH_NORMAL, {sp.normal.x[i], sp.normal.y[i], sp.normal.z[i]}});
        }
    }
    for (int i = 0; i < 4; ++i) {
      Ray& ray = new_rays[i];
      if (!ray.valid) continue;
      if (depth >= max_bounces || s1d[4][i] < roulette_factor[i]) {
        out.push_back({ray.tx, ray.ty, CH_COLOR, {ray.radiance[0], ray.radiance[1], ray.radiance[2]}});
      } else {
        float nt[3] = {new_throughput.x[i], new_throughput.y[i], new_throughput.z[i]};
        if (!(nt[0] != nt[0] || nt[1] != nt[1] || nt[2] != nt[2])) {
          ray.throughput[0] = nt[0], ray.throughput[1] = nt[1], ray.throughput[2] = nt[2];
        }
        spawned_rays.push_back(ray);
      }
    }
  } else {
    Ray final_rays[4];
    wray_into(sp.ray, final_rays);
    for (int i = 0; i < 4; ++i) {
      const Ray& ray = final_rays[i];
      if (!ray.valid) continue;
      out.push_back({ray.tx, ray.ty, depth == 0 ? CH_BACKGROUND : CH_COLOR,
                     {ray.radiance[0], ray.radiance[1], ray.radiance[2]}});
    }
  }
}

// ---- camera.rs -------------------------------------------------------------------------------------
WRay camera_get_rays(const RaynCamera& c, float scramble, const uint32_t* sample_nums, uint32_t tx, uint32_t ty, F4 u,
                     F4 v, F4 time, F4 ls0, F4 ls1) {
  V3 origin = seq_v3(c.origin, c.origin_velocity, time);  // self.origin.sample_at(time), camera.rs:90-92
  V3 at = seq_v3(c.at, c.at_velocity, time);
  V3 up = seq_v3(c.up, c.up_velocity, time);
  F4 hx = splat(c.half_size[0]), hy = splat(c.half_size[1]);
  V3 ro, rd;
  if (c.kind == RAYN_CAMERA_PINHOLE) {  // :81-114
    V3 bw = normalized(origin - at);
    V3 bu = normalized(cross(up, bw));
    V3 bv = cross(bw, bu);
    V3 lower_left = origin - bu * hx - bv * hy - bw;
    V3 horiz = bu * hx * splat(2.0f) * u;
    V3 verti = bv * hy * splat(2.0f) * v;
    ro = origin;
    rd = normalized(lower_left + horiz + verti - origin);
  } else if (c.kind == RAYN_CAMERA_THINLENS) {  // :168-208
    V3 focus = seq_v3(c.focus, c.focus_velocity, time);
    F4 focus_dist = mag(focus - origin);
    F4 aperture = seq_f(c.aperture, c.aperture_rate, time);
    V3 bw = normalized(origin - at);
    V3 bu = normalized(cross(up, bw));
    V3 bv = cross(bw, bu);
    V3 lower_left = origin - bu * hx * focus_dist - bv * hy * focus_dist - bw * focus_dist;
    V3 horiz = bu * hx * focus_dist * splat(2.0f) * u;
    V3 verti = bv * hy * focus_dist * splat(2.0f) * v;
    F4 dx, dy;
    concentric(ls0, ls1, &dx, &dy);
    dx = dx * aperture;
    dy = dy * aperture;
    V3 offset = bu * dx + bv * dy;
    ro = origin + offset;
    rd = normalized(lower_left + horiz + verti - ro);
  } else {  // orthographic :249-280
    F4 fx = splat(c.full_size[0]), fy = splat(c.full_size[1]);
    V3 bw = normalized(at - origin);
    V3 bu = normalized(cross(bw, up));
    V3 bv = cross(bu, bw);
    V3 lower_left = origin - bu * hx - bv * hy;
    V3 offset = bu * u * fx + bv * v * fy;
    ro = lower_left + offset;
    rd = bw;
  }
  WRay r;
  r.time = time;
  r.origin = ro;
  r.dir = rd;
  r.radiance = v3splat(0, 0, 0);
  r.throughput = v3splat(1, 1, 1);
  for (int i = 0; i < 4; ++i) {
    r.tx[i] = tx;
    r.ty[i] = ty;
    r.valid[i] = true;
    r.scramble[i] = scramble;
    r.sample[i] = sample_nums[i];
  }
  return r;
}

// ---- hitable.rs:170-210 ------------------------------------------------------------------------------
struct Hit {
  Ray ray;
  float t;
};
inline void closest_hit(const World& w, const WRay& ray, F4 t_max, const Thr& thr, int* ids, F4* dists,
                        int64_t* evals) {
  F4 closest = t_max;
  for (int i = 0; i < 4; ++i) ids[i] = -1;
  for (int id = 0; id < w.n_hit(); ++id) {
    F4 t = hitable_hit(w, id, ray, closest, thr, evals);
    alignas(16) float c[4];
    store4(c, closest);
    for (int i = 0; i < 4; ++i)
      if (t[i] < c[i]) {
        c[i] = t[i];
        ids[i] = id;
      }
    closest = load4(c);
  }
  *dists = closest;
}

struct QueueLog {
  int32_t* buf;
  int64_t cap;
  int64_t n;
};

// film.rs:439-627 for one tile
void render_tile(const World& w, const RaynFrameDesc& f, int tile_x, int tile_y, int tile_index, float* color,
                 float* alpha, float* background, float* normal, QueueLog* qlog, Counters& cnt) {
  const int W = f.width, H = f.height;
  const uint32_t x0 = tile_x * f.tile_w, y0 = tile_y * f.tile_h;
  const uint32_t x1 = (uint32_t)((int)(x0 + f.tile_w) < W ? x0 + f.tile_w : W);
  const uint32_t y1 = (uint32_t)((int)(y0 + f.tile_h) < H ? y0 + f.tile_h : H);
  const uint32_t tw = x1 - x0, th = y1 - y0;
  const int samples = f.samples, spp = 4 * samples, vm = f.volume_marches;
  const float ndc_x = 1.0f / (float)W, ndc_y = 1.0f / (float)H;
  Tables tab{spp, f.samples_1d, f.samples_2d};
  std::vector<float> tc(3 * tw * th, 0.0f), ta(tw * th, 0.0f), tb(3 * tw * th, 0.0f), tn(3 * tw * th, 0.0f);

  std::vector<WRay> spawned_wrays;
  std::vector<Ray> spawned_rays;
  std::vector<OutSample> new_samples;
  std::vector<std::vector<Hit>> bins(w.n_hit());
  const F4 time_range = splat(f.t1 - f.t0);

  for (uint32_t x = x0; x < x1; ++x)
    for (uint32_t y = y0; y < y1; ++y) {
      float scramble = f.scramble[x + y * (uint32_t)W];
      for (int samp = 0; samp < samples; ++samp) {
        uint32_t nums[4] = {4u * samp, 4u * samp + 1, 4u * samp + 2, 4u * samp + 3};
        float us[4], vs[4];
        for (int i = 0; i < 4; ++i)
          sample_uv(x, y, ndc_x, ndc_y, f.fis_inverse_cdf, tab.s2(0, nums[i], scramble, 0),
                    tab.s2(1, nums[i], scramble, 0), &us[i], &vs[i]);
        float sc4[4] = {scramble, scramble, scramble, scramble};
        F4 times = splat(f.t0) + time_range * tab.w1(nums, sc4, 0);
        F4 ls0 = tab.w2(0, nums, sc4, 1), ls1 = tab.w2(1, nums, sc4, 1);
        spawned_wrays.push_back(camera_get_rays(w.s->camera, scramble, nums, x - x0, y - y0, load4(us), load4(vs),
                                                times, ls0, ls1));
      }
    }

  for (int depth = 0;; ++depth) {
    if (spawned_wrays.empty()) break;
    for (auto& b : bins) b.clear();
    Thr thr{depth, &w.s->camera};
    for (const WRay& wray : spawned_wrays) {  // add_hits, hitable.rs:170-210
      int ids[4];
      F4 dists;
      closest_hit(w, wray, splat(w.s->consts.world_radius * 2.0f), thr, ids, &dists, &cnt.sdf_evals_extend);
      Ray rays[4];
      wray_into(wray, rays);
      for (int i = 0; i < 4; ++i) {
        if (rays[i].valid) cnt.extend_rays++;
        if (ids[i] >= 0 && rays[i].valid) bins[ids[i]].push_back({rays[i], dists[i]});
      }
    }
    spawned_wrays.clear();
    // process_hits, hitable.rs:94-133: pad every bin to x4 with invalid hits (t = 0)
    for (auto& b : bins)
      while (b.size() % 4 != 0) b.push_back({Ray::invalid(), 0.0f});
    if (qlog && qlog->buf) {
      int64_t total = 0;
      for (auto& b : bins) total += (int64_t)b.size();
      if (qlog->n + 3 + total <= qlog->cap) {
        qlog->buf[qlog->n++] = depth;
        qlog->buf[qlog->n++] = tile_index;
        qlog->buf[qlog->n++] = (int32_t)total;
        for (auto& b : bins)
          for (auto& h : b)
            qlog->buf[qlog->n++] = h.ray.valid ? (int32_t)((h.ray.tx * th + h.ray.ty) * spp + h.ray.sample) : -1;
      } else {
        qlog->n = qlog->cap + 1;  // overflow marker
      }
    }
    for (int obj = 0; obj < w.n_hit(); ++obj) {
      const RaynHitable& h = w.s->hitables[obj];
      for (size_t k = 0; k + 4 <= bins[obj].size(); k += 4) {
        Ray r4[4] = {bins[obj][k].ray, bins[obj][k + 1].ray, bins[obj][k + 2].ray, bins[obj][k + 3].ray};
        WHit hit{wray_from(r4), make4(bins[obj][k].t, bins[obj][k + 1].t, bins[obj][k + 2].t, bins[obj][k + 3].t)};
        ShadingPoint sp = h.kind == RAYN_HITABLE_SPHERE ? sphere_shading_info(h, hit)
                                                        : sdf_shading_info(h, w.s->consts, hit, thr);
        // film.rs:565-589
        F4 s1d[5], s2d[28];
        const int n1 = 3 + vm, n2 = 12 + 8 * vm;
        for (int set = 0; set < n1; ++set) s1d[set] = tab.w1(sp.ray.sample, sp.ray.scramble, 1 + set + depth * n1);
        for (int i = 0; i < n2; ++i)
          s2d[i] = tab.w2(i % 2, sp.ray.sample, sp.ray.scramble, 2 + i / 2 + depth * n2 / 2);
        integrate(w, f.max_bounces, vm, s1d, s2d, depth, h.material, sp, spawned_rays, new_samples, cnt);
      }
    }
    for (const OutSample& s : new_samples) {  // film.rs:604-606, :167-172
      size_t idx = s.tx + s.ty * tw;
      switch (s.channel) {
        case CH_COLOR:
          for (int k = 0; k < 3; ++k) tc[3 * idx + k] += s.v[k];
          break;
        case CH_ALPHA:
          ta[idx] += s.v[0];
          break;
        case CH_BACKGROUND:
          for (int k = 0; k < 3; ++k) tb[3 * idx + k] += s.v[k];
          break;
        case CH_NORMAL:
          for (int k = 0; k < 3; ++k) tn[3 * idx + k] += s.v[k];
          break;
      }
    }
    new_samples.clear();
    while (spawned_rays.size() % 4 != 0) spawned_rays.push_back(Ray::invalid());  // film.rs:608-610
    for (size_t k = 0; k + 4 <= spawned_rays.size(); k += 4) spawned_wrays.push_back(wray_from(&spawned_rays[k]));
    spawned_rays.clear();
  }
  // tile_finished / copy_from_tile, film.rs:82-98
  const float div = (float)spp;
  for (uint32_t x = 0; x < tw; ++x)
    for (uint32_t y = 0; y < th; ++y) {
      size_t ti = x + y * tw;
      size_t fi = (x0 + x) + (size_t)(y0 + y) * W;
      for (int k = 0; k < 3; ++k) {
        color[3 * fi + k] = tc[3 * ti + k] / div;
        background[3 * fi + k] = tb[3 * ti + k] / div;
        normal[3 * fi + k] = tn[3 * ti + k] / div;
      }
      alpha[fi] = ta[ti] / div;
    }
}

bool fp_contract_is_off() {
  // a*a = 1 + 2^-11 + 2^-24 rounds to 1 + 2^-11 when the product is rounded on its own;
  // a fused multiply-add keeps the 2^-24.
  volatile float a = 1.0f + 0x1p-12f, c = -(1.0f + 0x1p-11f);
  float x = a, z = c;
  F4 r = splat(x) * splat(x) + splat(z);
  float unf = r[0];
  float fused = dm::fma(x, x, z);
  return unf == 0.0f && fused == 0x1p-24f;
}

}  // namespace

// ==========================================================================================
// C entry points (test infrastructure)
// ==========================================================================================
extern "C" {

int32_t rayn_oracle_selfcheck(void) { return fp_contract_is_off() ? 0 : 1; }
int32_t rayn_oracle_muladd_fused(void) { return RAYN_MULADD_FUSED; }  // which A6 variant this library is (oracle/README.md)
void rayn_oracle_set_decoupled_lights(int32_t on) { g_decoupled_lights = on; }  // TEST-ONLY, see g_decoupled_lights

// Renders tiles with (tile_index % tile_stride) == tile_offset AND ((tile_index / tile_stride) % subsample_k) == 0.
// Planes are host pointers; untouched pixels keep their previous contents.
int32_t rayn_oracle_render_frame(const RaynSceneDesc* scene, const RaynFrameDesc* f, const RaynFilmPlanes* out,
                                 int32_t n_threads, int32_t subsample_k, int32_t* queue_log, int64_t queue_cap,
                                 int64_t* queue_n, int64_t* counters4, int64_t* tiles_rendered) {
  if (!scene || !f || !out) return RAYN_ERR_INVALID_ARG;
  if (f->volume_marches != 2) return RAYN_ERR_UNSUPPORTED;
  if (!fp_contract_is_off()) return RAYN_ERR_UNSUPPORTED;
  World w{scene};
  int ntx = (f->width + f->width % f->tile_w) / f->tile_w;    // film.rs:399-404
  int nty = (f->height + f->height % f->tile_h) / f->tile_h;
  int stride = f->tile_stride > 0 ? f->tile_stride : 1;
  if (subsample_k < 1) subsample_k = 1;
  std::vector<int> todo;
  if (f->tile_list) {  // explicit tile set (same meaning as in rayn_b200_render_frame)
    for (int i = 0; i < f->n_tile_list; ++i)
      if (f->tile_list[i] >= 0 && f->tile_list[i] < ntx * nty) todo.push_back(f->tile_list[i]);
  } else {
    for (int idx = 0; idx < ntx * nty; ++idx)
      if (idx % stride == f->tile_offset && ((idx / stride) % subsample_k) == 0) todo.push_back(idx);
  }
  QueueLog ql{queue_log, queue_cap, 0};
  Counters total;
  if (queue_log) n_threads = 1;
#ifdef _OPENMP
  if (n_threads > 0) omp_set_num_threads(n_threads);
#endif
#pragma omp parallel
  {
    Counters local;
#pragma omp for schedule(dynamic, 1)
    for (size_t k = 0; k < todo.size(); ++k) {
      int idx = todo[k];
      int tx = idx / nty, ty = idx % nty;
      if (tx * f->tile_w >= f->width || ty * f->tile_h >= f->height) continue;
      render_tile(w, *f, tx, ty, idx, out->color, out->alpha, out->background, out->normal, queue_log ? &ql : nullptr,
                  local);
    }
#pragma omp critical
    {
      total.extend_rays += local.extend_rays;
      total.shade_lanes += local.shade_lanes;
      total.shadow_rays += local.shadow_rays;
      total.sdf_evals_extend += local.sdf_evals_extend;
    }
  }
  if (queue_n) *queue_n = ql.n;
  if (counters4) {
    counters4[0] = total.extend_rays;
    counters4[1] = total.shade_lanes;
    counters4[2] = total.shadow_rays;
    counters4[3] = total.sdf_evals_extend;
  }
  if (tiles_rendered) *tiles_rendered = (int64_t)todo.size();
  return RAYN_OK;
}

// Film::save_to per-pixel arithmetic (film.rs:205-377), scalar f32 like the reference.
static inline float o_saturate(float x) { return fminf(fmaxf(x, 0.0f), 1.0f); }                 // spectrum.rs:35-40 (f32::max/min: NaN loses)
static inline float o_gamma(float x) { return dm::pow(x, 1.0f / 2.2f); }                         // spectrum.rs:30-32
static inline uint8_t o_u8(float v) {                                                            // `(v*255.0).min(255.0).max(0.0) as u8`
  float a = fmaxf(fminf(v * 255.0f, 255.0f), 0.0f);
  return (uint8_t)(int)a;
}
int32_t rayn_oracle_film_postprocess(int32_t mode, int32_t W, int32_t H, const RaynFilmPlanes* pl, uint8_t* out) {
  const int bpp = mode == RAYN_POST_COLOR_ALPHA ? 4 : (mode == RAYN_POST_ALPHA ? 1 : 3);
  for (int y = 0; y < H; ++y)
    for (int x = 0; x < W; ++x) {
      const size_t idx = (size_t)x + (size_t)(H - 1 - y) * W;  // film.rs:236
      uint8_t* d = out + ((size_t)x + (size_t)y * W) * bpp;
      for (int c = 0; c < 3 && mode != RAYN_POST_ALPHA; ++c) {
        float v;
        switch (mode) {
          case RAYN_POST_COLOR_PLUS_BACKGROUND: v = o_gamma(o_saturate(pl->color[3 * idx + c] + pl->background[3 * idx + c])); break;
          case RAYN_POST_COLOR_ALPHA: v = o_gamma(o_saturate(pl->color[3 * idx + c])); break;
          case RAYN_POST_COLOR_ONLY: v = o_gamma(pl->color[3 * idx + c]); break;
          case RAYN_POST_BACKGROUND: v = o_gamma(o_saturate(pl->background[3 * idx + c])); break;
          default: v = pl->normal[3 * idx + c] * 0.5f + 0.5f;
        }
        d[c] = o_u8(v);
      }
      if (mode == RAYN_POST_COLOR_ALPHA) d[3] = o_u8(pl->alpha[idx]);
      if (mode == RAYN_POST_ALPHA) d[0] = o_u8(pl->alpha[idx]);
    }
  return RAYN_OK;
}

int32_t rayn_oracle_kat_detmath(int32_t op, int64_t n, const float* a, const float* b, float* out) {
  for (int64_t i = 0; i < n; ++i) {
    float s, c;
    switch (op) {
      case 0: out[i] = dm::exp(a[i]); break;
      case 1: out[i] = dm::ln(a[i]); break;
      case 2: out[i] = dm::pow(a[i], b[i]); break;
      case 3: dm::sincos(a[i], &s, &c); out[i] = s; break;
      case 4: dm::sincos(a[i], &s, &c); out[i] = c; break;
      case 5: out[i] = dm::tan(a[i]); break;
      case 6: out[i] = dm::atan2(a[i], b[i]); break;
      case 7: out[i] = dm::powi5(a[i]); break;
      case 8: out[i] = dm::ln_fast(a[i]); break;
      default: return RAYN_ERR_INVALID_ARG;
    }
  }
  return RAYN_OK;
}

static inline V3 load_v3_packet(const float* p3, int64_t i, int64_t n) {
  float x[4], y[4], z[4];
  for (int l = 0; l < 4; ++l) {
    int64_t j = i + l < n ? i + l : n - 1;
    x[l] = p3[3 * j], y[l] = p3[3 * j + 1], z[l] = p3[3 * j + 2];
  }
  return {load4(x), load4(y), load4(z)};
}
static inline F4 load_f_packet(const float* p, int64_t i, int64_t n) {
  float x[4];
  for (int l = 0; l < 4; ++l) x[l] = p[i + l < n ? i + l : n - 1];
  return load4(x);
}
static inline void store_f_packet(float* p, int64_t i, int64_t n, F4 v) {
  for (int l = 0; l < 4 && i + l < n; ++l) p[i + l] = v[l];
}

int32_t rayn_oracle_kat_sdf_dist(const RaynHitable* sdf, int64_t n, const float* points3, float* out) {
  for (int64_t i = 0; i < n; i += 4) store_f_packet(out, i, n, sdf_dist(*sdf, load_v3_packet(points3, i, n)));
  return RAYN_OK;
}

struct ThrKatFn {
  float scale;
  int is_const;
  F4 at(F4 t) const { return is_const ? splat(scale) : splat(scale) * t; }
};

int32_t rayn_oracle_kat_sdf_hit(const RaynHitable* sdf, const RaynRenderConsts* consts, int64_t n,
                                const float* origins3, const float* dirs3, const float* t_max, float thr_scale,
                                int32_t thr_const, float* out_t) {
  ThrKatFn thr{thr_scale, thr_const};
  for (int64_t i = 0; i < n; i += 4)
    store_f_packet(out_t, i, n,
                   sdf_hit(*sdf, *consts, load_v3_packet(origins3, i, n), load_v3_packet(dirs3, i, n),
                           load_f_packet(t_max, i, n), thr, nullptr));
  return RAYN_OK;
}

int32_t rayn_oracle_kat_occluded(const RaynSceneDesc* scene, int64_t n, const float* start3, const float* end3,
                                 float* out) {
  World w{scene};
  for (int64_t i = 0; i < n; i += 4)
    store_f_packet(out, i, n, test_occluded(w, load_v3_packet(start3, i, n), load_v3_packet(end3, i, n), splat(0.0f)));
  return RAYN_OK;
}

// SphereLight::sample (light.rs:38-72): out_point3[n*3], out_pdf[n]
int32_t rayn_oracle_kat_light_sample(const RaynLight* light, int64_t n, const float* s0, const float* s1, const float* p3, float* out_point3,
                                     float* out_pdf) {
  for (int64_t i = 0; i < n; i += 4) {
    V3 pt, li;
    F4 pdf;
    light_sample(*light, load_f_packet(s0, i, n), load_f_packet(s1, i, n), load_v3_packet(p3, i, n), &pt, &li, &pdf);
    store_f_packet(out_pdf, i, n, pdf);
    for (int l = 0; l < 4 && i + l < n; ++l) {
      out_point3[3 * (i + l)] = pt.x[l], out_point3[3 * (i + l) + 1] = pt.y[l], out_point3[3 * (i + l) + 2] = pt.z[l];
    }
  }
  return RAYN_OK;
}
// SphereLight::sample_volume_scattering (light.rs:75-102): equi-angular distance + pdf
int32_t rayn_oracle_kat_light_sample_volume(const RaynLight* light, int64_t n, const float* sample, const float* o3, const float* d3,
                                            const float* t_max, float* out_t, float* out_pdf) {
  for (int64_t i = 0; i < n; i += 4) {
    F4 t, pdf;
    light_sample_volume(*light, load_f_packet(sample, i, n), load_v3_packet(o3, i, n), load_v3_packet(d3, i, n), load_f_packet(t_max, i, n), &t, &pdf);
    store_f_packet(out_t, i, n, t);
    store_f_packet(out_pdf, i, n, pdf);
  }
  return RAYN_OK;
}
// BSDF::scatter + BSDF::f (material.rs): for unit normals n3 and outgoing wo3, samples (s1d, u0..u3):
// out_wi3, out_f3 (the scatter event's f), out_pdf, out_feval3 = bsdf.f(wo, wi, n) as the integrator calls it.
int32_t rayn_oracle_kat_bsdf(const RaynMaterial* mat, int64_t n, const float* n3, const float* wo3, const float* s1d, const float* u4,
                             float* out_wi3, float* out_f3, float* out_pdf, float* out_feval3) {
  for (int64_t i = 0; i < n; i += 4) {
    ShadingPoint sp;
    sp.normal = load_v3_packet(n3, i, n);
    sp.basis = onb(sp.normal);
    V3 wo = load_v3_packet(wo3, i, n);
    F4 u[4];
    for (int k = 0; k < 4; ++k) {
      float tmp[4];
      for (int l = 0; l < 4; ++l) tmp[l] = u4[4 * (i + l < n ? i + l : n - 1) + k];
      u[k] = load4(tmp);
    }
    Scatter se = bsdf_scatter(*mat, wo, sp, load_f_packet(s1d, i, n), u);
    V3 fe = bsdf_f(*mat, wo, se.wi, sp.normal);
    store_f_packet(out_pdf, i, n, se.pdf);
    for (int l = 0; l < 4 && i + l < n; ++l) {
      const int64_t j = i + l;
      out_wi3[3 * j] = se.wi.x[l], out_wi3[3 * j + 1] = se.wi.y[l], out_wi3[3 * j + 2] = se.wi.z[l];
      out_f3[3 * j] = se.f.x[l], out_f3[3 * j + 1] = se.f.y[l], out_f3[3 * j + 2] = se.f.z[l];
      out_feval3[3 * j] = fe.x[l], out_feval3[3 * j + 1] = fe.y[l], out_feval3[3 * j + 2] = fe.z[l];
    }
  }
  return RAYN_OK;
}

int32_t rayn_oracle_kat_closest_hit(const RaynSceneDesc* scene, int32_t depth, int64_t n, const float* origins3,
                                    const float* dirs3, float* out_t, int32_t* out_obj) {
  World w{scene};
  Thr thr{depth, &scene->camera};
  for (int64_t i = 0; i < n; i += 4) {
    WRay r;
    r.origin = load_v3_packet(origins3, i, n);
    r.dir = load_v3_packet(dirs3, i, n);
    r.time = splat(0.0f);
    int ids[4];
    F4 d;
    closest_hit(w, r, splat(scene->consts.world_radius * 2.0f), thr, ids, &d, nullptr);
    store_f_packet(out_t, i, n, d);
    for (int l = 0; l < 4 && i + l < n; ++l) out_obj[i + l] = ids[l];
  }
  return RAYN_OK;
}

}  // extern "C"
