// rt_denoise.cuh — edge-avoiding a-trous wavelet filter of the film planes (Dammertz, Sewtz, Hanika, Lensch, HPG 2010).
// The exact statement (tap order, the float arithmetic, which taps are skipped) is at rayn_b200_film_denoise in
// include/rayn_b200.h; the CPU mirror in tests/film_mirror.cpp restates it and the GPU tests compare bit for bit.
//
// One kernel launch per level, one thread per pixel on 32x8 CTAs.  The guides are packed once into a float4
// (nx, ny, nz, a) plane and the colour ping-pongs between two float4 planes, so every tap is two 16-byte loads that
// mostly hit L1/L2 (neighbouring pixels share taps).
#pragma once
#include "rt_device.cuh"

namespace rt {

// Exact skip of dead taps.  dm::exp (detmath.h) returns +0 for every float argument x <= -103.972084f (bit pattern
// 0xc2cff1b5); -103.972076f (0xc2cff1b4) is the lowest argument with a nonzero result (the smallest denormal).  This
// is established on the device by tests/test_gpu_denoise.py, which evaluates dm::exp on every float in
// [-111, -103.972084] and finds +0 for all of them; below -110 dm::exp clamps its argument to -110, so the sweep covers
// every smaller argument too (including -inf).  Hence e > DENOISE_E_DEAD  =>  w = hk * exp(-e) = hk * (+0) = +0, and the
// skipped update `s += (+0) * c_q` is the identity on every accumulator: c_q is finite (non-finite taps are skipped
// first), so the product is +-0, and an accumulator that starts at +0 can never become -0 (round-to-nearest gives
// x + (-x) = +0), so adding +-0 leaves its bits unchanged.  `!(e <= DENOISE_E_DEAD)` also catches e = NaN, a tap the
// statement skips anyway.
#define DENOISE_E_DEAD 103.972076f
// e == 0 (identical colour and guides, always the centre tap) needs no exponential: dm::exp(-0.0f) is exactly 1.0f
// (tested on both sides), so w = hk * 1 = hk.

__device__ __forceinline__ bool dn_finite3(const float4 c) { return isfinite(c.x) && isfinite(c.y) && isfinite(c.z); }

// Luminance of the variance guide (rayn_b200_film_denoise_variance); the library builds with --fmad=false, so every product
// is rounded on its own as the header states.
__host__ __device__ __forceinline__ float dn_lum(float r, float g, float b) { return (0.2126f * r + 0.7152f * g) + 0.0722f * b; }

// floored q mod W, in [0, W): the column of tap q on a film that is periodic in x.  Only the taps near the seam divide.
__device__ __forceinline__ int dn_wrap(int q, int W) {
  if ((unsigned)q < (unsigned)W) return q;
  q %= W;
  return q < 0 ? q + W : q;
}

// planes -> float4 (r, g, b, 0) / (nx, ny, nz, a)
__global__ void __launch_bounds__(256) k_denoise_pack(long long npx, const float* __restrict__ c3, float4* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npx) return;
  out[i] = make_float4(c3[3 * i], c3[3 * i + 1], c3[3 * i + 2], 0.0f);
}
__global__ void __launch_bounds__(256) k_denoise_guides(long long npx, const float* __restrict__ n3, const float* __restrict__ a,
                                                        float4* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npx) return;
  out[i] = make_float4(n3[3 * i], n3[3 * i + 1], n3[3 * i + 2], a[i]);
}

// colour plane + its lum^2 moment plane -> float4 (r, g, b, v) with the level-0 variance of the pixel mean
// v = fmaxf(M - lum(c)^2, 0) / spp; kScale (rayn_b200_film_denoise_variance_scaled): v = (fmaxf(M - lum(c)^2, 0) * scale) / spp
template <bool kScale = false>
__global__ void __launch_bounds__(256) k_denoise_pack_var(long long npx, const float* __restrict__ c3, const float* __restrict__ m, float fspp,
                                                          float4* __restrict__ out, const float* __restrict__ scale = nullptr) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npx) return;
  const float r = c3[3 * i], g = c3[3 * i + 1], b = c3[3 * i + 2];
  const float l = dn_lum(r, g, b);
  float v = fmaxf(m[i] - l * l, 0.0f);
  if (kScale) v = v * scale[i];
  out[i] = make_float4(r, g, b, v / fspp);
}

// One level with step 2^level.  kOut3: the last level writes the interleaved rgb output plane instead of a float4 plane.
// kAlb (rayn_b200_film_denoise_albedo): a fourth edge-stopping term dl2 * il from the albedo guide, packed (r, g, b, 0) by
// k_denoise_pack; the kAlb = false instances never read `alb` or `il` and run the code of rayn_b200_film_denoise.
// kVar (rayn_b200_film_denoise_variance): src.w holds the pixel's variance v; a fifth term |lum(c_q) - lum(c_p)| * il_p with
// il_p = 1 / (sl * sqrt(g_p) + 1e-10), g_p the 3x3 prefilter of v, and the output's .w is the filtered variance
// (sum (w*w) v_q) / (sw*sw).  The prefilter is fused here: its 9 taps are neighbours of p that the 5x5 loop's first level
// reads too, so they are L1 hits, and no extra plane or launch is needed.  The kVar = false instances never read `sl`.
// kWrap (rayn_b200_film_denoise_wrap): the film is periodic in x, every tap column is taken floored-mod W; rows still skip.
template <bool kOut3, bool kAlb = false, bool kVar = false, bool kWrap = false>
__global__ void __launch_bounds__(256) k_denoise_level(int W, int H, int step, float ic, float in_, float ia, const float4* __restrict__ guide,
                                                       const float4* __restrict__ src, float4* __restrict__ dst4, float* __restrict__ dst3,
                                                       const float4* __restrict__ alb = nullptr, float il = 0.0f, float sl = 0.0f) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= W || y >= H) return;
  const size_t p = (size_t)y * W + x;
  const float4 cp = src[p];
  float4 o = cp;
  if (dn_finite3(cp)) {
    const float h[5] = {0.0625f, 0.25f, 0.375f, 0.25f, 0.0625f};
    const float4 gp = guide[p];
    const float4 lp = kAlb ? alb[p] : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    float sr = 0.0f, sg = 0.0f, sb = 0.0f, sw = 0.0f, sv = 0.0f;
    float lum_p = 0.0f, ilp = 0.0f;
    if (kVar) {
      lum_p = dn_lum(cp.x, cp.y, cp.z);
      const float k3[3] = {0.25f, 0.5f, 0.25f};
      float gs = 0.0f, gw = 0.0f;
#pragma unroll
      for (int dy = -1; dy <= 1; ++dy) {
        const int qy = y + dy;
        if (qy < 0 || qy >= H) continue;
#pragma unroll
        for (int dx = -1; dx <= 1; ++dx) {
          int qx = x + dx;
          if (kWrap) {
            qx = dn_wrap(qx, W);
          } else if (qx < 0 || qx >= W) {
            continue;
          }
          const float4 cq = src[(size_t)qy * W + qx];
          if (!dn_finite3(cq)) continue;
          const float kk = k3[dy + 1] * k3[dx + 1];
          gs += kk * cq.w;
          gw += kk;
        }
      }
      ilp = 1.0f / (sl * sqrtf(gs / gw) + 1e-10f);  // gw >= 0.25 (the centre tap is finite); ilp in [0, 1e10]
    }
#pragma unroll
    for (int dy = -2; dy <= 2; ++dy) {
      const int qy = y + step * dy;
      if (qy < 0 || qy >= H) continue;
      const float4* srow = src + (size_t)qy * W;
      const float4* grow = guide + (size_t)qy * W;
#pragma unroll
      for (int dx = -2; dx <= 2; ++dx) {
        int qx = x + step * dx;
        if (kWrap) {
          qx = dn_wrap(qx, W);
        } else if (qx < 0 || qx >= W) {
          continue;
        }
        const float4 cq = srow[qx];
        if (!dn_finite3(cq)) continue;
        const float4 gq = grow[qx];
        const float dr = cq.x - cp.x, dg = cq.y - cp.y, db = cq.z - cp.z;
        const float dc2 = (dr * dr + dg * dg) + db * db;
        const float nx = gq.x - gp.x, ny = gq.y - gp.y, nz = gq.z - gp.z;
        const float dn2 = (nx * nx + ny * ny) + nz * nz;
        const float da = gq.w - gp.w;
        const float da2 = da * da;
        float e = (dc2 * ic + dn2 * in_) + da2 * ia;
        if (kAlb) {
          // Every term of e is a product of a square (>= 0 or NaN) and a factor >= 0, so e is still a sum of non-negative
          // terms or NaN (0 * inf = NaN cannot occur: every factor is finite).  Hence both shortcuts hold unchanged: e == 0
          // still means exp(-e) = 1 exactly, and e > DENOISE_E_DEAD or NaN still means a skipped tap.  A non-finite albedo
          // component makes dl2 NaN or +inf, i.e. a NaN tap (skipped) or a dead one (weight +0), as in the statement.
          const float4 lq = alb[(size_t)qy * W + qx];
          const float ar = lq.x - lp.x, ag = lq.y - lp.y, ab = lq.z - lp.z;
          const float dl2 = (ar * ar + ag * ag) + ab * ab;
          e = e + dl2 * il;
        }
        if (kVar) {
          // |dl| >= 0 or NaN times ilp in [0, 1e10] (v >= 0, so g >= 0 or +inf, sqrt(+inf) * sl = +inf gives ilp = 0): the term
          // is >= 0 or NaN, never -0 < 0 or a 0 * inf, so e stays a sum of non-negative terms or NaN and both shortcuts hold
          // (the centre tap still has e = 0).  A luminance that overflows to +-inf makes the term NaN or +inf: skipped or dead.
          e = e + fabsf(dn_lum(cq.x, cq.y, cq.z) - lum_p) * ilp;
        }
        if (!(e <= DENOISE_E_DEAD)) continue;  // NaN (skipped by the statement) or a weight of exactly +0 (argument above)
        const float hk = h[dy + 2] * h[dx + 2];
        const float w = e == 0.0f ? hk : hk * dm::exp(-e);
        sr += w * cq.x;
        sg += w * cq.y;
        sb += w * cq.z;
        sw += w;
        if (kVar && !kOut3) {  // the last level writes the colour only
          // the statement adds only taps whose w*w is not +0 (so an infinite v_q never meets a zero weight); the dead taps
          // skipped above have w = +0 and so add nothing there either
          const float ww = w * w;
          if (ww != 0.0f) sv += ww * cq.w;
        }
      }
    }
    o = make_float4(sr / sw, sg / sw, sb / sw, kVar && !kOut3 ? sv / (sw * sw) : 0.0f);
  }
  if (kOut3) {
    dst3[3 * p] = o.x;
    dst3[3 * p + 1] = o.y;
    dst3[3 * p + 2] = o.z;
  } else {
    dst4[p] = o;
  }
}

// One level of the filter: the k_denoise_level instance of (last level, albedo guide, variance guide, periodic in x)
template <bool kAlb, bool kVar, bool kWrap>
inline void denoise_level(cudaStream_t st, bool last, int W, int H, int step, float ic, float in_, float ia, const float4* guide, const float4* src,
                          float4* dst4, float* dst3, const float4* alb, float il, float sl) {
  const dim3 blk(32, 8), grid((unsigned)((W + 31) / 32), (unsigned)((H + 7) / 8));
  if (last)
    k_denoise_level<true, kAlb, kVar, kWrap><<<grid, blk, 0, st>>>(W, H, step, ic, in_, ia, guide, src, nullptr, dst3, alb, il, sl);
  else
    k_denoise_level<false, kAlb, kVar, kWrap><<<grid, blk, 0, st>>>(W, H, step, ic, in_, ia, guide, src, dst4, nullptr, alb, il, sl);
}
template <bool kAlb, bool kVar>
inline void denoise_level(cudaStream_t st, bool wrap, bool last, int W, int H, int step, float ic, float in_, float ia, const float4* guide,
                          const float4* src, float4* dst4, float* dst3, const float4* alb, float il, float sl) {
  if (wrap)
    denoise_level<kAlb, kVar, true>(st, last, W, H, step, ic, in_, ia, guide, src, dst4, dst3, alb, il, sl);
  else
    denoise_level<kAlb, kVar, false>(st, last, W, H, step, ic, in_, ia, guide, src, dst4, dst3, alb, il, sl);
}

}  // namespace rt
