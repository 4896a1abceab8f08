// denoise_variance_oracle.cpp — CPU mirror of rayn_b200_film_denoise_variance (the statement is in include/rayn_b200.h).
// TEST INFRASTRUCTURE ONLY, built by tests/moments_oracle.py with g++ -ffp-contract=off, like tests/denoise_albedo_oracle.cpp,
// whose restatement this is with the variance term.  Every tap is evaluated; there is no shortcut for zero weights.
#include <math.h>
#include <stdint.h>

#include <vector>

#include "../include/rayn_b200.h"
#include "../rayn_b200/csrc/detmath.h"

namespace {

bool finite3(const float* c) { return isfinite(c[0]) && isfinite(c[1]) && isfinite(c[2]); }
float lum(const float* v) { return (0.2126f * v[0] + 0.7152f * v[1]) + 0.0722f * v[2]; }

// One level on (c: 3 floats, v: 1 float) per pixel.  il == 0: no albedo term; var: the variance term (sl finite).
void level(int W, int H, int step, float ic, float in_, float ia, float il, bool var, float sl, const float* n3, const float* a, const float* l3,
           const float* src, const float* vsrc, float* dst, float* vdst) {
  static const float h[5] = {0.0625f, 0.25f, 0.375f, 0.25f, 0.0625f};
  static const float k3[3] = {0.25f, 0.5f, 0.25f};
  for (int y = 0; y < H; ++y)
    for (int x = 0; x < W; ++x) {
      const size_t p = (size_t)y * W + x;
      const float* cp = src + 3 * p;
      if (!finite3(cp)) {
        dst[3 * p] = cp[0], dst[3 * p + 1] = cp[1], dst[3 * p + 2] = cp[2];
        vdst[p] = vsrc[p];
        continue;
      }
      float ilp = 0.0f, lp_ = 0.0f;
      if (var) {
        float gs = 0.0f, gw = 0.0f;
        for (int dy = -1; dy <= 1; ++dy)
          for (int dx = -1; dx <= 1; ++dx) {
            const int qx = x + dx, qy = y + dy;
            if (qx < 0 || qx >= W || qy < 0 || qy >= H) continue;
            const size_t q = (size_t)qy * W + qx;
            if (!finite3(src + 3 * q)) continue;
            const float kk = k3[dy + 1] * k3[dx + 1];
            gs += kk * vsrc[q];
            gw += kk;
          }
        ilp = 1.0f / (sl * sqrtf(gs / gw) + 1e-10f);
        lp_ = lum(cp);
      }
      const float* np_ = n3 + 3 * p;
      const float* lp = l3 ? l3 + 3 * p : nullptr;
      float sr = 0.0f, sg = 0.0f, sb = 0.0f, sw = 0.0f, sv = 0.0f;
      for (int dy = -2; dy <= 2; ++dy)
        for (int dx = -2; dx <= 2; ++dx) {
          const int qx = x + step * dx, qy = y + step * dy;
          if (qx < 0 || qx >= W || qy < 0 || qy >= H) continue;
          const size_t q = (size_t)qy * W + qx;
          const float* cq = src + 3 * q;
          if (!finite3(cq)) continue;
          const float* nq = n3 + 3 * q;
          const float dr = cq[0] - cp[0], dg = cq[1] - cp[1], db = cq[2] - cp[2];
          const float dc2 = (dr * dr + dg * dg) + db * db;
          const float nx = nq[0] - np_[0], ny = nq[1] - np_[1], nz = nq[2] - np_[2];
          const float dn2 = (nx * nx + ny * ny) + nz * nz;
          const float da = a[q] - a[p];
          const float da2 = da * da;
          float e = (dc2 * ic + dn2 * in_) + da2 * ia;
          if (il != 0.0f) {
            const float* lq = l3 + 3 * q;
            const float ar = lq[0] - lp[0], ag = lq[1] - lp[1], ab = lq[2] - lp[2];
            const float dl2 = (ar * ar + ag * ag) + ab * ab;
            e = e + dl2 * il;
          }
          if (var) e = e + fabsf(lum(cq) - lp_) * ilp;
          if (e != e) continue;
          const float hk = h[dy + 2] * h[dx + 2];
          const float w = hk * dm::exp(-e);
          sr += w * cq[0];
          sg += w * cq[1];
          sb += w * cq[2];
          sw += w;
          const float ww = w * w;
          if (ww != 0.0f) sv += ww * vsrc[q];
        }
      dst[3 * p] = sr / sw, dst[3 * p + 1] = sg / sw, dst[3 * p + 2] = sb / sw;
      vdst[p] = sv / (sw * sw);
    }
}

bool factor(float sigma, float* f) {
  if (!(sigma > 0.0f)) return false;
  *f = 1.0f / (sigma * sigma);
  return isfinite(*f);
}

}  // namespace

extern "C" {

int32_t rayn_oracle_muladd_fused(void) { return RAYN_MULADD_FUSED; }

// host planes only; returns RAYN_OK or RAYN_ERR_INVALID_ARG under the same rules as the library
int32_t rayn_oracle_film_denoise_variance(const RaynDenoiseDesc* d, float sigma_luminance, int32_t spp, const RaynMomentPlanes* m, float sigma_albedo,
                                          const float* albedo, int32_t W, int32_t H, const RaynFilmPlanes* in, const RaynFilmPlanes* out) {
  if (!m || !d || !in || !out || W <= 0 || H <= 0 || d->iterations < 1 || d->iterations > 8 || !in->normal || !in->alpha)
    return RAYN_ERR_INVALID_ARG;
  if ((in->color && !out->color) || (in->background && !out->background)) return RAYN_ERR_INVALID_ARG;
  if ((in->color && !m->color_lum2) || (in->background && !m->background_lum2) || spp < 1 || !(sigma_luminance > 0.0f))
    return RAYN_ERR_INVALID_ARG;
  float ic0, in_, ia, il = 0.0f;
  if ((albedo && !factor(sigma_albedo, &il)) || !factor(d->sigma_color, &ic0) || !isfinite(ldexpf(ic0, d->iterations - 1)) ||
      !factor(d->sigma_normal, &in_) || !factor(d->sigma_alpha, &ia))
    return RAYN_ERR_INVALID_ARG;
  const bool var = !isinf(sigma_luminance);
  const size_t n = (size_t)W * H;
  const float* srcs[2] = {in->color, in->background};
  const float* moms[2] = {m->color_lum2, m->background_lum2};
  float* dsts[2] = {out->color, out->background};
  for (int ch = 0; ch < 2; ++ch) {
    if (!srcs[ch]) continue;
    std::vector<float> cur(srcs[ch], srcs[ch] + 3 * n), next(3 * n), v(n, 0.0f), vnext(n);
    if (var)
      for (size_t p = 0; p < n; ++p) {
        const float l = lum(&cur[3 * p]);
        v[p] = fmaxf(moms[ch][p] - l * l, 0.0f) / (float)spp;
      }
    for (int i = 0; i < d->iterations; ++i) {
      level(W, H, 1 << i, ldexpf(ic0, i), in_, ia, il, var, sigma_luminance, in->normal, in->alpha, albedo, cur.data(), v.data(), next.data(),
            vnext.data());
      cur.swap(next);
      v.swap(vnext);
    }
    for (size_t k = 0; k < 3 * n; ++k) dsts[ch][k] = cur[k];
  }
  return RAYN_OK;
}

}  // extern "C"
