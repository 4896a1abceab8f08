// film_mirror.cpp — CPU mirrors of the film-plane passes of include/rayn_b200.h: the a-trous denoise in its four entry points
// (rayn_b200_film_denoise, _albedo, _variance, _variance_scaled) and rayn_b200_temporal_push.  TEST INFRASTRUCTURE ONLY, built
// by tests/mirrors.py with g++ -ffp-contract=off so that every float operation below is one IEEE rounding, as on the device
// (--fmad=false).  The exponential is detmath.h's dm::exp, shared with the kernels.  The filter is a plain restatement: it
// evaluates every tap, with no shortcut for zero weights.
#include <math.h>
#include <stdint.h>

#include <vector>

#include "../include/rayn_b200.h"
#include "../rayn_b200/csrc/detmath.h"

namespace {

bool finite3(const float* c) { return isfinite(c[0]) && isfinite(c[1]) && isfinite(c[2]); }
float lum(const float* v) { return (0.2126f * v[0] + 0.7152f * v[1]) + 0.0722f * v[2]; }

// One level on (c: 3 floats, v: 1 float) per pixel.  il == 0: no albedo term; !var: no luminance term.  With both off each
// tap's exponent is (dc2 * ic + dn2 * in) + da2 * ia, rayn_b200_film_denoise's.
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

// The filter behind every entry point, after that entry point's own argument rules: il != 0 adds the albedo term (albedo
// [3*W*H]); a finite sl adds the luminance term, with the level-0 variance from the moment planes m and spp, scaled per pixel
// by scale unless it is NULL.  Returns RAYN_OK or RAYN_ERR_INVALID_ARG under the rules every entry point shares.
int32_t denoise(const RaynDenoiseDesc* d, int32_t W, int32_t H, const RaynFilmPlanes* in, const RaynFilmPlanes* out, float il, const float* albedo,
                float sl, int32_t spp, const RaynMomentPlanes* m, const float* scale) {
  if (!d || !in || !out || W <= 0 || H <= 0 || d->iterations < 1 || d->iterations > 8 || !in->normal || !in->alpha) return RAYN_ERR_INVALID_ARG;
  if ((in->color && !out->color) || (in->background && !out->background)) return RAYN_ERR_INVALID_ARG;
  float ic0, in_, ia;
  if (!factor(d->sigma_color, &ic0) || !isfinite(ldexpf(ic0, d->iterations - 1)) || !factor(d->sigma_normal, &in_) || !factor(d->sigma_alpha, &ia))
    return RAYN_ERR_INVALID_ARG;
  const bool var = !isinf(sl);
  const size_t n = (size_t)W * H;
  const float* srcs[2] = {(const float*)in->color, (const float*)in->background};
  const float* moms[2] = {m ? (const float*)m->color_lum2 : nullptr, m ? (const float*)m->background_lum2 : nullptr};
  float* dsts[2] = {(float*)out->color, (float*)out->background};
  for (int ch = 0; ch < 2; ++ch) {
    if (!srcs[ch]) continue;
    std::vector<float> cur(srcs[ch], srcs[ch] + 3 * n), next(3 * n), v(n, 0.0f), vnext(n);
    if (var)
      for (size_t p = 0; p < n; ++p) {
        const float l = lum(&cur[3 * p]);
        float s = fmaxf(moms[ch][p] - l * l, 0.0f);
        if (scale) s = s * scale[p];
        v[p] = s / (float)spp;
      }
    for (int i = 0; i < d->iterations; ++i) {
      level(W, H, 1 << i, ldexpf(ic0, i), in_, ia, il, var, sl, (const float*)in->normal, (const float*)in->alpha, albedo, cur.data(), v.data(),
            next.data(), vnext.data());
      cur.swap(next);
      v.swap(vnext);
    }
    for (size_t k = 0; k < 3 * n; ++k) dsts[ch][k] = cur[k];
  }
  return RAYN_OK;
}

// the argument rules the two variance entry points add
bool variance_args(const RaynDenoiseDesc* d, float sigma_luminance, int32_t spp, const RaynMomentPlanes* m, float sigma_albedo, const float* albedo,
                   const RaynFilmPlanes* in, float* il) {
  *il = 0.0f;
  if (!m || !in || !d) return false;
  if ((in->color && !m->color_lum2) || (in->background && !m->background_lum2) || spp < 1 || !(sigma_luminance > 0.0f)) return false;
  return !albedo || factor(sigma_albedo, il);
}

// history plane indices, as rt_temporal.cuh
enum { TC = 0, TB = 3, TM = 6, TN = 8, TZ = 11, TLEN = 12, TS = 13 };

}  // namespace

extern "C" {

int32_t rayn_oracle_muladd_fused(void) { return RAYN_MULADD_FUSED; }

// 0 if a product and a sum are rounded on their own (the build has -ffp-contract=off), 1 if they were contracted
int32_t rayn_oracle_selfcheck(void) {
  volatile float va = 1.0f + 0x1p-12f, vc = -(1.0f + 0x1p-11f);
  const float a = va, c = vc;
  return a * a + c == 0.0f ? 0 : 1;
}

float rayn_oracle_exp(float x) { return dm::exp(x); }

// host planes only; each entry point returns RAYN_OK or RAYN_ERR_INVALID_ARG under the same rules as the library
int32_t rayn_oracle_film_denoise(const RaynDenoiseDesc* d, int32_t W, int32_t H, const RaynFilmPlanes* in, const RaynFilmPlanes* out) {
  return denoise(d, W, H, in, out, 0.0f, nullptr, INFINITY, 1, nullptr, nullptr);
}

int32_t rayn_oracle_film_denoise_albedo(const RaynDenoiseDesc* d, float sigma_albedo, const float* albedo, int32_t W, int32_t H,
                                        const RaynFilmPlanes* in, const RaynFilmPlanes* out) {
  float il;
  if (!albedo || !factor(sigma_albedo, &il)) return RAYN_ERR_INVALID_ARG;
  return denoise(d, W, H, in, out, il, albedo, INFINITY, 1, nullptr, nullptr);
}

int32_t rayn_oracle_film_denoise_variance(const RaynDenoiseDesc* d, float sigma_luminance, int32_t spp, const RaynMomentPlanes* m, float sigma_albedo,
                                          const float* albedo, int32_t W, int32_t H, const RaynFilmPlanes* in, const RaynFilmPlanes* out) {
  float il;
  if (!variance_args(d, sigma_luminance, spp, m, sigma_albedo, albedo, in, &il)) return RAYN_ERR_INVALID_ARG;
  return denoise(d, W, H, in, out, il, albedo, sigma_luminance, spp, m, nullptr);
}

int32_t rayn_oracle_film_denoise_variance_scaled(const RaynDenoiseDesc* d, float sigma_luminance, int32_t spp, const RaynMomentPlanes* m,
                                                 const float* scale, float sigma_albedo, const float* albedo, int32_t W, int32_t H,
                                                 const RaynFilmPlanes* in, const RaynFilmPlanes* out) {
  float il;
  if (!scale || !variance_args(d, sigma_luminance, spp, m, sigma_albedo, albedo, in, &il)) return RAYN_ERR_INVALID_ARG;
  return denoise(d, W, H, in, out, il, albedo, sigma_luminance, spp, m, scale);
}

// One push: hin / hout are 14 planes of W*H floats (hout must not alias hin); c, b, n [3*W*H], mc, mb [W*H], motion [4*W*H];
// outputs oc, ob [3*W*H], omc, omb, scale [W*H] (they may alias the inputs).
int32_t rayn_oracle_temporal_push(int32_t W, int32_t H, const RaynTemporalDesc* d, const float* hin, float* hout, const float* c, const float* b,
                                  const float* nrm, const float* mc, const float* mb, const float* motion, float* oc, float* ob, float* omc,
                                  float* omb, float* scale) {
  if (!d || W <= 0 || H <= 0 || W > (1 << 23) || H > (1 << 23) || !(d->alpha_min > 0.0f && d->alpha_min <= 1.0f) || !(d->sigma_depth > 0.0f) ||
      !(d->normal_cos >= -1.0f && d->normal_cos <= 1.0f) || (d->reset != 0 && d->reset != 1))
    return RAYN_ERR_INVALID_ARG;
  const size_t npx = (size_t)W * H;
  for (int y = 0; y < H; ++y)
    for (int x = 0; x < W; ++x) {
      const size_t p = (size_t)y * W + x;
      const float cur[8] = {c[3 * p], c[3 * p + 1], c[3 * p + 2], b[3 * p], b[3 * p + 1], b[3 * p + 2], mc[p], mb[p]};
      const float nx = nrm[3 * p], ny = nrm[3 * p + 1], nz = nrm[3 * p + 2];
      const float z = motion[4 * p + 2], zp = motion[4 * p + 3];
      float hv[10] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
      float nh = 0.0f;
      if (!d->reset && isfinite(zp)) {
        const float fx = (((float)x + 0.5f) + motion[4 * p]) - 0.5f, fy = (((float)y + 0.5f) + motion[4 * p + 1]) - 0.5f;
        const float x0 = floorf(fx), y0 = floorf(fy);
        const float ax = fx - x0, ay = fy - y0;
        float ws = 0.0f;
        for (int j = 0; j < 2; ++j)
          for (int i = 0; i < 2; ++i) {
            const float w = (i ? ax : 1.0f - ax) * (j ? ay : 1.0f - ay);
            const float qx = x0 + (float)i, qy = y0 + (float)j;
            if (w == 0.0f || w != w) continue;
            if (!(qx >= 0.0f && qx <= (float)(W - 1) && qy >= 0.0f && qy <= (float)(H - 1))) continue;
            const size_t q = (size_t)qy * W + (size_t)qx;
            const float* hq[14];
            for (int k = 0; k < 14; ++k) hq[k] = hin + k * npx + q;
            if (!(*hq[TLEN] > 0.0f)) continue;
            bool fin = true;
            for (int k = 0; k < 6; ++k) fin = fin && isfinite(*hq[TC + k]);
            if (!fin) continue;
            if (!isfinite(*hq[TZ]) || !(fabsf(*hq[TZ] - zp) <= d->sigma_depth * fabsf(zp))) continue;
            const float nd = (*hq[TN] * nx + *hq[TN + 1] * ny) + *hq[TN + 2] * nz;
            if (!(nd >= d->normal_cos)) continue;
            ws += w;
            for (int k = 0; k < 8; ++k) hv[k] += w * *hq[TC + k];
            hv[8] += w * *hq[TLEN];
            hv[9] += w * *hq[TS];
          }
        if (ws != 0.0f) {
          for (int k = 0; k < 10; ++k) hv[k] = hv[k] / ws;
          nh = hv[8];
        }
      }
      const float alpha = fmaxf(d->alpha_min, 1.0f / (nh + 1.0f));
      float o[8], s;
      if (alpha == 1.0f) {
        for (int k = 0; k < 8; ++k) o[k] = cur[k];
        s = 1.0f;
      } else {
        for (int k = 0; k < 8; ++k) o[k] = (1.0f - alpha) * hv[k] + alpha * cur[k];
        s = ((1.0f - alpha) * (1.0f - alpha)) * hv[9] + alpha * alpha;
      }
      for (int k = 0; k < 8; ++k) hout[k * npx + p] = o[k];
      hout[TN * npx + p] = nx, hout[(TN + 1) * npx + p] = ny, hout[(TN + 2) * npx + p] = nz;
      hout[TZ * npx + p] = z;
      hout[TLEN * npx + p] = nh + 1.0f;
      hout[TS * npx + p] = s;
      oc[3 * p] = o[0], oc[3 * p + 1] = o[1], oc[3 * p + 2] = o[2];
      ob[3 * p] = o[3], ob[3 * p + 1] = o[4], ob[3 * p + 2] = o[5];
      omc[p] = o[6], omb[p] = o[7];
      scale[p] = s;
    }
  return RAYN_OK;
}

}  // extern "C"
