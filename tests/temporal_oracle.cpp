// temporal_oracle.cpp — CPU mirrors of rayn_b200_temporal_push and rayn_b200_film_denoise_variance_scaled (the statements are
// in include/rayn_b200.h).  TEST INFRASTRUCTURE ONLY, built by tests/temporal_oracle.py with g++ -ffp-contract=off.
// It includes tests/denoise_variance_oracle.cpp unchanged and reuses its filter level; only the level-0 variance differs.
#include "denoise_variance_oracle.cpp"

namespace {

// history plane indices, as rt_temporal.cuh
enum { TC = 0, TB = 3, TM = 6, TN = 8, TZ = 11, TLEN = 12, TS = 13 };

}  // namespace

extern "C" {

// host planes only; the same argument rules as the library
int32_t rayn_oracle_film_denoise_variance_scaled(const RaynDenoiseDesc* d, float sigma_luminance, int32_t spp, const RaynMomentPlanes* m,
                                                 const float* scale, float sigma_albedo, const float* albedo, int32_t W, int32_t H,
                                                 const RaynFilmPlanes* in, const RaynFilmPlanes* out) {
  if (!scale || !m || !d || !in || !out || W <= 0 || H <= 0 || d->iterations < 1 || d->iterations > 8 || !in->normal || !in->alpha)
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
        v[p] = (fmaxf(moms[ch][p] - l * l, 0.0f) * scale[p]) / (float)spp;
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

// One push: hin / hout are 14 planes of W*H floats (hout must not alias hin); c, b, n [3*W*H], mc, mb [W*H], motion [4*W*H];
// outputs oc, ob [3*W*H], omc, omb, scale [W*H] (they may alias the inputs).
int32_t rayn_oracle_temporal_push(int32_t W, int32_t H, const RaynTemporalDesc* d, const float* hin, float* hout, const float* c, const float* b,
                                  const float* nrm, const float* mc, const float* mb, const float* motion, float* oc, float* ob, float* omc,
                                  float* omb, float* scale) {
  if (!d || W <= 0 || H <= 0 || !(d->alpha_min > 0.0f && d->alpha_min <= 1.0f) || !(d->sigma_depth > 0.0f) ||
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
