// rt_temporal.cuh — temporal accumulation of a frame sequence (rayn_b200_temporal_push; the exact statement is in
// include/rayn_b200.h, the CPU mirror in tests/temporal_oracle.cpp).
//
// One thread per pixel.  The history is 14 planes of W*H floats (structure of arrays, so every plane access of a warp is
// coalesced); a push reads one history and writes the other, so no thread reads a tap another thread is writing.
#pragma once
#include "rt_device.cuh"

namespace rt {

// history plane indices
enum { TH_C = 0, TH_B = 3, TH_M = 6, TH_N = 8, TH_Z = 11, TH_LEN = 12, TH_S = 13, TH_PLANES = 14 };

struct TemporalIo {
  const float *c, *b, *n, *mc, *mb, *motion;  // current frame
  float *oc, *ob, *omc, *omb, *scale;          // outputs (oc / ob may alias c / b)
};

__global__ void __launch_bounds__(256) k_temporal(int W, int H, RaynTemporalDesc d, const float* __restrict__ hin, float* __restrict__ hout,
                                                  TemporalIo io) {
  const long long npx = (long long)W * H;
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= npx) return;
  const int x = (int)(p % W), y = (int)(p / W);
  float cur[8];
  cur[0] = io.c[3 * p], cur[1] = io.c[3 * p + 1], cur[2] = io.c[3 * p + 2];
  cur[3] = io.b[3 * p], cur[4] = io.b[3 * p + 1], cur[5] = io.b[3 * p + 2];
  cur[6] = io.mc[p], cur[7] = io.mb[p];
  const float nx = io.n[3 * p], ny = io.n[3 * p + 1], nz = io.n[3 * p + 2];
  const float z = io.motion[4 * p + 2], zp = io.motion[4 * p + 3];
  float hv[10];  // colour 3, background 3, moments 2, n, s of the history
#pragma unroll
  for (int k = 0; k < 10; ++k) hv[k] = 0.0f;
  float nh = 0.0f;
  // a current pixel without a finite z_prev (no valid hit, or a non-finite record) takes no history
  if (!d.reset && isfinite(zp)) {
    const float fx = (((float)x + 0.5f) + io.motion[4 * p]) - 0.5f, fy = (((float)y + 0.5f) + io.motion[4 * p + 1]) - 0.5f;
    const float x0 = floorf(fx), y0 = floorf(fy);
    const float ax = fx - x0, ay = fy - y0;
    float ws = 0.0f;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const float w = (i ? ax : 1.0f - ax) * (j ? ay : 1.0f - ay);
        const float qxf = x0 + (float)i, qyf = y0 + (float)j;
        // NaN motion fails every comparison: no tap
        if (!(w != 0.0f) || !(qxf >= 0.0f && qxf <= (float)(W - 1) && qyf >= 0.0f && qyf <= (float)(H - 1))) continue;
        const size_t q = (size_t)qyf * W + (size_t)qxf;
        if (!(hin[TH_LEN * npx + q] > 0.0f)) continue;
        const float c0 = hin[TH_C * npx + q], c1 = hin[(TH_C + 1) * npx + q], c2 = hin[(TH_C + 2) * npx + q];
        const float b0 = hin[TH_B * npx + q], b1 = hin[(TH_B + 1) * npx + q], b2 = hin[(TH_B + 2) * npx + q];
        if (!(isfinite(c0) && isfinite(c1) && isfinite(c2) && isfinite(b0) && isfinite(b1) && isfinite(b2))) continue;
        if (!(fabsf(hin[TH_Z * npx + q] - zp) <= d.sigma_depth * fabsf(zp))) continue;  // false for a non-finite z_h
        const float nd = (hin[TH_N * npx + q] * nx + hin[(TH_N + 1) * npx + q] * ny) + hin[(TH_N + 2) * npx + q] * nz;
        if (!(nd >= d.normal_cos)) continue;
        ws += w;
        hv[0] += w * c0, hv[1] += w * c1, hv[2] += w * c2;
        hv[3] += w * b0, hv[4] += w * b1, hv[5] += w * b2;
        hv[6] += w * hin[TH_M * npx + q], hv[7] += w * hin[(TH_M + 1) * npx + q];
        hv[8] += w * hin[TH_LEN * npx + q], hv[9] += w * hin[TH_S * npx + q];
      }
    }
    if (ws != 0.0f) {
#pragma unroll
      for (int k = 0; k < 10; ++k) hv[k] = hv[k] / ws;
      nh = hv[8];
    }
  }
  const float alpha = fmaxf(d.alpha_min, 1.0f / (nh + 1.0f));
  float out[8], s;
  if (alpha == 1.0f) {
#pragma unroll
    for (int k = 0; k < 8; ++k) out[k] = cur[k];
    s = 1.0f;
  } else {
    const float beta = 1.0f - alpha;
#pragma unroll
    for (int k = 0; k < 8; ++k) out[k] = beta * hv[k] + alpha * cur[k];
    s = (beta * beta) * hv[9] + alpha * alpha;
  }
  io.oc[3 * p] = out[0], io.oc[3 * p + 1] = out[1], io.oc[3 * p + 2] = out[2];
  io.ob[3 * p] = out[3], io.ob[3 * p + 1] = out[4], io.ob[3 * p + 2] = out[5];
  io.omc[p] = out[6], io.omb[p] = out[7];
  io.scale[p] = s;
#pragma unroll
  for (int k = 0; k < 8; ++k) hout[k * npx + p] = out[k];
  hout[TH_N * npx + p] = nx, hout[(TH_N + 1) * npx + p] = ny, hout[(TH_N + 2) * npx + p] = nz;
  hout[TH_Z * npx + p] = z;
  hout[TH_LEN * npx + p] = nh + 1.0f;
  hout[TH_S * npx + p] = s;
}

}  // namespace rt
