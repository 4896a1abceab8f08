// rt_accum.cuh — device film accumulator for progressive / adaptive rendering (rayn_b200_accum_*).  The exact statement
// (fold, half-sample film, per-tile error, resolve) is at RaynAdaptiveDesc in include/rayn_b200.h; tests/accum_mirror.py
// restates it in numpy and the GPU tests compare bit for bit.  Every operation below is an explicit _rn intrinsic, so
// the result does not depend on the compiler's contraction flags.
//
// State layout (planar, like the film planes): S color [3*npx] | S alpha [npx] | S background [3*npx] | S normal [3*npx]
// | H [3*npx]  = 13 floats per pixel.  The round's planes m use the first 10 of those offsets.
#pragma once
#include "rt_device.cuh"

namespace rt {

#define ACC_T 256        // threads per CTA of k_accum_fold
#define ACC_CHUNK 1024   // e values staged in shared memory per step of the sequential tile sum

struct AccumTiles {  // per tile, indexed by tile index tile_x * n_tiles_y + tile_y
  double* E;
  long long* K;
  long long* Kh;
  int* rounds;
};

// One CTA per active tile (tiles[blockIdx.x]): folds the round's planes m into S and H, advances K / Kh / rounds, and
// computes E.  The e of every in-image pixel goes to shared memory in chunks of ACC_CHUNK in ascending pixel index, and
// thread 0 adds each chunk in that order in double: the strictly sequential sum of the statement.
__global__ void __launch_bounds__(ACC_T) k_accum_fold(int W, int H, int tile_w, int tile_h, int nty, const int* __restrict__ tiles, float n,
                                                      long long n_int, const float* __restrict__ m, float* __restrict__ S, AccumTiles ts) {
  __shared__ float erow[ACC_CHUNK];
  const size_t npx = (size_t)W * H;
  const int tile = tiles[blockIdx.x];
  const int tx = tile / nty, ty = tile - tx * nty;
  const int x0 = tx * tile_w, y0 = ty * tile_h;
  const int cw = min(x0 + tile_w, W) - x0, ch = min(y0 + tile_h, H) - y0, count = cw * ch;
  const int r = ts.rounds[tile];
  const bool upd_h = (r & 1) == 0, with_err = r + 1 >= 2;
  const long long K1 = ts.K[tile] + n_int, Kh1 = ts.Kh[tile] + (upd_h ? n_int : 0);
  const float fK = (float)K1, fKh = (float)Kh1;
  const float *mc = m, *ma = m + 3 * npx, *mb = m + 4 * npx, *mn = m + 7 * npx;
  float *Sc = S, *Sa = S + 3 * npx, *Sb = S + 4 * npx, *Sn = S + 7 * npx, *Hh = S + 10 * npx;
  double sum = 0.0;
  for (int c0 = 0; c0 < count; c0 += ACC_CHUNK) {
    const int c1 = min(c0 + ACC_CHUNK, count);
    for (int j = c0 + (int)threadIdx.x; j < c1; j += ACC_T) {
      const int yl = j / cw, xl = j - yl * cw;
      const size_t p = (size_t)(x0 + xl) + (size_t)(y0 + yl) * W;
      float sc[3], sb[3], hv[3];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float vc = mc[3 * p + c], vb = mb[3 * p + c];
        sc[c] = __fadd_rn(Sc[3 * p + c], __fmul_rn(vc, n));
        sb[c] = __fadd_rn(Sb[3 * p + c], __fmul_rn(vb, n));
        Sc[3 * p + c] = sc[c];
        Sb[3 * p + c] = sb[c];
        Sn[3 * p + c] = __fadd_rn(Sn[3 * p + c], __fmul_rn(mn[3 * p + c], n));
        hv[c] = Hh[3 * p + c];
        if (upd_h) {
          hv[c] = __fadd_rn(hv[c], __fmul_rn(__fadd_rn(vc, vb), n));
          Hh[3 * p + c] = hv[c];
        }
      }
      Sa[p] = __fadd_rn(Sa[p], __fmul_rn(ma[p], n));
      if (with_err) {
        float I[3], D[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          I[c] = __fdiv_rn(__fadd_rn(sc[c], sb[c]), fK);
          D[c] = fabsf(__fsub_rn(I[c], __fdiv_rn(hv[c], fKh)));
        }
        const float d = __fadd_rn(__fadd_rn(D[0], D[1]), D[2]);
        const float s = __fadd_rn(__fadd_rn(I[0], I[1]), I[2]);
        const float e = __fdiv_rn(d, __fsqrt_rn(fmaxf(s, 0x1p-10f)));
        erow[j - c0] = e != e ? __int_as_float(0x7f800000) : e;  // NaN counts as +inf
      }
    }
    if (!with_err) continue;  // CTA-uniform
    __syncthreads();
    if (threadIdx.x == 0)
      for (int k = 0; k < c1 - c0; ++k) sum = __dadd_rn(sum, (double)erow[k]);
    __syncthreads();
  }
  __syncthreads();  // every thread has read this tile's rounds / K / Kh
  if (threadIdx.x == 0) {
    ts.K[tile] = K1;
    ts.Kh[tile] = Kh1;
    ts.rounds[tile] = r + 1;
    ts.E[tile] = with_err ? __ddiv_rn(sum, (double)count) : __longlong_as_double(0x7ff0000000000000ll);
  }
}

// out.x[c] = S.x[c] / (float)K of the pixel's tile; 0 outside the tile grid (as k_zero_uncovered leaves a render).
__global__ void __launch_bounds__(256) k_accum_resolve(int W, int H, int tile_w, int tile_h, int ntx, int nty, const float* __restrict__ S,
                                                       const long long* __restrict__ K, float* color, float* alpha, float* background,
                                                       float* normal) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long npx = (long long)W * H;
  if (i >= npx) return;
  const int x = (int)(i % W), y = (int)(i / W);
  const int tx = x / tile_w, ty = y / tile_h;
  const bool covered = tx < ntx && ty < nty;
  const float fK = covered ? (float)K[tx * nty + ty] : 1.0f;
  auto put = [&](float* dst, const float* src, int nc) {
    if (!dst) return;
    for (int c = 0; c < nc; ++c) dst[nc * i + c] = covered ? __fdiv_rn(src[nc * i + c], fK) : 0.0f;
  };
  put(color, S, 3);
  put(alpha, S + 3 * npx, 1);
  put(background, S + 4 * npx, 3);
  put(normal, S + 7 * npx, 3);
}

}  // namespace rt
