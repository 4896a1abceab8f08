// host_inputs.cpp — host-side builders for the inputs the Rust host owns in rayn and hands
// to the renderer: the sampler tables, the per-pixel scramble plane, the filter
// importance-sampling table and the tile grid.  Pure CPU code, no CUDA.
//
// In a real drop-in the Rust side passes its own `Samples` / scramble / FIS buffers through
// RaynFrameDesc (include/rayn_b200.h); these builders exist so that the C++/Python stand-in
// hosts, the oracle and the CUDA path all consume the SAME inputs.  They restate algorithms
// that live in crates absent from the reference tree (SURVEY §8c) - unverified against the real
// crates, which is harmless for parity because the tables cross the ABI as data.
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../include/rayn_b200.h"

namespace {

// ---- quasi-rd (git ce11703) : Martin Roberts' R_d additive recurrence --------------------
// x_n = frac(0.5 + alpha * n), alpha_d = 1/phi_d, phi_d the generalised golden ratio.
// alpha is held as a 0.64 fixed-point fraction so `alpha * n mod 1` is exact for the huge
// per-set offsets `(offset + i) << 32` the reference uses (sampler.rs:23,28).
const uint64_t kAlpha1 = 0x9e3779b97f4a7c15ull;     // 1/phi_1 (golden ratio)
const uint64_t kAlpha2x = 0xc13fa9a902a6328full;    // 1/phi_2 (plastic number)
const uint64_t kAlpha2y = 0x91e10da5c79e7b1cull;    // 1/phi_2^2

inline float rd_value(uint64_t alpha, uint64_t n) {
  uint64_t frac = alpha * n + 0x8000000000000000ull;  // + 0.5, wraps mod 1
  // top 24 bits -> [0,1) float, exactly representable
  return (float)(frac >> 40) * (1.0f / 16777216.0f);
}

// ---- rand 0.7.2 SmallRng (= rand_pcg 0.2.1 Pcg64Mcg) seeded by rand_core 0.5.1
//      SeedableRng::seed_from_u64, then Standard f32: (next_u32() >> 8) * 2^-24 -------------
inline float small_rng_first_f32(uint64_t seed_u64) {
  const uint64_t MUL = 6364136223846793005ull, INC = 11634580027462260723ull;
  uint8_t seed[16];
  uint64_t state = seed_u64;
  for (int chunk = 0; chunk < 4; ++chunk) {
    state = state * MUL + INC;
    uint32_t xorshifted = (uint32_t)(((state >> 18) ^ state) >> 27);
    uint32_t rot = (uint32_t)(state >> 59);
    uint32_t x = (xorshifted >> rot) | (xorshifted << ((32 - rot) & 31));
    memcpy(seed + 4 * chunk, &x, 4);  // little endian
  }
  unsigned __int128 s;
  memcpy(&s, seed, 16);
  s |= 1;  // Mcg128Xsl64::new forces the state odd
  const unsigned __int128 MULT = ((unsigned __int128)2549297995355413924ull << 64) | 4865540595714422341ull;
  s = s * MULT;
  uint32_t rot = (uint32_t)(s >> 122);
  uint64_t xsl = (uint64_t)(s >> 64) ^ (uint64_t)s;
  uint64_t out = (xsl >> rot) | (xsl << ((64 - rot) & 63));
  uint32_t v = (uint32_t)out;
  return (float)(v >> 8) * (1.0f / 16777216.0f);
}

// ---- filter.rs:13-49 BlackmanHarris, math.rs:136-191 CDF, filter.rs:196-218 FIS::new ------
float blackman_harris(float radius, float p) {
  const float PI = 3.14159265358979323846f;
  const float A0 = 0.35875f, A1 = 0.48829f, A2 = 0.14128f, A3 = 0.01168f;
  const float TWOPI = PI * 2.0f, FOURPI = PI * 4.0f, SIXPI = PI * 6.0f;
  if (fabsf(p) > radius) return 0.0f;
  float x = fabsf(p / radius) * 0.5f + 0.5f;
  return A0 - A1 * cosf(TWOPI * x) + A2 * cosf(FOURPI * x) + A3 * cosf(SIXPI * x);
}

}  // namespace

extern "C" {

int32_t rayn_b200_host_rd_tables(int32_t spp, int32_t sets_1d, int32_t sets_2d, uint64_t offset, float* out_1d,
                                 float* out_2d) {
  return rayn_b200_host_rd_tables_at(spp, sets_1d, sets_2d, offset, 0, out_1d, out_2d);
}

// samples [first, first + spp) of every set: a later slice of the same sequence, for sample rounds of one film
int32_t rayn_b200_host_rd_tables_at(int32_t spp, int32_t sets_1d, int32_t sets_2d, uint64_t offset, uint64_t first, float* out_1d,
                                    float* out_2d) {
  if (spp <= 0 || sets_1d < 0 || sets_2d < 0 || (!out_1d && sets_1d) || (!out_2d && sets_2d) || first > (1ull << 32) - (uint64_t)spp)
    return RAYN_ERR_INVALID_ARG;
  for (int i = 0; i < sets_1d; ++i) {
    uint64_t base = ((offset + (uint64_t)i) << 32) + first;
    for (int n = 0; n < spp; ++n) out_1d[(size_t)spp * i + n] = rd_value(kAlpha1, base + (uint64_t)n + 1);
  }
  for (int i = 0; i < sets_2d; ++i) {
    uint64_t base = ((offset + (uint64_t)sets_1d + (uint64_t)i) << 32) + first;
    for (int n = 0; n < spp; ++n) {
      out_2d[(size_t)2 * spp * i + 2 * n + 0] = rd_value(kAlpha2x, base + (uint64_t)n + 1);
      out_2d[(size_t)2 * spp * i + 2 * n + 1] = rd_value(kAlpha2y, base + (uint64_t)n + 1);
    }
  }
  return RAYN_OK;
}

int32_t rayn_b200_host_scramble(int32_t width, int32_t height, float* out) {
  if (width <= 0 || height <= 0 || !out) return RAYN_ERR_INVALID_ARG;
  for (int y = 0; y < height; ++y)
    for (int x = 0; x < width; ++x)
      out[(size_t)x + (size_t)y * width] = small_rng_first_f32((uint64_t)((uint32_t)x + (uint32_t)y * (uint32_t)width));
  return RAYN_OK;
}

int32_t rayn_b200_host_fis_blackman_harris(float radius, float* out512) {
  if (!out512 || !(radius > 0.0f)) return RAYN_ERR_INVALID_ARG;
  const int N = RAYN_FIS_TABLE_SIZE;
  std::vector<float> item(N), weight(N), density(N);
  float weight_sum = 0.0f;
  for (int n = 0; n < N; ++n) {
    float t = (float)n / (float)(N - 1);
    float d = 0.0f * (1.0f - t) + radius * t;  // 0.0.lerp(f_rad, t)
    item[n] = d;
    weight[n] = blackman_harris(radius, d);
    weight_sum += weight[n];
  }
  for (int n = 0; n < N; ++n) weight[n] /= weight_sum;
  float cum = 0.0f;
  for (int n = 0; n < N; ++n) {
    cum += weight[n];
    density[n] = cum;
  }
  for (int n = N - 1; n >= 0; --n) {
    density[n] = 1.0f;
    if (weight[n] > 0.0f) break;
  }
  for (int n = 0; n < N; ++n) {
    float u = (float)n / (float)(N - 1);
    float v = item[N - 1];
    for (int k = 0; k < N; ++k)
      if (density[k] >= u) {
        v = item[k];
        break;
      }
    out512[n] = v;
  }
  return RAYN_OK;
}

int32_t rayn_b200_host_tile_grid(int32_t width, int32_t height, int32_t tile_w, int32_t tile_h, int32_t* n_tiles_x,
                                 int32_t* n_tiles_y) {
  if (width <= 0 || height <= 0 || tile_w <= 0 || tile_h <= 0) return RAYN_ERR_INVALID_ARG;
  // film.rs:399-404: (res + res % tile) / tile
  if (n_tiles_x) *n_tiles_x = (width + width % tile_w) / tile_w;
  if (n_tiles_y) *n_tiles_y = (height + height % tile_h) / tile_h;
  return RAYN_OK;
}

}  // extern "C"
