// motion_oracle.cpp — CPU mirror of the first-hit motion plane (include/rayn_b200.h, rayn_b200_render_motion).  TEST
// INFRASTRUCTURE ONLY: built by tests/temporal_oracle.py; nothing under rayn_b200/ may include, link or execute it.
//
// Like tests/albedo_oracle.cpp it includes tests/trap_oracle.cpp (and through it oracle/rayn_oracle.cpp) unchanged, calls the
// oracle's own sample_uv, camera_get_rays and closest_hit, and restates only the raygen loop of render_tile (film.rs:456-529)
// and the depth-0 fold threshold.  The projection of the header is written with the oracle's 4-lane Wec3 arithmetic.
// Build flags: those of oracle/Makefile (-ffp-contract=off is required, see there).
#include "trap_oracle.cpp"

namespace {

// proj(X, time) of the header, per lane
void project(const RaynCamera& c, int W, int H, V3 X, float time, F4* px, F4* py, F4* z) {
  const F4 t = splat(time);
  const V3 origin = seq_v3(c.origin, c.origin_velocity, t), at = seq_v3(c.at, c.at_velocity, t), up = seq_v3(c.up, c.up_velocity, t);
  const F4 hx = splat(c.half_size[0]), hy = splat(c.half_size[1]);
  const V3 r = X - origin;
  if (c.kind == RAYN_CAMERA_ORTHOGRAPHIC) {
    const V3 bw = normalized(at - origin);
    const V3 bu = normalized(cross(bw, up));
    const V3 bv = cross(bu, bw);
    *z = dot(r, bw);
    *px = ((dot(r, bu) + hx) / splat(c.full_size[0])) * splat((float)W);
    *py = ((dot(r, bv) + hy) / splat(c.full_size[1])) * splat((float)H);
  } else {
    const V3 bw = normalized(origin - at);
    const V3 bu = normalized(cross(up, bw));
    const V3 bv = cross(bw, bu);
    const F4 zz = -dot(r, bw);
    *z = zz;
    *px = ((dot(r, bu) / (zz * hx)) * splat(0.5f) + splat(0.5f)) * splat((float)W);
    *py = ((dot(r, bv) / (zz * hy)) * splat(0.5f) + splat(0.5f)) * splat((float)H);
  }
}

// per-sample records of one tile: rec[((y * W + x) * spp + s) * 4 + k]
// geo (optional): per sample (P.x, P.y, P.z, tau, u, v) for the float64 checks of tests/test_cpu_temporal.py
void motion_tile(const World& w, const RaynFrameDesc& f, float frame_dt, int tile_x, int tile_y, float* rec, float* geo) {
  const int W = f.width, H = f.height;
  const uint32_t x0 = tile_x * f.tile_w, y0 = tile_y * f.tile_h;
  const uint32_t x1 = (uint32_t)((int)(x0 + f.tile_w) < W ? x0 + f.tile_w : W);
  const uint32_t y1 = (uint32_t)((int)(y0 + f.tile_h) < H ? y0 + f.tile_h : H);
  const int samples = f.samples, spp = 4 * samples;
  const float ndc_x = 1.0f / (float)W, ndc_y = 1.0f / (float)H;
  Tables tab{spp, f.samples_1d, f.samples_2d};
  const F4 time_range = splat(f.t1 - f.t0);
  const Thr thr{0, &w.s->camera};
  const RaynCamera& cam = w.s->camera;
  int64_t evals = 0;
  for (uint32_t x = x0; x < x1; ++x)
    for (uint32_t y = y0; y < y1; ++y) {
      float scramble = f.scramble[x + y * (uint32_t)W];
      for (int samp = 0; samp < samples; ++samp) {
        uint32_t nums[4] = {4u * samp, 4u * samp + 1, 4u * samp + 2, 4u * samp + 3};
        float us[4], vs[4];
        for (int i = 0; i < 4; ++i)
          sample_uv(x, y, ndc_x, ndc_y, f.fis_inverse_cdf, tab.s2(0, nums[i], scramble, 0), tab.s2(1, nums[i], scramble, 0), &us[i], &vs[i]);
        float sc4[4] = {scramble, scramble, scramble, scramble};
        F4 times = splat(f.t0) + time_range * tab.w1(nums, sc4, 0);
        F4 ls0 = tab.w2(0, nums, sc4, 1), ls1 = tab.w2(1, nums, sc4, 1);
        const WRay wray = camera_get_rays(cam, scramble, nums, x - x0, y - y0, load4(us), load4(vs), times, ls0, ls1);
        int ids[4];
        F4 dists;
        closest_hit(w, wray, splat(w.s->consts.world_radius * 2.0f), thr, ids, &dists, &evals);
        const V3 P = point_at(wray, dists);
        const float tau = times[0];
        const F4 dt = splat(frame_dt);
        float vx[4] = {0, 0, 0, 0}, vy[4] = {0, 0, 0, 0}, vz[4] = {0, 0, 0, 0};
        bool moves[4] = {false, false, false, false};
        for (int i = 0; i < 4; ++i) {
          if (ids[i] < 0) continue;
          const RaynHitable& h = w.s->hitables[ids[i]];
          if (h.kind == RAYN_HITABLE_SPHERE && (h.center_velocity[0] != 0.0f || h.center_velocity[1] != 0.0f || h.center_velocity[2] != 0.0f)) {
            moves[i] = true;
            vx[i] = h.center_velocity[0], vy[i] = h.center_velocity[1], vz[i] = h.center_velocity[2];
          }
        }
        const V3 moved = P - V3{load4(vx) * dt, load4(vy) * dt, load4(vz) * dt};
        F4 px1, py1, z1, px0, py0, z0;
        project(cam, W, H, P, tau, &px1, &py1, &z1);
        // P' per lane: the moved point for moving spheres, P itself otherwise
        alignas(16) float pmx[4], pmy[4], pmz[4], ppx[4], ppy[4], ppz[4];
        store4(pmx, moved.x), store4(pmy, moved.y), store4(pmz, moved.z);
        store4(ppx, P.x), store4(ppy, P.y), store4(ppz, P.z);
        for (int i = 0; i < 4; ++i)
          if (moves[i]) ppx[i] = pmx[i], ppy[i] = pmy[i], ppz[i] = pmz[i];
        const V3 Pp = V3{load4(ppx), load4(ppy), load4(ppz)};
        project(cam, W, H, Pp, tau - frame_dt, &px0, &py0, &z0);
        for (int i = 0; i < 4; ++i) {
          float* out = rec + (((size_t)y * W + x) * spp + nums[i]) * 4;
          if (geo) {
            float* g = geo + (((size_t)y * W + x) * spp + nums[i]) * 6;
            g[0] = P.x[i], g[1] = P.y[i], g[2] = P.z[i], g[3] = tau, g[4] = us[i], g[5] = vs[i];
          }
          const bool valid = ids[i] >= 0 && (cam.kind == RAYN_CAMERA_ORTHOGRAPHIC || (z1[i] > 0.0f && z0[i] > 0.0f));
          if (valid) {
            out[0] = px0[i] - px1[i], out[1] = py0[i] - py1[i], out[2] = z1[i], out[3] = z0[i];
          } else {
            out[0] = 0.0f, out[1] = 0.0f, out[2] = NAN, out[3] = NAN;
          }
        }
      }
    }
}

}  // namespace

extern "C" {

// Per-sample records (float [W*H*spp*4], pixel-major, samples ascending) and the plane (float [4*W*H]) of the whole tile grid;
// pixels outside the grid have records (0, 0, NaN, NaN) and motion (0, 0, +inf, +inf).  subsample_k > 1 computes only the tiles
// whose index is a multiple of k (spot checks of large films); the other pixels stay as outside the grid.
// geo (may be NULL): float [W*H*spp*6], per sample the hit point, the camera time and the film coordinates (u, v) of its ray.
int32_t rayn_motion_oracle_render(const RaynSceneDesc* scene, const RaynFrameDesc* f, float frame_dt, float* per_sample, float* motion,
                                  int32_t n_threads, int32_t subsample_k, float* geo) {
  if (!scene || !f || !per_sample || !motion) return RAYN_ERR_INVALID_ARG;
  if (!fp_contract_is_off()) return RAYN_ERR_UNSUPPORTED;
  World w{scene};
  const int W = f->width, H = f->height, spp = 4 * f->samples;
  const int ntx = (W + W % f->tile_w) / f->tile_w, nty = (H + H % f->tile_h) / f->tile_h;  // film.rs:399-404
  for (size_t i = 0; i < (size_t)W * H * spp; ++i)
    per_sample[4 * i] = 0.0f, per_sample[4 * i + 1] = 0.0f, per_sample[4 * i + 2] = NAN, per_sample[4 * i + 3] = NAN;
  for (size_t i = 0; i < (size_t)W * H; ++i) motion[4 * i] = 0.0f, motion[4 * i + 1] = 0.0f, motion[4 * i + 2] = INFINITY, motion[4 * i + 3] = INFINITY;
#ifdef _OPENMP
  if (n_threads > 0) omp_set_num_threads(n_threads);
#endif
#pragma omp parallel for schedule(dynamic, 1)
  for (int idx = 0; idx < ntx * nty; ++idx) {
    const int tx = idx / nty, ty = idx % nty;
    if (tx * f->tile_w >= W || ty * f->tile_h >= H || (subsample_k > 1 && idx % subsample_k != 0)) continue;
    motion_tile(w, *f, frame_dt, tx, ty, per_sample, geo);
    const int xe = std::min((tx + 1) * f->tile_w, W), ye = std::min((ty + 1) * f->tile_h, H);
    for (int x = tx * f->tile_w; x < xe; ++x)
      for (int y = ty * f->tile_h; y < ye; ++y) {
        float acc[4] = {0.0f, 0.0f, 0.0f, 0.0f};
        int n = 0;
        for (int s = 0; s < spp; ++s) {
          const float* r = per_sample + (((size_t)y * W + x) * spp + s) * 4;
          if (r[2] != r[2]) continue;
          for (int k = 0; k < 4; ++k) acc[k] += r[k];
          ++n;
        }
        float* m = motion + 4 * ((size_t)y * W + x);
        if (n == 0) {
          m[0] = 0.0f, m[1] = 0.0f, m[2] = INFINITY, m[3] = INFINITY;
        } else {
          for (int k = 0; k < 4; ++k) m[k] = acc[k] / (float)n;
        }
      }
  }
  return RAYN_OK;
}

}  // extern "C"
