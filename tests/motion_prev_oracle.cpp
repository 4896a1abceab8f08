// motion_prev_oracle.cpp — CPU mirror of the motion plane against an explicit previous scene (include/rayn_b200.h,
// rayn_b200_render_motion_prev).  TEST INFRASTRUCTURE ONLY: built by tests/motion_prev_oracle.py; nothing under rayn_b200/ may
// include, link or execute it.
//
// It includes tests/motion_oracle.cpp (and through it tests/trap_oracle.cpp and oracle/rayn_oracle.cpp) unchanged and uses its
// `project`, the header's proj(X, time).  Like that mirror it restates only the raygen loop of render_tile (film.rs:456-529) and
// the depth-0 fold threshold, and calls the oracle's own sample_uv, camera_get_rays and closest_hit; both sphere centres are the
// oracle's seq_v3, which is how its sphere_hit forms a centre.
// Build flags: those of oracle/Makefile (-ffp-contract=off is required, see there).
#include "motion_oracle.cpp"

namespace {

bool moving(const RaynHitable& h) { return h.center_velocity[0] != 0.0f || h.center_velocity[1] != 0.0f || h.center_velocity[2] != 0.0f; }

// per-sample records of one tile against `prev`: rec[((y * W + x) * spp + s) * 4 + k]; geo as motion_tile's
void motion_prev_tile(const World& w, const RaynFrameDesc& f, float frame_dt, const RaynSceneDesc& prev, int tile_x, int tile_y, float* rec,
                      float* geo) {
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
        const float tau = times[0], tp = tau - frame_dt;
        // P' per lane: P + (c_prev(tp) - c(tau)) on a sphere that moved or moves, P itself otherwise
        alignas(16) float ppx[4], ppy[4], ppz[4];
        store4(ppx, P.x), store4(ppy, P.y), store4(ppz, P.z);
        for (int i = 0; i < 4; ++i) {
          if (ids[i] < 0) continue;
          const RaynHitable &h = w.s->hitables[ids[i]], &hp = prev.hitables[ids[i]];
          if (h.kind != RAYN_HITABLE_SPHERE || (!moving(hp) && !moving(h) && memcmp(hp.center, h.center, sizeof h.center) == 0)) continue;
          const V3 cp = seq_v3(hp.center, hp.center_velocity, splat(tp)), c = seq_v3(h.center, h.center_velocity, splat(tau));
          const float dcx = cp.x[0] - c.x[0], dcy = cp.y[0] - c.y[0], dcz = cp.z[0] - c.z[0];
          ppx[i] = ppx[i] + dcx, ppy[i] = ppy[i] + dcy, ppz[i] = ppz[i] + dcz;
        }
        const V3 Pp = V3{load4(ppx), load4(ppy), load4(ppz)};
        F4 px1, py1, z1, px0, py0, z0;
        project(cam, W, H, P, tau, &px1, &py1, &z1);
        project(prev.camera, W, H, Pp, tp, &px0, &py0, &z0);
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

// rayn_motion_oracle_render's outputs with rayn_b200_render_motion_prev's statement.  prev must match the scene (hitable count
// and kinds, camera kind), as the product call requires; RAYN_ERR_INVALID_ARG otherwise.
int32_t rayn_motion_prev_oracle_render(const RaynSceneDesc* scene, const RaynFrameDesc* f, float frame_dt, const RaynSceneDesc* prev,
                                       float* per_sample, float* motion, int32_t n_threads, int32_t subsample_k, float* geo) {
  if (!scene || !f || !per_sample || !motion) return RAYN_ERR_INVALID_ARG;
  if (!prev || !prev->hitables || prev->n_hitables != scene->n_hitables || prev->camera.kind != scene->camera.kind) return RAYN_ERR_INVALID_ARG;
  for (int j = 0; j < scene->n_hitables; ++j)
    if (prev->hitables[j].kind != scene->hitables[j].kind) return RAYN_ERR_INVALID_ARG;
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
    motion_prev_tile(w, *f, frame_dt, *prev, tx, ty, per_sample, geo);
    const int xe = std::min((tx + 1) * f->tile_w, W), ye = std::min((ty + 1) * f->tile_h, H);
    for (int x = tx * f->tile_w; x < xe; ++x)
      for (int y = ty * f->tile_h; y < ye; ++y) {  // k_motion_resolve: the mean over valid samples in sample order
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
