// albedo_oracle.cpp — CPU mirror of the first-hit albedo plane (include/rayn_b200.h, rayn_b200_render_albedo).  TEST
// INFRASTRUCTURE ONLY: built by tests/albedo_oracle.py; nothing under rayn_b200/ may include, link or execute it.
//
// It includes tests/trap_oracle.cpp (and through it oracle/rayn_oracle.cpp) unchanged and calls the oracle's own
// sample_uv, camera_get_rays and closest_hit; it restates only the raygen loop of render_tile (film.rs:456-529) and the
// depth-0 fold threshold (film.rs:540-551), then applies the albedo rule of the header to every camera sample.
// Build flags: those of oracle/Makefile (-ffp-contract=off is required, see there).
#include "trap_oracle.cpp"

namespace {

// per-sample albedos of one tile: a[((fy * W + fx) * spp + s) * 3 + c] for the tile's pixels, sample s, channel c
void albedo_tile(const World& w, const TrapTable& traps, const RaynFrameDesc& f, int tile_x, int tile_y, float* a) {
  const int W = f.width, H = f.height;
  const uint32_t x0 = tile_x * f.tile_w, y0 = tile_y * f.tile_h;
  const uint32_t x1 = (uint32_t)((int)(x0 + f.tile_w) < W ? x0 + f.tile_w : W);
  const uint32_t y1 = (uint32_t)((int)(y0 + f.tile_h) < H ? y0 + f.tile_h : H);
  const int samples = f.samples, spp = 4 * samples;
  const float ndc_x = 1.0f / (float)W, ndc_y = 1.0f / (float)H;
  Tables tab{spp, f.samples_1d, f.samples_2d};
  const F4 time_range = splat(f.t1 - f.t0);
  const Thr thr{0, &w.s->camera};
  int64_t evals = 0;
  for (uint32_t x = x0; x < x1; ++x)
    for (uint32_t y = y0; y < y1; ++y) {
      float scramble = f.scramble[x + y * (uint32_t)W];
      for (int samp = 0; samp < samples; ++samp) {  // film.rs:456-464: one 4-lane camera packet per iteration
        uint32_t nums[4] = {4u * samp, 4u * samp + 1, 4u * samp + 2, 4u * samp + 3};
        float us[4], vs[4];
        for (int i = 0; i < 4; ++i)
          sample_uv(x, y, ndc_x, ndc_y, f.fis_inverse_cdf, tab.s2(0, nums[i], scramble, 0), tab.s2(1, nums[i], scramble, 0), &us[i], &vs[i]);
        float sc4[4] = {scramble, scramble, scramble, scramble};
        F4 times = splat(f.t0) + time_range * tab.w1(nums, sc4, 0);
        F4 ls0 = tab.w2(0, nums, sc4, 1), ls1 = tab.w2(1, nums, sc4, 1);
        const WRay wray = camera_get_rays(w.s->camera, scramble, nums, x - x0, y - y0, load4(us), load4(vs), times, ls0, ls1);
        int ids[4];
        F4 dists;
        closest_hit(w, wray, splat(w.s->consts.world_radius * 2.0f), thr, ids, &dists, &evals);  // the depth-0 packet
        const V3 point = point_at(wray, dists);
        for (int i = 0; i < 4; ++i) {
          float* out = a + (((size_t)y * W + x) * spp + nums[i]) * 3;
          out[0] = out[1] = out[2] = 0.0f;  // Sky / Emissive hit or nothing hit
          if (ids[i] < 0) continue;
          const RaynHitable& h = w.s->hitables[ids[i]];
          const RaynMaterial& m = w.s->materials[h.material];
          if (m.kind != RAYN_MATERIAL_LAMBERTIAN && m.kind != RAYN_MATERIAL_DIELECTRIC) continue;
          const RaynAlbedoTrap* tp = traps[h.material];
          if (!tp) {
            out[0] = m.albedo[0], out[1] = m.albedo[1], out[2] = m.albedo[2];
            continue;
          }
          const F4 s = h.kind == RAYN_HITABLE_SPHERE ? splat(1.0f) : trap_coord(*tp, sdf_trap(h, point));
          const V3 alb = trap_albedo(*tp, s);
          out[0] = alb.x[i], out[1] = alb.y[i], out[2] = alb.z[i];
        }
      }
    }
}

}  // namespace

extern "C" {

// Per-sample albedos a_s (float [W*H*spp*3], pixel-major, samples ascending) and the plane (float [3*W*H]) of the whole tile
// grid; pixels outside the grid are 0 in both.  frame's tile selection is ignored, as in rayn_b200_render_albedo; subsample_k > 1
// computes only the tiles whose index is a multiple of k (for spot checks of large films), the others stay 0.
int32_t rayn_albedo_oracle_render(const RaynSceneDesc* scene, int32_t n_traps, const RaynAlbedoTrap* traps, const RaynFrameDesc* f,
                                  float* per_sample, float* albedo, int32_t n_threads, int32_t subsample_k) {
  if (!scene || !f || !per_sample || !albedo || n_traps < 0 || (n_traps > 0 && !traps)) return RAYN_ERR_INVALID_ARG;
  TrapTable table = {};
  for (int i = 0; i < n_traps; ++i) {
    if (traps[i].material < 0 || traps[i].material >= scene->n_materials) return RAYN_ERR_INVALID_ARG;
    table[traps[i].material] = &traps[i];
  }
  if (!fp_contract_is_off()) return RAYN_ERR_UNSUPPORTED;
  World w{scene};
  const int W = f->width, H = f->height, spp = 4 * f->samples;
  const int ntx = (W + W % f->tile_w) / f->tile_w, nty = (H + H % f->tile_h) / f->tile_h;  // film.rs:399-404
  memset(per_sample, 0, sizeof(float) * (size_t)W * H * spp * 3);
  memset(albedo, 0, sizeof(float) * (size_t)W * H * 3);
#ifdef _OPENMP
  if (n_threads > 0) omp_set_num_threads(n_threads);
#endif
#pragma omp parallel for schedule(dynamic, 1)
  for (int idx = 0; idx < ntx * nty; ++idx) {
    const int tx = idx / nty, ty = idx % nty;
    if (tx * f->tile_w >= W || ty * f->tile_h >= H || (subsample_k > 1 && idx % subsample_k != 0)) continue;
    albedo_tile(w, table, *f, tx, ty, per_sample);
    const int xe = std::min((tx + 1) * f->tile_w, W), ye = std::min((ty + 1) * f->tile_h, H);
    for (int x = tx * f->tile_w; x < xe; ++x)
      for (int y = ty * f->tile_h; y < ye; ++y)
        for (int c = 0; c < 3; ++c) {
          float acc = 0.0f;
          for (int s = 0; s < spp; ++s) acc += per_sample[(((size_t)y * W + x) * spp + s) * 3 + c];
          albedo[3 * ((size_t)y * W + x) + c] = acc / (float)spp;
        }
  }
  return RAYN_OK;
}

}  // extern "C"
