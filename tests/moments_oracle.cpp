// moments_oracle.cpp — CPU mirror of rayn_b200_render_frame_moments (the statement is in include/rayn_b200.h).  TEST
// INFRASTRUCTURE ONLY, built by tests/moments_oracle.py with the flags of oracle/Makefile (-ffp-contract=off is required).
// It includes tests/trap_oracle.cpp (and through it oracle/rayn_oracle.cpp) unchanged, so scenes with orbit traps render as
// there, and adds the lum^2 fold to the tile loop.
#include "trap_oracle.cpp"

namespace {

// lum(v) of the header: every product rounded on its own (no contraction)
inline float lum(const float* v) { return (0.2126f * v[0] + 0.7152f * v[1]) + 0.0722f * v[2]; }

// render_tile_traps() of tests/trap_oracle.cpp (the oracle's render_tile() with trap packets integrated per lane) with the
// lum^2 fold added to the CH_COLOR / CH_BACKGROUND cases of the new_samples loop: the same samples in the same order as the
// colour sums.  lum2_color / lum2_bg may be NULL.
void render_tile_moments(const World& w, const TrapTable& traps, const RaynFrameDesc& f, int tile_x, int tile_y, float* color,
                         float* alpha, float* background, float* normal, float* lum2_color, float* lum2_bg, Counters& cnt) {
  const int W = f.width, H = f.height;
  const uint32_t x0 = tile_x * f.tile_w, y0 = tile_y * f.tile_h;
  const uint32_t x1 = (uint32_t)((int)(x0 + f.tile_w) < W ? x0 + f.tile_w : W);
  const uint32_t y1 = (uint32_t)((int)(y0 + f.tile_h) < H ? y0 + f.tile_h : H);
  const uint32_t tw = x1 - x0, th = y1 - y0;
  const int samples = f.samples, spp = 4 * samples, vm = f.volume_marches;
  const float ndc_x = 1.0f / (float)W, ndc_y = 1.0f / (float)H;
  Tables tab{spp, f.samples_1d, f.samples_2d};
  std::vector<float> tc(3 * tw * th, 0.0f), ta(tw * th, 0.0f), tb(3 * tw * th, 0.0f), tn(3 * tw * th, 0.0f);
  std::vector<float> tmc(tw * th, 0.0f), tmb(tw * th, 0.0f);

  std::vector<WRay> spawned_wrays;
  std::vector<Ray> spawned_rays;
  std::vector<OutSample> new_samples;
  std::vector<std::vector<Hit>> bins(w.n_hit());
  const F4 time_range = splat(f.t1 - f.t0);

  for (uint32_t x = x0; x < x1; ++x)
    for (uint32_t y = y0; y < y1; ++y) {
      float scramble = f.scramble[x + y * (uint32_t)W];
      for (int samp = 0; samp < samples; ++samp) {
        uint32_t nums[4] = {4u * samp, 4u * samp + 1, 4u * samp + 2, 4u * samp + 3};
        float us[4], vs[4];
        for (int i = 0; i < 4; ++i)
          sample_uv(x, y, ndc_x, ndc_y, f.fis_inverse_cdf, tab.s2(0, nums[i], scramble, 0),
                    tab.s2(1, nums[i], scramble, 0), &us[i], &vs[i]);
        float sc4[4] = {scramble, scramble, scramble, scramble};
        F4 times = splat(f.t0) + time_range * tab.w1(nums, sc4, 0);
        F4 ls0 = tab.w2(0, nums, sc4, 1), ls1 = tab.w2(1, nums, sc4, 1);
        spawned_wrays.push_back(camera_get_rays(w.s->camera, scramble, nums, x - x0, y - y0, load4(us), load4(vs),
                                                times, ls0, ls1));
      }
    }

  for (int depth = 0;; ++depth) {
    if (spawned_wrays.empty()) break;
    for (auto& b : bins) b.clear();
    Thr thr{depth, &w.s->camera};
    for (const WRay& wray : spawned_wrays) {  // add_hits, hitable.rs:170-210
      int ids[4];
      F4 dists;
      closest_hit(w, wray, splat(w.s->consts.world_radius * 2.0f), thr, ids, &dists, &cnt.sdf_evals_extend);
      Ray rays[4];
      wray_into(wray, rays);
      for (int i = 0; i < 4; ++i) {
        if (rays[i].valid) cnt.extend_rays++;
        if (ids[i] >= 0 && rays[i].valid) bins[ids[i]].push_back({rays[i], dists[i]});
      }
    }
    spawned_wrays.clear();
    // process_hits, hitable.rs:94-133: pad every bin to x4 with invalid hits (t = 0)
    for (auto& b : bins)
      while (b.size() % 4 != 0) b.push_back({Ray::invalid(), 0.0f});
    for (int obj = 0; obj < w.n_hit(); ++obj) {
      const RaynHitable& h = w.s->hitables[obj];
      for (size_t k = 0; k + 4 <= bins[obj].size(); k += 4) {
        Ray r4[4] = {bins[obj][k].ray, bins[obj][k + 1].ray, bins[obj][k + 2].ray, bins[obj][k + 3].ray};
        WHit hit{wray_from(r4), make4(bins[obj][k].t, bins[obj][k + 1].t, bins[obj][k + 2].t, bins[obj][k + 3].t)};
        ShadingPoint sp = h.kind == RAYN_HITABLE_SPHERE ? sphere_shading_info(h, hit)
                                                        : sdf_shading_info(h, w.s->consts, hit, thr);
        // film.rs:565-589
        F4 s1d[5], s2d[28];
        const int n1 = 3 + vm, n2 = 12 + 8 * vm;
        for (int set = 0; set < n1; ++set) s1d[set] = tab.w1(sp.ray.sample, sp.ray.scramble, 1 + set + depth * n1);
        for (int i = 0; i < n2; ++i)
          s2d[i] = tab.w2(i % 2, sp.ray.sample, sp.ray.scramble, 2 + i / 2 + depth * n2 / 2);
        const RaynAlbedoTrap* tp = traps[h.material];
        if (!tp) {
          integrate(w, f.max_bounces, vm, s1d, s2d, depth, h.material, sp, spawned_rays, new_samples, cnt);
        } else {  // the albedo generator at this hit: the orbit trap at the shading point, s = 1 on an analytic sphere
          const F4 s = h.kind == RAYN_HITABLE_SPHERE ? splat(1.0f) : trap_coord(*tp, sdf_trap(h, sp.point));
          integrate_per_lane_albedo(w, f.max_bounces, vm, s1d, s2d, depth, h.material, trap_albedo(*tp, s), sp, spawned_rays,
                                    new_samples, cnt);
        }
      }
    }
    for (const OutSample& s : new_samples) {  // film.rs:604-606, :167-172
      size_t idx = s.tx + s.ty * tw;
      switch (s.channel) {
        case CH_COLOR:
          for (int k = 0; k < 3; ++k) tc[3 * idx + k] += s.v[k];
          tmc[idx] += lum(s.v) * lum(s.v);
          break;
        case CH_ALPHA:
          ta[idx] += s.v[0];
          break;
        case CH_BACKGROUND:
          for (int k = 0; k < 3; ++k) tb[3 * idx + k] += s.v[k];
          tmb[idx] += lum(s.v) * lum(s.v);
          break;
        case CH_NORMAL:
          for (int k = 0; k < 3; ++k) tn[3 * idx + k] += s.v[k];
          break;
      }
    }
    new_samples.clear();
    while (spawned_rays.size() % 4 != 0) spawned_rays.push_back(Ray::invalid());  // film.rs:608-610
    for (size_t k = 0; k + 4 <= spawned_rays.size(); k += 4) spawned_wrays.push_back(wray_from(&spawned_rays[k]));
    spawned_rays.clear();
  }
  // tile_finished / copy_from_tile, film.rs:82-98
  const float div = (float)spp;
  for (uint32_t x = 0; x < tw; ++x)
    for (uint32_t y = 0; y < th; ++y) {
      size_t ti = x + y * tw;
      size_t fi = (x0 + x) + (size_t)(y0 + y) * W;
      for (int k = 0; k < 3; ++k) {
        color[3 * fi + k] = tc[3 * ti + k] / div;
        background[3 * fi + k] = tb[3 * ti + k] / div;
        normal[3 * fi + k] = tn[3 * ti + k] / div;
      }
      alpha[fi] = ta[ti] / div;
      if (lum2_color) lum2_color[fi] = tmc[ti] / div;
      if (lum2_bg) lum2_bg[fi] = tmb[ti] / div;
    }
}

}  // namespace

extern "C" {

// rayn_trap_oracle_render_frame (same tile selection, trap list and return codes) with the moment planes; host pointers,
// untouched pixels keep their previous contents
int32_t rayn_moments_oracle_render_frame(const RaynSceneDesc* scene, int32_t n_traps, const RaynAlbedoTrap* traps, const RaynFrameDesc* f,
                                         const RaynFilmPlanes* out, float* lum2_color, float* lum2_bg, int32_t n_threads, int32_t subsample_k) {
  if (!scene || !f || !out || n_traps < 0 || (n_traps > 0 && !traps)) return RAYN_ERR_INVALID_ARG;
  TrapTable table = {};
  for (int i = 0; i < n_traps; ++i) {
    if (traps[i].material < 0 || traps[i].material >= scene->n_materials) return RAYN_ERR_INVALID_ARG;
    table[traps[i].material] = &traps[i];
  }
  if (f->volume_marches != 2) return RAYN_ERR_UNSUPPORTED;
  if (!fp_contract_is_off()) return RAYN_ERR_UNSUPPORTED;
  World w{scene};
  int ntx = (f->width + f->width % f->tile_w) / f->tile_w;  // film.rs:399-404
  int nty = (f->height + f->height % f->tile_h) / f->tile_h;
  int stride = f->tile_stride > 0 ? f->tile_stride : 1;
  if (subsample_k < 1) subsample_k = 1;
  std::vector<int> todo;
  if (f->tile_list) {
    for (int i = 0; i < f->n_tile_list; ++i)
      if (f->tile_list[i] >= 0 && f->tile_list[i] < ntx * nty) todo.push_back(f->tile_list[i]);
  } else {
    for (int idx = 0; idx < ntx * nty; ++idx)
      if (idx % stride == f->tile_offset && ((idx / stride) % subsample_k) == 0) todo.push_back(idx);
  }
#ifdef _OPENMP
  if (n_threads > 0) omp_set_num_threads(n_threads);
#endif
#pragma omp parallel
  {
    Counters local;
#pragma omp for schedule(dynamic, 1)
    for (size_t k = 0; k < todo.size(); ++k) {
      int idx = todo[k];
      int tx = idx / nty, ty = idx % nty;
      if (tx * f->tile_w >= f->width || ty * f->tile_h >= f->height) continue;
      render_tile_moments(w, table, *f, tx, ty, out->color, out->alpha, out->background, out->normal, lum2_color, lum2_bg, local);
    }
  }
  return g_lane_split_failed.exchange(0) ? RAYN_ERR_UNSUPPORTED : RAYN_OK;
}

}  // extern "C"
