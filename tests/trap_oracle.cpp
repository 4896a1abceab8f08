// trap_oracle.cpp — CPU oracle of the orbit-trap albedo (include/rayn_b200.h, RaynAlbedoTrap).  TEST INFRASTRUCTURE ONLY:
// built by tests/trap_oracle.py; nothing under rayn_b200/ may include, link or execute it.
//
// It extends the render oracle without changing it: oracle/rayn_oracle.cpp is included as it is, and this file adds
//   sdf_trap()        the trap on 4-lane packets, the same iterations as mandelbox_dist() / mandelbulb_dist() with a min fold;
//   trap_coord(), trap_albedo()   the palette;
//   integrate_per_lane_albedo()   integrate() (integrator.rs:47-205) with a per-lane albedo, from four runs of the
//                     oracle's own integrate() on a private copy of the material (see the function);
//   render_tile_traps()   render_tile() (film.rs:439-627) with one change: a packet whose material has a trap is integrated
//                     with integrate_per_lane_albedo().  (No queue log: the packet order is the oracle's, tested there.)
// Build flags: those of oracle/Makefile (-ffp-contract=off is required, see there).
#include "../oracle/rayn_oracle.cpp"

#include <array>
#include <atomic>

namespace {

using TrapTable = std::array<const RaynAlbedoTrap*, RAYN_MAX_MATERIALS>;  // trap of material m, or NULL
std::atomic<int> g_lane_split_failed{0};  // set if the four runs of integrate_per_lane_albedo ever disagree in shape

// Orbit trap per lane: the iterations of mandelbox_dist / mandelbulb_dist folding trap = (x < trap) ? x : trap, which is
// minps(x, trap) (a NaN x never replaces it).  Mandelbox: x = r2 of every iteration; Mandelbulb: every m a lane assigns, from
// the start value through its last iteration before bailout (escaped lanes keep their trap like their state).
inline F4 sdf_trap(const RaynHitable& h, V3 p) {
  F4 trap = splat(INFINITY);
  if (h.iterations <= 0) return trap;
  if (h.kind == RAYN_HITABLE_MANDELBULB) {
    V3 w = p;
    F4 dr = splat(1.0f);
    F4 m = dot(w, w);
    trap = f4min(m, trap);
    F4 bail2 = splat(h.bulb_bailout * h.bulb_bailout);
    F4 one = splat(1.0f);
    for (int i = 0; i < h.iterations; ++i) {
      F4 esc = cmp_gt(m, bail2);
      if (move_mask(esc) == 0xf) break;
      F4 m2 = m * m, m3 = m2 * m;
      F4 r = f4sqrt(m);
      F4 r7 = m3 * r;
      F4 ndr = fma4(splat(8.0f) * r7, dr, one);
      F4 a = w.z * w.z, b = m;
      F4 b2 = b * b, b3 = b2 * b, b4 = b2 * b2;
      F4 P = fma4(fma4(fma4(fma4(splat(128.0f), a, splat(-256.0f) * b), a, splat(160.0f) * b2), a, splat(-32.0f) * b3), a, b4);
      F4 A = fma4(fma4(fma4(splat(128.0f), a, splat(-192.0f) * b), a, splat(80.0f) * b2), a, splat(-8.0f) * b3);
      F4 ax = w.x * w.x;
      F4 q = fma4(w.x, w.x, w.y * w.y);
      F4 q2 = q * q, q3 = q2 * q, q4 = q2 * q2;
      F4 C = fma4(fma4(fma4(fma4(splat(128.0f), ax, splat(-256.0f) * q), ax, splat(160.0f) * q2), ax, splat(-32.0f) * q3), ax, q4);
      F4 B = fma4(fma4(fma4(splat(128.0f), ax, splat(-192.0f) * q), ax, splat(80.0f) * q2), ax, splat(-8.0f) * q3);
      F4 k = (w.z * A) / (q3 * f4sqrt(q));
      k = merge(cmp_gt(q, splat(0.0f)), k, splat(0.0f));
      V3 nw = {fma4(k, C, p.x), fma4(k, w.x * w.y * B, p.y), P + p.z};
      F4 nm = dot(nw, nw);
      w = v3merge(esc, w, nw);
      dr = merge(esc, dr, ndr);
      m = merge(esc, m, nm);
      trap = merge(esc, trap, f4min(nm, trap));
    }
    return trap;
  }
  V3 offset = p;
  F4 one = splat(1.0f);
  F4 dr = one;
  V3 l = v3broadcast(splat(h.box_l));
  V3 neg_l = -l;
  V3 two = v3broadcast(splat(2.0f));
  F4 scale = splat(h.scale);
  V3 scale_vec = v3broadcast(scale);
  F4 min_rad_sq = splat(h.min_rad_sq), fixed_rad_sq = splat(h.fixed_rad_sq);
  for (int i = 0; i < h.iterations; ++i) {
    p = v3mul_add(v3clamped(p, neg_l, l), two, -p);
    F4 r2 = mag_sq(p);
    trap = f4min(r2, trap);
    F4 mul = f4max(one, fixed_rad_sq / f4max(min_rad_sq, r2));
    p = p * mul;
    dr = dr * mul;
    p = v3mul_add(p, scale_vec, offset);
    dr = mul_add(-dr, scale, one);
  }
  return trap;
}
// palette coordinate s and albedo of a trap value (include/rayn_b200.h)
inline F4 trap_coord(const RaynAlbedoTrap& tp, F4 trap) {
  F4 lo = splat(tp.trap_lo), hi = splat(tp.trap_hi);
  F4 inner = merge(cmp_le(hi, trap), splat(1.0f), (trap - lo) / (hi - lo));
  return merge(cmp_gt(trap, lo), inner, splat(0.0f));
}
inline V3 trap_albedo(const RaynAlbedoTrap& tp, F4 s) {
  F4 r = splat(1.0f) - s;
  return {splat(tp.albedo_lo[0]) * r + splat(tp.albedo_hi[0]) * s, splat(tp.albedo_lo[1]) * r + splat(tp.albedo_hi[1]) * s,
          splat(tp.albedo_lo[2]) * r + splat(tp.albedo_hi[2]) * s};
}

// integrate() with lane i's albedo = albedo[i] for a Lambertian / Dielectric material.  Nothing in integrate() couples one lane's
// albedo to another lane: the light choice reads the sample tables, every BSDF term is per lane, and whether a lane ends
// (max_bounces, roulette on the INCOMING throughput) or spawns a ray does not depend on the albedo.  So run k of the
// oracle's own integrate(), with the material's constant albedo set to lane k's, gives lane k's results exactly, and the
// four runs push their outputs in the same order with the same lanes.  To tell the lanes apart, every run sees the packet
// with tile_coord.x = lane index; the merge takes entry j from the run of entry j's lane and restores the real coordinate.
void integrate_per_lane_albedo(const World& w, int max_bounces, int volume_marches, const F4* s1d, const F4* s2d, int depth,
                               int material, V3 albedo, const ShadingPoint& sp, std::vector<Ray>& spawned_rays,
                               std::vector<OutSample>& out, Counters& cnt) {
  RaynMaterial mats[RAYN_MAX_MATERIALS];
  memcpy(mats, w.s->materials, sizeof(RaynMaterial) * (size_t)w.s->n_materials);
  RaynSceneDesc scene = *w.s;
  scene.materials = mats;
  const World wk{&scene};
  ShadingPoint tagged = sp;
  for (uint32_t i = 0; i < 4; ++i) tagged.ray.tx[i] = i;
  std::vector<Ray> rays[4];
  std::vector<OutSample> samples[4];
  for (int k = 0; k < 4; ++k) {
    mats[material].albedo[0] = albedo.x[k], mats[material].albedo[1] = albedo.y[k], mats[material].albedo[2] = albedo.z[k];
    Counters scratch;
    integrate(wk, max_bounces, volume_marches, s1d, s2d, depth, material, tagged, rays[k], samples[k], k == 0 ? cnt : scratch);
  }
  for (int k = 1; k < 4; ++k)
    if (samples[k].size() != samples[0].size() || rays[k].size() != rays[0].size()) {
      g_lane_split_failed = 1;
      return;
    }
  for (size_t j = 0; j < samples[0].size(); ++j) {
    const uint32_t lane = samples[0][j].tx;
    OutSample o = samples[lane][j];
    if (o.tx != lane || o.channel != samples[0][j].channel || o.ty != samples[0][j].ty) g_lane_split_failed = 1;  // see above
    o.tx = sp.ray.tx[lane];
    out.push_back(o);
  }
  for (size_t j = 0; j < rays[0].size(); ++j) {
    const uint32_t lane = rays[0][j].tx;
    Ray r = rays[lane][j];
    if (r.tx != lane || r.sample != rays[0][j].sample) g_lane_split_failed = 1;
    r.tx = sp.ray.tx[lane];
    spawned_rays.push_back(r);
  }
}

// film.rs:439-627 for one tile: render_tile() of oracle/rayn_oracle.cpp with trap packets integrated per lane
void render_tile_traps(const World& w, const TrapTable& traps, const RaynFrameDesc& f, int tile_x, int tile_y, float* color,
                       float* alpha, float* background, float* normal, Counters& cnt) {
  const int W = f.width, H = f.height;
  const uint32_t x0 = tile_x * f.tile_w, y0 = tile_y * f.tile_h;
  const uint32_t x1 = (uint32_t)((int)(x0 + f.tile_w) < W ? x0 + f.tile_w : W);
  const uint32_t y1 = (uint32_t)((int)(y0 + f.tile_h) < H ? y0 + f.tile_h : H);
  const uint32_t tw = x1 - x0, th = y1 - y0;
  const int samples = f.samples, spp = 4 * samples, vm = f.volume_marches;
  const float ndc_x = 1.0f / (float)W, ndc_y = 1.0f / (float)H;
  Tables tab{spp, f.samples_1d, f.samples_2d};
  std::vector<float> tc(3 * tw * th, 0.0f), ta(tw * th, 0.0f), tb(3 * tw * th, 0.0f), tn(3 * tw * th, 0.0f);

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
          break;
        case CH_ALPHA:
          ta[idx] += s.v[0];
          break;
        case CH_BACKGROUND:
          for (int k = 0; k < 3; ++k) tb[3 * idx + k] += s.v[k];
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
    }
}

}  // namespace

extern "C" {

// rayn_oracle_render_frame with an orbit-trap list (rayn_b200_set_albedo_traps; trusted, the GPU library validates it) and
// without the queue log: tiles with (tile_index % tile_stride) == tile_offset AND ((tile_index / tile_stride) % subsample_k) == 0,
// or frame->tile_list.  Planes are host pointers; untouched pixels keep their previous contents.
int32_t rayn_trap_oracle_render_frame(const RaynSceneDesc* scene, int32_t n_traps, const RaynAlbedoTrap* traps, const RaynFrameDesc* f,
                                      const RaynFilmPlanes* out, int32_t n_threads, int32_t subsample_k, int64_t* counters4,
                                      int64_t* tiles_rendered) {
  if (!scene || !f || !out || n_traps < 0 || (n_traps > 0 && !traps)) return RAYN_ERR_INVALID_ARG;
  TrapTable table = {};
  for (int i = 0; i < n_traps; ++i) {
    if (traps[i].material < 0 || traps[i].material >= scene->n_materials) return RAYN_ERR_INVALID_ARG;
    table[traps[i].material] = &traps[i];
  }
  if (f->volume_marches != 2) return RAYN_ERR_UNSUPPORTED;
  if (!fp_contract_is_off()) return RAYN_ERR_UNSUPPORTED;
  World w{scene};
  int ntx = (f->width + f->width % f->tile_w) / f->tile_w;    // film.rs:399-404
  int nty = (f->height + f->height % f->tile_h) / f->tile_h;
  int stride = f->tile_stride > 0 ? f->tile_stride : 1;
  if (subsample_k < 1) subsample_k = 1;
  std::vector<int> todo;
  if (f->tile_list) {  // explicit tile set (same meaning as in rayn_b200_render_frame)
    for (int i = 0; i < f->n_tile_list; ++i)
      if (f->tile_list[i] >= 0 && f->tile_list[i] < ntx * nty) todo.push_back(f->tile_list[i]);
  } else {
    for (int idx = 0; idx < ntx * nty; ++idx)
      if (idx % stride == f->tile_offset && ((idx / stride) % subsample_k) == 0) todo.push_back(idx);
  }
  Counters total;
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
      render_tile_traps(w, table, *f, tx, ty, out->color, out->alpha, out->background, out->normal, local);
    }
#pragma omp critical
    {
      total.extend_rays += local.extend_rays;
      total.shade_lanes += local.shade_lanes;
      total.shadow_rays += local.shadow_rays;
      total.sdf_evals_extend += local.sdf_evals_extend;
    }
  }
  if (counters4) {
    counters4[0] = total.extend_rays;
    counters4[1] = total.shade_lanes;
    counters4[2] = total.shadow_rays;
    counters4[3] = total.sdf_evals_extend;
  }
  if (tiles_rendered) *tiles_rendered = (int64_t)todo.size();
  return g_lane_split_failed.exchange(0) ? RAYN_ERR_UNSUPPORTED : RAYN_OK;
}

int32_t rayn_trap_oracle_kat_sdf_trap(const RaynHitable* sdf, int64_t n, const float* points3, float* out) {
  for (int64_t i = 0; i < n; i += 4) store_f_packet(out, i, n, sdf_trap(*sdf, load_v3_packet(points3, i, n)));
  return RAYN_OK;
}

// palette coordinate s and albedo of trap values
int32_t rayn_trap_oracle_kat_trap_albedo(const RaynAlbedoTrap* tp, int64_t n, const float* trap, float* out_s, float* out_albedo3) {
  for (int64_t i = 0; i < n; i += 4) {
    const F4 s = trap_coord(*tp, load_f_packet(trap, i, n));
    const V3 a = trap_albedo(*tp, s);
    alignas(16) float ax[4], ay[4], az[4], sv[4];
    store4(sv, s), store4(ax, a.x), store4(ay, a.y), store4(az, a.z);
    for (int k = 0; k < 4 && i + k < n; ++k) {
      out_s[i + k] = sv[k];
      out_albedo3[3 * (i + k)] = ax[k], out_albedo3[3 * (i + k) + 1] = ay[k], out_albedo3[3 * (i + k) + 2] = az[k];
    }
  }
  return RAYN_OK;
}

}  // extern "C"
