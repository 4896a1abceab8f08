// render_mirror.cpp — CPU mirrors of the render passes of include/rayn_b200.h: the film with orbit-trap albedos
// (RaynAlbedoTrap) and optional luminance moments (rayn_b200_render_frame_moments), the first-hit albedo plane
// (rayn_b200_render_albedo) and the motion plane (rayn_b200_render_motion, rayn_b200_render_motion_prev).  TEST
// INFRASTRUCTURE ONLY: built by tests/mirrors.py; nothing under rayn_b200/ may include, link or execute it.
//
// It extends the render oracle without changing it: oracle/rayn_oracle.cpp is included as it is, and its own sample_uv,
// camera_get_rays, closest_hit and integrate() do the work.  This file adds
//   sdf_trap()        the trap on 4-lane packets, the same iterations as mandelbox_dist() / mandelbulb_dist() with a min fold;
//   trap_coord(), trap_albedo()   the palette;
//   integrate_per_lane_albedo()   integrate() (integrator.rs:47-205) with a per-lane albedo, from four runs of the
//                     oracle's own integrate() on a private copy of the material (see the function);
//   camera_packet()   the raygen of render_tile (film.rs:456-464) for one pixel and one sample packet;
//   render_tile_traps()   render_tile() (film.rs:439-627) with two changes: a packet whose material has a trap is integrated
//                     with integrate_per_lane_albedo(), and the lum^2 fold of the moment planes.  (No queue log: the packet
//                     order is the oracle's, tested there.)
//   first_hit_tile()  the depth-0 closest hit of every camera packet of a tile, handed to a per-lane rule (albedo, motion);
//   select_tiles(), for_tiles()   which tiles a pass computes, and the OpenMP loop over them.
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
// the albedo generator at a hit: the orbit trap at the point, s = 1 on an analytic sphere
inline V3 hit_trap_albedo(const RaynAlbedoTrap& tp, const RaynHitable& h, V3 point) {
  return trap_albedo(tp, h.kind == RAYN_HITABLE_SPHERE ? splat(1.0f) : trap_coord(tp, sdf_trap(h, point)));
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

// lum(v) of the header: every product rounded on its own (no contraction)
inline float lum(const float* v) { return (0.2126f * v[0] + 0.7152f * v[1]) + 0.0722f * v[2]; }

// pixels [x0, x1) x [y0, y1) of tile (tile_x, tile_y), clipped to the film
struct TileRect {
  uint32_t x0, y0, x1, y1;
  TileRect(const RaynFrameDesc& f, int tile_x, int tile_y)
      : x0(tile_x * f.tile_w), y0(tile_y * f.tile_h),
        x1((uint32_t)((int)(x0 + f.tile_w) < f.width ? x0 + f.tile_w : f.width)),
        y1((uint32_t)((int)(y0 + f.tile_h) < f.height ? y0 + f.tile_h : f.height)) {}
};

// film.rs:456-464: the 4-lane camera packet of sample packet samp at pixel (x, y) of tile t; us, vs and times
// (the lanes' film coordinates and camera times) for callers that need them
WRay camera_packet(const World& w, const RaynFrameDesc& f, const Tables& tab, uint32_t x, uint32_t y, const TileRect& t, int samp,
                   float* us, float* vs, F4* times) {
  const float scramble = f.scramble[x + y * (uint32_t)f.width];
  uint32_t nums[4] = {4u * samp, 4u * samp + 1, 4u * samp + 2, 4u * samp + 3};
  for (int i = 0; i < 4; ++i)
    sample_uv(x, y, 1.0f / (float)f.width, 1.0f / (float)f.height, f.fis_inverse_cdf, tab.s2(0, nums[i], scramble, 0),
              tab.s2(1, nums[i], scramble, 0), &us[i], &vs[i]);
  float sc4[4] = {scramble, scramble, scramble, scramble};
  *times = splat(f.t0) + splat(f.t1 - f.t0) * tab.w1(nums, sc4, 0);
  F4 ls0 = tab.w2(0, nums, sc4, 1), ls1 = tab.w2(1, nums, sc4, 1);
  return camera_get_rays(w.s->camera, scramble, nums, x - t.x0, y - t.y0, load4(us), load4(vs), *times, ls0, ls1);
}

// film.rs:439-627 for one tile: render_tile() of oracle/rayn_oracle.cpp with trap packets integrated per lane, and the lum^2
// fold in the CH_COLOR / CH_BACKGROUND cases of the new_samples loop (the same samples in the same order as the colour sums).
// lum2_color / lum2_bg may be NULL.
void render_tile_traps(const World& w, const TrapTable& traps, const RaynFrameDesc& f, int tile_x, int tile_y, const RaynFilmPlanes& out,
                       float* lum2_color, float* lum2_bg, Counters& cnt) {
  const TileRect t(f, tile_x, tile_y);
  const uint32_t tw = t.x1 - t.x0, th = t.y1 - t.y0;
  const int samples = f.samples, spp = 4 * samples, vm = f.volume_marches;
  Tables tab{spp, f.samples_1d, f.samples_2d};
  std::vector<float> tc(3 * tw * th, 0.0f), ta(tw * th, 0.0f), tb(3 * tw * th, 0.0f), tn(3 * tw * th, 0.0f);
  std::vector<float> tmc(tw * th, 0.0f), tmb(tw * th, 0.0f);

  std::vector<WRay> spawned_wrays;
  std::vector<Ray> spawned_rays;
  std::vector<OutSample> new_samples;
  std::vector<std::vector<Hit>> bins(w.n_hit());

  for (uint32_t x = t.x0; x < t.x1; ++x)
    for (uint32_t y = t.y0; y < t.y1; ++y)
      for (int samp = 0; samp < samples; ++samp) {
        float us[4], vs[4];
        F4 times;
        spawned_wrays.push_back(camera_packet(w, f, tab, x, y, t, samp, us, vs, &times));
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
        if (!tp)
          integrate(w, f.max_bounces, vm, s1d, s2d, depth, h.material, sp, spawned_rays, new_samples, cnt);
        else
          integrate_per_lane_albedo(w, f.max_bounces, vm, s1d, s2d, depth, h.material, hit_trap_albedo(*tp, h, sp.point), sp,
                                    spawned_rays, new_samples, cnt);
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
  float *color = (float*)out.color, *alpha = (float*)out.alpha, *background = (float*)out.background, *normal = (float*)out.normal;
  const float div = (float)spp;
  for (uint32_t x = 0; x < tw; ++x)
    for (uint32_t y = 0; y < th; ++y) {
      size_t ti = x + y * tw;
      size_t fi = (t.x0 + x) + (size_t)(t.y0 + y) * f.width;
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

// The depth-0 packets of one tile (film.rs:456-551): for every camera packet, the oracle's closest_hit at depth 0, then
// rule(x, y, first sample number, wray, ids, dists, us, vs, times) for its four lanes.
template <class Rule>
void first_hit_tile(const World& w, const RaynFrameDesc& f, int tile_x, int tile_y, Rule&& rule) {
  const TileRect t(f, tile_x, tile_y);
  Tables tab{4 * f.samples, f.samples_1d, f.samples_2d};
  const Thr thr{0, &w.s->camera};
  int64_t evals = 0;
  for (uint32_t x = t.x0; x < t.x1; ++x)
    for (uint32_t y = t.y0; y < t.y1; ++y)
      for (int samp = 0; samp < f.samples; ++samp) {
        float us[4], vs[4];
        F4 times;
        const WRay wray = camera_packet(w, f, tab, x, y, t, samp, us, vs, &times);
        int ids[4];
        F4 dists;
        closest_hit(w, wray, splat(w.s->consts.world_radius * 2.0f), thr, ids, &dists, &evals);
        rule(x, y, 4 * samp, wray, ids, dists, us, vs, times);
      }
}

// The tile indices a pass computes, on the grid of film.rs:399-404 (nty tiles per column).  A render honours frame->tile_list,
// or else takes (idx % tile_stride) == tile_offset, and keeps every subsample_k-th of those (idx / stride); first-hit passes
// ignore the tile selection, as the product does, and keep every subsample_k-th index.
struct Tiles {
  std::vector<int> todo;
  int nty;
};
Tiles select_tiles(const RaynFrameDesc& f, bool render, int subsample_k) {
  const int ntx = (f.width + f.width % f.tile_w) / f.tile_w, nty = (f.height + f.height % f.tile_h) / f.tile_h;
  const int stride = render && f.tile_stride > 0 ? f.tile_stride : 1, offset = render ? f.tile_offset : 0;
  if (subsample_k < 1) subsample_k = 1;
  Tiles t{{}, nty};
  if (render && f.tile_list) {  // explicit tile set (same meaning as in rayn_b200_render_frame)
    for (int i = 0; i < f.n_tile_list; ++i)
      if (f.tile_list[i] >= 0 && f.tile_list[i] < ntx * nty) t.todo.push_back(f.tile_list[i]);
  } else {
    for (int idx = 0; idx < ntx * nty; ++idx)
      if (idx % stride == offset && ((idx / stride) % subsample_k) == 0) t.todo.push_back(idx);
  }
  return t;
}

// fn(tile_x, tile_y, counters) for every selected tile on the grid, in parallel; returns the sum of the counters
template <class Fn>
Counters for_tiles(const RaynFrameDesc& f, const Tiles& tiles, int n_threads, Fn&& fn) {
  Counters total;
#ifdef _OPENMP
  if (n_threads > 0) omp_set_num_threads(n_threads);
#endif
#pragma omp parallel
  {
    Counters local;
#pragma omp for schedule(dynamic, 1)
    for (size_t k = 0; k < tiles.todo.size(); ++k) {
      const int tx = tiles.todo[k] / tiles.nty, ty = tiles.todo[k] % tiles.nty;
      if (tx * f.tile_w >= f.width || ty * f.tile_h >= f.height) continue;
      fn(tx, ty, local);
    }
#pragma omp critical
    {
      total.extend_rays += local.extend_rays;
      total.shade_lanes += local.shade_lanes;
      total.shadow_rays += local.shadow_rays;
      total.sdf_evals_extend += local.sdf_evals_extend;
    }
  }
  return total;
}

// the trap list of rayn_b200_set_albedo_traps (trusted, the GPU library validates it) as a per-material table
bool trap_table(const RaynSceneDesc* scene, int32_t n_traps, const RaynAlbedoTrap* traps, TrapTable* table) {
  if (n_traps < 0 || (n_traps > 0 && !traps)) return false;
  *table = {};
  for (int i = 0; i < n_traps; ++i) {
    if (traps[i].material < 0 || traps[i].material >= scene->n_materials) return false;
    (*table)[traps[i].material] = &traps[i];
  }
  return true;
}

bool moving(const RaynHitable& h) { return h.center_velocity[0] != 0.0f || h.center_velocity[1] != 0.0f || h.center_velocity[2] != 0.0f; }

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

// The motion record (dx, dy, z, z_prev) of every lane of a depth-0 packet: P' is P on a hit that does not move, otherwise
//   prev == NULL (rayn_b200_render_motion, the uploaded scene run backwards): P - v*dt on a moving sphere;
//   prev given (rayn_b200_render_motion_prev): P + (c_prev(tau - dt) - c(tau)) on a sphere that moved or moves, projected
//   with prev's camera.
void motion_records(const World& w, const RaynSceneDesc* prev, int W, int H, float frame_dt, V3 P, float tau, const int* ids, float* rec[4]) {
  const RaynCamera& cam = w.s->camera;
  const float tp = tau - frame_dt;
  alignas(16) float ppx[4], ppy[4], ppz[4];
  store4(ppx, P.x), store4(ppy, P.y), store4(ppz, P.z);
  for (int i = 0; i < 4; ++i) {
    if (ids[i] < 0) continue;
    const RaynHitable& h = w.s->hitables[ids[i]];
    if (h.kind != RAYN_HITABLE_SPHERE) continue;
    if (!prev) {
      if (!moving(h)) continue;
      ppx[i] = ppx[i] - h.center_velocity[0] * frame_dt, ppy[i] = ppy[i] - h.center_velocity[1] * frame_dt,
      ppz[i] = ppz[i] - h.center_velocity[2] * frame_dt;
    } else {
      const RaynHitable& hp = prev->hitables[ids[i]];
      if (!moving(hp) && !moving(h) && memcmp(hp.center, h.center, sizeof h.center) == 0) continue;
      const V3 cp = seq_v3(hp.center, hp.center_velocity, splat(tp)), c = seq_v3(h.center, h.center_velocity, splat(tau));
      ppx[i] = ppx[i] + (cp.x[0] - c.x[0]), ppy[i] = ppy[i] + (cp.y[0] - c.y[0]), ppz[i] = ppz[i] + (cp.z[0] - c.z[0]);
    }
  }
  F4 px1, py1, z1, px0, py0, z0;
  project(cam, W, H, P, tau, &px1, &py1, &z1);
  project(prev ? prev->camera : cam, W, H, V3{load4(ppx), load4(ppy), load4(ppz)}, tp, &px0, &py0, &z0);
  for (int i = 0; i < 4; ++i) {
    const bool valid = ids[i] >= 0 && (cam.kind == RAYN_CAMERA_ORTHOGRAPHIC || (z1[i] > 0.0f && z0[i] > 0.0f));
    float* out = rec[i];
    if (valid) {
      out[0] = px0[i] - px1[i], out[1] = py0[i] - py1[i], out[2] = z1[i], out[3] = z0[i];
    } else {
      out[0] = 0.0f, out[1] = 0.0f, out[2] = NAN, out[3] = NAN;
    }
  }
}

}  // namespace

extern "C" {

// rayn_oracle_render_frame with an orbit-trap list and optional moment planes (lum2_color, lum2_bg may be NULL), without the
// queue log; tiles as select_tiles.  Planes are host pointers; untouched pixels keep their previous contents.
int32_t rayn_mirror_render_frame(const RaynSceneDesc* scene, int32_t n_traps, const RaynAlbedoTrap* traps, const RaynFrameDesc* f,
                                 const RaynFilmPlanes* out, float* lum2_color, float* lum2_bg, int32_t n_threads, int32_t subsample_k,
                                 int64_t* counters4, int64_t* tiles_rendered) {
  TrapTable table;
  if (!scene || !f || !out || !trap_table(scene, n_traps, traps, &table)) return RAYN_ERR_INVALID_ARG;
  if (f->volume_marches != 2) return RAYN_ERR_UNSUPPORTED;
  if (!fp_contract_is_off()) return RAYN_ERR_UNSUPPORTED;
  const World w{scene};
  const Tiles tiles = select_tiles(*f, true, subsample_k);
  const Counters total = for_tiles(*f, tiles, n_threads, [&](int tx, int ty, Counters& cnt) {
    render_tile_traps(w, table, *f, tx, ty, *out, lum2_color, lum2_bg, cnt);
  });
  if (counters4) {
    counters4[0] = total.extend_rays;
    counters4[1] = total.shade_lanes;
    counters4[2] = total.shadow_rays;
    counters4[3] = total.sdf_evals_extend;
  }
  if (tiles_rendered) *tiles_rendered = (int64_t)tiles.todo.size();
  return g_lane_split_failed.exchange(0) ? RAYN_ERR_UNSUPPORTED : RAYN_OK;
}

// Per-sample albedos a_s (float [W*H*spp*3], pixel-major, samples ascending) and the plane (float [3*W*H]) of the whole tile
// grid; pixels outside the grid are 0 in both, as are the tiles that subsample_k > 1 leaves out.
int32_t rayn_mirror_render_albedo(const RaynSceneDesc* scene, int32_t n_traps, const RaynAlbedoTrap* traps, const RaynFrameDesc* f,
                                  float* per_sample, float* albedo, int32_t n_threads, int32_t subsample_k) {
  TrapTable table;
  if (!scene || !f || !per_sample || !albedo || !trap_table(scene, n_traps, traps, &table)) return RAYN_ERR_INVALID_ARG;
  if (!fp_contract_is_off()) return RAYN_ERR_UNSUPPORTED;
  const World w{scene};
  const int W = f->width, H = f->height, spp = 4 * f->samples;
  memset(per_sample, 0, sizeof(float) * (size_t)W * H * spp * 3);
  memset(albedo, 0, sizeof(float) * (size_t)W * H * 3);
  for_tiles(*f, select_tiles(*f, false, subsample_k), n_threads, [&](int tx, int ty, Counters&) {
    first_hit_tile(w, *f, tx, ty, [&](uint32_t x, uint32_t y, int s0, const WRay& wray, const int* ids, F4 dists, const float*, const float*, F4) {
      const V3 point = point_at(wray, dists);
      for (int i = 0; i < 4; ++i) {
        float* out = per_sample + (((size_t)y * W + x) * spp + s0 + i) * 3;  // stays 0: Sky / Emissive hit or nothing hit
        if (ids[i] < 0) continue;
        const RaynHitable& h = w.s->hitables[ids[i]];
        const RaynMaterial& m = w.s->materials[h.material];
        if (m.kind != RAYN_MATERIAL_LAMBERTIAN && m.kind != RAYN_MATERIAL_DIELECTRIC) continue;
        if (const RaynAlbedoTrap* tp = table[h.material]) {
          const V3 alb = hit_trap_albedo(*tp, h, point);
          out[0] = alb.x[i], out[1] = alb.y[i], out[2] = alb.z[i];
        } else {
          out[0] = m.albedo[0], out[1] = m.albedo[1], out[2] = m.albedo[2];
        }
      }
    });
    const TileRect t(*f, tx, ty);
    for (uint32_t x = t.x0; x < t.x1; ++x)  // k_albedo_resolve: the sum in sample order / spp
      for (uint32_t y = t.y0; y < t.y1; ++y)
        for (int c = 0; c < 3; ++c) {
          float acc = 0.0f;
          for (int s = 0; s < spp; ++s) acc += per_sample[(((size_t)y * W + x) * spp + s) * 3 + c];
          albedo[3 * ((size_t)y * W + x) + c] = acc / (float)spp;
        }
  });
  return RAYN_OK;
}

// Per-sample records (float [W*H*spp*4], pixel-major, samples ascending) and the plane (float [4*W*H]) of the whole tile grid,
// against prev (rayn_b200_render_motion_prev) or, with prev NULL, the uploaded scene run backwards (rayn_b200_render_motion).
// Pixels outside the grid, and in the tiles that subsample_k > 1 leaves out, have records (0, 0, NaN, NaN) and motion
// (0, 0, +inf, +inf).  prev must match the scene (hitable count and kinds, camera kind), as the product call requires;
// RAYN_ERR_INVALID_ARG otherwise.  geo (may be NULL): float [W*H*spp*6], per sample the hit point, the camera time and the
// film coordinates (u, v) of its ray.
int32_t rayn_mirror_render_motion(const RaynSceneDesc* scene, const RaynFrameDesc* f, float frame_dt, const RaynSceneDesc* prev, float* per_sample,
                                  float* motion, int32_t n_threads, int32_t subsample_k, float* geo) {
  if (!scene || !f || !per_sample || !motion) return RAYN_ERR_INVALID_ARG;
  if (prev) {
    if (!prev->hitables || prev->n_hitables != scene->n_hitables || prev->camera.kind != scene->camera.kind) return RAYN_ERR_INVALID_ARG;
    for (int j = 0; j < scene->n_hitables; ++j)
      if (prev->hitables[j].kind != scene->hitables[j].kind) return RAYN_ERR_INVALID_ARG;
  }
  if (!fp_contract_is_off()) return RAYN_ERR_UNSUPPORTED;
  const World w{scene};
  const int W = f->width, H = f->height, spp = 4 * f->samples;
  for (size_t i = 0; i < (size_t)W * H * spp; ++i)
    per_sample[4 * i] = 0.0f, per_sample[4 * i + 1] = 0.0f, per_sample[4 * i + 2] = NAN, per_sample[4 * i + 3] = NAN;
  for (size_t i = 0; i < (size_t)W * H; ++i) motion[4 * i] = 0.0f, motion[4 * i + 1] = 0.0f, motion[4 * i + 2] = INFINITY, motion[4 * i + 3] = INFINITY;
  for_tiles(*f, select_tiles(*f, false, subsample_k), n_threads, [&](int tx, int ty, Counters&) {
    first_hit_tile(w, *f, tx, ty, [&](uint32_t x, uint32_t y, int s0, const WRay& wray, const int* ids, F4 dists, const float* us, const float* vs, F4 times) {
      const V3 P = point_at(wray, dists);
      const size_t r0 = ((size_t)y * W + x) * spp + s0;
      float* rec[4] = {per_sample + 4 * r0, per_sample + 4 * (r0 + 1), per_sample + 4 * (r0 + 2), per_sample + 4 * (r0 + 3)};
      motion_records(w, prev, W, H, frame_dt, P, times[0], ids, rec);
      for (int i = 0; geo && i < 4; ++i) {
        float* g = geo + (r0 + i) * 6;
        g[0] = P.x[i], g[1] = P.y[i], g[2] = P.z[i], g[3] = times[0], g[4] = us[i], g[5] = vs[i];
      }
    });
    const TileRect t(*f, tx, ty);
    for (uint32_t x = t.x0; x < t.x1; ++x)
      for (uint32_t y = t.y0; y < t.y1; ++y) {  // k_motion_resolve: the mean over valid samples in sample order
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
  });
  return RAYN_OK;
}

int32_t rayn_mirror_kat_sdf_trap(const RaynHitable* sdf, int64_t n, const float* points3, float* out) {
  for (int64_t i = 0; i < n; i += 4) store_f_packet(out, i, n, sdf_trap(*sdf, load_v3_packet(points3, i, n)));
  return RAYN_OK;
}

// palette coordinate s and albedo of trap values
int32_t rayn_mirror_kat_trap_albedo(const RaynAlbedoTrap* tp, int64_t n, const float* trap, float* out_s, float* out_albedo3) {
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
