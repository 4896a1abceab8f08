// metallic_mirror.cpp — CPU mirror of the Metallic material of include/rayn_b200.h (RAYN_MATERIAL_METALLIC): its f and scatter,
// and through them the oracle's film, the render mirror's film (orbit traps, moments) and the first-hit albedo plane of scenes
// with metals.  TEST INFRASTRUCTURE ONLY: built by tests/metallic_mirrors.py; nothing under rayn_b200/ may include, link or
// execute it.
//
// It extends the render mirror and the oracle without changing either: tests/render_mirror.cpp (which includes
// oracle/rayn_oracle.cpp) is included as it is.  Their film loops call integrate(...) and the render mirror's
// integrate_per_lane_albedo(...) with the sample sets as non-const F4 arrays; the overloads declared below take `F4*` where the
// originals take `const F4*`, so overload resolution picks them for those calls (an identity conversion beats a qualification
// conversion).  For every material that is not a metal they call the originals with the same arguments, so every other kind
// renders exactly as before (tested: films of the configs through this library equal the oracle's bit for bit).  For a metal
// they run integrate() with the metal's BSDF: metal_f and metal_scatter below, the statement of the header, in the oracle's
// 4-lane arithmetic.  An orbit-trap palette reaches a metal the way it reaches the other kinds: the render mirror's per-lane
// split substitutes each lane's albedo into a copy of the material, and a metal reads its albedo as F0.
// Build flags: those of oracle/Makefile (-ffp-contract=off is required, see there).
#include <stdint.h>

#include <vector>

#include "../include/rayn_b200.h"

namespace {
struct F4;
struct V3;
struct World;
struct ShadingPoint;
struct Ray;
struct OutSample;
struct Counters;
void integrate(const World& w, int max_bounces, int volume_marches, F4* s1d, F4* s2d, int depth, int material, ShadingPoint sp,
               std::vector<Ray>& spawned_rays, std::vector<OutSample>& out, Counters& cnt);
void integrate_per_lane_albedo(const World& w, int max_bounces, int volume_marches, F4* s1d, F4* s2d, int depth, int material, V3 albedo,
                               const ShadingPoint& sp, std::vector<Ray>& spawned_rays, std::vector<OutSample>& out, Counters& cnt);
}  // namespace

#include "render_mirror.cpp"

namespace {

bool metal_receives_light(const RaynMaterial& m) { return receives_light(m) || m.kind == RAYN_MATERIAL_METALLIC; }

// f(first, second, n), called as bsdf.f(wo, wi, n): the Dielectric's f (oracle bsdf_f) without its diffuse term, with
// f_schlick(dotv, F0[c]) per channel
V3 metal_f(const RaynMaterial& m, V3 first, V3 second, V3 n) {
  F4 zero = splat(0.0f), two = splat(2.0f);
  F4 rough = splat(m.roughness);
  F4 dotv = f4max(zero, dot(first, n));
  V3 half = normalized(second + first);
  F4 cos_alpha = f4powf(f4max(zero, dot(half, n)), rough);
  F4 spec_factor = cos_alpha * (rough + two) / (two * splat(kPI));
  return {spec_factor * f_schlick(dotv, splat(m.albedo[0])), spec_factor * f_schlick(dotv, splat(m.albedo[1])),
          spec_factor * f_schlick(dotv, splat(m.albedo[2]))};
}
// scatter: the Dielectric's specular branch (oracle bsdf_scatter), always taken; s1d and s2d[0..1] are not read
Scatter metal_scatter(const RaynMaterial& m, V3 wo, const ShadingPoint& sp, const F4* s2d) {
  F4 one = splat(1.0f), two = splat(2.0f);
  F4 rough = splat(m.roughness);
  V3 norm = sp.normal;
  F4 cosv = f4abs(dot(norm, wo));
  V3 spec_sample = cosine_power(s2d[2], s2d[3], rough);
  V3 reflection = reflected(wo, norm);
  M3 basis = onb(reflection);
  V3 spec_bounce = normalized(basis * spec_sample);
  F4 cos_alpha_pow = f4max(f4powf(spec_sample.z, rough), splat(kEPSILON));
  F4 spec_pdf = (rough + one) / splat(kTWO_PI) * cos_alpha_pow;
  F4 spec_coeff = (rough + two) / splat(kTWO_PI) * cos_alpha_pow;
  F4 below_horizon = cmp_lt(dot(norm, spec_bounce), splat(0.0f));
  spec_coeff = merge(below_horizon, splat(0.0f), spec_coeff);
  Scatter se;
  se.wi = spec_bounce;
  se.f = {spec_coeff * f_schlick(cosv, splat(m.albedo[0])), spec_coeff * f_schlick(cosv, splat(m.albedo[1])),
          spec_coeff * f_schlick(cosv, splat(m.albedo[2]))};
  se.pdf = spec_pdf;
  return se;
}
// any kind's BSDF: the metal's, else the oracle's
V3 any_bsdf_f(const RaynMaterial& m, V3 first, V3 second, V3 n) {
  return m.kind == RAYN_MATERIAL_METALLIC ? metal_f(m, first, second, n) : bsdf_f(m, first, second, n);
}
Scatter any_bsdf_scatter(const RaynMaterial& m, V3 wo, const ShadingPoint& sp, F4 s1d, const F4* s2d) {
  return m.kind == RAYN_MATERIAL_METALLIC ? metal_scatter(m, wo, sp, s2d) : bsdf_scatter(m, wo, sp, s1d, s2d);
}

// surface_sample_one_light of the oracle with the metal's f
V3 metal_surface_sample_one_light(const World& w, int light_idx, F4 s0, F4 s1, const ShadingPoint& sp, const RaynMaterial& mat) {
  V3 end_point, li;
  F4 pdf;
  light_sample(w.s->lights[light_idx], s0, s1, sp.point, &end_point, &li, &pdf);
  V3 wo = -sp.ray.dir;
  V3 wi = end_point - sp.point;
  F4 dist = mag(wi);
  wi = wi / dist;
  V3 occlude_point = sp.point + sp.normal * f4signum(dot(sp.normal, wi)) * sp.offset_by;
  F4 occluded = test_occluded(w, occlude_point, end_point, sp.ray.time);
  V3 f = metal_f(mat, wo, wi, sp.normal) * f4max(dot(sp.normal, wi), splat(0.0f));
  F4 transmission = w.s->volume.has_extinction ? f4exp(splat(-w.s->volume.coeff_extinction) * dist) : splat(1.0f);
  return li * f * transmission * occluded / pdf;
}

// the oracle's integrate() for a material that receives light, with the metal's f and scatter (the decoupled-lights test
// switch of the oracle is not mirrored: it is never set on a parity path)
void metal_integrate(const World& w, int max_bounces, int volume_marches, const F4* s1d, const F4* s2d, int depth, int material,
                     ShadingPoint sp, std::vector<Ray>& spawned_rays, std::vector<OutSample>& out, Counters& cnt) {
  V3 wo = -sp.ray.dir;
  const RaynMaterial& mat = w.s->materials[material];
  const RaynVolume& vol = w.s->volume;
  const int nl = w.n_lights();
  F4 volume_transmission = vol.has_extinction ? f4exp(splat(-vol.coeff_extinction) * sp.t) : splat(1.0f);
  sp.ray.radiance = sp.ray.radiance + bsdf_le(mat, wo) * sp.ray.throughput * volume_transmission;
  for (int i = 0; i < 4; ++i) cnt.shade_lanes += sp.ray.valid[i] ? 1 : 0;
  if (nl > 0) {
    F4 correction = splat((float)nl / 4.0f);
    for (int i = 0; i < 4; ++i) {
      V3 li = metal_surface_sample_one_light(w, light_index(s1d[0][i], nl), s2d[0 + i * 2], s2d[1 + i * 2], sp, mat);
      sp.ray.radiance = sp.ray.radiance + li * sp.ray.throughput * correction * volume_transmission;
      cnt.shadow_rays += 4;
    }
  }
  if (vol.has_scattering && nl > 0) {
    F4 rho_s = splat(vol.coeff_scattering);
    for (int march = 0; march < volume_marches; ++march) {
      F4 correction = splat((float)nl / 4.0f / (float)volume_marches);
      for (int i = 0; i < 4; ++i) {
        int li_idx = light_index(s1d[march + 1][i], nl);
        F4 t;
        V3 li = volume_sample_one_light(w, li_idx, s2d[8 + 8 * march + i * 2], s2d[8 + 8 * march + i * 2 + 1], s1d[1], sp.ray.origin,
                                        sp.ray.dir, sp.t, sp.ray.time, &t);
        F4 transmission = vol.has_extinction ? f4exp(splat(-vol.coeff_extinction) * t) : splat(1.0f);
        sp.ray.radiance = sp.ray.radiance + li * sp.ray.throughput * correction * rho_s * transmission;
        cnt.shadow_rays += 4;
      }
    }
  }
  Scatter se = metal_scatter(mat, wo, sp, s2d + 8 + 8 * volume_marches);
  F4 ndl = f4abs(dot(se.wi, sp.normal));
  V3 new_throughput = sp.ray.throughput * volume_transmission * se.f * ndl / se.pdf;
  F4 roulette_factor;
  if (depth > 2) {
    roulette_factor = f4max(splat(1.0f) - component_max(sp.ray.throughput), splat(0.05f));
    new_throughput = new_throughput / (splat(1.0f) - roulette_factor);
  } else {
    roulette_factor = splat(0.0f);
  }
  WRay nr = create_rays(sp, se.wi);
  Ray new_rays[4];
  wray_into(nr, new_rays);
  if (depth == 0) {
    for (int i = 0; i < 4; ++i)
      if (new_rays[i].valid) {
        out.push_back({new_rays[i].tx, new_rays[i].ty, CH_ALPHA, {1.0f, 0, 0}});
        out.push_back({new_rays[i].tx, new_rays[i].ty, CH_NORMAL, {sp.normal.x[i], sp.normal.y[i], sp.normal.z[i]}});
      }
  }
  for (int i = 0; i < 4; ++i) {
    Ray& ray = new_rays[i];
    if (!ray.valid) continue;
    if (depth >= max_bounces || s1d[4][i] < roulette_factor[i]) {
      out.push_back({ray.tx, ray.ty, CH_COLOR, {ray.radiance[0], ray.radiance[1], ray.radiance[2]}});
    } else {
      float nt[3] = {new_throughput.x[i], new_throughput.y[i], new_throughput.z[i]};
      if (!(nt[0] != nt[0] || nt[1] != nt[1] || nt[2] != nt[2])) ray.throughput[0] = nt[0], ray.throughput[1] = nt[1], ray.throughput[2] = nt[2];
      spawned_rays.push_back(ray);
    }
  }
}

void integrate(const World& w, int max_bounces, int volume_marches, F4* s1d, F4* s2d, int depth, int material, ShadingPoint sp,
               std::vector<Ray>& spawned_rays, std::vector<OutSample>& out, Counters& cnt) {
  const F4 *c1 = s1d, *c2 = s2d;
  if (w.s->materials[material].kind == RAYN_MATERIAL_METALLIC)
    metal_integrate(w, max_bounces, volume_marches, c1, c2, depth, material, sp, spawned_rays, out, cnt);
  else
    integrate(w, max_bounces, volume_marches, c1, c2, depth, material, sp, spawned_rays, out, cnt);  // the oracle's
}

// the render mirror's integrate_per_lane_albedo (see there) with the runs going through integrate() above
void integrate_per_lane_albedo(const World& w, int max_bounces, int volume_marches, F4* s1d, F4* s2d, int depth, int material, V3 albedo,
                               const ShadingPoint& sp, std::vector<Ray>& spawned_rays, std::vector<OutSample>& out, Counters& cnt) {
  const F4 *c1 = s1d, *c2 = s2d;
  if (w.s->materials[material].kind != RAYN_MATERIAL_METALLIC)
    return integrate_per_lane_albedo(w, max_bounces, volume_marches, c1, c2, depth, material, albedo, sp, spawned_rays, out, cnt);
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
    metal_integrate(wk, max_bounces, volume_marches, c1, c2, depth, material, tagged, rays[k], samples[k], k == 0 ? cnt : scratch);
  }
  for (int k = 1; k < 4; ++k)
    if (samples[k].size() != samples[0].size() || rays[k].size() != rays[0].size()) {
      g_lane_split_failed = 1;
      return;
    }
  for (size_t j = 0; j < samples[0].size(); ++j) {
    const uint32_t lane = samples[0][j].tx;
    OutSample o = samples[lane][j];
    if (o.tx != lane || o.channel != samples[0][j].channel || o.ty != samples[0][j].ty) g_lane_split_failed = 1;
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

}  // namespace

extern "C" {

// rayn_mirror_render_albedo with the metal among the kinds that receive light: its a_s is F0, or the trap palette
int32_t rayn_metal_render_albedo(const RaynSceneDesc* scene, int32_t n_traps, const RaynAlbedoTrap* traps, const RaynFrameDesc* f, float* per_sample,
                                 float* albedo, int32_t n_threads, int32_t subsample_k) {
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
        if (!metal_receives_light(m)) continue;
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

// rayn_oracle_kat_bsdf for every kind, the metal included
int32_t rayn_metal_kat_bsdf(const RaynMaterial* mat, int64_t n, const float* n3, const float* wo3, const float* s1d, const float* u4, float* out_wi3,
                            float* out_f3, float* out_pdf, float* out_feval3) {
  for (int64_t i = 0; i < n; i += 4) {
    ShadingPoint sp;
    sp.normal = load_v3_packet(n3, i, n);
    sp.basis = onb(sp.normal);
    V3 wo = load_v3_packet(wo3, i, n);
    F4 u[4];
    for (int k = 0; k < 4; ++k) {
      float tmp[4];
      for (int l = 0; l < 4; ++l) tmp[l] = u4[4 * (i + l < n ? i + l : n - 1) + k];
      u[k] = load4(tmp);
    }
    Scatter se = any_bsdf_scatter(*mat, wo, sp, load_f_packet(s1d, i, n), u);
    V3 fe = any_bsdf_f(*mat, wo, se.wi, sp.normal);
    store_f_packet(out_pdf, i, n, se.pdf);
    for (int l = 0; l < 4 && i + l < n; ++l) {
      const int64_t j = i + l;
      out_wi3[3 * j] = se.wi.x[l], out_wi3[3 * j + 1] = se.wi.y[l], out_wi3[3 * j + 2] = se.wi.z[l];
      out_f3[3 * j] = se.f.x[l], out_f3[3 * j + 1] = se.f.y[l], out_f3[3 * j + 2] = se.f.z[l];
      out_feval3[3 * j] = fe.x[l], out_feval3[3 * j + 1] = fe.y[l], out_feval3[3 * j + 2] = fe.z[l];
    }
  }
  return RAYN_OK;
}

}  // extern "C"
