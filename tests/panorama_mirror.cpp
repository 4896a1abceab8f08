// panorama_mirror.cpp — CPU mirrors of the equirectangular camera of include/rayn_b200.h (RAYN_CAMERA_EQUIRECTANGULAR): its rays,
// its motion-plane projection, and through them the film, albedo and motion passes of a panorama.  TEST INFRASTRUCTURE ONLY:
// built by tests/panorama_mirrors.py; nothing under rayn_b200/ may include, link or execute it.
//
// It extends the render mirror and the oracle without changing either: tests/render_mirror.cpp (which includes
// oracle/rayn_oracle.cpp) is included as it is.  Their raygen calls camera_get_rays(camera, scramble, nums, ...) with `nums` a
// non-const uint32_t[4]; the overload declared below takes `uint32_t*` where the oracle's takes `const uint32_t*`, so overload
// resolution picks it for those calls (an identity conversion beats a qualification conversion).  It returns the oracle's packet
// with the panorama's origin and direction for an equirectangular camera, and the oracle's packet unchanged for every other
// kind.  So the oracle's render_tile() and the render mirror's film and albedo passes render panoramas here, and the three
// reference cameras exactly as before.  The motion pass needs the panorama projection inside its per-lane rule, so
// rayn_pano_render_motion restates rayn_mirror_render_motion's driver and rule with it.
// Build flags: those of oracle/Makefile (-ffp-contract=off is required, see there).
#include <stdint.h>

#include "../include/rayn_b200.h"

namespace {
struct F4;
struct WRay;
WRay camera_get_rays(const RaynCamera& c, float scramble, uint32_t* sample_nums, uint32_t tx, uint32_t ty, F4 u, F4 v, F4 time, F4 ls0, F4 ls1);
}  // namespace

#include "render_mirror.cpp"

namespace {

// the oracle's camera packet, with camera_ray's equirectangular branch (include/rayn_b200.h) per lane for a panorama
WRay camera_get_rays(const RaynCamera& c, float scramble, uint32_t* sample_nums, uint32_t tx, uint32_t ty, F4 u, F4 v, F4 time, F4 ls0, F4 ls1) {
  const uint32_t* nums = sample_nums;
  WRay r = camera_get_rays(c, scramble, nums, tx, ty, u, v, time, ls0, ls1);
  if (c.kind != RAYN_CAMERA_EQUIRECTANGULAR) return r;
  const V3 origin = seq_v3(c.origin, c.origin_velocity, time), at = seq_v3(c.at, c.at_velocity, time), up = seq_v3(c.up, c.up_velocity, time);
  const V3 bw = normalized(origin - at);
  const V3 bu = normalized(cross(up, bw));
  const V3 bv = cross(bw, bu);
  F4 sp, cp, st, ct;
  f4sincos((u - splat(0.5f)) * splat(kTWO_PI), &sp, &cp);
  f4sincos((v - splat(0.5f)) * splat(kPI), &st, &ct);
  r.origin = origin;
  r.dir = normalized(bu * (ct * sp) + bv * st - bw * (ct * cp));
  return r;
}

// proj(X, time) of the motion-plane statement, per lane: the equirectangular branch, else the render mirror's project()
void project_any(const RaynCamera& c, int W, int H, V3 X, float time, F4* px, F4* py, F4* z) {
  if (c.kind != RAYN_CAMERA_EQUIRECTANGULAR) return project(c, W, H, X, time, px, py, z);
  const F4 t = splat(time);
  const V3 origin = seq_v3(c.origin, c.origin_velocity, t), at = seq_v3(c.at, c.at_velocity, t), up = seq_v3(c.up, c.up_velocity, t);
  const V3 r = X - origin;
  const V3 bw = normalized(origin - at);
  const V3 bu = normalized(cross(up, bw));
  const V3 bv = cross(bw, bu);
  const F4 xr = dot(r, bu), yr = dot(r, bv), zr = -dot(r, bw);
  *z = mag(r);
  *px = (f4atan2(xr, zr) / splat(kTWO_PI) + splat(0.5f)) * splat((float)W);
  *py = (f4atan2(yr, f4sqrt(xr * xr + zr * zr)) / splat(kPI) + splat(0.5f)) * splat((float)H);
}

// motion_records() of the render mirror with project_any(), and dx the short way round the seam for a panorama
void pano_motion_records(const World& w, const RaynSceneDesc* prev, int W, int H, float frame_dt, V3 P, float tau, const int* ids, float* rec[4]) {
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
  project_any(cam, W, H, P, tau, &px1, &py1, &z1);
  project_any(prev ? prev->camera : cam, W, H, V3{load4(ppx), load4(ppy), load4(ppz)}, tp, &px0, &py0, &z0);
  for (int i = 0; i < 4; ++i) {
    const bool valid = ids[i] >= 0 && (cam.kind == RAYN_CAMERA_ORTHOGRAPHIC || (z1[i] > 0.0f && z0[i] > 0.0f));
    float* out = rec[i];
    if (valid) {
      float dx = px0[i] - px1[i];
      if (cam.kind == RAYN_CAMERA_EQUIRECTANGULAR) {
        const float hw = (float)W * 0.5f;
        dx = dx > hw ? dx - (float)W : (dx < -hw ? dx + (float)W : dx);
      }
      out[0] = dx, out[1] = py0[i] - py1[i], out[2] = z1[i], out[3] = z0[i];
    } else {
      out[0] = 0.0f, out[1] = 0.0f, out[2] = NAN, out[3] = NAN;
    }
  }
}

// lanes of v that are inside [0, n) into p3 [3n]
void store_v3_lanes(float* p3, int64_t i, int64_t n, const V3& v) {
  alignas(16) float x[4], y[4], z[4];
  store4(x, v.x), store4(y, v.y), store4(z, v.z);
  for (int k = 0; k < 4 && i + k < n; ++k) p3[3 * (i + k)] = x[k], p3[3 * (i + k) + 1] = y[k], p3[3 * (i + k) + 2] = z[k];
}

}  // namespace

extern "C" {

// rayn_mirror_render_motion (same arguments and outputs) for any camera kind, the equirectangular one included
int32_t rayn_pano_render_motion(const RaynSceneDesc* scene, const RaynFrameDesc* f, float frame_dt, const RaynSceneDesc* prev, float* per_sample,
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
      pano_motion_records(w, prev, W, H, frame_dt, P, times[0], ids, rec);
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

// the camera packet's rays for n film positions (u, v) at one camera time (lane 0's, like every lane of a packet), lens samples
// 0.5 (the lens centre) -> ro3, rd3 [3n]
int32_t rayn_pano_kat_camera_rays(const RaynCamera* cam, int64_t n, const float* u, const float* v, float time, float* ro3, float* rd3) {
  if (!cam || n < 0 || !u || !v || !ro3 || !rd3) return RAYN_ERR_INVALID_ARG;
  uint32_t nums[4] = {0, 1, 2, 3};
  for (int64_t i = 0; i < n; i += 4) {
    const WRay r = camera_get_rays(*cam, 0.0f, nums, 0, 0, load_f_packet(u, i, n), load_f_packet(v, i, n), splat(time), splat(0.5f), splat(0.5f));
    store_v3_lanes(ro3, i, n, r.origin);
    store_v3_lanes(rd3, i, n, r.dir);
  }
  return RAYN_OK;
}

// proj(X, time) of the motion-plane statement for n points -> out3 [3n] (px, py, z per point)
int32_t rayn_pano_kat_project(const RaynCamera* cam, int32_t W, int32_t H, int64_t n, const float* points3, float time, float* out3) {
  if (!cam || n < 0 || !points3 || !out3) return RAYN_ERR_INVALID_ARG;
  for (int64_t i = 0; i < n; i += 4) {
    F4 px, py, z;
    project_any(*cam, W, H, load_v3_packet(points3, i, n), time, &px, &py, &z);
    store_v3_lanes(out3, i, n, V3{px, py, z});
  }
  return RAYN_OK;
}

}  // extern "C"
