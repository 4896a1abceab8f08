// rt_motion.cuh — the first-hit motion plane (rayn_b200_render_motion; the exact statement is in include/rayn_b200.h).
//
// The pass runs the render's own k_raygen and depth-0 closest-hit stage, like the albedo pass (rt_albedo.cuh), then:
//   k_motion_paths    one thread per path: the hit point projected at the previous and the current time, into a float4 per
//                     path of a pass buffer that is idle here (PassBufs::rad, which only the shading kernels read); with an
//                     albedo plane, also k_albedo_paths's value into PassBufs::nrm, so one march serves both guides;
//   k_motion_resolve  one thread per pixel: the sequential mean over the pixel's valid samples, in sample order.
// rayn_b200_render_motion_prev runs k_motion_paths_prev instead of k_motion_paths: the same body with the previous frame's
// camera and sphere centres (DevPrev) in place of the current scene run backwards.
#pragma once
#include "rt_albedo.cuh"

namespace rt {

// What rayn_b200_render_motion_prev reads of the previous frame's scene, in a 516-byte device buffer the call writes.  It is
// not a kernel parameter: k_motion_paths's block (DevScene, DevFrame, PassBufs, frame_dt) is 3844 bytes, and this would take
// it past the 4 KB that rt_kernels.cuh's scene limits are sized for.
struct DevPrev {
  RaynCamera cam;
  float center[RAYN_MAX_HITABLES][3];
  float velocity[RAYN_MAX_HITABLES][3];
  uint32_t still;  // bit j: hitable j is a sphere with a zero velocity in both scenes and the same centre bit for bit (P' = P)
};

// Film position (px, py) in pixels and view depth z of point X for camera c at `time`: the inverse of camera_ray's
// pixel -> (u, v) map (the thin lens through its lens centre).  The one projection both times go through.
RT_D void camera_project(const RaynCamera& c, int W, int H, f3 X, float time, float* px, float* py, float* z) {
  const f3 origin = seq3(c.origin, c.origin_velocity, time), at = seq3(c.at, c.at_velocity, time), up = seq3(c.up, c.up_velocity, time);
  const float hx = c.half_size[0], hy = c.half_size[1];
  const f3 r = X - origin;
  if (c.kind == RAYN_CAMERA_ORTHOGRAPHIC) {
    const f3 bw = normalized(at - origin);
    const f3 bu = normalized(cross(bw, up));
    const f3 bv = cross(bu, bw);
    *z = dot(r, bw);
    *px = ((dot(r, bu) + hx) / c.full_size[0]) * (float)W;
    *py = ((dot(r, bv) + hy) / c.full_size[1]) * (float)H;
  } else {
    const f3 bw = normalized(origin - at);
    const f3 bu = normalized(cross(up, bw));
    const f3 bv = cross(bw, bu);
    const float zz = -dot(r, bw);
    *z = zz;
    *px = ((dot(r, bu) / (zz * hx)) * 0.5f + 0.5f) * (float)W;
    *py = ((dot(r, bv) / (zz * hy)) * 0.5f + 0.5f) * (float)H;
  }
}

// Path g's record (dx, dy, z, z_prev), or (0, 0, NaN, NaN) for an invalid sample; with albedo, a_s as k_albedo_paths.
// kPrev: the previous projection and a sphere hit's previous position come from *pv (rayn_b200_render_motion_prev).
template <bool kAlb, bool kPrev>
RT_D void motion_path(const DevScene& sc, const DevFrame& fr, const PassBufs& pb, float frame_dt, const DevPrev* __restrict__ pv) {
  const int ts = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const TileGeom tg = tile_geom(fr, pb.tile_ids[ts]);
  if (i >= tg.npaths) return;
  const size_t g = (size_t)ts * pb.R + i;
  const int key = pb.q_key[g];
  float4 rec = make_float4(0.0f, 0.0f, __int_as_float(0x7fffffff), __int_as_float(0x7fffffff));
  f3 a = mk3(0.0f, 0.0f, 0.0f);
  if (key >= 0) {
    const RaynHitable& h = sc.hit[key];
    const float4 o4 = pb.o_time[g], d4 = pb.d_t[g];
    const f3 P = fma3s(mk3(d4.x, d4.y, d4.z), d4.w, mk3(o4.x, o4.y, o4.z));  // as k_albedo_paths / k_normals
    // lane 0 of the camera packet: its o_time.w is the time raygen evaluated the camera at (depth 0: nothing moved it)
    const float tau = (i & 3) ? pb.o_time[g - (i & 3)].w : o4.w;
    f3 Pp = P;
    if constexpr (kPrev) {  // P + (c_prev(tau - dt) - c(tau)), both centres as the extend stage forms them
      if (h.kind == RAYN_HITABLE_SPHERE && !((pv->still >> key) & 1u))
        Pp = P + (seq3(pv->center[key], pv->velocity[key], tau - frame_dt) - sphere_center(h, tau));
    } else {
      if (sphere_moves(h)) Pp = P - ld3(h.center_velocity) * frame_dt;
    }
    float px1, py1, z1, px0, py0, z0;
    camera_project(sc.cam, fr.W, fr.H, P, tau, &px1, &py1, &z1);
    camera_project(kPrev ? pv->cam : sc.cam, fr.W, fr.H, Pp, tau - frame_dt, &px0, &py0, &z0);
    if (sc.cam.kind == RAYN_CAMERA_ORTHOGRAPHIC || (z1 > 0.0f && z0 > 0.0f)) rec = make_float4(px0 - px1, py0 - py1, z1, z0);
    if (kAlb) {
      const RaynMaterial& mat = sc.mat[h.material];
      if (receives_light(mat)) {
        if ((sc.trap_mask >> h.material) & 1u) {
          float s = 1.0f;
          if (h.kind != RAYN_HITABLE_SPHERE) s = trap_coord(sc.trap[h.material], sdf_trap(h, P));
          a = trap_albedo(sc.trap[h.material], s);
        } else {
          a = ld3(mat.albedo);
        }
      }
    }
  }
  pb.rad[g] = rec;
  if (kAlb) pb.nrm[g] = make_float4(a.x, a.y, a.z, 0.0f);
}

template <bool kAlb>
__global__ void __launch_bounds__(256) k_motion_paths(const __grid_constant__ DevScene sc, const DevFrame fr, const PassBufs pb, float frame_dt) {
  motion_path<kAlb, false>(sc, fr, pb, frame_dt, nullptr);
}

// rayn_b200_render_motion_prev; its own kernel, so that k_motion_paths's parameter block and code stay as they are
template <bool kAlb>
__global__ void __launch_bounds__(256) k_motion_paths_prev(const __grid_constant__ DevScene sc, const DevFrame fr, const PassBufs pb, float frame_dt,
                                                           const DevPrev* __restrict__ pv) {
  motion_path<kAlb, true>(sc, fr, pb, frame_dt, pv);
}

// motion[4 pix + k] = (((+0 + r_a[k]) + r_b[k]) + ...) / (float)n over the pixel's valid samples (z not NaN), sample order;
// n = 0: (0, 0, +inf, +inf)
__global__ void __launch_bounds__(256) k_motion_resolve(const DevFrame fr, const PassBufs pb, const float4* __restrict__ rec, float* __restrict__ motion) {
  const int ts = blockIdx.y, pl = blockIdx.x * blockDim.x + threadIdx.x;
  const TileGeom tg = tile_geom(fr, pb.tile_ids[ts]);
  if (pl >= tg.tw * tg.th) return;
  const int xl = pl / tg.th, yl = pl - xl * tg.th;
  const size_t pix = (size_t)(tg.x0 + xl) + (size_t)(tg.y0 + yl) * fr.W;
  const float4* __restrict__ src = rec + (size_t)ts * pb.R + (size_t)pl * fr.spp;
  float sx = 0.0f, sy = 0.0f, sz = 0.0f, sp = 0.0f;
  int n = 0;
  for (int s = 0; s < fr.spp; ++s) {
    const float4 v = src[s];
    if (v.z != v.z) continue;
    sx += v.x;
    sy += v.y;
    sz += v.z;
    sp += v.w;
    ++n;
  }
  float* __restrict__ m = motion + 4 * pix;
  if (n == 0) {
    m[0] = 0.0f, m[1] = 0.0f, m[2] = INFINITY, m[3] = INFINITY;
  } else {
    const float div = (float)n;
    m[0] = sx / div, m[1] = sy / div, m[2] = sz / div, m[3] = sp / div;
  }
}

// pixels outside the tile grid: (0, 0, +inf, +inf)
__global__ void __launch_bounds__(256) k_motion_clear(long long npx, float* __restrict__ motion) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npx) return;
  float* __restrict__ m = motion + 4 * i;
  m[0] = 0.0f, m[1] = 0.0f, m[2] = INFINITY, m[3] = INFINITY;
}

}  // namespace rt
