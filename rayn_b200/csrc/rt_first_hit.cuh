// rt_first_hit.cuh — the first-hit passes: the albedo plane (rayn_b200_render_albedo) and the motion plane
// (rayn_b200_render_motion, rayn_b200_render_motion_prev); the exact statements are in include/rayn_b200.h.
//
// A pass runs the render's own k_raygen and depth-0 closest-hit stage (k_scan_live, k_extend_spheres / k_extend_march), so
// every path's q_key / d_t holds exactly the hit the render shades at depth 0.  Then:
//   k_first_hit_paths  one thread per path, into float4s per path of pass buffers that are idle here: the motion record
//                      (the hit point projected at the previous and the current time) into PassBufs::rad, which only the
//                      shading kernels read, and the albedo the hit's BSDF reads at depth 0 into PassBufs::nrm, which only
//                      k_normals writes, at a later stage; one march serves both guides;
//   k_motion_resolve   one thread per pixel: the sequential mean over the pixel's valid samples, in sample order;
//   k_albedo_resolve   one thread per pixel: the sequential sum of the pixel's spp contiguous paths, in sample order, / spp.
#pragma once
#include "rt_kernels.cuh"

namespace rt {

// What rayn_b200_render_motion_prev reads of the previous frame's scene, in a 516-byte device buffer the call writes.  It is
// not a kernel parameter: k_first_hit_paths's block without it (DevScene, DevFrame, PassBufs, frame_dt) is 3844 bytes, and
// this would take it past the 4 KB that rt_kernels.cuh's scene limits are sized for.
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
  } else if (c.kind == RAYN_CAMERA_EQUIRECTANGULAR) {  // z is the distance; px, py invert the angles of camera_ray
    const f3 bw = normalized(origin - at);
    const f3 bu = normalized(cross(up, bw));
    const f3 bv = cross(bw, bu);
    const float xr = dot(r, bu), yr = dot(r, bv), zr = -dot(r, bw);
    *z = mag(r);
    *px = (dm::atan2(xr, zr) / RT_TWO_PI + 0.5f) * (float)W;
    *py = (dm::atan2(yr, sqrtf(xr * xr + zr * zr)) / RT_PI + 0.5f) * (float)H;
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

// The albedo a_s of a depth-0 hit on h at point P (fma3s(d, t, o), the point k_normals evaluates): RaynMaterial.albedo, or
// the orbit-trap palette at s = trap_coord(trap(P)) (s = 1 on an analytic sphere); (0, 0, 0) for Sky / Emissive hits.  Only
// SDF hits whose material has a trap run the (scalar) trap evaluation.
RT_D f3 first_hit_albedo(const DevScene& sc, const RaynHitable& h, f3 P) {
  const RaynMaterial& mat = sc.mat[h.material];
  if (!receives_light(mat)) return mk3(0.0f, 0.0f, 0.0f);
  if (!((sc.trap_mask >> h.material) & 1u)) return ld3(mat.albedo);
  const float s = h.kind != RAYN_HITABLE_SPHERE ? trap_coord(sc.trap[h.material], sdf_trap(h, P)) : 1.0f;
  return trap_albedo(sc.trap[h.material], s);
}

// Path g's records.  kMotion: (dx, dy, z, z_prev) into pb.rad, or (0, 0, NaN, NaN) for an invalid sample; kPrev: the previous
// projection and a sphere hit's previous position come from *pv (rayn_b200_render_motion_prev), else from the uploaded scene
// run backwards.  kAlb: a_s into pb.nrm, (0, 0, 0) for rays that hit nothing.
template <bool kMotion, bool kAlb, bool kPrev>
__global__ void __launch_bounds__(256) k_first_hit_paths(const __grid_constant__ DevScene sc, const DevFrame fr, const PassBufs pb, float frame_dt,
                                                         const DevPrev* __restrict__ pv) {
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
    const f3 P = fma3s(mk3(d4.x, d4.y, d4.z), d4.w, mk3(o4.x, o4.y, o4.z));  // as k_normals
    if constexpr (kMotion) {
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
      if (sc.cam.kind == RAYN_CAMERA_ORTHOGRAPHIC || (z1 > 0.0f && z0 > 0.0f)) {
        float dx = px0 - px1;
        if (sc.cam.kind == RAYN_CAMERA_EQUIRECTANGULAR) {  // the short way round the seam
          const float hw = (float)fr.W * 0.5f;
          dx = dx > hw ? dx - (float)fr.W : (dx < -hw ? dx + (float)fr.W : dx);
        }
        rec = make_float4(dx, py0 - py1, z1, z0);
      }
    }
    if constexpr (kAlb) a = first_hit_albedo(sc, h, P);
  }
  if constexpr (kMotion) pb.rad[g] = rec;
  if constexpr (kAlb) pb.nrm[g] = make_float4(a.x, a.y, a.z, 0.0f);
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

// albedo[3 pix + c] = (((+0 + a_0[c]) + a_1[c]) + ...) / (float)spp over the pixel's paths pl*spp .. pl*spp + spp-1 (sample order)
__global__ void __launch_bounds__(256) k_albedo_resolve(const DevFrame fr, const PassBufs pb, const float4* __restrict__ a, float* __restrict__ albedo) {
  const int ts = blockIdx.y, pl = blockIdx.x * blockDim.x + threadIdx.x;
  const TileGeom tg = tile_geom(fr, pb.tile_ids[ts]);
  if (pl >= tg.tw * tg.th) return;
  const int xl = pl / tg.th, yl = pl - xl * tg.th;
  const size_t pix = (size_t)(tg.x0 + xl) + (size_t)(tg.y0 + yl) * fr.W;
  const float4* __restrict__ src = a + (size_t)ts * pb.R + (size_t)pl * fr.spp;
  float r = 0.0f, gr = 0.0f, b = 0.0f;
  for (int s = 0; s < fr.spp; ++s) {
    const float4 v = src[s];
    r += v.x;
    gr += v.y;
    b += v.z;
  }
  const float div = (float)fr.spp;
  albedo[3 * pix] = r / div;
  albedo[3 * pix + 1] = gr / div;
  albedo[3 * pix + 2] = b / div;
}

}  // namespace rt
