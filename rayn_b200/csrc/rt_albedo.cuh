// rt_albedo.cuh — the first-hit albedo plane (rayn_b200_render_albedo; the exact statement is in include/rayn_b200.h).
//
// The pass runs the render's own k_raygen and depth-0 closest-hit stage (k_scan_live, k_extend_spheres / k_extend_march),
// so every path's q_key / d_t holds exactly the hit the render shades at depth 0.  Then:
//   k_albedo_paths    one thread per path: the albedo the hit's BSDF reads at depth 0 (hit_albedo's rule), into a float4 per
//                     path of a pass buffer that is idle here (PassBufs::nrm, which only k_normals writes, at a later stage);
//   k_albedo_resolve  one thread per pixel: the sequential sum of the pixel's spp contiguous paths, in sample order, / spp.
#pragma once
#include "rt_kernels.cuh"

namespace rt {

// The albedo a_s of path g's depth-0 hit: RaynMaterial.albedo, or the orbit-trap palette at s = trap_coord(trap(p)) with p the
// point k_normals evaluates (s = 1 on an analytic sphere); (0, 0, 0) for Sky / Emissive hits and for rays that hit nothing.
// Only SDF hits whose material has a trap run the (scalar) trap evaluation.
__global__ void __launch_bounds__(256) k_albedo_paths(const __grid_constant__ DevScene sc, const DevFrame fr, const PassBufs pb, float4* __restrict__ out) {
  const int ts = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const TileGeom tg = tile_geom(fr, pb.tile_ids[ts]);
  if (i >= tg.npaths) return;
  const size_t g = (size_t)ts * pb.R + i;
  const int key = pb.q_key[g];
  f3 a = mk3(0.0f, 0.0f, 0.0f);
  if (key >= 0) {
    const RaynHitable& h = sc.hit[key];
    const RaynMaterial& mat = sc.mat[h.material];
    if (receives_light(mat)) {
      if ((sc.trap_mask >> h.material) & 1u) {
        float s = 1.0f;
        if (h.kind != RAYN_HITABLE_SPHERE) {
          const float4 o4 = pb.o_time[g], d4 = pb.d_t[g];
          const f3 point = fma3s(mk3(d4.x, d4.y, d4.z), d4.w, mk3(o4.x, o4.y, o4.z));  // as k_normals
          s = trap_coord(sc.trap[h.material], sdf_trap(h, point));
        }
        a = trap_albedo(sc.trap[h.material], s);
      } else {
        a = ld3(mat.albedo);
      }
    }
  }
  out[g] = make_float4(a.x, a.y, a.z, 0.0f);
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
