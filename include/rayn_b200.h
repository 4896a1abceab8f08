/*
 * rayn_b200.h — C ABI of the H100-native wavefront path tracer that replaces the
 * render hot path of fu5ha/rayn (reference @ 6486a86).
 *
 * The ONE reference call this boundary replaces is
 *     Film::render_frame_into(world, camera, integrator, filter, tile_size,
 *                             frame, time_range, samples)
 * (reference src/film.rs:382-395, called once per frame from src/main.rs:64-73).
 *
 * The reference has no FFI: its extension surface is Rust traits with `dyn` objects
 * (src/hitable.rs:8-18, src/material.rs:11-38, src/light.rs:5-17, src/camera.rs:5-19).
 * Trait objects cannot cross to a GPU, so every trait implementor the reference ships
 * becomes a tagged plain-old-data descriptor here.  Insertion ORDER of hitables,
 * materials and lights is semantic (closest-hit fold order src/hitable.rs:177-198,
 * bin order src/hitable.rs:116-133) and is preserved.
 *
 * Everything is plain C: fixed-width ints, floats, pointers and sizes.  No exception
 * ever unwinds across this boundary; every call returns a status code
 * (the reference panics / unwraps instead: src/main.rs:32,45,96, src/film.rs:127,667).
 *
 * A Rust `extern "C"` block for this header is mechanical; INTEGRATION.md shows it.
 */
#ifndef RAYN_B200_H
#define RAYN_B200_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RAYN_B200_ABI_VERSION 2

/* ---- limits (fixed so the scene fits a kernel-parameter block) -------------------
 * CONTRACT CHANGE vs the reference: its stores are unbounded `Vec<Box<dyn ..>>` (src/hitable.rs:143,
 * src/material.rs:58, src/world.rs:7-13).  Here the whole scene rides in the 4 KB kernel-parameter constant bank
 * (warp-uniform operands then cost no load), which caps the counts; setup.rs needs 7 / 4 / 5.  upload_scene returns
 * RAYN_ERR_INVALID_ARG beyond these.                                                                              */
#define RAYN_MAX_HITABLES 16
#define RAYN_MAX_MATERIALS 16
#define RAYN_MAX_LIGHTS 16
#define RAYN_FIS_TABLE_SIZE 512 /* FILTER_TABLE_SIZE, src/filter.rs:187 */

/* ---- status codes ---------------------------------------------------------------- */
typedef enum RaynStatus {
  RAYN_OK = 0,
  RAYN_ERR_INVALID_ARG = 1,
  RAYN_ERR_UNSUPPORTED = 2, /* representable in rayn, not in this build (e.g. vm != 2)   */
  RAYN_ERR_CUDA = 3,
  RAYN_ERR_OOM = 4,
  RAYN_ERR_NO_SCENE = 5,
  RAYN_ERR_NO_DEVICE = 6,
  RAYN_ERR_NCCL = 7      /* NCCL missing (dlopen) or a collective failed                    */
} RaynStatus;

/* ---- Hitable (src/hitable.rs:8-18) ------------------------------------------------ */
typedef enum RaynHitableKind {
  RAYN_HITABLE_SPHERE = 0,     /* Sphere<TR>, src/sphere.rs:7-21 (constant centre)          */
  RAYN_HITABLE_MANDELBOX = 1,  /* TracedSDF<MandelBox>, src/sdf.rs:12-23,104-141            */
  RAYN_HITABLE_MANDELBULB = 2  /* TracedSDF<Mandelbulb>: AUTHORED here, not in the reference */
} RaynHitableKind;

typedef struct RaynHitable {
  int32_t kind;     /* RaynHitableKind                                                     */
  int32_t material; /* MaterialHandle, index into materials[] (src/material.rs:55-56)      */
  /* Sphere::new(centre, radius, material), src/sphere.rs:14-20                            */
  float center[3];
  float radius;
  /* MandelBox::new(iterations, BoxFold::new(l), SphereFold::new(min_r, fixed_r), scale),
   * src/sdf.rs:113-123,150-158,171-179.  The two radii are stored SQUARED, computed by the
   * host in f32 exactly as SphereFold::new does (src/sdf.rs:173-174).                     */
  int32_t iterations;
  float box_l;
  float min_rad_sq;
  float fixed_rad_sq;
  float scale;
  /* Mandelbulb (authored): power is fixed to 8 in this build; bailout radius.             */
  int32_t bulb_power;
  float bulb_bailout;
  /* Sphere<TR> with a time-varying centre (SURVEY §8f rank 4): centre(t) = center + center_velocity * t,
   * i.e. what the closure `|t| center + velocity * t` gives through `impl WSequenced<Wec3> for Fn(f32)->Vec3`
   * (src/animation.rs:62-67) - which evaluates the closure at LANE 0's time for the whole 4-lane packet.
   * All-zero velocity = the constant `impl_inherent_wsequenced` path (animation.rs:52).               */
  float center_velocity[3];
} RaynHitable;

/* ---- Material / BSDF (src/material.rs:11-38) -------------------------------------- */
typedef enum RaynMaterialKind {
  RAYN_MATERIAL_LAMBERTIAN = 0, /* src/material.rs:86-142                                   */
  RAYN_MATERIAL_DIELECTRIC = 1, /* src/material.rs:144-257; roughness = REMAPPED exponent   */
  RAYN_MATERIAL_SKY = 2,        /* src/material.rs:394-449                                  */
  RAYN_MATERIAL_EMISSIVE = 3    /* src/material.rs:451-520                                  */
} RaynMaterialKind;

typedef struct RaynMaterial {
  int32_t kind;
  float albedo[3];     /* Lambertian / Dielectric                                          */
  float roughness;     /* Dielectric: the Phong exponent AFTER new_remap (material.rs:167-174) */
  float sky_top[3];    /* Sky::new(top, bottom)                                            */
  float sky_bottom[3];
  float emission[3];   /* Emissive::new_splat                                              */
} RaynMaterial;

/* ---- Orbit-trap albedo: a per-hit albedo generator for SDF surfaces -----------------------------------------------
 * rayn's Lambertian<AG> and Dielectric<AG, RG> take an `albedo_gen: WShadingParamGenerator<WSrgb>` evaluated per shading
 * point (material.rs:75-83,91-115,150-192); RaynMaterial.albedo is its constant implementor.  This is the one other
 * generator kind built here: an orbit-trap palette, the classic way of colouring fractal surfaces.  Exact statement, in
 * float, no contraction:
 *   point   p = fma3s(d, t, o) of the hit: the point whose normal get_shading_info estimates (sdf.rs:85-101)
 *   trap    trap(h, p) starts at +inf and folds trap = (x < trap) ? x : trap (a NaN never replaces it), where x is
 *     Mandelbox:  for each iteration MandelBox::dist runs at p, r2 = mag_sq of the box-folded point (ultraviolet dot with
 *                 the build's mul_add: mul_add(x, x, mul_add(y, y, z * z))), before the min_rad_sq clamp (sdf.rs:181-187)
 *     Mandelbulb: every m = dot(w, w) the estimator assigns: m = dot(p, p) at the start, then the m of each iteration it
 *                 runs before bailout (iteration i runs while i < iterations && !(m > bailout^2))
 *     iterations = 0 (either fractal): trap = +inf
 *   palette s = !(trap > trap_lo) ? 0 : (trap >= trap_hi ? 1 : (trap - trap_lo) / (trap_hi - trap_lo));
 *           a hit on an analytic sphere whose material has a trap has s = 1 (no orbit)
 *   albedo  albedo[c] = albedo_lo[c] * (1 - s) + albedo_hi[c] * s, with (1 - s) computed once
 * The albedo replaces RaynMaterial.albedo wherever that hit's BSDF reads it: the Lambertian f and scatter f, and the
 * Dielectric diffuse term of f (next-event estimation) and of scatter.  Normals, offsets, sample dimensions, packet
 * composition, light choice and the alpha / normal channels do not change; trap evaluations are not counted in
 * RaynStats.sdf_evals_normals.                                                                                      */
typedef struct RaynAlbedoTrap {
  int32_t material;                 /* index into the uploaded scene's materials: LAMBERTIAN or DIELECTRIC, one entry per material */
  float trap_lo, trap_hi;           /* finite, trap_lo < trap_hi                                                                   */
  float albedo_lo[3], albedo_hi[3]; /* finite                                                                                      */
} RaynAlbedoTrap;

/* ---- Light (src/light.rs:5-17): SphereLight::new(pos, rad, emission) :27-34 -------- */
typedef struct RaynLight {
  float pos[3];
  float rad;
  float emission[3];
} RaynLight;

/* ---- Camera (src/camera.rs:5-19) --------------------------------------------------- */
typedef enum RaynCameraKind {
  RAYN_CAMERA_PINHOLE = 0,     /* src/camera.rs:42-119  */
  RAYN_CAMERA_THINLENS = 1,    /* src/camera.rs:121-213 */
  RAYN_CAMERA_ORTHOGRAPHIC = 2 /* src/camera.rs:215-285 */
} RaynCameraKind;

/* The derived fields are what the reference constructors store (camera.rs:52-72,
 * 133-157,227-241); the HOST computes them (tan etc. are host-side f32 libm there too),
 * so they are inputs on both sides of a parity comparison.                               */
typedef struct RaynCamera {
  int32_t kind;
  float half_size[2];    /* (half_width, half_height)                                      */
  float full_size[2];    /* orthographic only                                              */
  float half_pixel_size; /* half_height / res.y, or pixel_size / 2 for orthographic        */
  float origin[3];
  float at[3];
  float up[3];
  float focus[3];        /* thin lens: focus point                                         */
  float aperture;        /* thin lens                                                      */
  /* linear-in-time camera parameters, same closure semantics as RaynHitable.center_velocity
   * (camera.rs:90-92,177-182,258-260 sample origin/at/up/focus at the packet's time): a closure-backed
   * WSequenced<Wec3> is evaluated at LANE 0's time (animation.rs:62-67).                                  */
  float origin_velocity[3];
  float at_velocity[3];
  float up_velocity[3];
  float focus_velocity[3];
  /* EXTENSION, no reference counterpart: aperture(t) = aperture + aperture_rate * t0 (lane-0 time).  The reference
   * implements closure-backed WSequenced only for Fn(f32)->Vec3; an f32 parameter can only be a constant there
   * (impl_wsequenced_for_sequenced, animation.rs:51-53).  Keep 0 for reference behaviour.                       */
  float aperture_rate;
} RaynCamera;

/* ---- VolumeParams (src/volume.rs:2-5): Option<f32> pairs --------------------------- */
typedef struct RaynVolume {
  int32_t has_scattering;
  float coeff_scattering;
  int32_t has_extinction;
  float coeff_extinction;
} RaynVolume;

/* ---- compile-time constants of the reference that leak into the hot path ----------- */
typedef struct RaynRenderConsts {
  float world_radius;      /* WORLD_RADIUS, src/setup.rs:33 (t_max = 2x, film.rs:556)      */
  float sdf_detail_scale;  /* SDF_DETAIL_SCALE, src/setup.rs:37                            */
  int32_t max_marches;     /* MAX_MARCHES = 256, src/sdf.rs:9                              */
  int32_t max_vis_marches; /* MAX_VIS_MARCHES = 100, src/sdf.rs:10                         */
} RaynRenderConsts;

/* ---- World (src/world.rs:7-13) + the selected camera ------------------------------- */
typedef struct RaynSceneDesc {
  int32_t n_hitables;
  const RaynHitable* hitables;
  int32_t n_materials;
  const RaynMaterial* materials;
  int32_t n_lights;
  const RaynLight* lights;
  RaynCamera camera;
  RaynVolume volume;
  RaynRenderConsts consts;
} RaynSceneDesc;

typedef enum RaynMemSpace { RAYN_MEM_HOST = 0, RAYN_MEM_DEVICE = 1 } RaynMemSpace;

/* ---- one call of render_frame_into (src/film.rs:382-395) --------------------------- */
typedef struct RaynFrameDesc {
  int32_t width, height;   /* Film.res                                                     */
  int32_t tile_w, tile_h;  /* tile_size; main.rs passes 16x16                              */
  int32_t samples;         /* SAMPLES; spp = 4*samples (film.rs:439,463-464)               */
  int32_t max_bounces;     /* PathTracingIntegrator.max_bounces (integrator.rs:33-36)      */
  int32_t volume_marches;  /* must be 2: samples_1d[3],[4] are hard-wired (integrator.rs:138,175) */
  int32_t frame;           /* only labels the sample tables here                           */
  float t0, t1;            /* time_range (film.rs:390,454,509-512)                         */
  /* Host-owned sampler state (src/sampler.rs:11-15), passed so seeds match by construction */
  int32_t sets_1d;         /* >= 1 + (mb+1)*(3+vm)   (film.rs:431, integrator.rs:39-41)    */
  int32_t sets_2d;         /* >= 2 + (mb+1)*(12+8vm) (film.rs:432, integrator.rs:43-45)    */
  const float* samples_1d; /* [spp * sets_1d]                                              */
  const float* samples_2d; /* [2 * spp * sets_2d]                                          */
  const float* scramble;   /* [width*height], per-pixel Cranley-Patterson shift (film.rs:460-461) */
  const float* fis_inverse_cdf; /* [512], FilterImportanceSampler (filter.rs:189-218)      */
  int32_t input_space;     /* RaynMemSpace of the four pointers above                      */
  /* multi-GPU sharding: this call renders tiles with (tile_index % tile_stride) == tile_offset,
   * tile_index = tile_x * n_tiles_y + tile_y (film.rs:401-425).  1-GPU: stride 1, offset 0. */
  int32_t tile_offset;
  int32_t tile_stride;
  /* optional explicit shard: if tile_list != NULL (HOST pointer, n_tile_list entries, each a
   * tile_index, ascending) it replaces offset/stride.  Lets the host pick any interleave,
   * e.g. the diagonal (tile_x + tile_y) % N that balances centre-weighted fractal scenes.      */
  const int32_t* tile_list;
  int32_t n_tile_list;
} RaynFrameDesc;

/* ---- Film channel planes (src/film.rs:103-120), row-major, y up, already / spp ------
 * Any plane pointer may be NULL: that channel is not written, like a Film<N> created without it
 * (film.rs:175-203; add_sample ignores absent channels, film.rs:167-172).                  */
typedef struct RaynFilmPlanes {
  float* color;      /* [3*W*H] Srgb                                                       */
  float* alpha;      /* [W*H]                                                              */
  float* background; /* [3*W*H]                                                            */
  float* normal;     /* [3*W*H] WorldNormal                                                */
  int32_t space;     /* RaynMemSpace                                                       */
} RaynFilmPlanes;

typedef struct RaynConfig {
  int32_t device;            /* CUDA device ordinal                                        */
  int64_t max_paths_per_pass;/* queue capacity in paths; 0 = default                       */
  int32_t flags;             /* RAYN_FLAG_*                                                */
} RaynConfig;

#define RAYN_FLAG_TIMING 1       /* record per-kernel CUDA-event times into RaynStats      */
#define RAYN_FLAG_SIMPLE_MARCH 2 /* TEST BUILD ONLY (-DRAYN_LEGACY_KERNELS, librayn_b200_legacy.so): round-1 v0
                                    one-thread-per-ray kernels; RAYN_ERR_UNSUPPORTED in the product library */

#define RAYN_FLAG_NO_FOLD_ALL 64 /* keep the closest-hit fold in insertion order even for [spheres] Mandelbox [spheres] scenes  */
#define RAYN_FLAG_NO_DIV3 32     /* never select the three-operation sphere-fold division (see rayn_b200_debug_sdf_variant) */
#define RAYN_FLAG_NO_GRAPH 16    /* launch every kernel directly; by default small single-pass frames (launch bound) are
                                    captured once into a CUDA graph and replayed with one launch                */

#define RAYN_STAT_KERNELS 12
typedef struct RaynStats {
  int64_t launches;                 /* kernels launched by the last render call            */
  int64_t passes;                   /* tile passes                                         */
  int64_t paths;                    /* camera paths generated = samples rendered           */
  int64_t extend_rays;              /* rays through K2 (closest hit), all depths           */
  int64_t shade_lanes;              /* valid lanes shaded, all depths                      */
  int64_t shadow_rays;              /* shadow segments tested (K5)                         */
  int64_t sdf_evals_extend;         /* SDF dist() evaluations inside K2                    */
  int64_t sdf_evals_shadow;         /* SDF dist() evaluations inside K5                    */
  float kernel_ms[RAYN_STAT_KERNELS];   /* RAYN_FLAG_TIMING: summed device ms per kernel   */
  int64_t kernel_launches[RAYN_STAT_KERNELS];
  float total_ms;                   /* device ms of the last render call (events)          */
  int64_t sdf_evals_normals;        /* SDF dist() evaluations of get_shading_info (4 per SDF shading lane) */
  int64_t bulb_iters_extend;        /* Mandelbulb iterations actually run inside K2 (data dependent)       */
  int64_t bulb_iters_shadow;        /* ... inside K5                                                       */
  int64_t reserved_;                /* 1 when the last frame ran as ONE CUDA-graph launch (captured or replayed) */
  int64_t march_trips_extend;       /* warp-level distance-evaluation trips of K2: sdf_evals_extend / (64 * trips) = busy march slots */
  int64_t march_trips_shadow;       /* ... of K5                                                                                      */
} RaynStats;

/* indices into kernel_ms / kernel_launches */
enum {
  RAYN_K_RAYGEN = 0,
  RAYN_K_EXTEND = 1,
  RAYN_K_BIN = 2,
  RAYN_K_SHADE_PRE = 3,
  RAYN_K_SHADOW = 4,
  RAYN_K_SHADE_POST = 5,
  RAYN_K_COMPACT = 6,
  RAYN_K_RESOLVE = 7,
  RAYN_K_MISC = 8,
  RAYN_K_NORMALS = 9,
  RAYN_K_EXTEND_SPHERES = 10,
  RAYN_K_GATHER = 11
};

typedef struct RaynContext RaynContext;

/* ---- lifecycle --------------------------------------------------------------------- */
int32_t rayn_b200_abi_version(void);
/* 1 if this library was built with `wide` f32x4::mul_add FUSED (rayn built with -C target-feature=+fma), 0 for the
 * default: unfused, what a stock `cargo run --release` of the reference produces (oracle/README.md A6).          */
int32_t rayn_b200_muladd_fused(void);
int32_t rayn_b200_create(const RaynConfig* cfg, RaynContext** out_ctx);
void rayn_b200_destroy(RaynContext* ctx);
const char* rayn_b200_last_error(const RaynContext* ctx); /* ctx may be NULL: global slot */

/* World -> device.  Replaces the `&world` argument of film.rs:384.                      */
int32_t rayn_b200_upload_scene(RaynContext* ctx, const RaynSceneDesc* scene);
/* Replaces the orbit-trap list of the current scene (n = 0 clears it; traps may be NULL then).  upload_scene clears it,
 * so a caller that never calls this renders exactly as before.  RAYN_ERR_NO_SCENE before an upload; RAYN_ERR_INVALID_ARG
 * for a bad entry (material index out of range, Sky / Emissive material, duplicate material, n < 0 or
 * > RAYN_MAX_MATERIALS, non-finite value, trap_lo >= trap_hi); the list is unchanged then.  Render calls with
 * RAYN_FLAG_SIMPLE_MARCH (legacy test kernels) and a non-empty list return RAYN_ERR_UNSUPPORTED.                     */
int32_t rayn_b200_set_albedo_traps(RaynContext* ctx, int32_t n, const RaynAlbedoTrap* traps);

/* The drop-in for Film::render_frame_into (film.rs:382-628) + tile_finished (:660-691).
 * Host pointers: inputs are copied H2D and planes D2H inside the call.
 * Device pointers: nothing is copied; planes are written in place on the device.        */
int32_t rayn_b200_render_frame(RaynContext* ctx, const RaynFrameDesc* frame,
                               const RaynFilmPlanes* out);

int32_t rayn_b200_get_stats(const RaynContext* ctx, RaynStats* out);

/* ---- luminance second moments: a variance AOV (rayn_b200_film_denoise_variance, or an external filter) ----------------
 * rayn_b200_render_frame plus two planes [W*H] (row-major, y up) in memory space `space`, which must equal out->space.
 * In float, no contraction, with every product rounded on its own:
 *   lum(v) = (0.2126f*v0 + 0.7152f*v1) + 0.0722f*v2
 *   color_lum2 = (((+0 + lum(x_0)*lum(x_0)) + lum(x_1)*lum(x_1)) + ...) / (float)spp
 * for every pixel of the tile grid (film.rs:399-404), the sum over the pixel's Color samples x_k in the order the film adds its
 * Color samples (the reference's wavefront order, the order of the colour sums); background_lum2 the same over its Background
 * samples.  Pixels outside the tile grid are 0 (device planes are cleared there, like the film planes).  A path adds at most
 * one Color or Background sample, so this is the mean over the spp paths of the squared path luminance (0 for a path that
 * added none): a film channel that adds like the others, so films of different sample counts combine by weighted averaging;
 * with the film's mean and spp it gives the variance.  The film planes equal render_frame's bit for bit.  Any plane pointer
 * of `out` or `moments` may be NULL, but not all six.  The tile selection, graph capture and asynchrony rules are render_frame's.
 * RAYN_FLAG_SIMPLE_MARCH: RAYN_ERR_UNSUPPORTED.                                                                           */
typedef struct RaynMomentPlanes {
  float* color_lum2;      /* [W*H] */
  float* background_lum2; /* [W*H] */
  int32_t space;          /* RaynMemSpace */
} RaynMomentPlanes;
int32_t rayn_b200_render_frame_moments(RaynContext* ctx, const RaynFrameDesc* frame, const RaynFilmPlanes* out,
                                       const RaynMomentPlanes* moments);

/* ---- first-hit albedo plane: an AOV for denoisers (rayn_b200_film_denoise_albedo, or an external one beside the
 * normal plane) -----------------------------------------------------------------------------------------------------
 * albedo[3*W*H] (row-major, y up, like the film planes) in memory space `space` (RaynMemSpace).  In float, no contraction:
 * for every pixel of the tile grid (film.rs:399-404) and every camera sample s = 0..spp-1 (spp = 4*frame->samples), the
 * ray render_frame generates for that sample (same tables, scramble, filter, time and lens; the camera takes the time of
 * lane 0 of its 4-sample packet) is traced to its closest hit with the DEPTH-0 fold of render_frame (hitable.rs:170-198,
 * threshold film.rs:540-551), which is render_frame's depth-0 hit exactly (moving spheres at lane 0's time of the extend
 * packet, which at depth 0 is samples 4k..4k+3 of the pixel).  Its albedo a_s is
 *   Lambertian or Dielectric hit: the albedo the BSDF reads at depth 0, i.e. RaynMaterial.albedo, or for a material with
 *     an orbit trap lo*(1 - s') + hi*s' (RaynAlbedoTrap) with s' = trap_coord(trap(p)), p = dir.mul_add(t, origin) the hit
 *     point (ray.rs:22-24), s' = 1 on an analytic sphere;
 *   Sky or Emissive hit, or nothing hit: (0, 0, 0).
 * albedo[3p+c] = (((+0 + a_0[c]) + a_1[c]) + ... + a_{spp-1}[c]) / (float)spp, summed in ascending sample order; pixels
 * outside the tile grid are 0.  frame->tile_list / tile_offset / tile_stride are ignored (the whole grid is rendered); all
 * other frame checks are render_frame's.  RAYN_FLAG_SIMPLE_MARCH: RAYN_ERR_UNSUPPORTED.  Synchronous; replaces RaynStats
 * like a render (k_first_hit_paths counts under RAYN_K_NORMALS, k_albedo_resolve under RAYN_K_RESOLVE); never captured
 * into a CUDA graph, and later renders are unaffected.
 * Property (tested): if every Lambertian / Dielectric material has albedo (1, 1, 1) and there are no traps, every channel
 * equals render_frame's alpha plane bit for bit, for the same frame: alpha is nA / spp with nA the count of depth-0
 * Lambertian / Dielectric hits, and a sum of nA ones is nA exactly.                                                 */
int32_t rayn_b200_render_albedo(RaynContext* ctx, const RaynFrameDesc* frame, float* albedo /* [3*W*H] */, int32_t space);

/* ---- screen-space motion of the first hit: the reprojection input of rayn_b200_temporal_push ----------------------------
 * motion[4*W*H] (row-major, y up; per pixel dx, dy, z, z_prev) and optionally albedo[3*W*H], both in memory space `space`.
 * Every camera sample s of a pixel of the tile grid is traced to render_frame's depth-0 hit exactly as in
 * rayn_b200_render_albedo (same rays, same fold; frame->tile_list / tile_offset / tile_stride are ignored).  With tau the
 * time of lane 0 of the sample's camera packet (the time raygen evaluates the camera at), in float, no contraction beyond the
 * build's mul_add (fma3s / dot / cross / normalized of rt_device.cuh):
 *   P  = fma3s(d, t, o)                                     the hit point, as rayn_b200_render_albedo forms it
 *   P' = (P.x - v.x*frame_dt, P.y - v.y*frame_dt, P.z - v.z*frame_dt)   if the hit is a sphere with a non-zero
 *        center_velocity v (each product rounded on its own); P' = P otherwise
 *   proj(X, time) with the scene camera's origin, at, up evaluated at `time` as camera_ray does (a zero velocity keeps the
 *        base value itself) and r = X - origin:
 *     pinhole / thin lens (through the lens centre): bw = normalized(origin - at), bu = normalized(cross(up, bw)),
 *        bv = cross(bw, bu), z = -dot(r, bw), px = ((dot(r, bu) / (z * hx)) * 0.5f + 0.5f) * (float)W,
 *        py = ((dot(r, bv) / (z * hy)) * 0.5f + 0.5f) * (float)H
 *     orthographic: bw = normalized(at - origin), bu = normalized(cross(bw, up)), bv = cross(bu, bw), z = dot(r, bw),
 *        px = ((dot(r, bu) + hx) / full_size[0]) * (float)W, py = ((dot(r, bv) + hy) / full_size[1]) * (float)H
 *     (hx, hy = half_size): the inverse of camera_ray's pixel -> (u, v) map, px = u * W, in film pixels
 *   (px1, py1, z)      = proj(P, tau),  (px0, py0, z_prev) = proj(P', tau - frame_dt)
 *   the sample is VALID if it hit something and, for a pinhole / thin-lens camera, z > 0 and z_prev > 0; its record is
 *   (px0 - px1, py0 - py1, z, z_prev), and an invalid sample's record is (0, 0, NaN, NaN) (so a NaN z also counts invalid).
 * motion[4p + k] = (((+0 + r_a[k]) + r_b[k]) + ...) / (float)n over the n valid samples of the pixel in ascending sample
 * order; a pixel with n = 0, or outside the tile grid, is (0, 0, +inf, +inf), which never matches a history tap.
 * Both projections are the same function, so a static camera and a static scene give dx = dy = +0 and z_prev == z exactly
 * (tested).  If albedo != NULL it is rayn_b200_render_albedo's plane for the same frame, bit for bit, from the same march.
 * frame_dt must be finite.  RAYN_FLAG_SIMPLE_MARCH: RAYN_ERR_UNSUPPORTED.  Synchronous; stats and graph rules are
 * rayn_b200_render_albedo's (k_first_hit_paths counts under RAYN_K_NORMALS, k_motion_resolve under RAYN_K_RESOLVE).       */
int32_t rayn_b200_render_motion(RaynContext* ctx, const RaynFrameDesc* frame, float frame_dt, float* motion /* [4*W*H] */,
                                float* albedo /* [3*W*H] or NULL */, int32_t space);

/* ---- screen-space motion against the previous frame's scene: animation that is not one linear scene ------------------------
 * rayn_b200_render_motion measures motion by running the uploaded scene backwards, which is exact only when one upload
 * describes the whole sequence.  A host that uploads a new scene per frame (curved camera paths, closures sampled per frame,
 * an interactive camera) passes here the scene `prev` that frame k-1 was rendered with.  The call reads only prev->camera
 * and prev->hitables[j].kind, .center and .center_velocity.  Everything is rayn_b200_render_motion's statement (same rays,
 * fold, tau, validity, records and resolve; albedo as there), except the previous position and projection:
 *   P' = P + (c_prev_j(tau - frame_dt) - c_j(tau))   for a hit on sphere hitable j, each operation rounded on its own, with
 *        c_j(t) = seq(center, center_velocity, t) of the uploaded hitable and c_prev_j that of prev's, each formed as the
 *        extend stage forms a sphere centre: base + v*t per component (product, then sum, each rounded), or the base itself
 *        if v is zero; tau - frame_dt is rounded once and used for both the centre and the camera;
 *   P' = P   for an SDF hit (there is no SDF motion), and for a sphere whose velocity is zero in both scenes and whose centres
 *        are equal bit for bit;
 *   (px0, py0, z_prev) = proj(P', tau - frame_dt) with prev->camera in place of the scene camera: its origin, at and up
 *        evaluated at tau - frame_dt as camera_ray does, and its own half_size / full_size, so a zoom between frames
 *        reprojects correctly; (px1, py1, z) = proj(P, tau) with the uploaded camera, as in rayn_b200_render_motion.
 * Identity (tested): if prev describes the uploaded scene and no sphere moves, the plane equals rayn_b200_render_motion's bit
 * for bit, since both projections are then the same function of the same operands.  A moving sphere whose linear parameters
 * are unchanged still moves: its hits differ from rayn_b200_render_motion's only by rounding (c(tau - frame_dt) - c(tau)
 * against -v*frame_dt).
 * RAYN_ERR_INVALID_ARG: prev NULL, prev->hitables NULL, a non-finite frame_dt, prev->n_hitables different from the uploaded
 * scene's, a hitable kind that differs, or a camera kind that differs (a cut to another camera type is a history reset, not
 * motion).  RAYN_FLAG_SIMPLE_MARCH: RAYN_ERR_UNSUPPORTED.  Synchronous; stats and graph rules are rayn_b200_render_motion's
 * (k_first_hit_paths counts under RAYN_K_NORMALS).                                                                           */
int32_t rayn_b200_render_motion_prev(RaynContext* ctx, const RaynFrameDesc* frame, float frame_dt, const RaynSceneDesc* prev,
                                     float* motion /* [4*W*H] */, float* albedo /* [3*W*H] or NULL */, int32_t space);

/* ---- multi-GPU: film tiles shard across GPUs, NCCL only for the final film gather -------------------------
 * The reference's only parallelism is one rayon task per tile over shared read-only state (film.rs:640-649); the
 * multi-GPU form of that is one context per GPU, each rendering the tiles `(tile_x + tile_y) % world == rank`
 * (interleaved: fractal scenes are centre-weighted), and ONE all-gather of dense tile slabs at the end of the frame.
 * The context owns the NCCL communicator (SURVEY §8b "Threading"):
 *   one process per GPU : rank 0 calls comm_unique_id, the host distributes the 128 bytes by any means, every rank
 *                         calls comm_init_rank on its context;
 *   one process, n GPUs : comm_init_all(ctxs, n)  (ncclCommInitAll), then render_frame_multi.
 * NCCL is dlopen()ed ("libnccl.so.2") at the first comm call: the library has no link-time NCCL dependency.      */
#define RAYN_COMM_ID_BYTES 128
int32_t rayn_b200_comm_unique_id(uint8_t out_id[RAYN_COMM_ID_BYTES]);
int32_t rayn_b200_comm_init_rank(RaynContext* ctx, const uint8_t id[RAYN_COMM_ID_BYTES], int32_t rank, int32_t world);
int32_t rayn_b200_comm_init_all(RaynContext* const* ctxs, int32_t n);
int32_t rayn_b200_comm_destroy(RaynContext* ctx);
int32_t rayn_b200_comm_info(const RaynContext* ctx, int32_t* rank, int32_t* world); /* world 0 = no communicator */
/* the shard of `rank`: ascending tile indices with (tile_x + tile_y) % world == rank.  Returns the count (or the
 * needed capacity if cap is too small / out is NULL); < 0 on bad arguments.  Pure host arithmetic.                */
int32_t rayn_b200_shard_tiles(int32_t width, int32_t height, int32_t tile_w, int32_t tile_h, int32_t rank,
                              int32_t world, int32_t* out, int32_t cap);
/* render_frame for a context that holds a communicator: renders this rank's shard (frame->tile_list / tile_offset /
 * tile_stride are ignored), then all-gathers, so EVERY rank ends with the complete film in `out`, bit-identical to
 * the 1-GPU film.  Pack, ncclAllGather and unpack are enqueued on the render stream: no host synchronisation
 * between render and gather.  DEVICE planes must be non-NULL for all four channels.                               */
int32_t rayn_b200_render_frame_sharded(RaynContext* ctx, const RaynFrameDesc* frame, const RaynFilmPlanes* out);
/* the gather alone, for planes already rendered with the rank's shard (device pointers, asynchronous on the context's
 * stream; rayn_b200_sync waits).                                                                                  */
int32_t rayn_b200_film_gather(RaynContext* ctx, int32_t width, int32_t height, int32_t tile_w, int32_t tile_h,
                              const RaynFilmPlanes* planes_dev);
int32_t rayn_b200_sync(RaynContext* ctx);
/* one process driving n GPUs (contexts from comm_init_all, same scene uploaded to each): renders all shards
 * concurrently, gathers, and returns the film of ctxs[0] in `out` (HOST planes).  frame inputs must be HOST pointers. */
int32_t rayn_b200_render_frame_multi(RaynContext* const* ctxs, int32_t n, const RaynFrameDesc* frame,
                                     const RaynFilmPlanes* out);

/* ---- explicit slab helpers (device pointers): what the gather is made of; kept for hosts that bring their own
 * transport.  pack: copies the listed tiles out of full-size planes into a dense slab
 *       [n_tiles][10][tile_w*tile_h] (channel order: color rgb, alpha, bg rgb, normal xyz)
 * unpack: scatters one rank's slab back into full-size planes.                           */
int64_t rayn_b200_film_slab_floats(int32_t tile_w, int32_t tile_h, int32_t n_tiles);
/* tile_list: HOST pointer to n_tiles tile indices (the shard whose slab this is) */
int32_t rayn_b200_film_pack_tiles(RaynContext* ctx, int32_t width, int32_t height, int32_t tile_w,
                                  int32_t tile_h, const int32_t* tile_list, int32_t n_tiles,
                                  const RaynFilmPlanes* planes_dev, float* slab_dev);
int32_t rayn_b200_film_unpack_tiles(RaynContext* ctx, int32_t width, int32_t height, int32_t tile_w,
                                    int32_t tile_h, const int32_t* tile_list, int32_t n_tiles,
                                    const float* slab_dev, const RaynFilmPlanes* planes_dev);

/* ---- film post-process: the per-pixel arithmetic of Film::save_to (src/film.rs:205-377) -----
 * (SURVEY §8f rank 3: the step AFTER the path; PNG encoding itself stays host I/O.)
 * Writes the pixel buffer the reference hands to the `image` crate: rows top to bottom
 * (y flipped, film.rs:236), 8 bits per sample, `(v*255).min(255).max(0) as u8`.             */
typedef enum RaynPostMode {
  RAYN_POST_COLOR_PLUS_BACKGROUND = 0, /* RGB8  (col+bg).saturated().gamma_corrected(2.2)  film.rs:253-274 */
  RAYN_POST_COLOR_ALPHA = 1,           /* RGBA8 col.saturated().gamma_corrected(2.2), a    film.rs:230-252 */
  RAYN_POST_COLOR_ONLY = 2,            /* RGB8  col.gamma_corrected(2.2)  (no saturate)    film.rs:275-293 */
  RAYN_POST_BACKGROUND = 3,            /* RGB8  bg.saturated().gamma_corrected(2.2)        film.rs:300-325 */
  RAYN_POST_WORLD_NORMAL = 4,          /* RGB8  n*0.5 + 0.5                                film.rs:326-350 */
  RAYN_POST_ALPHA = 5                  /* L8    a                                          film.rs:351-372 */
} RaynPostMode;
/* planes->space says where the float planes live; out_space where `out` lives (RaynMemSpace).
 * out holds width*height*{3,4,3,3,3,1} bytes.                                                */
int32_t rayn_b200_film_postprocess(RaynContext* ctx, int32_t mode, int32_t width, int32_t height,
                                   const RaynFilmPlanes* planes, uint8_t* out, int32_t out_space);

/* ---- film denoise: edge-avoiding a-trous wavelet filter (Dammertz et al., HPG 2010; PAPERS.md) -----------------
 * Filters the color and background planes of a rendered film, guided by its normal and alpha planes, which the
 * reference only writes out for an external denoiser (film.rs:326-372).  Level i = 0..iterations-1 uses step 2^i and
 * the 5x5 taps q = p + 2^i (dx, dy), dx, dy in -2..2, kernel h = {1/16, 1/4, 3/8, 1/4, 1/16}; level 0 reads `in`,
 * each later level reads the previous one, the last writes `out`.  Per tap, in float and in this order:
 *   dc2 = (dr*dr + dg*dg) + db*db of c_q - c_p,  dn2 the same of n_q - n_p,  da2 = (a_q - a_p)^2
 *   e = (dc2*ic_i + dn2*in) + da2*ia,  w = h[dy+2]*h[dx+2] * exp(-e)     (exp: detmath.h)
 *   ic_i = ldexpf(1/(sigma_color^2), i),  in = 1/sigma_normal^2,  ia = 1/sigma_alpha^2
 * output = (sum w*c_q) / (sum w), taps visited dy outer, dx inner, ascending.  Taps outside the image, taps with a
 * non-finite colour component and taps whose e is NaN are skipped; a pixel whose own colour is non-finite is copied.
 * A sigma must be > 0 (+inf disables its term) and large enough that every factor is finite; else
 * RAYN_ERR_INVALID_ARG.  in->normal and in->alpha are required; in->color / in->background are optional, each one
 * present needs the matching out plane.  out->color / out->background may be the same pointers as in's.
 * in->space and out->space are RaynMemSpace each.  Device planes on both sides: asynchronous on the context's
 * stream (rayn_b200_sync waits); otherwise the call copies, filters and returns with the result in place.
 * Scratch is stream-ordered (cudaMallocAsync) and released within the call.                                    */
typedef struct RaynDenoiseDesc {
  int32_t iterations; /* levels L, 1..8 (step 2^i)               */
  float sigma_color;  /* > 0; +inf disables the term             */
  float sigma_normal;
  float sigma_alpha;
} RaynDenoiseDesc;
int32_t rayn_b200_film_denoise(RaynContext* ctx, const RaynDenoiseDesc* desc, int32_t width, int32_t height,
                               const RaynFilmPlanes* in, const RaynFilmPlanes* out);
/* The same filter with an albedo guide (e.g. rayn_b200_render_albedo's plane): per tap, with
 *   dl2 = (dr*dr + dg*dg) + db*db of albedo_q - albedo_p,   il = 1/sigma_albedo^2 (the same at every level),
 *   e = ((dc2*ic_i + dn2*in) + da2*ia) + dl2*il
 * and everything else as in rayn_b200_film_denoise (sigma, skip, aliasing, space and asynchrony rules).  `albedo` is a
 * [3*W*H] plane in in->space; NULL is RAYN_ERR_INVALID_ARG.  sigma_albedo must be > 0 with a finite 1/sigma^2; at +inf the
 * term is NOT added, and the call equals rayn_b200_film_denoise bit for bit.  A tap whose albedo has a non-finite
 * component gets a NaN e (skipped) or e = +inf (weight +0).                                                         */
int32_t rayn_b200_film_denoise_albedo(RaynContext* ctx, const RaynDenoiseDesc* desc, float sigma_albedo, const float* albedo,
                                      int32_t width, int32_t height, const RaynFilmPlanes* in, const RaynFilmPlanes* out);
/* The same filter guided by each pixel's variance (after Schied et al., SVGF, HPG 2017; PAPERS.md).  Each colour plane X
 * (color, background) is filtered with its moment plane M (color_lum2, background_lum2 of rayn_b200_render_frame_moments for
 * a film of `spp` samples per pixel), lum() as stated there.  Every pixel carries (c, v); in float, in this order:
 *   level 0:  v_p = fmaxf(M_p - lum(c_p)*lum(c_p), 0.0f) / (float)spp        (the variance of the pixel mean)
 *   level i, pixel p with finite colour:
 *     g_p  = (sum k*v_q) / (sum k) over the 3x3 taps q = p + (dx, dy), dx, dy in -1..1 (unit spacing, every level),
 *            dy outer, dx inner, ascending, k = K[dy+1]*K[dx+1], K = {0.25, 0.5, 0.25}, skipping taps outside the image
 *            and taps with a non-finite colour component
 *     il_p = 1.0f / (sigma_luminance * sqrtf(g_p) + 1e-10f)
 *     per tap of the 5x5 filter: e = e_0 + fabsf(lum(c_q) - lum(c_p)) * il_p, where e_0 is the e of rayn_b200_film_denoise,
 *            or of rayn_b200_film_denoise_albedo when albedo != NULL; w, the skips and the colour output are unchanged
 *     v'_p = (sum (w*w)*v_q) / (sw*sw), sw = sum w, the sum in tap order over the taps that are not skipped and whose w*w
 *            is not +0
 *   a pixel whose colour is non-finite is copied, colour and variance.  The last level writes the colour only.
 * e stays a sum of non-negative terms or NaN (il_p is in [0, 1e10]), so the centre tap has e = 0 and w = h*h as before.
 * sigma_luminance must be > 0; at +inf the term is not added, v is not formed, and the call equals
 * rayn_b200_film_denoise (albedo NULL) or rayn_b200_film_denoise_albedo bit for bit.  albedo may be NULL (no albedo term);
 * otherwise sigma_albedo follows rayn_b200_film_denoise_albedo.  spp >= 1.  `moments` lives in in->space
 * (moments->space == in->space); a present input colour plane without its moment plane is RAYN_ERR_INVALID_ARG, as are
 * spp < 1 and a bad sigma.  The aliasing, space and asynchrony rules are rayn_b200_film_denoise's.                       */
int32_t rayn_b200_film_denoise_variance(RaynContext* ctx, const RaynDenoiseDesc* desc, float sigma_luminance, int32_t spp,
                                        const RaynMomentPlanes* moments, float sigma_albedo, const float* albedo, int32_t width,
                                        int32_t height, const RaynFilmPlanes* in, const RaynFilmPlanes* out);
/* rayn_b200_film_denoise_variance with a per-pixel variance scale (e.g. rayn_b200_temporal_push's var_scale, for a film that
 * is a blend of frames): level 0 becomes
 *   v_p = (fmaxf(M_p - lum(c_p)*lum(c_p), 0.0f) * scale_p) / (float)spp
 * and everything else is unchanged.  var_scale [W*H] lives in in->space; NULL is RAYN_ERR_INVALID_ARG.  With var_scale == 1
 * everywhere the call equals rayn_b200_film_denoise_variance bit for bit (x * 1 == x), and at sigma_luminance = +inf the
 * scale is not read.                                                                                                       */
int32_t rayn_b200_film_denoise_variance_scaled(RaynContext* ctx, const RaynDenoiseDesc* desc, float sigma_luminance, int32_t spp,
                                               const RaynMomentPlanes* moments, const float* var_scale, float sigma_albedo,
                                               const float* albedo, int32_t width, int32_t height, const RaynFilmPlanes* in,
                                               const RaynFilmPlanes* out);

/* ---- temporal accumulation of a frame sequence (the temporal half of SVGF, Schied et al. 2017; PAPERS.md) ---------------
 * A RaynTemporal holds the reprojectable history of one W x H film: per pixel colour 3, background 3, the 2 moments,
 * normal 3, z 1, history length n 1 and s 1, twice (14 floats per pixel each, allocated at create so render-pass sizing sees
 * them; a push reads one and writes the other).  A new history has n = 0 everywhere.
 * temporal_push(in, moments, motion): `in` is the current frame (color, background, normal required; alpha unused),
 * `moments` its lum^2 planes (rayn_b200_render_frame_moments), `motion` its rayn_b200_render_motion plane.  Per pixel
 * p = (x, y), in float, no contraction:
 *   reset = 0 and z_prev finite:  fx = (((float)x + 0.5f) + dx) - 0.5f, fy likewise; x0 = floorf(fx), y0 = floorf(fy), ax = fx - x0, ay = fy - y0;
 *     taps (x0 + i, y0 + j), j outer, i inner, in {0, 1}, weight w = (i ? ax : 1 - ax) * (j ? ay : 1 - ay).  A tap is USED if
 *     w != 0, it is inside the image (compared in float), its history n > 0, its colour and background are finite, z_h is
 *     finite and fabsf(z_h - z_prev) <= sigma_depth * fabsf(z_prev) (|z_prev| serves orthographic views, whose z may be
 *     <= 0; z_h is tested on its own because sigma_depth = +inf, or an overflowing product, would otherwise pass a history
 *     without a hit, z_h = +inf) and ((nx_h*nx + ny_h*ny) + nz_h*nz) >= normal_cos (n the current normal).
 *     ws = sum w, and every history value X (colour, background, moments, n, s) is X_h = (sum w*X_q) / ws, sums in tap order
 *     over the used taps.  No used tap: n_h = 0.
 *   reset = 1, or z_prev not finite (a pixel without a valid hit: motion (0, 0, +inf, +inf)):  n_h = 0.
 *   alpha = fmaxf(alpha_min, 1.0f / (n_h + 1.0f));
 *   alpha == 1 (always when n_h = 0): every output is the current frame's value bit for bit, n' = n_h + 1, s' = 1;
 *   otherwise, for colour, background and both moments: x' = (1 - alpha) * x_h + alpha * x,  n' = n_h + 1,
 *     s' = ((1 - alpha) * (1 - alpha)) * s_h + alpha * alpha.
 * s' is the sum of squared blend weights, and for frames with independent noise max(M' - lum(c')^2, 0) * s' / spp is an
 * UPPER BOUND on the variance of the blended pixel mean.  It is exact when no pixel resamples its history (integer motion,
 * every used tap with weight 1; a cumulative mean, alpha_min -> 0 on a static view, gives s' = 1/n').  Under sub-pixel
 * motion the bilinear taps average the independent noise of neighbouring history pixels (sum w^2 < sum w of their variance)
 * while s_h is interpolated linearly, so the true variance is smaller: about 0.78 of the bound at 0.1 px per frame, 0.60 at
 * 0.5 px and 0.46 at (0.5, 0.5) px, with alpha_min 0.2 (tested).  The bound holds by Minkowski's and Jensen's inequalities.
 * The push writes c', b' to out, M' to out_moments and s' to var_scale, and stores c', b', M', n', s' with the current normal
 * and z in the history.  out may alias in (each pixel reads only its own input).  Every plane and var_scale is required and
 * in one memory space (in->space); host planes are staged and the call is synchronous, device planes run asynchronously on
 * the context's stream (rayn_b200_sync waits).  RAYN_ERR_INVALID_ARG for a NULL plane, mixed spaces, or a bad desc.
 * temporal_create: width and height in [1, 2^23] and width * height <= 2^31, else RAYN_ERR_INVALID_ARG.  Up to 2^23 every
 * pixel centre (float)x + 0.5f is exact, so a static pixel reads its own history; beyond it x + 0.5f rounds and the push
 * would read a neighbour's.                                                                                               */
typedef struct RaynTemporal RaynTemporal;
typedef struct RaynTemporalDesc {
  float alpha_min;    /* (0, 1]: the smallest blend weight of the new frame                */
  float sigma_depth;  /* > 0: relative depth tolerance of a history tap                     */
  float normal_cos;   /* [-1, 1]: least dot product of history and current normal           */
  int32_t reset;      /* 1: ignore the history (scene cut, first frame)                     */
} RaynTemporalDesc;
int32_t rayn_b200_temporal_create(RaynContext* ctx, int32_t width, int32_t height, RaynTemporal** out);
void rayn_b200_temporal_destroy(RaynTemporal* t);
int32_t rayn_b200_temporal_push(RaynContext* ctx, RaynTemporal* t, const RaynTemporalDesc* desc, const RaynFilmPlanes* in,
                                const RaynMomentPlanes* moments, const float* motion, const RaynFilmPlanes* out,
                                const RaynMomentPlanes* out_moments, float* var_scale);

/* ---- progressive / adaptive rendering: a device film accumulator refined in sample rounds -----------------------
 * Per-tile stopping rule after Dammertz, Hanika, Keller, Lensch (WSCG 2009; PAPERS.md): a tile's error compares the
 * film of all its samples with the film of half of them (the rounds it rendered first, third, ...), weighted by
 * 1/sqrt(I).  accum_create allocates all device state (13 floats per pixel, the round's 10 planes per pixel, per tile
 * K, Kh, rounds, E), so render-pass sizing sees it.  Tile index = tile_x * n_tiles_y + tile_y on the grid of
 * film.rs:399-404 (including its partial-tile quirk).
 *
 * accum_round(frame, desc): the ACTIVE tiles, chosen per tile before the round, are those with
 *     rounds < max_rounds && (rounds < min_rounds || !(E <= threshold))
 * They are rendered with `frame` (its tile_list / tile_offset / tile_stride are ignored) into the accumulator's own
 * device planes m (already / spp), then folded in.  width, height and tile size must equal the accumulator's.
 * A tile that stops never resumes, so all active tiles share one sample history: the CALLER passes tables for the
 * samples they have not seen yet, i.e. rayn_b200_{host,device}_rd_tables_at with first_sample = the sum of spp of the
 * earlier rounds (= `samples` of an active tile in accum_tiles).  The library cannot check this.  Active tiles whose
 * round counts differ (a desc changed between rounds) are RAYN_ERR_INVALID_ARG.  Synchronous (the tile errors pick
 * the next round's tiles).  *out_tiles_rendered (may be NULL) = active tiles; 0 = every tile has stopped, nothing ran.
 * Exact statement, float unless marked, no contraction; n = (float)(4 * frame->samples); for every in-image pixel of
 * an active tile:
 *   S.x[c] = S.x[c] + m.x[c] * n          for color (3), alpha (1), background (3), normal (3)
 *   if the tile's rounds is even before the round:  H[c] = H[c] + (m.color[c] + m.background[c]) * n
 * per tile: K += 4*samples, Kh += 4*samples if H was updated (int64), rounds += 1.  A round that would take K past
 * 2^24 is RAYN_ERR_INVALID_ARG (so (float)K is exact).  Then, for tiles with rounds >= 2, per pixel:
 *   I[c] = (S.color[c] + S.background[c]) / (float)K,   A[c] = H[c] / (float)Kh
 *   d = (|I0-A0| + |I1-A1|) + |I2-A2|,   s = (I0 + I1) + I2,   e = d / sqrtf(fmaxf(s, 0x1p-10f));  NaN e -> +inf
 *   E = (double sum of (double)e over the tile's in-image pixels in ascending pixel index x + y*width, strictly
 *        sequential) / (double)count
 * Tiles with fewer than 2 rounds have E = +inf.  A negative threshold never stops a tile (E is never negative):
 * uniform progressive rendering.
 * accum_resolve: out.x[c] = S.x[c] / (float)K of the pixel's tile; pixels outside the tile grid are 0.  After one round
 * of power-of-two spp this is render_frame's film bit for bit.  Planes are host or device (out->space), any may be
 * NULL; synchronous.  RAYN_ERR_INVALID_ARG before the first round.
 * accum_tiles: host arrays of n_tiles_x * n_tiles_y entries (either may be NULL): E and samples (= K) per tile.   */
typedef struct RaynAccum RaynAccum;
typedef struct RaynAdaptiveDesc {
  int32_t min_rounds; /* >= 2: every tile gets at least this many rounds                            */
  int32_t max_rounds; /* >= min_rounds: no tile gets more                                           */
  float threshold;    /* not NaN: a tile stops once its error E <= threshold; < 0 = never (uniform)  */
} RaynAdaptiveDesc;
int32_t rayn_b200_accum_create(RaynContext* ctx, int32_t width, int32_t height, int32_t tile_w, int32_t tile_h,
                               RaynAccum** out);
void rayn_b200_accum_destroy(RaynAccum* acc);
int32_t rayn_b200_accum_round(RaynContext* ctx, RaynAccum* acc, const RaynFrameDesc* frame,
                              const RaynAdaptiveDesc* desc, int32_t* out_tiles_rendered);
int32_t rayn_b200_accum_tiles(RaynContext* ctx, const RaynAccum* acc, double* err, int64_t* samples);
int32_t rayn_b200_accum_resolve(RaynContext* ctx, const RaynAccum* acc, const RaynFilmPlanes* out);

/* ---- host-side input builders (pure CPU; stand in for crates the Rust host owns) ----
 * quasi-rd R_d tables (sampler.rs:18-37), rand SmallRng scramble (film.rs:460-461),
 * FilterImportanceSampler::new(BlackmanHarris) (filter.rs:13-49,196-218).               */
int32_t rayn_b200_host_rd_tables(int32_t spp, int32_t sets_1d, int32_t sets_2d, uint64_t offset,
                                 float* out_1d, float* out_2d);
/* samples [first_sample, first_sample + spp) of the same sequences: element n of set i is the R_d value at index
 * ((offset + i) << 32) + first_sample + n + 1 (2D sets offset by sets_1d, as above); rd_tables is first_sample = 0.
 * first_sample + spp > 2^32 is RAYN_ERR_INVALID_ARG.  For sample rounds of one film (rayn_b200_accum_round).       */
int32_t rayn_b200_host_rd_tables_at(int32_t spp, int32_t sets_1d, int32_t sets_2d, uint64_t offset, uint64_t first_sample,
                                    float* out_1d, float* out_2d);
/* the same in device memory (DEVICE pointers, bit-identical to the host builder), synchronous */
int32_t rayn_b200_device_rd_tables_at(RaynContext* ctx, int32_t spp, int32_t sets_1d, int32_t sets_2d, uint64_t offset,
                                      uint64_t first_sample, float* out_1d_dev, float* out_2d_dev);
int32_t rayn_b200_host_scramble(int32_t width, int32_t height, float* out);
int32_t rayn_b200_host_fis_blackman_harris(float radius, float* out512);
/* the same tables / scramble plane generated directly in device memory (DEVICE pointers; bit-identical
 * to the host builders) - saves uploading W*H floats of scramble per frame (133 MB at 8K)           */
int32_t rayn_b200_device_frame_inputs(RaynContext* ctx, int32_t width, int32_t height, int32_t spp, int32_t sets_1d,
                                      int32_t sets_2d, uint64_t offset, float* out_1d_dev, float* out_2d_dev,
                                      float* scramble_dev);
/* tile count per film.rs:399-404 (including its partial-tile quirk) */
int32_t rayn_b200_host_tile_grid(int32_t width, int32_t height, int32_t tile_w, int32_t tile_h,
                                 int32_t* n_tiles_x, int32_t* n_tiles_y);

/* ---- kernel-level known-answer entry points (device execution, host pointers) -------
 * Used by tests to compare single stages against the oracle lane by lane.              */
/* op: 0 exp, 1 ln, 2 pow(a,b), 3 sin, 4 cos, 5 tan, 6 atan2(a,b), 7 powi5, 8 ln_fast    */
int32_t rayn_b200_kat_detmath(RaynContext* ctx, int32_t op, int64_t n, const float* a,
                              const float* b, float* out);
/* SDF::dist (sdf.rs:125-141) */
int32_t rayn_b200_kat_sdf_dist(RaynContext* ctx, const RaynHitable* sdf, int64_t n,
                               const float* points3, float* out);
/* the same through the packed two-point estimator the march kernels run (rt_sdf2.cuh); variant < 0 = the one the
 * scheduler would pick for this hitable, else force 0 generic Mandelbox / 1 12-iteration fast / 2 n-iteration fast / 3 Mandelbulb /
 * 4, 5 = 1, 2 with the three-operation sphere-fold division (RAYN_ERR_INVALID_ARG unless its exhaustive check passes here) */
int32_t rayn_b200_kat_sdf_dist2(RaynContext* ctx, const RaynHitable* sdf, int32_t variant, int64_t n,
                                const float* points3, float* out);
/* trap(sdf, p) per point (RaynAlbedoTrap above), through the device function k_normals evaluates */
int32_t rayn_b200_kat_sdf_trap(RaynContext* ctx, const RaynHitable* sdf, int64_t n, const float* points3, float* out);
/* Newton division of the Mandelbox sphere fold vs IEEE division: number of x among the n consecutive floats starting
 * at bit pattern first_bits for which num / x differs (must be 0 wherever the fast variants are selected)           */
int32_t rayn_b200_kat_fastdiv(RaynContext* ctx, float num, uint32_t first_bits, int64_t n, int64_t* out_mismatches);
/* detmath op (as kat_detmath) at every 32-bit pattern v as its first operand, b the second (swap != 0: b first, v second),
 * inputs generated on the device: out_hashes256[c] = sum over the v with v >> 24 == c of
 * splitmix64(((uint64_t)v << 32) | bits of the result)  mod 2^64; a NaN of powi5 counts as 0x7fc00000 (its payload is
 * the hardware's, detmath.h)                                                                                          */
int32_t rayn_b200_kat_detmath_sweep(RaynContext* ctx, int32_t op, float b, int32_t swap, uint64_t* out_hashes256);
/* TracedSDF::hit (sdf.rs:59-83).  thr(t) = thr_scale * t, or thr_scale if thr_const != 0 */
int32_t rayn_b200_kat_sdf_hit(RaynContext* ctx, const RaynHitable* sdf,
                              const RaynRenderConsts* consts, int64_t n, const float* origins3,
                              const float* dirs3, const float* t_max, float thr_scale,
                              int32_t thr_const, float* out_t);
/* HitableStore::test_occluded over the uploaded scene (hitable.rs:164-168) */
int32_t rayn_b200_kat_occluded(RaynContext* ctx, int64_t n, const float* start3,
                               const float* end3, float* out);
/* HitableStore::add_hits closest-hit fold over the uploaded scene (hitable.rs:170-198):
 * out_t[i], out_obj[i] (-1 = nothing hit).  depth selects the threshold closure
 * (film.rs:540-551).                                                                     */
int32_t rayn_b200_kat_closest_hit(RaynContext* ctx, int32_t depth, int64_t n,
                                  const float* origins3, const float* dirs3, float* out_t,
                                  int32_t* out_obj);

/* SphereLight::sample (light.rs:38-72) and ::sample_volume_scattering (:75-102) per lane */
int32_t rayn_b200_kat_light_sample(RaynContext* ctx, const RaynLight* light, int64_t n, const float* s0,
                                   const float* s1, const float* points3, float* out_point3, float* out_pdf);
int32_t rayn_b200_kat_light_sample_volume(RaynContext* ctx, const RaynLight* light, int64_t n,
                                          const float* sample, const float* origins3, const float* dirs3,
                                          const float* t_max, float* out_t, float* out_pdf);
/* BSDF::scatter + BSDF::f (material.rs): normals3/wo3 unit vectors, s1d[n], u4[4n] ->
 * out_wi3, out_f3 (scatter event f), out_pdf, out_feval3 = bsdf.f(wo, wi, n) as integrator.rs:230 calls it */
int32_t rayn_b200_kat_bsdf(RaynContext* ctx, const RaynMaterial* mat, int64_t n, const float* normals3,
                           const float* wo3, const float* s1d, const float* u4, float* out_wi3,
                           float* out_f3, float* out_pdf, float* out_feval3);

/* Which march-kernel specialisation upload_scene selected for hitable `hitable_index` of the current scene: -1 analytic sphere,
 * 0 generic Mandelbox, 1 / 2 packed Mandelbox (12 / n iterations), 3 Mandelbulb, 4 / 5 = 1 / 2 with the three-operation
 * sphere-fold division, which upload_scene selects only after dividing by EVERY float in [min_rad_sq, fixed_rad_sq] on this
 * device and finding all quotients equal to IEEE division; -2 = bad index / no scene                                      */
int32_t rayn_b200_debug_sdf_variant(const RaynContext* ctx, int32_t hitable_index);

/* Packet-order debugging (SURVEY F6): when enabled, render_frame records for every depth
 * and tile the shading queue (path id per slot, -1 = padding) into an internal host log. */
int32_t rayn_b200_debug_enable_queue_log(RaynContext* ctx, int32_t enable);
/* returns number of int32 entries; copies up to cap entries.
 * Layout: repeated records { depth, tile_index, n_slots, slot[0..n_slots) }.             */
int64_t rayn_b200_debug_read_queue_log(RaynContext* ctx, int32_t* out, int64_t cap);

#ifdef __cplusplus
}
#endif
#endif /* RAYN_B200_H */
