// rayn_host.hpp — C++ host side above the C ABI: the stand-in for rayn's Rust host
// (src/setup.rs scene API, src/world.rs, src/film.rs Film, src/main.rs driver), written in C++
// because the image has no Rust toolchain (SURVEY F4).  Same names and argument meaning as the
// reference constructors; every object flattens to the POD descriptors of include/rayn_b200.h.
#pragma once
#include <cmath>
#include <cstdint>
#include <memory>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "../../include/rayn_b200.h"

namespace rayn {

struct Vec3 {  // ultraviolet::Vec3, host-side constants only
  float x = 0, y = 0, z = 0;
  Vec3() = default;
  Vec3(float x_, float y_, float z_) : x(x_), y(y_), z(z_) {}
  static Vec3 zero() { return {}; }
  Vec3 operator*(float s) const { return {x * s, y * s, z * s}; }
  Vec3 normalized() const {
    const float m = std::sqrt(x * x + y * y + z * z);
    return {x / m, y / m, z / m};
  }
  void store(float* p) const { p[0] = x, p[1] = y, p[2] = z; }
};
using Srgb = Vec3;  // spectrum.rs newtype
// A Sequenced<Vec3> parameter: constant, or linear in time (stands for the closure `|t| base + velocity * t`,
// animation.rs:55-68; evaluated at lane 0's time of a packet like every closure-backed WSequenced, :62-67).
struct Seq3 {
  Vec3 base, velocity;
  Seq3(Vec3 b) : base(b) {}  // NOLINT: constants convert implicitly, like `impl Sequenced<Vec3> for Vec3`
  Seq3(Vec3 b, Vec3 v) : base(b), velocity(v) {}
};
inline Seq3 Linear(Vec3 base, Vec3 velocity) { return Seq3(base, velocity); }
using MaterialHandle = int;
using CameraHandle = int;

// ---- materials (material.rs) ------------------------------------------------------------
// An albedo generator (rayn's albedo_gen, material.rs:75-83) that colours an SDF surface by orbit trap: the trap value at the
// hit, mapped from [trap_lo, trap_hi] onto lo .. hi and clamped; analytic spheres get hi (include/rayn_b200.h, RaynAlbedoTrap).
struct OrbitTrapAlbedo {
  float trap_lo, trap_hi;
  Srgb lo, hi;
};
struct Material {
  RaynMaterial pod{};
  bool has_trap = false;
  RaynAlbedoTrap trap{};  // material index filled in by MaterialStore::add_material
 protected:
  void set_albedo(const Srgb& a) { a.store(pod.albedo); }
  void set_albedo(const OrbitTrapAlbedo& t) {  // the constant is albedo_hi, what a trap material gives on analytic spheres
    t.hi.store(pod.albedo);
    has_trap = true;
    trap.trap_lo = t.trap_lo, trap.trap_hi = t.trap_hi;
    t.lo.store(trap.albedo_lo), t.hi.store(trap.albedo_hi);
  }
};
struct Lambertian : Material {  // material.rs:91-100
  template <class A>
  explicit Lambertian(A albedo) {
    pod.kind = RAYN_MATERIAL_LAMBERTIAN;
    set_albedo(albedo);
  }
};
struct Dielectric : Material {  // material.rs:150-175
  template <class A>
  Dielectric(A albedo, float roughness_exponent) {
    pod.kind = RAYN_MATERIAL_DIELECTRIC;
    set_albedo(albedo);
    pod.roughness = roughness_exponent;
  }
  template <class A>
  static Dielectric new_remap(A albedo, float roughness) {  // :167-174
    float r = 1.0f - roughness;
    r = 1.0f + r * r * r * r * 300.0f;
    return Dielectric(albedo, r);
  }
};
// A glossy conductor with coloured Fresnel (include/rayn_b200.h, RAYN_MATERIAL_METALLIC): an EXTENSION with no reference
// counterpart.  F0 per channel in albedo, or an orbit-trap palette; the exponent remap is the Dielectric's.
struct Metallic : Material {
  template <class A>
  Metallic(A f0, float roughness_exponent) {
    pod.kind = RAYN_MATERIAL_METALLIC;
    set_albedo(f0);
    pod.roughness = roughness_exponent;
  }
  template <class A>
  static Metallic new_remap(A f0, float roughness) { return Metallic(f0, Dielectric::new_remap(Srgb(0, 0, 0), roughness).pod.roughness); }
};
struct Sky : Material {  // material.rs:394-404
  Sky(Srgb top, Srgb bottom) {
    pod.kind = RAYN_MATERIAL_SKY;
    top.store(pod.sky_top);
    bottom.store(pod.sky_bottom);
  }
};
struct Emissive : Material {  // material.rs:451-469
  explicit Emissive(Srgb emission) {
    pod.kind = RAYN_MATERIAL_EMISSIVE;
    emission.store(pod.emission);
    pod.albedo[0] = pod.albedo[1] = pod.albedo[2] = 0.5f;  // inner LambertianBSDF, :482-484
  }
  static Emissive new_splat(Srgb emission) { return Emissive(emission); }
};
struct MaterialStore {  // material.rs:58-73
  std::vector<RaynMaterial> items;
  std::vector<RaynAlbedoTrap> traps;  // orbit-trap albedos, one per material that has one (rayn_b200_set_albedo_traps)
  MaterialHandle add_material(const Material& m) {
    items.push_back(m.pod);
    const MaterialHandle h = (MaterialHandle)items.size() - 1;
    if (m.has_trap) {
      traps.push_back(m.trap);
      traps.back().material = h;
    }
    return h;
  }
};

// ---- hitables (sphere.rs, sdf.rs) ----------------------------------------------------------
struct Hitable {
  RaynHitable pod{};
};
struct Sphere : Hitable {  // sphere.rs:14-20
  Sphere(Seq3 center, float radius, MaterialHandle material) {
    pod.kind = RAYN_HITABLE_SPHERE;
    pod.material = material;
    center.base.store(pod.center);
    center.velocity.store(pod.center_velocity);
    pod.radius = radius;
  }
};
struct BoxFold {  // sdf.rs:150-158
  float l;
  explicit BoxFold(float side_length) : l(side_length) {}
};
struct SphereFold {  // sdf.rs:171-179
  float min_rad_sq, fixed_rad_sq;
  SphereFold(float min_radius, float fixed_radius) : min_rad_sq(min_radius * min_radius), fixed_rad_sq(fixed_radius * fixed_radius) {}
};
struct MandelBox {  // sdf.rs:113-123
  int iterations;
  BoxFold box_fold;
  SphereFold sphere_fold;
  float scale;
  MandelBox(int it, BoxFold b, SphereFold s, float sc) : iterations(it), box_fold(b), sphere_fold(s), scale(sc) {}
};
struct Mandelbulb {  // AUTHORED: not in the reference (SURVEY F1)
  int iterations;
  int power;
  float bailout;
  explicit Mandelbulb(int it, int pw = 8, float bail = 2.0f) : iterations(it), power(pw), bailout(bail) {}
};
struct TracedSDF : Hitable {  // sdf.rs:12-21
  TracedSDF(const MandelBox& s, MaterialHandle material) {
    pod.kind = RAYN_HITABLE_MANDELBOX;
    pod.material = material;
    pod.iterations = s.iterations;
    pod.box_l = s.box_fold.l;
    pod.min_rad_sq = s.sphere_fold.min_rad_sq;
    pod.fixed_rad_sq = s.sphere_fold.fixed_rad_sq;
    pod.scale = s.scale;
  }
  TracedSDF(const Mandelbulb& s, MaterialHandle material) {
    pod.kind = RAYN_HITABLE_MANDELBULB;
    pod.material = material;
    pod.iterations = s.iterations;
    pod.bulb_power = s.power;
    pod.bulb_bailout = s.bailout;
  }
};
struct HitableStore {  // hitable.rs:143-153
  std::vector<RaynHitable> items;
  void push(const Hitable& h) { items.push_back(h.pod); }
  size_t len() const { return items.size(); }
};

// ---- lights (light.rs) ----------------------------------------------------------------------
struct SphereLight {  // light.rs:27-34
  RaynLight pod{};
  SphereLight(Vec3 pos, float rad, Srgb emission) {
    pos.store(pod.pos);
    pod.rad = rad;
    emission.store(pod.emission);
  }
};

// ---- cameras (camera.rs) ----------------------------------------------------------------------
struct Camera {
  RaynCamera pod{};
};
inline void fov_half(float rx, float ry, float vfov, float* hw, float* hh) {  // camera.rs:59-63
  const float theta = vfov * 3.14159265358979323846f / 180.0f;
  *hh = std::tan(theta / 2.0f);
  *hw = (rx / ry) * *hh;
}
struct PinholeCamera : Camera {  // camera.rs:52-72
  PinholeCamera(float rx, float ry, float vfov, Seq3 origin, Seq3 at, Seq3 up) {
    pod.kind = RAYN_CAMERA_PINHOLE;
    fov_half(rx, ry, vfov, &pod.half_size[0], &pod.half_size[1]);
    pod.half_pixel_size = pod.half_size[1] / ry;
    origin.base.store(pod.origin), at.base.store(pod.at), up.base.store(pod.up);
    origin.velocity.store(pod.origin_velocity), at.velocity.store(pod.at_velocity), up.velocity.store(pod.up_velocity);
  }
};
struct ThinLensCamera : Camera {  // camera.rs:133-157
  ThinLensCamera(float rx, float ry, float vfov, float aperture, Seq3 origin, Seq3 at, Seq3 up, Seq3 focus, float aperture_rate = 0.0f) {
    pod.kind = RAYN_CAMERA_THINLENS;
    fov_half(rx, ry, vfov, &pod.half_size[0], &pod.half_size[1]);
    pod.half_pixel_size = pod.half_size[1] / ry;
    pod.aperture = aperture;
    pod.aperture_rate = aperture_rate;
    origin.base.store(pod.origin), at.base.store(pod.at), up.base.store(pod.up), focus.base.store(pod.focus);
    origin.velocity.store(pod.origin_velocity), at.velocity.store(pod.at_velocity), up.velocity.store(pod.up_velocity);
    focus.velocity.store(pod.focus_velocity);
  }
};
struct OrthographicCamera : Camera {  // camera.rs:227-241
  OrthographicCamera(float rx, float ry, float vertical_size, Seq3 origin, Seq3 at, Seq3 up) {
    pod.kind = RAYN_CAMERA_ORTHOGRAPHIC;
    const float aspect = rx / ry;
    pod.full_size[0] = vertical_size * aspect, pod.full_size[1] = vertical_size;
    pod.half_size[0] = pod.full_size[0] / 2.0f, pod.half_size[1] = pod.full_size[1] / 2.0f;
    pod.half_pixel_size = (vertical_size / ry) / 2.0f;
    origin.base.store(pod.origin), at.base.store(pod.at), up.base.store(pod.up);
    origin.velocity.store(pod.origin_velocity), at.velocity.store(pod.at_velocity), up.velocity.store(pod.up_velocity);
  }
};
// A 360-degree equirectangular panorama (include/rayn_b200.h, RAYN_CAMERA_EQUIRECTANGULAR): an EXTENSION with no reference
// counterpart.  half_pixel_size is the angular half pixel, as rayn_b200/scene.py EquirectangularCamera computes it.
struct EquirectangularCamera : Camera {
  EquirectangularCamera(float ry, Seq3 origin, Seq3 at, Seq3 up) {
    pod.kind = RAYN_CAMERA_EQUIRECTANGULAR;
    pod.half_pixel_size = (3.14159265358979323846f / ry) / 2.0f;
    origin.base.store(pod.origin), at.base.store(pod.at), up.base.store(pod.up);
    origin.velocity.store(pod.origin_velocity), at.velocity.store(pod.at_velocity), up.velocity.store(pod.up_velocity);
  }
};
// true if the tile grid of film.rs:399-404 leaves the last columns of a film `width` pixels wide out (0 < width % tile_w <
// tile_w / 2): a panorama would show a black strip at the seam
inline bool panorama_width_uncovered(int width, int tile_w) {
  const int r = width % tile_w;
  return 0 < r && 2 * r < tile_w;
}
struct CameraStore {  // camera.rs:24-40
  std::vector<RaynCamera> items;
  CameraHandle add_camera(const Camera& c) {
    items.push_back(c.pod);
    return (CameraHandle)items.size() - 1;
  }
  const RaynCamera& get(CameraHandle h) const { return items.at((size_t)h); }
};

struct VolumeParams {  // volume.rs:2-5 (Option<f32> pairs)
  bool has_scattering = false, has_extinction = false;
  float coeff_scattering = 0, coeff_extinction = 0;
};

struct World {  // world.rs:7-13
  HitableStore hitables;
  std::vector<SphereLight> lights;
  MaterialStore materials;
  CameraStore cameras;
  VolumeParams volume_params;
  RaynRenderConsts consts{100.0f, 0.5f, 256, 100};  // setup.rs:33,37; sdf.rs:9-10
};

struct PathTracingIntegrator {  // integrator.rs:33-45
  int max_bounces, volume_marches;
  int requested_1d_sample_sets() const { return (max_bounces + 1) * (3 + volume_marches); }
  int requested_2d_sample_sets() const { return (max_bounces + 1) * (12 + 8 * volume_marches); }
};
struct BlackmanHarrisFilter {  // filter.rs:13-27
  float radius = 1.5f;
};

inline void check(int32_t rc, RaynContext* ctx) {
  if (rc != RAYN_OK) throw std::runtime_error(std::string("rayn_b200 error ") + std::to_string(rc) + ": " + rayn_b200_last_error(ctx));
}

// film.rs:175-203.  Four channel planes (Color, Alpha, Background, WorldNormal), row-major, y up.
class Film {
 public:
  Film(int w, int h, int device = 0) : w_(w), h_(h) {
    RaynConfig cfg{device, 0, 0};
    check(rayn_b200_create(&cfg, &ctx_), nullptr);
    color.assign((size_t)3 * w * h, 0.0f), alpha.assign((size_t)w * h, 0.0f);
    background.assign((size_t)3 * w * h, 0.0f), normal.assign((size_t)3 * w * h, 0.0f);
  }
  ~Film() { rayn_b200_destroy(ctx_); }
  Film(const Film&) = delete;
  Film& operator=(const Film&) = delete;

  // film.rs:382-395.  moments: the same render with its luminance second moments (rayn_b200_render_frame_moments) into
  // color_lum2 / background_lum2, for denoise_variance; the film planes are the same.
  void render_frame_into(const World& world, CameraHandle camera, const PathTracingIntegrator& integrator, const BlackmanHarrisFilter& filter,
                         int tile_w, int tile_h, int frame, float t0, float t1, int samples, bool moments = false) {
    const int spp = 4 * samples;
    const int sets_1d = 1 + integrator.requested_1d_sample_sets();  // film.rs:431
    const int sets_2d = 2 + integrator.requested_2d_sample_sets();  // film.rs:432
    std::vector<float> s1((size_t)spp * sets_1d), s2((size_t)2 * spp * sets_2d), scr((size_t)w_ * h_), fis(RAYN_FIS_TABLE_SIZE);
    check(rayn_b200_host_rd_tables(spp, sets_1d, sets_2d, (uint64_t)frame, s1.data(), s2.data()), ctx_);  // film.rs:434
    check(rayn_b200_host_scramble(w_, h_, scr.data()), ctx_);                                              // film.rs:460-461
    check(rayn_b200_host_fis_blackman_harris(filter.radius, fis.data()), ctx_);                            // film.rs:429
    upload_scene(world, camera);
    RaynFrameDesc f = frame_desc(integrator, tile_w, tile_h, frame, t0, t1, samples, sets_1d, sets_2d);
    f.samples_1d = s1.data(), f.samples_2d = s2.data(), f.scramble = scr.data(), f.fis_inverse_cdf = fis.data();
    RaynFilmPlanes p{color.data(), alpha.data(), background.data(), normal.data(), RAYN_MEM_HOST};
    spp_ = spp;
    if (moments) {
      color_lum2.assign((size_t)w_ * h_, 0.0f), background_lum2.assign((size_t)w_ * h_, 0.0f);
      const RaynMomentPlanes m{color_lum2.data(), background_lum2.data(), RAYN_MEM_HOST};
      check(rayn_b200_render_frame_moments(ctx_, &f, &p, &m), ctx_);
    } else {
      color_lum2.clear(), background_lum2.clear();
      check(rayn_b200_render_frame(ctx_, &f, &p), ctx_);
    }
    rayn_b200_get_stats(ctx_, &stats);
    ++progressive_epoch;  // film.rs:657
  }
  // Progressive render in rounds of 4*samples spp on a device film accumulator: every tile keeps rendering until its
  // error E <= threshold, after at least min_rounds and at most max_rounds rounds (rayn_b200_accum_round).  Each round's
  // tables are the next spp samples of the frame's sequences.  Leaves the film in the planes, the per-tile errors and
  // samples in tile_errors / tile_samples; returns the number of rounds rendered.
  int render_adaptive(const World& world, CameraHandle camera, const PathTracingIntegrator& integrator, const BlackmanHarrisFilter& filter,
                      int tile_w, int tile_h, int frame, float t0, float t1, int samples, int min_rounds, int max_rounds, float threshold) {
    const int spp = 4 * samples;
    const int sets_1d = 1 + integrator.requested_1d_sample_sets(), sets_2d = 2 + integrator.requested_2d_sample_sets();
    std::vector<float> s1((size_t)spp * sets_1d), s2((size_t)2 * spp * sets_2d), scr((size_t)w_ * h_), fis(RAYN_FIS_TABLE_SIZE);
    check(rayn_b200_host_scramble(w_, h_, scr.data()), ctx_);
    check(rayn_b200_host_fis_blackman_harris(filter.radius, fis.data()), ctx_);
    upload_scene(world, camera);
    RaynFrameDesc f = frame_desc(integrator, tile_w, tile_h, frame, t0, t1, samples, sets_1d, sets_2d);
    f.samples_1d = s1.data(), f.samples_2d = s2.data(), f.scramble = scr.data(), f.fis_inverse_cdf = fis.data();
    const RaynAdaptiveDesc d{min_rounds, max_rounds, threshold};
    RaynAccum* acc = nullptr;
    check(rayn_b200_accum_create(ctx_, w_, h_, tile_w, tile_h, &acc), ctx_);
    int rounds = 0;
    try {
      for (uint64_t first = 0;; first += (uint64_t)spp) {
        check(rayn_b200_host_rd_tables_at(spp, sets_1d, sets_2d, (uint64_t)frame, first, s1.data(), s2.data()), ctx_);
        int32_t n = 0;
        check(rayn_b200_accum_round(ctx_, acc, &f, &d, &n), ctx_);
        if (n == 0) break;
        ++rounds;
        ++progressive_epoch;  // film.rs:657
        rayn_b200_get_stats(ctx_, &stats);
      }
      RaynFilmPlanes p{color.data(), alpha.data(), background.data(), normal.data(), RAYN_MEM_HOST};
      check(rayn_b200_accum_resolve(ctx_, acc, &p), ctx_);
      int ntx = 0, nty = 0;
      check(rayn_b200_host_tile_grid(w_, h_, tile_w, tile_h, &ntx, &nty), ctx_);
      tile_errors.assign((size_t)ntx * nty, 0.0), tile_samples.assign((size_t)ntx * nty, 0);
      check(rayn_b200_accum_tiles(ctx_, acc, tile_errors.data(), tile_samples.data()), ctx_);
    } catch (...) {
      rayn_b200_accum_destroy(acc);
      throw;
    }
    rayn_b200_accum_destroy(acc);
    return rounds;
  }
  // First-hit albedo plane of the frame (rayn_b200_render_albedo) into `albedo`: the first 4*samples camera samples of the
  // frame's sequences.
  void render_albedo(const World& world, CameraHandle camera, const PathTracingIntegrator& integrator, const BlackmanHarrisFilter& filter,
                     int tile_w, int tile_h, int frame, float t0, float t1, int samples) {
    const int spp = 4 * samples;
    const int sets_1d = 1 + integrator.requested_1d_sample_sets(), sets_2d = 2 + integrator.requested_2d_sample_sets();
    std::vector<float> s1((size_t)spp * sets_1d), s2((size_t)2 * spp * sets_2d), scr((size_t)w_ * h_), fis(RAYN_FIS_TABLE_SIZE);
    check(rayn_b200_host_rd_tables(spp, sets_1d, sets_2d, (uint64_t)frame, s1.data(), s2.data()), ctx_);
    check(rayn_b200_host_scramble(w_, h_, scr.data()), ctx_);
    check(rayn_b200_host_fis_blackman_harris(filter.radius, fis.data()), ctx_);
    upload_scene(world, camera);
    RaynFrameDesc f = frame_desc(integrator, tile_w, tile_h, frame, t0, t1, samples, sets_1d, sets_2d);
    f.samples_1d = s1.data(), f.samples_2d = s2.data(), f.scramble = scr.data(), f.fis_inverse_cdf = fis.data();
    albedo.assign((size_t)3 * w_ * h_, 0.0f);
    check(rayn_b200_render_albedo(ctx_, &f, albedo.data(), RAYN_MEM_HOST), ctx_);
  }
  // Edge-avoiding a-trous filter of color and background in place, guided by normal and alpha (rayn_b200_film_denoise).
  void denoise(int iterations, float sigma_color, float sigma_normal, float sigma_alpha) {
    const RaynDenoiseDesc d{iterations, sigma_color, sigma_normal, sigma_alpha};
    RaynFilmPlanes p{color.data(), alpha.data(), background.data(), normal.data(), RAYN_MEM_HOST};
    check(rayn_b200_film_denoise(ctx_, &d, w_, h_, &p, &p), ctx_);
  }
  // ... also guided by the albedo plane of render_albedo (rayn_b200_film_denoise_albedo)
  void denoise_albedo(int iterations, float sigma_color, float sigma_normal, float sigma_alpha, float sigma_albedo) {
    const RaynDenoiseDesc d{iterations, sigma_color, sigma_normal, sigma_alpha};
    RaynFilmPlanes p{color.data(), alpha.data(), background.data(), normal.data(), RAYN_MEM_HOST};
    check(rayn_b200_film_denoise_albedo(ctx_, &d, sigma_albedo, albedo.data(), w_, h_, &p, &p), ctx_);
  }
  // ... guided by each pixel's variance from the moments of render_frame_into(..., moments = true) and the film's spp
  // (rayn_b200_film_denoise_variance), and by the albedo plane of render_albedo if with_albedo.  The moments describe the
  // unfiltered film, so they are dropped once it is filtered (like rayn_b200.film.Film.denoise).
  void denoise_variance(int iterations, float sigma_color, float sigma_normal, float sigma_alpha, float sigma_luminance, bool with_albedo,
                        float sigma_albedo) {
    if (color_lum2.empty()) throw std::runtime_error("denoise_variance needs a render_frame_into(..., moments = true) first");
    if (with_albedo && albedo.empty()) throw std::runtime_error("denoise_variance with the albedo guide needs render_albedo first");
    const RaynDenoiseDesc d{iterations, sigma_color, sigma_normal, sigma_alpha};
    RaynFilmPlanes p{color.data(), alpha.data(), background.data(), normal.data(), RAYN_MEM_HOST};
    const RaynMomentPlanes m{color_lum2.data(), background_lum2.data(), RAYN_MEM_HOST};
    check(rayn_b200_film_denoise_variance(ctx_, &d, sigma_luminance, spp_, &m, sigma_albedo, with_albedo ? albedo.data() : nullptr, w_, h_, &p, &p),
          ctx_);
    color_lum2.clear(), background_lum2.clear();
  }
  // Any of the filters above on a panorama's film, periodic in x (rayn_b200_film_denoise_wrap): sigma_luminance = +inf is the
  // filter without the variance term, with_albedo adds the albedo guide of render_albedo.
  void denoise_wrap(int iterations, float sigma_color, float sigma_normal, float sigma_alpha, float sigma_luminance, bool with_albedo,
                    float sigma_albedo) {
    const bool var = !std::isinf(sigma_luminance);
    if (var && color_lum2.empty()) throw std::runtime_error("denoise_wrap with the variance term needs a render_frame_into(..., moments = true) first");
    if (with_albedo && albedo.empty()) throw std::runtime_error("denoise_wrap with the albedo guide needs render_albedo first");
    const RaynDenoiseDesc d{iterations, sigma_color, sigma_normal, sigma_alpha};
    RaynFilmPlanes p{color.data(), alpha.data(), background.data(), normal.data(), RAYN_MEM_HOST};
    const RaynMomentPlanes m{color_lum2.data(), background_lum2.data(), RAYN_MEM_HOST};
    check(rayn_b200_film_denoise_wrap(ctx_, &d, sigma_luminance, spp_, var ? &m : nullptr, nullptr, sigma_albedo,
                                      with_albedo ? albedo.data() : nullptr, w_, h_, &p, &p),
          ctx_);
    if (var) color_lum2.clear(), background_lum2.clear();
  }
  int width() const { return w_; }
  int height() const { return h_; }
  std::vector<float> color, alpha, background, normal;
  std::vector<float> albedo;          // render_albedo: [3*W*H]
  std::vector<float> color_lum2, background_lum2;  // render_frame_into(..., moments = true): [W*H] each
  std::vector<double> tile_errors;    // render_adaptive: E per tile index tile_x * n_tiles_y + tile_y
  std::vector<int64_t> tile_samples;  // ... and samples per pixel
  RaynStats stats{};
  int progressive_epoch = 0;

 private:
  void upload_scene(const World& world, CameraHandle camera) {
    std::vector<RaynLight> lights;
    for (const auto& l : world.lights) lights.push_back(l.pod);
    RaynSceneDesc sc{};
    sc.n_hitables = (int)world.hitables.items.size(), sc.hitables = world.hitables.items.data();
    sc.n_materials = (int)world.materials.items.size(), sc.materials = world.materials.items.data();
    sc.n_lights = (int)lights.size(), sc.lights = lights.data();
    sc.camera = world.cameras.get(camera);
    sc.volume = RaynVolume{world.volume_params.has_scattering, world.volume_params.coeff_scattering, world.volume_params.has_extinction,
                           world.volume_params.coeff_extinction};
    sc.consts = world.consts;
    check(rayn_b200_upload_scene(ctx_, &sc), ctx_);
    if (!world.materials.traps.empty())
      check(rayn_b200_set_albedo_traps(ctx_, (int32_t)world.materials.traps.size(), world.materials.traps.data()), ctx_);
  }
  RaynFrameDesc frame_desc(const PathTracingIntegrator& integrator, int tile_w, int tile_h, int frame, float t0, float t1, int samples, int sets_1d,
                           int sets_2d) const {
    RaynFrameDesc f{};
    f.width = w_, f.height = h_, f.tile_w = tile_w, f.tile_h = tile_h, f.samples = samples;
    f.max_bounces = integrator.max_bounces, f.volume_marches = integrator.volume_marches, f.frame = frame, f.t0 = t0, f.t1 = t1;
    f.sets_1d = sets_1d, f.sets_2d = sets_2d;
    f.input_space = RAYN_MEM_HOST, f.tile_offset = 0, f.tile_stride = 1;
    return f;
  }
  int w_, h_;
  int spp_ = 0;  // samples per pixel of the last render_frame_into
  RaynContext* ctx_ = nullptr;
};

}  // namespace rayn
