// main.cpp — stand-in for rayn's src/main.rs + src/setup.rs on top of the C ABI.
//   rayn_host [--config 1..5] [--res W H] [--samples S] [--bounces B] [--adaptive THRESHOLD [--rounds MAX]] [--denoise L]
//             [--denoise-albedo] [--denoise-variance] [--orbit-trap LO HI R0 G0 B0 R1 G1 B1] [--out file.ppm] [--dump planes.bin]
// --denoise-albedo (with --denoise) renders the first-hit albedo plane as rayn_b200.film.Film does and guides the filter with it.
// --denoise-variance (with --denoise, not with --adaptive) renders the frame with its luminance moments and weights each
// pixel's colour by its own variance, as rayn_b200.film.Film does with a "moments" channel; combinable with --denoise-albedo.
// --orbit-trap colours the fractal of configs 2-5 by orbit trap: albedo (R0 G0 B0) at trap LO, (R1 G1 B1) at HI
// (include/rayn_b200.h, RaynAlbedoTrap; tools/trap_range.py prints a range for config 3).
// Renders one frame (frame 1, shutter 1/24 at 24 fps: main.rs:47-49,61-62), prints the reference's
// "Done in {s} seconds." line (main.rs:79-82) and writes the display image with the formula of
// Film::save_to (film.rs:253-267): (color + background).saturated().gamma_corrected(2.2), y flipped.
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "rayn_host.hpp"

using namespace rayn;

static constexpr float WORLD_RADIUS = 100.0f;    // setup.rs:33
static constexpr int FRACTAL_ITERATIONS = 12;    // setup.rs:44
// --denoise sigmas: the library's defaults (rayn_b200/film.py DENOISE_DEFAULTS, picked in DESIGN.md §4b)
static constexpr float kDenoiseSigmaColor = 2.5f, kDenoiseSigmaNormal = 0.4f, kDenoiseSigmaAlpha = 0.5f;
// --denoise-albedo: rayn_b200/film.py DENOISE_ALBEDO_SIGMA and ALBEDO_SAMPLES (picked in DESIGN.md §4e)
static constexpr float kDenoiseAlbedoSigma = 0.2f;
static constexpr int kAlbedoSamples = 16;
// --denoise-variance: rayn_b200/film.py DENOISE_LUMINANCE_SIGMA and DENOISE_VARIANCE_SIGMA_COLOR (picked in DESIGN.md §4f)
static constexpr float kDenoiseLuminanceSigma = 4.0f, kDenoiseVarianceSigmaColor = INFINITY;

// --adaptive: the library's defaults (rayn_b200/film.py ADAPTIVE_THRESHOLD / ADAPTIVE_MAX_ROUNDS, picked in DESIGN.md §4c)
static constexpr float kAdaptiveThreshold = 0.025f;
static constexpr int kAdaptiveMaxRounds = 32;

// setup.rs:46-169; `fractal` 0 = Mandelbox (the reference scene), 1 = authored Mandelbulb
// trap: the fractal's albedo generator (--orbit-trap), NULL = the reference's constant grey
static CameraHandle setup(World& world, float rx, float ry, bool volume, int fractal, bool thinlens, const OrbitTrapAlbedo* trap = nullptr) {
  if (volume) world.volume_params = VolumeParams{true, true, 0.25f, 0.035f};                      // :55-60
  const MaterialHandle sky = world.materials.add_material(Sky(Srgb(0.3f, 0.4f, 0.6f), Srgb(0.2f, 0.3f, 0.6f) * 0.05f));  // :63-69
  world.hitables.push(Sphere(Vec3(0, 0, 0), WORLD_RADIUS, sky));                                  // :71
  const MaterialHandle grey = trap ? world.materials.add_material(Dielectric::new_remap(*trap, 0.6f))
                                   : world.materials.add_material(Dielectric::new_remap(Srgb(0.2f, 0.2f, 0.2f), 0.6f));  // :76
  if (fractal == 0)
    world.hitables.push(TracedSDF(MandelBox(FRACTAL_ITERATIONS, BoxFold(1.0f), SphereFold(0.01f, 1.9f), -2.1f), grey));  // :78-86
  else
    world.hitables.push(TracedSDF(Mandelbulb(8, 8, 2.0f), grey));
  const Srgb green = Srgb(1.5f, 4.5f, 3.0f).normalized(), blue = Srgb(1.5f, 3.0f, 4.5f).normalized();  // :99-100
  const MaterialHandle blue_emissive = world.materials.add_material(Emissive::new_splat(blue * 3.0f));
  const MaterialHandle green_emissive = world.materials.add_material(Emissive::new_splat(green * 3.0f));
  const std::pair<Vec3, float> light_pairs[2] = {{Vec3(1.2f, -1.2f, 1.2f), 0.15f}, {Vec3(-1.2f, 1.2f, 1.2f), 0.15f}};  // :106-109
  for (const auto& lp : light_pairs) {
    Vec3 green_pos = lp.first;
    green_pos.y *= -1.0f;
    world.lights.push_back(SphereLight(green_pos, lp.second, green * 40.0f));
    world.lights.push_back(SphereLight(lp.first, lp.second, blue * 40.0f));
    world.hitables.push(Sphere(green_pos, lp.second - 0.01f, green_emissive));
    world.hitables.push(Sphere(lp.first, lp.second - 0.01f, blue_emissive));
  }
  world.lights.push_back(SphereLight(Vec3::zero(), 0.25f, green * 20.0f));                        // :121
  world.hitables.push(Sphere(Vec3::zero(), 0.24f, green_emissive));                               // :122
  const Vec3 origin = Vec3(-0.45f, 0.2f, 2.0f) * 2.25f;                                           // :134
  if (thinlens) return world.cameras.add_camera(ThinLensCamera(rx, ry, 60.0f, 0.05f, origin, Vec3(0, 0, 0), Vec3(0, 1, 0), Vec3(0, 0, 0)));
  return world.cameras.add_camera(PinholeCamera(rx, ry, 60.0f, origin, Vec3(0, 0, 0), Vec3(0, 1, 0)));  // :129-141
}

static CameraHandle setup_single_sphere(World& world, float rx, float ry) {  // BASELINE config 1
  const MaterialHandle sky = world.materials.add_material(Sky(Srgb(0.3f, 0.4f, 0.6f), Srgb(0.2f, 0.3f, 0.6f) * 0.05f));
  world.hitables.push(Sphere(Vec3(0, 0, 0), WORLD_RADIUS, sky));
  const MaterialHandle grey = world.materials.add_material(Dielectric::new_remap(Srgb(0.2f, 0.2f, 0.2f), 0.6f));
  world.hitables.push(Sphere(Vec3(0, 0, 0), 1.0f, grey));
  world.lights.push_back(SphereLight(Vec3(1.2f, 1.2f, 1.2f), 0.15f, Srgb(1, 1, 1) * 40.0f));
  return world.cameras.add_camera(PinholeCamera(rx, ry, 60.0f, Vec3(-0.45f, 0.2f, 2.0f) * 2.25f, Vec3(0, 0, 0), Vec3(0, 1, 0)));
}

int main(int argc, char** argv) {
  int config = 3, W = 1280, H = 720, samples = 2, bounces = 3;  // setup.rs:16,22,30 defaults
  int denoise = 0;  // a-trous levels run after the render, before --out / --dump; 0 = off
  bool denoise_albedo = false, denoise_variance = false;
  bool adaptive = false;  // --adaptive: rounds of --samples each until every tile's error <= threshold (at most --rounds)
  float threshold = kAdaptiveThreshold;
  int max_rounds = kAdaptiveMaxRounds;
  bool res_set = false, samples_set = false, bounces_set = false;
  const char *out = nullptr, *dump = nullptr, *dump_scene = nullptr;
  bool orbit_trap = false;
  OrbitTrapAlbedo trap{0.0f, 1.0f, Srgb(0, 0, 0), Srgb(0, 0, 0)};
  for (int i = 1; i < argc; ++i) {
    if (!strcmp(argv[i], "--config") && i + 1 < argc) config = atoi(argv[++i]);
    else if (!strcmp(argv[i], "--res") && i + 2 < argc) W = atoi(argv[++i]), H = atoi(argv[++i]), res_set = true;
    else if (!strcmp(argv[i], "--samples") && i + 1 < argc) samples = atoi(argv[++i]), samples_set = true;
    else if (!strcmp(argv[i], "--bounces") && i + 1 < argc) bounces = atoi(argv[++i]), bounces_set = true;
    else if (!strcmp(argv[i], "--out") && i + 1 < argc) out = argv[++i];
    else if (!strcmp(argv[i], "--dump") && i + 1 < argc) dump = argv[++i];
    else if (!strcmp(argv[i], "--dump-scene") && i + 1 < argc) dump_scene = argv[++i];
    else if (!strcmp(argv[i], "--denoise") && i + 1 < argc) denoise = atoi(argv[++i]);
    else if (!strcmp(argv[i], "--denoise-albedo")) denoise_albedo = true;
    else if (!strcmp(argv[i], "--denoise-variance")) denoise_variance = true;
    else if (!strcmp(argv[i], "--adaptive") && i + 1 < argc) adaptive = true, threshold = (float)atof(argv[++i]);
    else if (!strcmp(argv[i], "--rounds") && i + 1 < argc) max_rounds = atoi(argv[++i]);
    else if (!strcmp(argv[i], "--orbit-trap") && i + 8 < argc) {
      float v[8];
      for (int k = 0; k < 8; ++k) v[k] = (float)atof(argv[++i]);
      trap = OrbitTrapAlbedo{v[0], v[1], Srgb(v[2], v[3], v[4]), Srgb(v[5], v[6], v[7])};
      orbit_trap = true;
    } else {
      fprintf(stderr, "usage: rayn_host [--config 1..5] [--res W H] [--samples S] [--bounces B] [--adaptive THRESHOLD [--rounds MAX]] "
                      "[--denoise L [--denoise-albedo] [--denoise-variance]] [--orbit-trap LO HI R0 G0 B0 R1 G1 B1] [--out f.ppm] [--dump f.bin]\n");
      return 2;
    }
  }
  if (denoise < 0 || denoise > 8) { fprintf(stderr, "--denoise takes 1..8 levels (0 = off)\n"); return 2; }
  if (denoise_albedo && !denoise) { fprintf(stderr, "--denoise-albedo needs --denoise L\n"); return 2; }
  if (denoise_variance && !denoise) { fprintf(stderr, "--denoise-variance needs --denoise L\n"); return 2; }
  if (denoise_variance && adaptive) { fprintf(stderr, "--denoise-variance needs one render: the adaptive accumulator keeps no moments\n"); return 2; }
  if (max_rounds < 2) { fprintf(stderr, "--rounds takes at least 2 rounds\n"); return 2; }
  static const int cfg_res[6][2] = {{0, 0}, {256, 256}, {1024, 1024}, {1920, 1080}, {2048, 2048}, {7680, 4320}};
  static const int cfg_samples[6] = {0, 1, 32, 128, 64, 256}, cfg_bounces[6] = {0, 2, 4, 8, 4, 8};
  if (config < 1 || config > 5) { fprintf(stderr, "config must be 1..5\n"); return 2; }
  if (orbit_trap && config == 1) { fprintf(stderr, "--orbit-trap colours the fractal of configs 2-5\n"); return 2; }
  if (!res_set) W = cfg_res[config][0], H = cfg_res[config][1];
  if (!samples_set) samples = cfg_samples[config];
  if (!bounces_set) bounces = cfg_bounces[config];
  try {
    World world;
    const CameraHandle camera = config == 1 ? setup_single_sphere(world, (float)W, (float)H)
                                            : setup(world, (float)W, (float)H, config == 4, config == 3 ? 0 : 1, config == 4,
                                                    orbit_trap ? &trap : nullptr);
    if (dump_scene) {  // flattened World as raw PODs (no GPU needed): hitables | materials | lights | camera | volume
      FILE* f = fopen(dump_scene, "wb");
      if (!f) { perror(dump_scene); return 1; }
      fwrite(world.hitables.items.data(), sizeof(RaynHitable), world.hitables.items.size(), f);
      fwrite(world.materials.items.data(), sizeof(RaynMaterial), world.materials.items.size(), f);
      for (const auto& l : world.lights) fwrite(&l.pod, sizeof(RaynLight), 1, f);
      fwrite(&world.cameras.get(camera), sizeof(RaynCamera), 1, f);
      const RaynVolume v{world.volume_params.has_scattering, world.volume_params.coeff_scattering, world.volume_params.has_extinction,
                         world.volume_params.coeff_extinction};
      fwrite(&v, sizeof v, 1, f);
      fclose(f);
      return 0;
    }
    Film film(W, H);
    const PathTracingIntegrator integrator{bounces, 2};  // main.rs:53-56
    const BlackmanHarrisFilter filter{1.5f};             // main.rs:51
    const int frame = 1, frame_rate = 24;
    const float frame_start = (float)frame * (1.0f / (float)frame_rate), frame_end = frame_start + 1.0f / 24.0f;  // main.rs:61-62
    const auto t0 = std::chrono::steady_clock::now();
    if (adaptive) {
      const int rounds = film.render_adaptive(world, camera, integrator, filter, 16, 16, frame, frame_start, frame_end, samples, 2, max_rounds, threshold);
      const double secs = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
      printf("Done in %.3f seconds.\n", secs);  // main.rs:79-82
      int64_t total = 0, done = 0;
      for (size_t t = 0; t < film.tile_samples.size(); ++t) total += film.tile_samples[t], done += film.tile_errors[t] <= (double)threshold;
      printf("%dx%d, %d rounds of %d spp, %d bounces: %.1f spp per tile on average, %lld of %zu tiles below E = %g\n", W, H, rounds, 4 * samples,
             bounces, (double)total / (double)std::max<size_t>(film.tile_samples.size(), 1), (long long)done, film.tile_samples.size(), threshold);
    } else {
      film.render_frame_into(world, camera, integrator, filter, 16, 16, frame, frame_start, frame_end, samples, denoise_variance);
      const double secs = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
      printf("Done in %.3f seconds.\n", secs);  // main.rs:79-82
      printf("%dx%d, %d spp, %d bounces: %.2f Msamples/s (device %.1f ms, %lld kernel launches)\n", W, H, 4 * samples, bounces,
             (double)film.stats.paths / secs / 1e6, film.stats.total_ms, (long long)film.stats.launches);
    }
    if (denoise_albedo)
      film.render_albedo(world, camera, integrator, filter, 16, 16, frame, frame_start, frame_end,
                         std::min(adaptive ? samples * max_rounds : samples, kAlbedoSamples));
    if (denoise_variance) {
      film.denoise_variance(denoise, kDenoiseVarianceSigmaColor, kDenoiseSigmaNormal, kDenoiseSigmaAlpha, kDenoiseLuminanceSigma, denoise_albedo,
                            kDenoiseAlbedoSigma);
    } else if (denoise_albedo) {
      film.denoise_albedo(denoise, kDenoiseSigmaColor, kDenoiseSigmaNormal, kDenoiseSigmaAlpha, kDenoiseAlbedoSigma);
    } else if (denoise) {
      film.denoise(denoise, kDenoiseSigmaColor, kDenoiseSigmaNormal, kDenoiseSigmaAlpha);
    }
    if (dump) {
      FILE* f = fopen(dump, "wb");
      if (!f) { perror(dump); return 1; }
      fwrite(film.color.data(), 4, film.color.size(), f), fwrite(film.alpha.data(), 4, film.alpha.size(), f);
      fwrite(film.background.data(), 4, film.background.size(), f), fwrite(film.normal.data(), 4, film.normal.size(), f);
      fclose(f);
    }
    if (out) {
      FILE* f = fopen(out, "wb");
      if (!f) { perror(out); return 1; }
      fprintf(f, "P6\n%d %d\n255\n", W, H);
      for (int y = H - 1; y >= 0; --y)  // film.rs:236 y flip
        for (int x = 0; x < W; ++x)
          for (int c = 0; c < 3; ++c) {
            const size_t i = 3 * ((size_t)x + (size_t)y * W) + c;
            float v = film.color[i] + film.background[i];  // film.rs:262
            v = std::pow(std::fmin(std::fmax(v, 0.0f), 1.0f), 1.0f / 2.2f);
            fputc((int)std::fmin(std::fmax(v * 255.0f, 0.0f), 255.0f), f);
          }
      fclose(f);
    }
  } catch (const std::exception& e) {
    fprintf(stderr, "rayn_host: %s\n", e.what());
    return 1;
  }
  return 0;
}
