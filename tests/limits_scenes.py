"""Scenes at the limits of include/rayn_b200.h (16 hitables, 16 materials, 16 lights), scenes with exact ties, boundary
sample tables and the many-light direct-illumination scene with its float64 closed form.  Shared by test_cpu_limits.py
and test_gpu_limits.py.  Every random choice is seeded, so every scene is reproducible."""
import numpy as np

from rayn_b200 import (BoxFold, CameraStore, Dielectric, Emissive, HitableStore, Lambertian, Linear, MandelBox, Mandelbulb,
                       MaterialStore, PathTracingIntegrator, PinholeCamera, Sky, Sphere, SphereFold, SphereLight, Srgb, TracedSDF,
                       Vec3, VolumeParams, World, configs)
from rayn_b200 import _lib as L
from rayn_b200.film import FrameInputs
from rayn_b200.scene import OrbitTrapAlbedo

TR = configs.frame_time_range(1)
N = 16  # RAYN_MAX_HITABLES == RAYN_MAX_MATERIALS == RAYN_MAX_LIGHTS
CAMERA_ORIGIN = Vec3(-0.45, 0.2, 2.0) * 2.25  # setup.rs:134
VOLUME = VolumeParams(0.25, 0.035)            # setup.rs:55-60
# kinds of materials 1..15 (material 0 is the sky): every kind present, material 15 is trap-able, the shape-A Mandelbox (8) is shaded
KINDS = "DLEDLDELDLDELDL"
TRAPPABLE = [m for m in range(1, N) if KINDS[m - 1] in "LD"]
TRAP_RANGE = (0.05, 2.5)  # wide enough for every Mandelbox and Mandelbulb below; constant outside it


def _materials(rng, traps):
    mats = MaterialStore()
    mats.add_material(Sky(Srgb(0.3, 0.4, 0.6), Srgb(0.2, 0.3, 0.6) * 0.05))
    for m in range(1, N):
        kind = KINDS[m - 1]
        albedo = Srgb(*rng.uniform(0.1, 0.9, 3))
        if kind in "LD" and traps:
            albedo = OrbitTrapAlbedo(*TRAP_RANGE, rng.uniform(0.05, 0.95, 3), rng.uniform(0.05, 0.95, 3))
        if kind == "L":
            mats.add_material(Lambertian(albedo))
        elif kind == "D":
            mats.add_material(Dielectric.new_remap(albedo, float(rng.uniform(0.2, 0.9))))
        else:
            mats.add_material(Emissive.new_splat(Srgb(*rng.uniform(0.5, 3.0, 3))))
    return mats


def _lights(rng, n=N):
    """n sphere lights on a shell around the fractals, each with its own radius and colour"""
    out = []
    for _ in range(n):
        d = rng.normal(size=3)
        p = d / np.linalg.norm(d) * rng.uniform(2.2, 3.2)
        out.append(SphereLight(Vec3(*p), float(rng.uniform(0.08, 0.25)), Srgb(*rng.uniform(5.0, 40.0, 3))))
    return out


def _small_sphere(rng, material, moving=False):
    c = Vec3(*rng.uniform(-1.6, 1.6, 3))
    if moving:
        c = Linear(c, Vec3(*rng.uniform(-12.0, 12.0, 3)))  # up to ~0.5 units over the shutter
    return Sphere(c, float(rng.uniform(0.12, 0.4)), material)


def _world(hitables, lights, mats, res, volume):
    cams = CameraStore()
    cam = cams.add_camera(PinholeCamera(res, 60.0, CAMERA_ORIGIN, Vec3(0, 0, 0), Vec3(0, 1, 0)))
    return cam, World(hitables, lights, mats, cams, VOLUME if volume else VolumeParams(None, None))


def reference_box():
    return MandelBox(configs.FRACTAL_ITERATIONS, BoxFold(1.0), SphereFold(0.01, 1.9), -2.1)  # setup.rs:84


def shape_a(res, volume, traps=False, seed=1):
    """setup.rs's shape at the limit: [sky sphere, 7 spheres, reference Mandelbox, 7 spheres], 16 materials, 16 lights"""
    rng = np.random.default_rng(seed)
    mats = _materials(rng, traps)
    hits = HitableStore()
    hits.push(Sphere(Vec3(0, 0, 0), configs.WORLD_RADIUS, 0))
    for m in range(1, 8):
        hits.push(_small_sphere(rng, m))
    hits.push(TracedSDF(reference_box(), 8))
    for m in range(9, N):
        hits.push(_small_sphere(rng, m))
    return _world(hits, _lights(rng), mats, res, volume)


# the 15 (16) SDFs of shape B: (kind, iterations, scale) - Mandelboxes with the reference fold constants at 12 iterations
# (variant 4, or 1 without the three-operation division) and at other counts (5 / 2), one with box_l = 0 that fails
# sdf_box_fast_ok (generic variant 0), and Mandelbulbs (3); scales differ so that they overlap around the origin
B_SDFS = [("box", 12, -2.1), ("bulb", 8, 0), ("box", 7, -1.8), ("bulb", 5, 0), ("box", 12, -2.4), ("box0", 6, -2.0),
          ("bulb", 3, 0), ("box", 9, -1.6), ("box", 12, -1.9), ("bulb", 10, 0), ("box", 4, -2.6), ("bulb", 6, 0),
          ("box", 12, -2.2), ("box", 15, -2.0), ("bulb", 4, 0), ("box", 10, -2.3)]
B_VARIANTS = {"box": {1, 2, 4, 5}, "box0": {0}, "bulb": {3}}


def _b_sdf(kind, iters, scale):
    if kind == "bulb":
        return Mandelbulb(iters, 8, 2.0)
    return MandelBox(iters, BoxFold(0.0 if kind == "box0" else 1.0), SphereFold(0.01, 1.9), scale)


def shape_b(res, volume, sky=True, traps=False, seed=2):
    """many SDFs: a sky sphere and 15 SDF hitables, or (sky=False) 16 SDFs and no sphere, so that missed rays are dropped;
    every hitable has its own material.  Without a sky sphere material 0 (Sky) shades the first SDF."""
    rng = np.random.default_rng(seed)
    mats = _materials(rng, traps)
    hits = HitableStore()
    if sky:
        hits.push(Sphere(Vec3(0, 0, 0), configs.WORLD_RADIUS, 0))
    for k, (kind, iters, scale) in enumerate(B_SDFS[:N - 1] if sky else B_SDFS):
        hits.push(TracedSDF(_b_sdf(kind, iters, scale), k + 1 if sky else k))
    return _world(hits, _lights(rng), mats, res, volume)


def b_kinds(sky=True):
    """[(hitable index, kind in B_VARIANTS)] of shape B's SDFs"""
    off = 1 if sky else 0
    return [(k + off, kind) for k, (kind, _, _) in enumerate(B_SDFS[:N - 1] if sky else B_SDFS)]


def shape_c(res, volume, seed=3):
    """moving spheres at the limit: a sky sphere and 15 spheres with non-zero centre velocity (no SDF)"""
    rng = np.random.default_rng(seed)
    mats = _materials(rng, False)
    hits = HitableStore()
    hits.push(Sphere(Vec3(0, 0, 0), configs.WORLD_RADIUS, 0))
    for m in range(1, N):
        hits.push(_small_sphere(rng, m, moving=True))
    return _world(hits, _lights(rng), mats, res, volume)


def spheres_only(seed=4):
    """16 static spheres around the origin (sky sphere first): the scene of the float64 closest-hit check"""
    rng = np.random.default_rng(seed)
    mats = _materials(rng, False)
    hits = HitableStore()
    hits.push(Sphere(Vec3(0, 0, 0), configs.WORLD_RADIUS, 0))
    for m in range(1, N):
        hits.push(_small_sphere(rng, m))
    return _world(hits, _lights(rng), mats, (32, 32), False)


SHAPES = {"A": shape_a, "B": shape_b, "B16": lambda res, volume, **kw: shape_b(res, volume, sky=False, **kw), "C": shape_c}


def inputs(res, samples, max_bounces, frame=1):
    integ = PathTracingIntegrator(max_bounces, 2)
    return integ, FrameInputs(res[0], res[1], samples, integ, frame=frame)


# ---- exact ties ------------------------------------------------------------------------------------------------------
def _tie_base(res):
    """config 3 (setup.rs, no volume) with two spare materials: a Lambertian for the first copy, an Emissive for the second"""
    cam, world = configs.setup(res, volume=False, fractal="mandelbox")
    first = world.materials.add_material(Lambertian(Srgb(0.7, 0.5, 0.3)))
    second = world.materials.add_material(Emissive.new_splat(Srgb(0.5, 2.0, 3.0)))
    return cam, world, first, second


def tie_scene(kind, res, second_material=None):
    """-> (camera, world, index of the later duplicate).  kind:
      spheres_before / spheres_after / spheres_across: two identical spheres before, after or on both sides of the Mandelbox;
      boxes_adjacent / boxes_separated: two identical Mandelboxes, next to each other or with a sphere between them.
    The first copy has a Lambertian, the later one an Emissive (second_material: another material for it)."""
    cam, world, first, second = _tie_base(res)
    second = second if second_material is None else world.materials.add_material(second_material)
    items = world.hitables.items
    sky, box, emitters = items[0], items[1], items[2:]
    at = Vec3(-0.45, 0.35, 2.6)  # between the camera and the Mandelbox, in the middle of the view
    s1, s2 = Sphere(at, 0.4, first), Sphere(at, 0.4, second)
    b1, b2 = TracedSDF(box.sdf, first), TracedSDF(box.sdf, second)
    order = {"spheres_before": [sky, s1, s2, box], "spheres_after": [sky, box, s1, s2], "spheres_across": [sky, s1, box, s2],
             "boxes_adjacent": [sky, b1, b2], "boxes_separated": [sky, b1, emitters[0], b2]}[kind]
    later = s2 if kind.startswith("spheres") else b2
    world.hitables.items = order + [e for e in emitters if e not in order]
    return cam, world, world.hitables.items.index(later)


def light_tie_scene(res):
    """config 3 with a sphere exactly where a light is (same centre and radius) and every light listed twice"""
    cam, world = configs.setup(res, volume=True, fractal="mandelbox")
    lights = world.lights
    grey = world.hitables.items[1].material
    world.hitables.push(Sphere(Vec3(*lights[0].pos), float(lights[0].rad), grey))
    world.lights = [SphereLight(Vec3(*l.pos), float(l.rad), Srgb(*l.emission)) for l in lights for _ in range(2)]
    return cam, world


# ---- boundary sample tables --------------------------------------------------------------------------------------------
ONE_MINUS = np.float32(1) - np.float32(2.0 ** -24)  # the largest float below 1


def boundary_values(materials=()):
    """The sample values at which the path changes branch: 0, 2^-24, 0.5 - 2^-25, 0.5, 1 - 2^-24; k/n and its neighbouring
    floats for n = 1..16 (floor(s * n_lights), the concentric map and the FIS lookup); the Schlick fresnel at normal
    incidence (0.04, the Dielectric lobe choice) and its neighbours; the roulette factors 0.05 and 1 - max channel of every
    albedo the throughput can take after one bounce."""
    f = np.float32
    vals = [f(0.0), f(2.0 ** -24), f(0.5) - f(2.0 ** -25), f(0.5), ONE_MINUS]
    for n in range(1, 17):
        for k in range(n + 1):
            x = f(k) / f(n)
            vals += [np.nextafter(x, f(0)), x, np.nextafter(x, f(1))]
    for x in (f(0.04) + f(0.96) * f(0.0), f(0.05)):
        vals += [np.nextafter(x, f(0)), x, np.nextafter(x, f(1))]
    for m in materials:
        a = getattr(m, "albedo", None)
        if a is not None:
            vals.append(f(1.0) - f(np.max(a)))
    v = np.unique(np.array(vals, np.float32))
    return v[(v >= 0) & (v < 1)]


def set_families(integrator):
    """1-D / 2-D set indices of each dimension family, by the layout of oracle/rayn_oracle.cpp and rt_kernels.cuh::slot_ctx:
    1-D set 0 = camera time, set 1 + depth * n1 + k (k = 0: surface light choice, 1..vm: volume light choices, 1 also the
    volume sample, vm + 1: BSDF lobe, vm + 2: roulette); 2-D set 0 = camera / FIS, 1 = lens, 2 + depth * n2h + k (k < 4:
    surface light samples, 4 .. 4 + 4 vm: volume light samples, then two BSDF sets).  -> {family: (sets_1d, sets_2d)}"""
    vm, mb = integrator.volume_marches, integrator.max_bounces
    n1, n2h = 3 + vm, (12 + 8 * vm) // 2
    depths = range(mb + 1)
    s1 = lambda ks: [1 + d * n1 + k for d in depths for k in ks]  # noqa: E731
    s2 = lambda ks: [2 + d * n2h + k for d in depths for k in ks]  # noqa: E731
    return {"camera": ([0], [0]), "lens": ([], [1]), "light_choice": (s1(range(1 + vm)), []), "volume": (s1([1]), s2(range(4, 4 + 4 * vm))),
            "light_sample": ([], s2(range(4))), "bsdf": (s1([vm + 1]), s2(range(4 + 4 * vm, n2h))), "roulette": (s1([vm + 2]), [])}


def boundary_tables(inp, values, seed, family=None, integrator=None, scramble=None):
    """Overwrites inp's sample tables with values drawn (seeded) from `values`: all of them, or only the sets of one
    dimension family (set_families).  scramble: a constant for the whole scramble plane (None keeps SmallRng's)."""
    rng = np.random.default_rng(seed)
    spp = inp.spp
    if family is None:
        inp.samples_1d[:] = rng.choice(values, inp.samples_1d.size)
        inp.samples_2d[:] = rng.choice(values, inp.samples_2d.size)
    else:
        sets_1d, sets_2d = set_families(integrator)[family]
        for s in sets_1d:
            inp.samples_1d[s * spp:(s + 1) * spp] = rng.choice(values, spp)
        for s in sets_2d:
            inp.samples_2d[2 * s * spp:2 * (s + 1) * spp] = rng.choice(values, 2 * spp)
    if scramble is not None:
        inp.scramble[:] = np.float32(scramble)
    return inp


# The path reads every sample as fract(table + scramble[pixel]) (sampler.rs, dm::fract).  With a constant scramble plane of
# 0 (no rotation) or 1 - 2^-24 (every read wraps), these table values read as exactly 0 and 1 - 2^-24:
# 0 + 0 = 0, (1 - 2^-24) + 0 = 1 - 2^-24;  2^-24 + (1 - 2^-24) = 1 -> 0, 0 + (1 - 2^-24) = 1 - 2^-24.
EXTREME_TABLE_VALUES = {0.0: (0.0, ONE_MINUS), float(ONE_MINUS): (np.float32(2.0 ** -24), 0.0)}


def extreme_family_tables(inp, family, integrator, scramble, seed):
    """one dimension family reads only 0 and 1 - 2^-24 (scramble: a key of EXTREME_TABLE_VALUES, set on the whole plane);
    the other families read their R_d values, rotated by the same constant"""
    values = np.array(EXTREME_TABLE_VALUES[scramble], np.float32)
    return boundary_tables(inp, values, seed, family=family, integrator=integrator, scramble=scramble)


# ---- many-light direct illumination and its closed form ------------------------------------------------------------------
CF_RES = (8, 8)
CF_ALBEDO = (0.6, 0.45, 0.3)


def closed_form_scene(seed=5):
    """A Lambertian unit sphere filling a pinhole camera's view (every camera ray hits it, also at the edge of the filter
    footprint), lit by 16 sphere lights that are fully above the horizon of every visible point; no sky sphere, no volume."""
    rng = np.random.default_rng(seed)
    mats, hits = MaterialStore(), HitableStore()
    hits.push(Sphere(Vec3(0, 0, 0), 1.0, mats.add_material(Lambertian(Srgb(*CF_ALBEDO)))))
    lights = []
    for _ in range(N):
        theta, phi = rng.uniform(0.0, np.radians(30.0)), rng.uniform(0.0, 2 * np.pi)
        d = np.array([np.sin(theta) * np.cos(phi), np.sin(theta) * np.sin(phi), np.cos(theta)])
        lights.append(SphereLight(Vec3(*(d * rng.uniform(3.5, 5.0))), float(rng.uniform(0.1, 0.3)), Srgb(*rng.uniform(2.0, 20.0, 3))))
    cams = CameraStore()
    cam = cams.add_camera(PinholeCamera(CF_RES, 16.0, Vec3(0.0, 0.0, 3.0), Vec3(0, 0, 0), Vec3(0, 1, 0)))
    return cam, World(hits, lights, mats, cams, VolumeParams(None, None))


def closed_form_film(world, camera, fis, m=48):
    """float64 expected colour of every pixel: (albedo / pi) sum_j E_j with E_j = pi L_j (r_j / d_j)^2 cos(theta_j) (the
    irradiance of a sphere source fully above the horizon), averaged over the pixel's filter footprint by a midpoint
    quadrature of m x m points through the FIS inverse-CDF table (film.rs sample_uv).  -> [H, W, 3]"""
    cam = world.cameras.get(camera)
    w, h = int(cam.res[0]), int(cam.res[1])
    inv = np.asarray(fis, np.float64)

    def fis_sample(u):  # filter.rs:222-235 in float64
        u = 2.0 * (u - 0.5)
        mult = np.where(u < 0.0, -1.0, 1.0)
        a = np.minimum(np.abs(u), 0.99999) * (L.RAYN_FIS_TABLE_SIZE - 1)
        i = np.floor(a).astype(int)
        return mult * (inv[i] + (inv[i + 1] - inv[i]) * (a - i))

    off = fis_sample((np.arange(m) + 0.5) / m)
    origin, at, up = (np.asarray(v[0], np.float64) for v in (cam.origin, cam.at, cam.up))
    bw = (origin - at) / np.linalg.norm(origin - at)
    bu = np.cross(up, bw); bu /= np.linalg.norm(bu)
    bv = np.cross(bw, bu)
    hx, hy = float(cam.half_width), float(cam.half_height)
    lower_left = origin - bu * hx - bv * hy - bw
    lights = [(np.asarray(l.pos, np.float64), float(l.rad), np.asarray(l.emission, np.float64)) for l in world.lights]
    albedo = np.asarray(world.materials.items[0].albedo, np.float64)
    out = np.zeros((h, w, 3))
    for y in range(h):
        for x in range(w):
            u = ((x + 0.5 + off)[:, None] / w) * np.ones((1, m))
            v = ((y + 0.5 + off)[None, :] / h) * np.ones((m, 1))
            d = lower_left + bu[None, None] * (2 * hx * u)[..., None] + bv[None, None] * (2 * hy * v)[..., None] - origin
            d /= np.linalg.norm(d, axis=-1, keepdims=True)
            b = d @ origin
            disc = b * b - (origin @ origin - 1.0)
            assert (disc > 0).all(), "a camera ray of the footprint misses the sphere"
            p = origin + d * (-b - np.sqrt(disc))[..., None]
            n = p  # unit sphere at the origin
            e = np.zeros(p.shape)
            for c, r, le in lights:
                to = c - p
                dist = np.linalg.norm(to, axis=-1)
                cos = np.sum(to * n, axis=-1) / dist
                assert (np.arccos(np.clip(cos, -1, 1)) + np.arcsin(r / dist) < np.pi / 2).all(), "light not above the horizon"
                e += np.pi * le * ((r / dist) ** 2 * cos)[..., None]
            out[y, x] = (albedo / np.pi * e).reshape(-1, 3).mean(0)
    return out


def closed_form_check(films, expected):
    """films: K colour planes [H, W, 3] of independent frames.  -> (worst per-pixel |z|, |z| of the film-wide mean), z in units
    of the standard error estimated from the spread between frames."""
    f = np.stack([np.asarray(x, np.float64).reshape(expected.shape) for x in films])
    k = len(f)
    mean, se = f.mean(0), f.std(0, ddof=1) / np.sqrt(k)
    z_px = np.abs(mean - expected) / np.maximum(se, 1e-12)
    wide = f.mean(axis=(1, 2))  # [K, 3]
    z_all = np.abs(wide.mean(0) - expected.mean(axis=(0, 1))) / np.maximum(wide.std(0, ddof=1) / np.sqrt(k), 1e-12)
    return float(z_px.max()), float(z_all.max())
