"""Host-side mirror of rayn's scene API (reference src/setup.rs, src/world.rs and the
constructors of the Hitable / Material / Light / Camera implementors).

Same names and argument meaning as the reference so that a scene script reads like
`setup.rs`; every object flattens into the plain-old-data descriptors of
include/rayn_b200.h (trait objects cannot cross a C ABI, SURVEY F5).  All host arithmetic is
done in numpy float32 to mirror the reference's f32 constructors.
"""
import ctypes as C
import math

import numpy as np

from . import _lib as L

f32 = np.float32


def _v3(v):
    a = np.asarray(v, dtype=np.float32).reshape(3)
    return a


class Vec3:
    """ultraviolet::Vec3 (host-side, constants only)."""

    def __init__(self, x, y, z):
        self.v = np.array([x, y, z], dtype=np.float32)

    @staticmethod
    def zero():
        return Vec3(0.0, 0.0, 0.0)

    def __mul__(self, s):
        return Vec3(*(self.v * f32(s)))

    def normalized(self):
        m = np.sqrt(np.sum(self.v * self.v, dtype=np.float32), dtype=np.float32)
        return Vec3(*(self.v / m))

    def copy(self):
        return Vec3(*self.v)

    @property
    def x(self):
        return self.v[0]

    @property
    def y(self):
        return self.v[1]

    @property
    def z(self):
        return self.v[2]


class Srgb(Vec3):
    """spectrum.rs Srgb newtype over Vec3."""

    def __mul__(self, s):
        return Srgb(*(self.v * f32(s)))

    def normalized(self):
        n = Vec3.normalized(self)
        return Srgb(*n.v)


def _arr(x):
    return x.v if isinstance(x, Vec3) else _v3(x)


class Linear:
    """A `Sequenced` parameter that is linear in time: value(t) = base + velocity * t.  Stands for the closure
    `move |t| base + velocity * t` a rayn scene would pass (animation.rs:55-68).  Like every closure-backed WSequenced it is
    evaluated at lane 0's time for a whole 4-lane packet (animation.rs:62-67).

    Any other closure `f(t) -> Vec3` (or a 3-sequence) may be passed where a scene takes a Linear, but only linear-in-time
    parameters cross the C ABI: each render uploads the closure's chord over its time range (Linear.chord)."""

    def __init__(self, base, velocity):
        self.base, self.velocity = base, velocity

    @staticmethod
    def chord(f, t0, t1):
        """The Linear that equals closure f at the shutter ends t0 and t1 (each rounded to float32 first, as the renderer
        takes them): velocity = (f(t1) - f(t0)) / (t1 - t0) and base = f(t0) - velocity * t0, computed in float64 and then
        rounded to float32; for t1 == t0, velocity 0 and base f(t0).  An approximation of rayn, which evaluates the closure at
        every packet's lane-0 time: the chord is exact at t0 and t1 only (up to the float32 rounding of base, velocity and
        the renderer's base + velocity * t), and in between it is the straight line between them."""
        t0, t1 = float(np.float32(t0)), float(np.float32(t1))
        a = np.asarray(_arr(f(t0)), np.float64)
        if t1 == t0:
            return Linear(a.astype(np.float32), np.zeros(3, np.float32))
        v = (np.asarray(_arr(f(t1)), np.float64) - a) / (t1 - t0)
        return Linear((a - v * t0).astype(np.float32), v.astype(np.float32))


def _is_closure(x):
    return callable(x) and not isinstance(x, (Vec3, Linear))


def _seq(x):
    """-> (base[3], velocity[3]) for a constant or Linear Vec3 parameter; a closure is kept as it is (see _at)."""
    if _is_closure(x):
        return x
    if isinstance(x, Linear):
        return _arr(x.base), _arr(x.velocity)
    return _arr(x), np.zeros(3, np.float32)


def _at(p, time_range):
    """-> (base[3], velocity[3]) of a parameter _seq made, for one render over time_range: a closure's chord there."""
    if not _is_closure(p):
        return p
    if time_range is None:
        raise ValueError("a scene with closure parameters needs the render's time_range to flatten (Linear.chord)")
    return _seq(Linear.chord(p, time_range[0], time_range[1]))


# ---- materials (material.rs) ---------------------------------------------------------------
class OrbitTrapAlbedo:
    """An albedo generator (rayn's `albedo_gen: WShadingParamGenerator<WSrgb>`, material.rs:75-83) that colours an SDF surface
    by orbit trap: the smallest squared radius the distance estimator's iteration reaches at the hit point (Mandelbox: the r2
    its sphere fold divides by; Mandelbulb: |w|^2), mapped linearly from [trap_lo, trap_hi] onto albedo_lo .. albedo_hi and
    clamped.  Hits on analytic spheres take albedo_hi.  The exact statement is in include/rayn_b200.h (RaynAlbedoTrap).
    Pass it as the albedo of Lambertian(...), Dielectric(...) or Dielectric.new_remap(...), or as the F0 of Metallic(...)."""

    def __init__(self, trap_lo, trap_hi, albedo_lo, albedo_hi):
        self.trap_lo, self.trap_hi = f32(trap_lo), f32(trap_hi)
        self.albedo_lo, self.albedo_hi = _arr(albedo_lo), _arr(albedo_hi)
        if not (np.isfinite(self.trap_lo) and np.isfinite(self.trap_hi) and self.trap_lo < self.trap_hi):
            raise ValueError(f"OrbitTrapAlbedo needs finite trap_lo < trap_hi, got {trap_lo}, {trap_hi}")
        if not (np.isfinite(self.albedo_lo).all() and np.isfinite(self.albedo_hi).all()):
            raise ValueError("OrbitTrapAlbedo needs finite albedos")

    def trap_desc(self, material):
        t = L.RaynAlbedoTrap()
        t.material = int(material)
        t.trap_lo, t.trap_hi = float(self.trap_lo), float(self.trap_hi)
        t.albedo_lo[:] = self.albedo_lo.tolist()
        t.albedo_hi[:] = self.albedo_hi.tolist()
        return t


def _albedo(albedo):
    """-> (constant albedo[3], OrbitTrapAlbedo or None).  A trap material's constant is albedo_hi (what analytic spheres get)."""
    if isinstance(albedo, OrbitTrapAlbedo):
        return albedo.albedo_hi.copy(), albedo
    return _arr(albedo), None


def _remap_roughness(roughness):
    """Roughness in [0,1] -> Phong exponent, material.rs:167-174 (Dielectric::new_remap), in float32."""
    r = f32(1.0) - f32(roughness)
    return f32(1.0) + r * r * r * r * f32(300.0)


class Lambertian:  # material.rs:91-100
    def __init__(self, albedo):
        self.albedo, self.albedo_gen = _albedo(albedo)

    def flatten(self):
        m = L.RaynMaterial()
        m.kind = L.MATERIAL_LAMBERTIAN
        m.albedo[:] = self.albedo.tolist()
        return m


class Dielectric:  # material.rs:150-175
    def __init__(self, albedo, roughness_exponent):
        self.albedo, self.albedo_gen = _albedo(albedo)
        self.roughness = f32(roughness_exponent)

    @staticmethod
    def new_remap(albedo, roughness):
        """Roughness in [0,1] -> Phong exponent, material.rs:167-174."""
        return Dielectric(albedo, _remap_roughness(roughness))

    def flatten(self):
        m = L.RaynMaterial()
        m.kind = L.MATERIAL_DIELECTRIC
        m.albedo[:] = self.albedo.tolist()
        m.roughness = float(self.roughness)
        return m


class Metallic:
    """A glossy conductor with coloured Fresnel: the Dielectric's Phong specular lobe with Schlick F0 per channel and no
    diffuse term.  An extension with no reference counterpart (rayn's material.rs carries a Metallic only as commented-out
    code); the exact statement is in include/rayn_b200.h (RAYN_MATERIAL_METALLIC).  f0 may be an OrbitTrapAlbedo: the palette
    then replaces F0 at every hit."""

    def __init__(self, f0, roughness_exponent):
        self.albedo, self.albedo_gen = _albedo(f0)
        self.roughness = f32(roughness_exponent)

    @property
    def f0(self):
        return self.albedo

    @staticmethod
    def new_remap(f0, roughness):
        """Roughness in [0,1] -> Phong exponent, as Dielectric.new_remap."""
        return Metallic(f0, _remap_roughness(roughness))

    def flatten(self):
        m = L.RaynMaterial()
        m.kind = L.MATERIAL_METALLIC
        m.albedo[:] = self.albedo.tolist()
        m.roughness = float(self.roughness)
        return m


class Sky:  # material.rs:394-404
    def __init__(self, top, bottom):
        self.top, self.bottom = _arr(top), _arr(bottom)

    def flatten(self):
        m = L.RaynMaterial()
        m.kind = L.MATERIAL_SKY
        m.sky_top[:] = self.top.tolist()
        m.sky_bottom[:] = self.bottom.tolist()
        return m


class Emissive:  # material.rs:451-469
    def __init__(self, emission):
        self.emission = _arr(emission)

    @staticmethod
    def new_splat(emission):
        return Emissive(emission)

    def flatten(self):
        m = L.RaynMaterial()
        m.kind = L.MATERIAL_EMISSIVE
        m.emission[:] = self.emission.tolist()
        m.albedo[:] = [0.5, 0.5, 0.5]  # inner LambertianBSDF, material.rs:482-484
        return m


class MaterialStore:  # material.rs:58-73
    def __init__(self):
        self.items = []

    def add_material(self, material):
        self.items.append(material)
        return len(self.items) - 1  # MaterialHandle


# ---- hitables (sphere.rs, sdf.rs) --------------------------------------------------------------
class Sphere:  # sphere.rs:14-20 (centre: constant, Linear or a closure f(t) -> Vec3)
    def __init__(self, center, radius, material):
        # a closure centre is kept as it is, with center_velocity None
        self.center, self.center_velocity = (center, None) if _is_closure(center) else _seq(center)
        self.radius, self.material = f32(radius), int(material)

    def has_closures(self):
        return self.center_velocity is None

    def flatten(self, time_range=None):
        """time_range: the render's (t0, t1), needed if the centre is a closure (its chord there is uploaded)"""
        center, velocity = _at(self.center, time_range) if self.has_closures() else (self.center, self.center_velocity)
        h = L.RaynHitable()
        h.kind = L.HITABLE_SPHERE
        h.material = self.material
        h.center[:] = center.tolist()
        h.center_velocity[:] = velocity.tolist()
        h.radius = float(self.radius)
        return h


class BoxFold:  # sdf.rs:150-158
    def __init__(self, side_length):
        self.l = f32(side_length)


class SphereFold:  # sdf.rs:171-179 (radii stored squared, in f32)
    def __init__(self, min_radius, fixed_radius):
        self.min_rad_sq = f32(min_radius) * f32(min_radius)
        self.fixed_rad_sq = f32(fixed_radius) * f32(fixed_radius)


class MandelBox:  # sdf.rs:113-123
    def __init__(self, iterations, box_fold, sphere_fold, scale):
        self.iterations, self.box_fold, self.sphere_fold, self.scale = int(iterations), box_fold, sphere_fold, f32(scale)


class Mandelbulb:
    """AUTHORED power-8 Mandelbulb distance estimator; no reference counterpart (SURVEY F1)."""

    def __init__(self, iterations, power=8, bailout=2.0):
        self.iterations, self.power, self.bailout = int(iterations), int(power), f32(bailout)


class TracedSDF:  # sdf.rs:12-21
    def __init__(self, sdf, material):
        self.sdf, self.material = sdf, int(material)

    def has_closures(self):
        return False

    def flatten(self, time_range=None):
        """time_range is not used: an SDF has no time-varying parameter"""
        h = L.RaynHitable()
        h.material = self.material
        s = self.sdf
        if isinstance(s, MandelBox):
            h.kind = L.HITABLE_MANDELBOX
            h.iterations = s.iterations
            h.box_l = float(s.box_fold.l)
            h.min_rad_sq = float(s.sphere_fold.min_rad_sq)
            h.fixed_rad_sq = float(s.sphere_fold.fixed_rad_sq)
            h.scale = float(s.scale)
        elif isinstance(s, Mandelbulb):
            h.kind = L.HITABLE_MANDELBULB
            h.iterations = s.iterations
            h.bulb_power = s.power
            h.bulb_bailout = float(s.bailout)
        else:
            raise TypeError(f"unsupported SDF {type(s).__name__}")
        return h


class HitableStore:  # hitable.rs:143-153
    def __init__(self):
        self.items = []

    def push(self, hitable):
        self.items.append(hitable)

    def __len__(self):
        return len(self.items)


# ---- lights (light.rs) ----------------------------------------------------------------------------
class SphereLight:  # light.rs:27-34
    def __init__(self, pos, rad, emission):
        self.pos, self.rad, self.emission = _arr(pos), f32(rad), _arr(emission)

    def flatten(self):
        l = L.RaynLight()
        l.pos[:] = self.pos.tolist()
        l.rad = float(self.rad)
        l.emission[:] = self.emission.tolist()
        return l


# ---- cameras (camera.rs) ----------------------------------------------------------------------------
def _store_seq(c, time_range, origin, at, up, focus=None):
    origin, at, up = _at(origin, time_range), _at(at, time_range), _at(up, time_range)
    c.origin[:], c.origin_velocity[:] = origin[0].tolist(), origin[1].tolist()
    c.at[:], c.at_velocity[:] = at[0].tolist(), at[1].tolist()
    c.up[:], c.up_velocity[:] = up[0].tolist(), up[1].tolist()
    if focus is not None:
        focus = _at(focus, time_range)
        c.focus[:], c.focus_velocity[:] = focus[0].tolist(), focus[1].tolist()


class _Camera:
    """The sequenced parameters of a camera (origin, at, up and a thin lens's focus): constants, Linear or closures; a
    closure's chord over the render's time_range is what flatten(time_range) stores."""

    def has_closures(self):
        return any(_is_closure(p) for p in (self.origin, self.at, self.up, getattr(self, "focus", None)))


def _fov_half(resolution, vfov):
    theta = f32(vfov) * f32(math.pi) / f32(180.0)
    # f32::tan -> libm tanf; numpy's float32 tan is 1 ulp off for 30 degrees, so round the double result instead
    half_height = f32(math.tan(float(theta / f32(2.0))))
    aspect = f32(resolution[0]) / f32(resolution[1])
    half_width = aspect * half_height
    return f32(half_width), f32(half_height)


class PinholeCamera(_Camera):  # camera.rs:52-72
    def __init__(self, resolution, vfov, origin, at, up):
        self.res = (f32(resolution[0]), f32(resolution[1]))
        self.half_width, self.half_height = _fov_half(self.res, vfov)
        self.half_pixel_size = self.half_height / self.res[1]
        self.origin, self.at, self.up = _seq(origin), _seq(at), _seq(up)

    def flatten(self, time_range=None):
        c = L.RaynCamera()
        c.kind = L.CAMERA_PINHOLE
        c.half_size[:] = [float(self.half_width), float(self.half_height)]
        c.half_pixel_size = float(self.half_pixel_size)
        _store_seq(c, time_range, self.origin, self.at, self.up)
        return c


class ThinLensCamera(_Camera):  # camera.rs:133-157
    def __init__(self, resolution, vfov, aperture, origin, at, up, focus):
        self.res = (f32(resolution[0]), f32(resolution[1]))
        self.half_width, self.half_height = _fov_half(self.res, vfov)
        self.half_pixel_size = self.half_height / self.res[1]
        self.aperture, self.aperture_rate = (f32(aperture.base), f32(aperture.velocity)) if isinstance(aperture, Linear) else (f32(aperture), f32(0.0))
        self.origin, self.at, self.up, self.focus = _seq(origin), _seq(at), _seq(up), _seq(focus)

    def flatten(self, time_range=None):
        c = L.RaynCamera()
        c.kind = L.CAMERA_THINLENS
        c.half_size[:] = [float(self.half_width), float(self.half_height)]
        c.half_pixel_size = float(self.half_pixel_size)
        _store_seq(c, time_range, self.origin, self.at, self.up, self.focus)
        c.aperture = float(self.aperture)
        c.aperture_rate = float(self.aperture_rate)
        return c


class OrthographicCamera(_Camera):  # camera.rs:227-241
    def __init__(self, resolution, vertical_size, origin, at, up):
        self.res = (f32(resolution[0]), f32(resolution[1]))
        aspect = self.res[0] / self.res[1]
        self.size = (f32(vertical_size) * aspect, f32(vertical_size))
        self.pixel_size = f32(vertical_size) / self.res[1]
        self.origin, self.at, self.up = _seq(origin), _seq(at), _seq(up)

    def flatten(self, time_range=None):
        c = L.RaynCamera()
        c.kind = L.CAMERA_ORTHOGRAPHIC
        c.half_size[:] = [float(self.size[0] / f32(2.0)), float(self.size[1] / f32(2.0))]
        c.full_size[:] = [float(self.size[0]), float(self.size[1])]
        c.half_pixel_size = float(self.pixel_size / f32(2.0))
        _store_seq(c, time_range, self.origin, self.at, self.up)
        return c


class EquirectangularCamera(_Camera):
    """A 360-degree equirectangular panorama (include/rayn_b200.h, RAYN_CAMERA_EQUIRECTANGULAR): an EXTENSION with no
    reference counterpart.  u spans the full turn about `up` (the screen centre looks at `at`), v runs from the -up pole to the
    +up pole; origin, at and up may each be a constant, Linear or a closure, as for PinholeCamera.  Its film is periodic in x:
    Film denoises and accumulates it across the seam."""

    def __init__(self, resolution, origin, at, up):
        self.res = (f32(resolution[0]), f32(resolution[1]))
        self.half_pixel_size = f32(f32(math.pi) / self.res[1]) / f32(2.0)  # the angular half pixel
        self.origin, self.at, self.up = _seq(origin), _seq(at), _seq(up)

    def flatten(self, time_range=None):
        c = L.RaynCamera()
        c.kind = L.CAMERA_EQUIRECTANGULAR
        c.half_pixel_size = float(self.half_pixel_size)
        _store_seq(c, time_range, self.origin, self.at, self.up)
        return c


class CameraStore:  # camera.rs:24-40
    def __init__(self):
        self.items = []

    def add_camera(self, camera):
        self.items.append(camera)
        return len(self.items) - 1  # CameraHandle

    def get(self, handle):
        return self.items[handle]


class VolumeParams:  # volume.rs:2-5
    def __init__(self, coeff_scattering=None, coeff_extinction=None):
        self.coeff_scattering, self.coeff_extinction = coeff_scattering, coeff_extinction


class RenderConsts:
    """Compile-time constants of the reference that leak into the hot path (setup.rs:33,37; sdf.rs:9-10)."""

    def __init__(self, world_radius=100.0, sdf_detail_scale=0.5, max_marches=256, max_vis_marches=100):
        self.world_radius, self.sdf_detail_scale = world_radius, sdf_detail_scale
        self.max_marches, self.max_vis_marches = max_marches, max_vis_marches


class World:  # world.rs:7-13
    def __init__(self, hitables, lights, materials, cameras, volume_params, consts=None):
        self.hitables, self.lights, self.materials, self.cameras = hitables, lights, materials, cameras
        self.volume_params = volume_params
        self.consts = consts or RenderConsts()

    def has_closures(self, camera_handle):
        """True if a sphere centre or a sequenced parameter of the camera is a closure f(t) -> Vec3 (Linear.chord)."""
        return self.cameras.get(camera_handle).has_closures() or any(h.has_closures() for h in self.hitables.items)

    def flatten(self, camera_handle, time_range=None):
        """-> (RaynSceneDesc, keepalive).  Order of hitables / materials / lights is preserved.  time_range: the render's
        (t0, t1); a closure parameter is uploaded as its chord over it (Linear.chord), and without it raises ValueError.
        A scene without closures flattens the same whatever time_range."""
        nh, nm, nl = len(self.hitables.items), len(self.materials.items), len(self.lights)
        hit = (L.RaynHitable * max(nh, 1))(*[h.flatten(time_range) for h in self.hitables.items])
        mat = (L.RaynMaterial * max(nm, 1))(*[m.flatten() for m in self.materials.items])
        lig = (L.RaynLight * max(nl, 1))(*[l.flatten() for l in self.lights])
        d = L.RaynSceneDesc()
        d.n_hitables, d.hitables = nh, C.cast(hit, C.POINTER(L.RaynHitable))
        d.n_materials, d.materials = nm, C.cast(mat, C.POINTER(L.RaynMaterial))
        d.n_lights, d.lights = nl, C.cast(lig, C.POINTER(L.RaynLight))
        d.camera = self.cameras.get(camera_handle).flatten(time_range)
        v = self.volume_params
        d.volume.has_scattering = 0 if v.coeff_scattering is None else 1
        d.volume.coeff_scattering = float(v.coeff_scattering or 0.0)
        d.volume.has_extinction = 0 if v.coeff_extinction is None else 1
        d.volume.coeff_extinction = float(v.coeff_extinction or 0.0)
        d.consts.world_radius = float(self.consts.world_radius)
        d.consts.sdf_detail_scale = float(self.consts.sdf_detail_scale)
        d.consts.max_marches = int(self.consts.max_marches)
        d.consts.max_vis_marches = int(self.consts.max_vis_marches)
        return d, (hit, mat, lig)

    def albedo_traps(self):
        """-> [RaynAlbedoTrap]: one entry per material whose albedo is an OrbitTrapAlbedo (rayn_b200_set_albedo_traps)."""
        return [m.albedo_gen.trap_desc(i) for i, m in enumerate(self.materials.items) if getattr(m, "albedo_gen", None) is not None]


class PathTracingIntegrator:  # integrator.rs:33-45
    def __init__(self, max_bounces, volume_marches=2):
        self.max_bounces, self.volume_marches = int(max_bounces), int(volume_marches)

    def requested_1d_sample_sets(self):
        return (self.max_bounces + 1) * (3 + self.volume_marches)

    def requested_2d_sample_sets(self):
        return (self.max_bounces + 1) * (12 + 8 * self.volume_marches)


class BlackmanHarrisFilter:  # filter.rs:13-27
    def __init__(self, radius=1.5):
        self.radius = float(radius)
