"""rayn_b200 — H100-native wavefront path tracer behind rayn's render-path interface.

Package layout (only what the hot path needs):
  csrc/      CUDA kernels (sm_90a), C-ABI implementation, deterministic math, host input builders
  _lib.py    ctypes binding of include/rayn_b200.h
  scene.py   host mirror of rayn's scene API (setup.rs / world.rs constructors) -> POD descriptors
  film.py    Film.render_frame_into (film.rs:382-395) and the Renderer handle
  configs.py setup.rs scene + the five BASELINE configs
  dist.py    tile sharding across GPUs + NCCL film gather
  build.py   in-tree nvcc build of librayn_b200.so
"""
from .scene import (BlackmanHarrisFilter, BoxFold, CameraStore, Dielectric, Emissive, EquirectangularCamera, HitableStore, Lambertian, Linear,  # noqa: F401
                    MandelBox, Mandelbulb, MaterialStore, Metallic, OrbitTrapAlbedo, OrthographicCamera, PathTracingIntegrator, PinholeCamera,
                    RenderConsts, Sky, Sphere, SphereFold, SphereLight, Srgb, ThinLensCamera, TracedSDF, Vec3,
                    VolumeParams, World)
from .film import Film, FrameInputs, Renderer  # noqa: F401
