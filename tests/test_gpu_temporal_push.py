"""The temporal push on the device at sizes the CPU mirrors are slow at: rendered frames reprojected through
Renderer.render_motion / render_motion_prev and Renderer.temporal_push at 640x360 (the check of
test_cpu_temporal_reprojection.py), and the film-width limit of rayn_b200_temporal_create: 2^23 + 1 is rejected, and a
2^23 x 1 film reads every static pixel's own history.  Also the device against the mirror bit for bit where only the
finite-z_h rule keeps a history without a hit out: sigma_depth = +inf, and 3e38 with huge depths."""
import numpy as np
import pytest

from rayn_b200 import _lib as L

import mirrors
import test_cpu_temporal_push as tp
import test_cpu_temporal_reprojection as rp
from helpers import assert_bit_equal

pytestmark = pytest.mark.gpu
MAX_SIDE = 1 << 23


@pytest.mark.parametrize("motion", rp.MOTIONS)
def test_history_lands_on_the_same_surface_point_at_640x360(renderer, motion):
    """device motion planes and device pushes; the hit points come from the CPU mirror.  With 4 samples (16 spp, as
    FrameInputs.spp = 4 x samples) the median error of the correct convention is 0.13 to 0.15 pixel footprints and every
    wrong one is at least 4.0x worse (measured with the mirrors, whose planes and pushes the device equals bit for bit)."""
    W, H = 640, 360
    fr = rp.render_pair(motion, W, H, 4, device=renderer)
    for i in (0, 1):
        assert_bit_equal(fr[f"plane{i}"], fr[f"mirror_plane{i}"], f"{motion} motion plane {i}")
    t = renderer.temporal_create(W, H)
    try:
        rp.check(rp.scores(lambda *a: renderer.temporal_push(t, *a), fr), 0.2)
    finally:
        t.close()


def test_create_rejects_films_beyond_two_to_the_23(renderer):
    for W, H in ((MAX_SIDE + 1, 1), (1, MAX_SIDE + 1)):
        with pytest.raises(L.RaynError) as e:
            renderer.temporal_create(W, H)
        assert e.value.code == L.RAYN_ERR_INVALID_ARG


def test_widest_film_reads_its_own_history(renderer):
    """a 2^23 x 1 film, zero motion, equal depths and normals: frame A, then colour 0 with alpha_min 0.5 gives exactly 0.5 A
    at every x (the largest x is 2^23 - 1, whose x + 0.5f is still exact)"""
    W, H = MAX_SIDE, 1
    rng = np.random.default_rng(23)
    a = {k: rng.uniform(0.25, 2.0, (H, W, 3)).astype(np.float32) for k in ("color", "background")}
    a["color"][0, :, 0] = np.arange(W, dtype=np.float32) + 1.0  # each pixel's own index: a neighbour's value differs
    nrm = np.zeros((H, W, 3), np.float32)
    nrm[..., 2] = 1.0
    mom = rng.uniform(0.25, 2.0, (H, W, 2)).astype(np.float32)
    mv = np.zeros((H, W, 4), np.float32)
    mv[..., 2:] = 2.0
    t = renderer.temporal_create(W, H)
    try:
        out, om, s = renderer.temporal_push(t, dict(a, normal=nrm), mom, mv, 0.5, 0.1, 0.5)
        for k in ("color", "background"):
            assert_bit_equal(out[k], a[k], k)
        assert_bit_equal(om, mom, "moments")
        assert (s == 1).all()
        zero = np.zeros((H, W, 3), np.float32)
        out, om, s = renderer.temporal_push(t, {"color": zero, "background": zero, "normal": nrm}, np.zeros_like(mom), mv, 0.5, 0.1, 0.5)
        for k in ("color", "background"):
            assert_bit_equal(out[k], a[k] * np.float32(0.5), k)
        assert_bit_equal(om, mom * np.float32(0.5), "moments")
        assert (s == 0.5).all()
    finally:
        t.close()


@pytest.mark.parametrize("sigma_depth", [3e38, np.inf])
def test_history_without_a_hit_is_never_used(renderer, sigma_depth):
    """a sky history (z_h = +inf) next to a hit: sigma_depth * |z_prev| is +inf, and frame 2 still comes back unchanged"""
    W, H = 4, 3
    (p0, m0, mv0), (p1, m1, mv1) = tp.sky_then_hit(W, H, np.random.default_rng(4))
    t = renderer.temporal_create(W, H)
    try:
        renderer.temporal_push(t, p0, m0, mv0, 0.2, sigma_depth, -1.0)
        out, om, s = renderer.temporal_push(t, p1, m1, mv1, 0.2, sigma_depth, -1.0)
    finally:
        t.close()
    assert_bit_equal(out["color"], p1["color"]), assert_bit_equal(out["background"], p1["background"]), assert_bit_equal(om, m1)
    assert (s == 1).all()


@pytest.mark.parametrize("sigma_depth", [3e38, np.inf])
def test_edge_sequence_equals_the_mirror_with_an_overflowing_depth_test(renderer, sigma_depth):
    """16 pushes of the CPU edge inputs (pixels without a hit, huge depths, non-finite motion, landings on the borders, a reset)
    at every alpha_min and normal_cos of the CPU descriptors: device and mirror agree bit for bit on every output"""
    W, H = 37, 23
    rng = np.random.default_rng(17)
    mirror = mirrors.TemporalMirror(W, H)
    t = renderer.temporal_create(W, H)
    try:
        for k in range(2 * len(tp.DESCS)):
            cur, nrm, motion = tp.edge_frame(W, H, rng)
            planes = {"color": cur[0:3].T.reshape(H, W, 3), "background": cur[3:6].T.reshape(H, W, 3), "normal": nrm.T.reshape(H, W, 3)}
            mom, mv = cur[6:8].T.reshape(H, W, 2), motion.T.reshape(H, W, 4)
            alpha_min, _, normal_cos = tp.DESCS[k % len(tp.DESCS)]
            reset = k == 9
            out, om, s = renderer.temporal_push(t, planes, mom, mv, alpha_min, sigma_depth, normal_cos, reset)
            rc, ref, rom, rs = mirror.push(planes, mom, mv, alpha_min, sigma_depth, normal_cos, reset)
            assert rc == L.RAYN_OK
            for key in ("color", "background"):
                assert_bit_equal(out[key], ref[key], f"push {k} {key}")
            assert_bit_equal(om, rom, f"push {k} moments"), assert_bit_equal(s, rs, f"push {k} var_scale")
    finally:
        t.close()
