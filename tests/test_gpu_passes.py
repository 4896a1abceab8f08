"""Renders of several passes keep two passes in flight, alternating between two pass sets on two streams (api.cu:
render_enqueue).  The passes cover disjoint tiles, so the film and the order-free stats must not depend on how many passes a
frame is split into, on which stream a pass ran, or on whether the frame ran serially on one stream (RAYN_FLAG_TIMING).
Covered: 1, 2, 3 and 5 passes (an odd count leaves one stream a lone last pass) on configs 1, 3 and 4, host- and
device-space films, moments, a sharded render, an accum_round, and renders followed by a first-hit pass on one context."""
import ctypes as C

import numpy as np
import pytest

from rayn_b200 import _lib as L
from rayn_b200 import configs
from rayn_b200.film import FrameInputs, Renderer, make_frame_desc

from helpers import CH, assert_bit_equal, small_config

pytestmark = pytest.mark.gpu
TR = configs.frame_time_range(1)
RES, TILE, SAMPLES = (96, 64), (16, 16), 1
N_TILES = (RES[0] // TILE[0]) * (RES[1] // TILE[1])  # 24
R = TILE[0] * TILE[1] * 4 * SAMPLES                  # paths per tile
TILES_PER_PASS = {1: 0, 2: 12, 3: 8, 5: 5}            # passes -> tiles per pass (0: the default budget, one pass)
# the stats that do not depend on scheduling (march trips do: a drained slot's last trips depend on its neighbours)
ORDER_FREE = ("paths", "extend_rays", "shadow_rays", "sdf_evals_extend", "sdf_evals_shadow", "sdf_evals_normals", "bulb_iters_extend",
              "bulb_iters_shadow")


def renderer(c, passes, flags=0):
    r = Renderer(0, max_paths_per_pass=TILES_PER_PASS[passes] * R, flags=flags)
    r.upload_scene(c["world"], c["camera"])
    return r


def host_render(c, inp, passes, flags=0, moments=False):
    r = renderer(c, passes, flags)
    try:
        f = r.render_host(inp, TILE, c["integrator"], TR, moments=moments)
        st = r.stats()
    finally:
        r.close()
    assert st.passes == passes
    return f, {k: getattr(st, k) for k in ORDER_FREE}


@pytest.mark.parametrize("cfg,bounces", [(1, 2), (3, 3), (4, 2)])
def test_pass_count_does_not_change_the_film_or_the_stats(cfg, bounces):
    c, inp = small_config(cfg, RES, SAMPLES, bounces)
    ref, ref_st = host_render(c, inp, 1)
    assert ref_st["paths"] == RES[0] * RES[1] * 4 * SAMPLES
    for passes in (2, 3, 5):
        f, st = host_render(c, inp, passes)
        for ch in CH:
            assert_bit_equal(f[ch], ref[ch], f"config {cfg}, {passes} passes: {ch}")
        assert st == ref_st, f"config {cfg}, {passes} passes"
    # the serial one-stream order of a timed render gives the same film
    f, st = host_render(c, inp, 5, flags=L.FLAG_TIMING)
    for ch in CH:
        assert_bit_equal(f[ch], ref[ch], f"config {cfg}, timed: {ch}")
    assert st == ref_st


def test_moments_over_several_passes():
    c, inp = small_config(3, RES, SAMPLES, 3)
    ref, _ = host_render(c, inp, 1, moments=True)
    for passes in (2, 5):
        f, _ = host_render(c, inp, passes, moments=True)
        for ch in CH + ("moments",):
            assert_bit_equal(f[ch], ref[ch], f"{passes} passes: {ch}")


def device_planes(torch, w, h):
    film = torch.zeros(10 * w * h, dtype=torch.float32, device="cuda:0")
    npx = w * h
    p = L.RaynFilmPlanes(film[:3 * npx].data_ptr(), film[3 * npx:4 * npx].data_ptr(), film[4 * npx:7 * npx].data_ptr(),
                         film[7 * npx:].data_ptr(), L.MEM_DEVICE)
    return film, p


def as_host(film, w, h):
    a = film.cpu().numpy()
    npx = w * h
    return {"color": a[:3 * npx], "alpha": a[3 * npx:4 * npx], "background": a[4 * npx:7 * npx], "normal": a[7 * npx:]}


def test_device_space_film_over_several_passes():
    torch = pytest.importorskip("torch")
    from rayn_b200.dist import device_frame_desc
    c, inp = small_config(3, RES, SAMPLES, 3)
    ref, _ = host_render(c, inp, 1)
    inputs_dev = [torch.from_numpy(a).to("cuda:0") for a in inp.arrays()]
    fd = device_frame_desc(inputs_dev, RES[0], RES[1], TILE, c["samples"], c["integrator"], 1, TR, (inp.sets_1d, inp.sets_2d))
    for passes in (3, 5):
        r = renderer(c, passes)
        try:
            film, p = device_planes(torch, *RES)
            r.render(fd, p)
            assert r.stats().passes == passes
            got = as_host(film, *RES)  # the render returned: the whole film is on the device, on any stream
        finally:
            r.close()
        for ch in CH:
            assert_bit_equal(got[ch], ref[ch].ravel(), f"{passes} passes: {ch}")


def test_sharded_render_over_several_passes():
    """render_frame_sharded on a one-rank communicator: the shard's passes, then the gather, then the copy-out."""
    c, inp = small_config(3, RES, SAMPLES, 3)
    ref, _ = host_render(c, inp, 1)
    lib = L.lib()
    r = renderer(c, 5)
    try:
        ident = (C.c_uint8 * L.COMM_ID_BYTES)()
        L.check(lib.rayn_b200_comm_unique_id(ident))
        L.check(lib.rayn_b200_comm_init_rank(r.ctx, ident, 0, 1), r.ctx)
        npx = RES[0] * RES[1]
        host = {k: np.zeros(n * npx, np.float32) for k, n in (("color", 3), ("alpha", 1), ("background", 3), ("normal", 3))}
        hp = L.RaynFilmPlanes(*(host[k].ctypes.data for k in CH), L.MEM_HOST)
        fd = make_frame_desc(RES[0], RES[1], TILE, c["samples"], c["integrator"], 1, TR, tuple(a.ctypes.data for a in inp.arrays()), L.MEM_HOST,
                             0, 1, (inp.sets_1d, inp.sets_2d))
        L.check(lib.rayn_b200_render_frame_sharded(r.ctx, C.byref(fd), C.byref(hp)), r.ctx)
        assert r.stats().passes == 5
        L.check(lib.rayn_b200_comm_destroy(r.ctx), r.ctx)
    finally:
        r.close()
    for ch in CH:
        assert_bit_equal(host[ch], ref[ch].ravel(), ch)


def test_accum_round_over_several_passes():
    c = configs.baseline_config(3, res=RES, samples=SAMPLES, max_bounces=3)
    out = []
    for passes in (1, 3):
        r = renderer(c, passes)
        try:
            acc = r.accum_create(RES[0], RES[1], TILE)
            for k in range(3):
                inp = FrameInputs(RES[0], RES[1], SAMPLES, c["integrator"], first_sample=4 * SAMPLES * k)
                f = make_frame_desc(RES[0], RES[1], TILE, SAMPLES, c["integrator"], 1, TR, tuple(a.ctypes.data for a in inp.arrays()), L.MEM_HOST,
                                    sets=(inp.sets_1d, inp.sets_2d))
                r.accum_round(acc, f, 2, 4, -1.0)
                if k == 0:
                    assert r.stats().passes == passes
            out.append((r.accum_tiles(acc), r.accum_resolve(acc)))
            acc.close()
        finally:
            r.close()
    (e0, k0), f0 = out[0]
    (e1, k1), f1 = out[1]
    assert np.array_equal(e0.view(np.uint64), e1.view(np.uint64)) and np.array_equal(k0, k1)
    for ch in CH:
        assert_bit_equal(f1[ch], f0[ch], ch)


def test_renders_then_albedo_on_one_context():
    """Two renders of several passes and then a first-hit pass, back to back on one context, against fresh one-pass
    contexts: the albedo pass (one stream) reuses the first pass set after the two-stream renders."""
    c, inp = small_config(3, RES, SAMPLES, 3)
    inp2 = FrameInputs(RES[0], RES[1], SAMPLES, c["integrator"], frame=2)
    refs = [host_render(c, i, 1)[0] for i in (inp, inp2)]
    r1 = renderer(c, 1)
    try:
        ref_alb = r1.render_albedo(inp, TILE, c["integrator"], TR)
    finally:
        r1.close()
    r = renderer(c, 5)
    try:
        got = [r.render_host(i, TILE, c["integrator"], TR) for i in (inp, inp2)]
        assert r.stats().passes == 5
        alb = r.render_albedo(inp, TILE, c["integrator"], TR)
        again = r.render_host(inp, TILE, c["integrator"], TR)
    finally:
        r.close()
    for g, ref in zip(got + [again], refs + refs[:1]):
        for ch in CH:
            assert_bit_equal(g[ch], ref[ch], ch)
    assert_bit_equal(alb, ref_alb, "albedo")
