"""Progressive / adaptive rendering on the device film accumulator (rayn_b200_accum_*, rt_accum.cuh) against the CPU
oracle folded with the numpy mirror (tests/accum_mirror.py), bit for bit: the active tiles of every round, every tile's
E and K, and the film.  Also the device sample-range tables, the one-round corollary, threshold extremes, completion,
memory spaces, pass-size invariance, argument errors, Film.render_adaptive and rayn_host --adaptive."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from rayn_b200 import _lib as L
from rayn_b200 import configs
from rayn_b200.film import Film, FrameInputs, Renderer, adaptive_desc, make_frame_desc

import accum_mirror as am
from helpers import CH, assert_bit_equal, small_config

pytestmark = pytest.mark.gpu
TR = configs.frame_time_range(1)


def frame_for(inp, integrator, tile):
    ptrs = tuple(a.ctypes.data for a in inp.arrays())
    return make_frame_desc(inp.width, inp.height, tile, inp.samples, integrator, inp.frame, TR, ptrs, L.MEM_HOST,
                           sets=(inp.sets_1d, inp.sets_2d))


def run_round(renderer, acc, c, samples, first, desc, frame=1):
    w, h = acc.width, acc.height
    inp = FrameInputs(w, h, samples, c["integrator"], frame=frame, first_sample=first)
    return renderer.accum_round(acc, frame_for(inp, c["integrator"], acc.tile_size), *desc), inp


def uniform_rounds(renderer, c, res, tile, samples, rounds):
    acc = renderer.accum_create(res[0], res[1], tile)
    for r in range(rounds):
        run_round(renderer, acc, c, samples, r * 4 * samples, (2, rounds, -1.0))
    return acc


@pytest.mark.parametrize("spp,first", [(4, 0), (16, 37), (12, 2 ** 32 - 12), (1, 2 ** 32 - 1), (64, 1000)])
def test_device_tables_at_equal_host(renderer, spp, first):
    import torch
    s1, s2 = 5, 7
    d1, d2 = torch.full((spp * s1,), float("nan"), device="cuda"), torch.full((2 * spp * s2,), float("nan"), device="cuda")
    torch.cuda.synchronize()
    L.check(L.lib().rayn_b200_device_rd_tables_at(renderer.ctx, spp, s1, s2, 3, first, d1.data_ptr(), d2.data_ptr()), renderer.ctx)
    h1, h2 = np.empty(spp * s1, np.float32), np.empty(2 * spp * s2, np.float32)
    fp = C.POINTER(C.c_float)
    assert L.host_lib().rayn_b200_host_rd_tables_at(spp, s1, s2, 3, first, h1.ctypes.data_as(fp), h2.ctypes.data_as(fp)) == L.RAYN_OK
    assert_bit_equal(d1.cpu().numpy(), h1, "1d")
    assert_bit_equal(d2.cpu().numpy(), h2, "2d")
    assert L.lib().rayn_b200_device_rd_tables_at(renderer.ctx, spp, s1, s2, 3, 2 ** 32 - spp + 1, d1.data_ptr(), d2.data_ptr()) == L.RAYN_ERR_INVALID_ARG


@pytest.mark.parametrize("n", [1, 3, 4])
@pytest.mark.parametrize("samples", [1, 2, 4])
def test_one_round_resolves_to_render_frame(renderer, n, samples):
    """One round of power-of-two spp: (m * 2^k) / 2^k == m, so the accumulated film is render_frame's bit for bit.  40x37
    with 16x16 tiles drops the last partial row of tiles (film.rs:399-404), which must stay 0."""
    c, inp = small_config(n, (40, 37), samples, 3)
    renderer.upload_scene(c["world"], c["camera"])
    ref = renderer.render_host(inp, (16, 16), c["integrator"], TR)
    acc = renderer.accum_create(40, 37, (16, 16))
    assert renderer.accum_round(acc, frame_for(inp, c["integrator"], (16, 16)), 2, 4, -1.0) == acc.n_tiles == 3 * 2
    got = renderer.accum_resolve(acc)
    for ch in CH:
        assert_bit_equal(got[ch], ref[ch], f"cfg{n} {samples} samples {ch}")
    assert not got["color"].reshape(37, 40, 3)[32:].any()


@pytest.mark.parametrize("n,res,tile,mb", [(1, (37, 23), (8, 8), 2), (3, (64, 48), (16, 16), 3), (3, (37, 23), (8, 8), 2),
                                           (4, (37, 23), (8, 8), 2), (4, (64, 48), (16, 16), 2)])
def test_rounds_against_oracle_and_mirror(renderer, oracle, n, res, tile, mb):
    """Every round is re-rendered by the oracle on the same tile list and tables and folded by the mirror.  From round 3
    the threshold is the 30th percentile of the tiles' E after round 2, so some tiles stop at min_rounds and others go on."""
    c = configs.baseline_config(n, res=res, samples=1, max_bounces=mb)
    integ, (w, h) = c["integrator"], res
    renderer.upload_scene(c["world"], c["camera"])
    acc = renderer.accum_create(w, h, tile)
    m = am.AccumMirror(w, h, *tile)
    min_r, max_r, thr = 2, 6, -1.0
    history = []
    for r in range(max_r + 1):
        if r == 2:
            thr = float(np.float32(np.percentile(m.E, 30)))
        act = m.active(min_r, max_r, thr)
        first = int(m.K[act[0]]) if act else 0
        _, k_before = renderer.accum_tiles(acc)
        got, inp = run_round(renderer, acc, c, 1, first, (min_r, max_r, thr))
        assert got == len(act), f"round {r}"
        err, k = renderer.accum_tiles(acc)
        assert np.flatnonzero(k != k_before).tolist() == act, f"round {r}: active tiles"
        history.append(len(act))
        if not act:
            break
        o, _ = oracle.render(c["world"], c["camera"], inp, tile, integ, TR, tile_list=act)
        m.fold(o, act, 1)
        assert np.array_equal(k, m.K), f"round {r}: K"
        assert np.array_equal(err.view(np.uint64), m.E.view(np.uint64)), f"round {r}: E {err} vs {m.E}"
    print(f"cfg{n} {res} tiles {tile}: active tiles per round {history}, threshold {thr:.4g}")
    assert (m.rounds == min_r).any() and (m.rounds > min_r).any(), m.rounds
    final = renderer.accum_resolve(acc)
    want = m.resolve()
    for ch in CH:
        assert_bit_equal(final[ch], want[ch], f"final {ch}")
    acc.close()


def test_threshold_extremes_completion_and_nan(renderer):
    c = configs.baseline_config(1, res=(40, 24), samples=1, max_bounces=2)
    renderer.upload_scene(c["world"], c["camera"])
    acc = renderer.accum_create(40, 24, (8, 8))
    counts = [run_round(renderer, acc, c, 1, 4 * r, (2, 4, -1.0))[0] for r in range(5)]
    assert counts == [acc.n_tiles] * 4 + [0]  # threshold < 0: every tile gets max_rounds
    err, k = renderer.accum_tiles(acc)
    assert (k == 16).all() and np.isfinite(err).all()
    before = renderer.accum_resolve(acc)
    assert run_round(renderer, acc, c, 1, 16, (2, 4, -1.0))[0] == 0  # after completion: nothing rendered or changed
    err2, k2 = renderer.accum_tiles(acc)
    after = renderer.accum_resolve(acc)
    assert np.array_equal(err.view(np.uint64), err2.view(np.uint64)) and np.array_equal(k, k2)
    for ch in CH:
        assert_bit_equal(after[ch], before[ch], ch)
    acc2 = renderer.accum_create(40, 24, (8, 8))
    counts = [run_round(renderer, acc2, c, 1, 4 * r, (3, 6, np.inf))[0] for r in range(4)]
    assert counts == [acc2.n_tiles] * 3 + [0]  # threshold +inf: every tile stops at min_rounds
    assert (renderer.accum_tiles(acc2)[1] == 12).all()
    with pytest.raises(L.RaynError) as e:
        run_round(renderer, acc2, c, 1, 12, (3, 6, float("nan")))
    assert e.value.code == L.RAYN_ERR_INVALID_ARG
    acc.close(), acc2.close()


def test_resolve_host_device_and_null_planes(renderer):
    import torch
    c = configs.baseline_config(3, res=(48, 32), samples=1, max_bounces=3)
    renderer.upload_scene(c["world"], c["camera"])
    acc = uniform_rounds(renderer, c, (48, 32), (16, 16), 1, 3)
    ref = renderer.accum_resolve(acc)
    npx = 48 * 32
    dev = {k: torch.full(((1 if k == "alpha" else 3) * npx,), float("nan"), device="cuda") for k in CH}
    torch.cuda.synchronize()
    renderer.accum_resolve(acc, L.RaynFilmPlanes(*(dev[k].data_ptr() for k in CH), L.MEM_DEVICE))
    for k in CH:
        assert_bit_equal(dev[k].cpu().numpy(), ref[k], f"device {k}")
    host = {k: np.full_like(ref[k], np.nan) for k in CH}
    renderer.accum_resolve(acc, L.RaynFilmPlanes(host["color"].ctypes.data, None, None, host["normal"].ctypes.data, L.MEM_HOST))
    assert_bit_equal(host["color"], ref["color"], "color")
    assert_bit_equal(host["normal"], ref["normal"], "normal")
    assert np.isnan(host["alpha"]).all() and np.isnan(host["background"]).all()  # NULL planes: nothing written
    renderer.accum_resolve(acc, L.RaynFilmPlanes(None, None, None, None, L.MEM_HOST))
    acc.close()


def test_pass_size_invariance():
    """A pass budget of two 8x8 tiles at 4 spp splits every round into several passes: same tiles, errors and film."""
    c = configs.baseline_config(3, res=(40, 32), samples=1, max_bounces=3)
    out = []
    for cap in (0, 600):
        r = Renderer(0, max_paths_per_pass=cap)
        try:
            r.upload_scene(c["world"], c["camera"])
            acc = r.accum_create(40, 32, (8, 8))
            run_round(r, acc, c, 1, 0, (2, 4, 0.3))
            passes = r.stats().passes  # of the first round, which renders every tile
            for k in range(1, 4):
                run_round(r, acc, c, 1, 4 * k, (2, 4, 0.3))  # an active tile has rendered k rounds of 4 spp before round k
            out.append((r.accum_tiles(acc), r.accum_resolve(acc), passes))
            acc.close()
        finally:
            r.close()
    (e0, k0), f0, p0 = out[0]
    (e1, k1), f1, p1 = out[1]
    assert p1 > p0
    assert np.array_equal(e0.view(np.uint64), e1.view(np.uint64)) and np.array_equal(k0, k1)
    for ch in CH:
        assert_bit_equal(f1[ch], f0[ch], ch)


def test_argument_errors(renderer):
    lib = L.lib()
    c = configs.baseline_config(1, res=(32, 16), samples=1, max_bounces=2)
    renderer.upload_scene(c["world"], c["camera"])
    h = C.c_void_p()
    for args in [(0, 16, 8, 8), (32, 16, 0, 8), (32, -1, 8, 8)]:
        assert lib.rayn_b200_accum_create(renderer.ctx, *args, C.byref(h)) == L.RAYN_ERR_INVALID_ARG
    assert lib.rayn_b200_accum_create(renderer.ctx, 32, 16, 8, 8, None) == L.RAYN_ERR_INVALID_ARG
    acc = renderer.accum_create(32, 16, (8, 8))
    planes = L.RaynFilmPlanes(None, None, None, None, L.MEM_HOST)
    assert lib.rayn_b200_accum_resolve(renderer.ctx, acc.handle, C.byref(planes)) == L.RAYN_ERR_INVALID_ARG  # before any round
    inp = FrameInputs(32, 16, 1, c["integrator"])
    good = frame_for(inp, c["integrator"], (8, 8))
    n = C.c_int32(-1)

    def call(frame=good, desc=adaptive_desc(2, 4, 0.1), a=acc.handle):
        return lib.rayn_b200_accum_round(renderer.ctx, a, C.byref(frame) if frame is not None else None,
                                         C.byref(desc) if desc is not None else None, C.byref(n))
    for d in [adaptive_desc(1, 4, 0.1), adaptive_desc(3, 2, 0.1), adaptive_desc(2, 4, float("nan"))]:
        assert call(desc=d) == L.RAYN_ERR_INVALID_ARG
    assert call(desc=None) == L.RAYN_ERR_INVALID_ARG and call(frame=None) == L.RAYN_ERR_INVALID_ARG
    assert call(a=None) == L.RAYN_ERR_INVALID_ARG
    for field, value in [("width", 40), ("height", 8), ("tile_w", 16), ("tile_h", 4)]:
        f = frame_for(inp, c["integrator"], (8, 8))
        setattr(f, field, value)
        assert call(frame=f) == L.RAYN_ERR_INVALID_ARG, field
    f = frame_for(inp, c["integrator"], (8, 8))
    f.samples = (1 << 22) + 1  # K would pass 2^24
    assert call(frame=f) == L.RAYN_ERR_INVALID_ARG
    assert renderer.accum_tiles(acc)[1].sum() == 0  # nothing was folded by the refused calls
    assert call() == L.RAYN_OK and n.value == acc.n_tiles  # the accumulator and the context still work
    acc.close()


def test_rendering_is_unchanged_by_adaptive_rounds(renderer):
    from test_cpu_oracle import GOLD, GOLD_SUFFIX, GOLDEN_CASES
    name = "cfg3_32x32_8spp_3b"
    n, res, samples, mb = GOLDEN_CASES[name]
    gold = np.load(os.path.join(GOLD, name + GOLD_SUFFIX + ".npz"))
    c, inp = small_config(n, res, samples, mb)
    renderer.upload_scene(c["world"], c["camera"])
    acc = uniform_rounds(renderer, c, (48, 40), (8, 8), 1, 3)
    renderer.upload_scene(c["world"], c["camera"])
    after = renderer.render_host(inp, (16, 16), c["integrator"], TR)
    for ch in CH:
        assert_bit_equal(after[ch], gold[ch], f"after {ch}")
    acc.close()


def manual_adaptive(renderer, c, res, tile, samples, min_r, max_r, thr, frame=1):
    """The accumulator driven with host tables (FrameInputs first_sample), as a reference for the device-table drivers."""
    renderer.upload_scene(c["world"], c["camera"])
    acc = renderer.accum_create(res[0], res[1], tile)
    first, rounds = 0, 0
    while run_round(renderer, acc, c, samples, first, (min_r, max_r, thr), frame)[0]:
        first += 4 * samples
        rounds += 1
    film, (err, k) = renderer.accum_resolve(acc), renderer.accum_tiles(acc)
    acc.close()
    return rounds, film, err, k


def test_film_render_adaptive_with_preview_then_denoise(renderer):
    c = configs.baseline_config(3, res=(40, 32), samples=1, max_bounces=3)
    f = Film(("color", "alpha", "background", "normal"), (40, 32))
    seen = []
    rounds = f.render_adaptive(c["world"], c["camera"], c["integrator"], None, (8, 8), 1, TR, 1, min_rounds=2, max_rounds=5,
                               threshold=0.3, on_round=lambda film: seen.append((film.channels["color"].copy(), film.tile_samples.copy())))
    assert rounds == len(seen) >= 2 and f.progressive_epoch == rounds
    assert all(s[0].shape == (32, 40, 3) for s in seen)
    assert (np.diff([s[1].sum() for s in seen]) > 0).all()
    ref_rounds, ref, err, k = manual_adaptive(renderer, c, (40, 32), (8, 8), 1, 2, 5, 0.3)
    assert rounds == ref_rounds
    assert np.array_equal(f.tile_errors.view(np.uint64), err.view(np.uint64)) and np.array_equal(f.tile_samples, k)
    for ch in CH:
        assert_bit_equal(f.channels[ch].reshape(-1), ref[ch], f"render_adaptive {ch}")
    assert_bit_equal(seen[-1][0], f.channels["color"], "the last preview is the final film")
    before = f.channels["color"].copy()
    f.denoise(3)
    assert f.channels["color"].shape == (32, 40, 3) and not np.array_equal(before, f.channels["color"])


def test_cpp_host_adaptive_flag(renderer, tmp_path):
    from rayn_b200 import build
    exe = os.path.join(os.path.dirname(build.OUT), "rayn_host")
    args = [exe, "--config", "3", "--res", "48", "32", "--samples", "1", "--bounces", "3", "--adaptive", "0.3", "--rounds", "4"]
    r = subprocess.run(args + ["--dump", str(tmp_path / "a.bin"), "--out", str(tmp_path / "a.ppm")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert "Done in" in r.stdout and "rounds of 4 spp" in r.stdout, r.stdout
    assert (tmp_path / "a.ppm").stat().st_size == len(b"P6\n48 32\n255\n") + 48 * 32 * 3
    npx = 48 * 32
    raw = np.fromfile(tmp_path / "a.bin", np.float32)
    c = configs.baseline_config(3, res=(48, 32), samples=1, max_bounces=3)
    _, ref, _, _ = manual_adaptive(renderer, c, (48, 32), (16, 16), 1, 2, 4, 0.3)
    assert_bit_equal(raw[:3 * npx], ref["color"], "rayn_host --adaptive color")
    assert_bit_equal(raw[4 * npx:7 * npx], ref["background"], "rayn_host --adaptive background")
    r = subprocess.run(args + ["--denoise", "3", "--dump", str(tmp_path / "d.bin")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    den = np.fromfile(tmp_path / "d.bin", np.float32)
    assert_bit_equal(den[3 * npx:4 * npx], raw[3 * npx:4 * npx], "alpha untouched by --denoise")
    assert not np.array_equal(den[:3 * npx], raw[:3 * npx])
