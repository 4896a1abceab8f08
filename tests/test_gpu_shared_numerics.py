"""The device against the shared-numerics data of tests/test_cpu_shared_numerics.py: detmath over every 32-bit input of every
sweep in tests/golden/detmath_sweep.json (device = host, bit for bit, NaN payloads included but powi5's), the special-operand
table,
and the device R_d tables and scramble plane against their Python-int statements."""
import ctypes as C

import numpy as np
import pytest

from rayn_b200 import _lib as L
from test_cpu_shared_numerics import (BIG, SCRAMBLE_SHAPES, big_sample_pixels, golden, rd_cases, rd_statement, scramble_statement,
                                      special_cases, sweep_ids, sweep_by_name, u2f)

pytestmark = pytest.mark.gpu
u32 = np.uint32


def device_sweep(renderer, s):
    out = (C.c_uint64 * 256)()
    L.check(L.lib().rayn_b200_kat_detmath_sweep(renderer.ctx, s["op"], u2f(int(s["fixed"], 16)), 1 if s["swap"] else 0, out), renderer.ctx)
    return [f"0x{v:016x}" for v in out]


def first_difference(renderer, oracle, s, chunk):
    """the first input of the chunk whose device and host result bits differ"""
    v = np.arange(chunk << 24, (chunk + 1) << 24, dtype=np.uint64).astype(np.uint32).view(np.float32)
    fixed = np.full(v.size, u2f(int(s["fixed"], 16)), np.float32)
    a, b = (fixed, v) if s["swap"] else (v, fixed)
    d, h = renderer.kat_detmath(s["op"], a, b), oracle.kat_detmath(s["op"], a, b)
    same = d.view(u32) == h.view(u32)
    if s["op"] == 7:
        same |= np.isnan(d) & np.isnan(h)
    bad = np.flatnonzero(~same)
    if bad.size == 0:
        return "no differing input (the hashes themselves differ)"
    i = bad[0]
    return f"{bad.size} inputs differ, first ({a[i]!r}, {b[i]!r}): device 0x{int(d.view(u32)[i]):08x}, host 0x{int(h.view(u32)[i]):08x}"


@pytest.mark.parametrize("name", sweep_ids())
def test_device_sweep_equals_host_over_every_input(renderer, oracle, name):
    s = sweep_by_name(name)
    got = device_sweep(renderer, s)
    bad = [c for c in range(256) if got[c] != s["hashes"][c]]
    assert not bad, f"{name}: {len(bad)} chunks differ; chunk 0x{bad[0]:02x}: {first_difference(renderer, oracle, s, bad[0])}"


def test_device_special_values_equal_host(renderer, oracle):
    for op in sorted({c[1] for c in special_cases()}):
        cases = [c for c in special_cases() if c[1] == op]
        a, b = np.array([c[2] for c in cases], np.float32), np.array([c[3] for c in cases], np.float32)
        d, h = renderer.kat_detmath(op, a, b), oracle.kat_detmath(op, a, b)
        same = d.view(u32) == h.view(u32)
        if op == 7:  # powi5 is float multiplies: its NaN payload is the hardware's (detmath.h)
            same |= np.isnan(d) & np.isnan(h)
        bad = np.flatnonzero(~same)
        assert bad.size == 0, [(cases[i], hex(int(d.view(u32)[i])), hex(int(h.view(u32)[i]))) for i in bad]


def test_device_sweep_rejects_bad_arguments(renderer):
    out = (C.c_uint64 * 256)()
    assert L.lib().rayn_b200_kat_detmath_sweep(renderer.ctx, 9, 0.0, 0, out) == L.RAYN_ERR_INVALID_ARG
    assert L.lib().rayn_b200_kat_detmath_sweep(renderer.ctx, 0, 0.0, 0, None) == L.RAYN_ERR_INVALID_ARG


@pytest.mark.skipif(L.MULADD_FUSED or L.LEGACY, reason="already inside a variant run")
def test_fused_mul_add_variant_shared_numerics():
    """the transcendentals use no mul_add, so the _fma library's sweeps must give the same hashes"""
    from test_gpu_parity import _run_suite_variant
    out = _run_suite_variant({"RAYN_MULADD_FUSED": "1"}, ["tests/test_gpu_shared_numerics.py", "-k", "not variant"])
    assert " passed" in out


def test_device_rd_tables_match_the_statement(renderer):
    import torch
    for spp, s1, s2, off, first in rd_cases():
        d1 = torch.full((max(spp * s1, 1),), float("nan"), device="cuda")
        d2 = torch.full((max(2 * spp * s2, 1),), float("nan"), device="cuda")
        torch.cuda.synchronize()
        L.check(L.lib().rayn_b200_device_rd_tables_at(renderer.ctx, spp, s1, s2, off, first, d1.data_ptr(), d2.data_ptr()), renderer.ctx)
        w1, w2 = rd_statement(spp, s1, s2, off, first)
        case = (spp, s1, s2, off, first)
        assert np.array_equal(d1.cpu().numpy()[:spp * s1].view(u32), w1.view(u32)), f"1d tables at {case}"
        assert np.array_equal(d2.cpu().numpy()[:2 * spp * s2].view(u32), w2.view(u32)), f"2d tables at {case}"


def _device_scramble(renderer, w, h):
    import torch
    sc = torch.full((w * h,), float("nan"), device="cuda")
    torch.cuda.synchronize()
    L.check(L.lib().rayn_b200_device_frame_inputs(renderer.ctx, w, h, 1, 0, 0, 0, None, None, sc.data_ptr()), renderer.ctx)
    return sc


def test_device_scramble_matches_the_statement(renderer):
    for w, h in SCRAMBLE_SHAPES:
        got = _device_scramble(renderer, w, h).cpu().numpy()
        want = np.array([scramble_statement(i) for i in range(w * h)], np.float32)
        assert np.array_equal(got.view(u32), want.view(u32)), (w, h)
    import torch
    idx = big_sample_pixels()
    got = _device_scramble(renderer, *BIG)[torch.from_numpy(idx).cuda()].cpu().numpy()
    want = np.array([scramble_statement(int(i)) for i in idx], np.float32)
    assert np.array_equal(got.view(u32), want.view(u32))
