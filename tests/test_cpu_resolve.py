"""The numpy statement of the film resolve (tests/resolve_ref.py) and the path records its GPU known-answer tests use
(test_gpu_geometry.py): the statement against a plain per-pixel loop, the records' key patterns, the coverage of the case
list, and that the cases fail a resolve whose sort is unstable or whose sums run in sample order."""
import numpy as np
import pytest

import resolve_ref as rr

F = np.float32
SMALL = [(c, a) for c, a in rr.kat_cases() if a["tile"][0] * a["tile"][1] * 4 * a["samples"] * len(a["tile_ids"]) <= 300000]


def loop_resolve(case):
    """pixel by pixel with Python's stable sorted() and one float32 addition at a time"""
    w, h, (tw, th), spp = case["width"], case["height"], case["tile"], 4 * case["samples"]
    planes, mom = rr.fresh_planes(w, h)
    R = tw * th * spp
    for k, t in enumerate(case["tile_ids"]):
        x0, y0, cw, ch = rr.tile_rect(w, h, tw, th, t)
        for pl in range(cw * ch):
            pix = (x0 + pl // ch) + (y0 + pl % ch) * w
            g = [k * R + pl * spp + s for s in range(spp)]
            s0 = [int(case["nrm0"][i, 3:4].view(np.uint32)[0]) for i in g]
            a = sorted([i for i, s in zip(g, s0) if s], key=lambda i: int(case["nrm0"][i, 3:4].view(np.uint32)[0]))
            b = sorted([i for i in g if case["term"][i] >> 30], key=lambda i: (int(case["term"][i] >> 22) & 0xFF, int(case["term"][i]) & 0x3FFFFF))
            with np.errstate(all="ignore"):
                for c in range(3):
                    acc = F(0)
                    for i in a:
                        acc = F(acc + case["nrm0"][i, c])
                    planes["normal"][3 * pix + c] = acc / F(spp)
                    for kind, name in ((1, "color"), (2, "background")):
                        acc = F(0)
                        for i in b:
                            if case["term"][i] >> 30 == kind:
                                acc = F(acc + case["rad"][i, c])
                        planes[name][3 * pix + c] = acc / F(spp)
                planes["alpha"][pix] = F(len(a)) / F(spp)
                for kind in (1, 2):
                    acc = F(0)
                    for i in b:
                        if case["term"][i] >> 30 == kind:
                            r, gg, bb = case["rad"][i, :3]
                            lum = (F(0.2126) * r + F(0.7152) * gg) + F(0.0722) * bb
                            acc = F(acc + lum * lum)
                    mom[kind - 1][pix] = acc / F(spp)
    return planes, mom


def same(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return bool(((a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))).all())


def run(case, **kw):
    planes, mom = rr.fresh_planes(case["width"], case["height"])
    rr.resolve(case, planes, mom, **kw)
    return planes, mom


def films_equal(x, y):
    return all(same(x[0][k], y[0][k]) for k in x[0]) and same(x[1], y[1])


@pytest.mark.parametrize("pattern", rr.PATTERNS)
def test_statement_equals_a_plain_loop(pattern):
    for seed, (tile, samples, mb, n_hit) in enumerate([((3, 2), 17, 5, 3), ((1, 1), 1, 0, 0), ((2, 3), 9, 254, 16)]):
        w, h = 2 * tile[0] - tile[0] // 2 if tile[0] > 1 else 2, 2 * tile[1] - tile[1] // 2 if tile[1] > 1 else 2
        ntx, nty = rr.tile_grid(w, h, *tile)
        case = rr.make_case(w, h, tile, samples, mb, n_hit, list(range(ntx * nty))[::-1], pattern, seed, specials=seed == 2)
        assert films_equal(run(case), loop_resolve(case)), (pattern, tile)


def test_records_follow_their_patterns():
    spp = 260
    for pattern in ("asc", "desc", "equal", "chunk", "digit_low", "digit_mid", "digit_top", "max"):
        case = rr.make_case(3, 2, (2, 1), spp // 4, 7, 0, [0, 1], pattern, 5)
        R = 2 * spp
        QS = R
        for pl in range(2):
            g = np.arange(pl * spp, (pl + 1) * spp)
            t = case["term"][g]
            v = np.flatnonzero(t >> 30)
            key = (t[v] & 0x3FFFFFFF).astype(np.int64)
            depth, slot = key >> 22, key & 0x3FFFFF
            assert (slot < QS).all() and (depth <= 7).all()
            s0 = case["nrm0"][g, 3].view(np.uint32)
            assert ((s0 == 0) | (s0 <= QS)).all()
            if len(v) < 2:
                continue
            if pattern == "asc":
                assert (np.diff(key) >= 0).all()
            if pattern == "desc":
                assert (np.diff(key) <= 0).all() and (np.diff(key) < 0).any()
            if pattern == "equal":
                assert (key == key[0]).all()
            if pattern == "max":
                assert key.max() == (7 << 22) | (QS - 1)
            if pattern == "chunk" and len(v) > 32:
                ch = v // 32
                for c in np.unique(ch):
                    assert (np.diff(key[ch == c]) >= 0).all()
                    lanes = v[ch == c] % 32
                    if c + 1 in ch and len(v) < spp:
                        assert lanes.max() < 31  # invalid lanes before the boundary
                        assert key[ch == c + 1][0] < key[ch == c][-1]  # the keys fall across it
            if pattern.startswith("digit"):
                packed = (depth << case["slot_bits"]) | slot
                passes, dbits = rr.sort_plan(case["slot_bits"] + case["depth_bits"])
                diff = np.bitwise_or.reduce(packed ^ packed[0])
                shift = {"digit_low": 0, "digit_mid": dbits * (passes // 2), "digit_top": dbits * (passes - 1)}[pattern]
                assert diff & ~(((1 << dbits) - 1) << shift) == 0, (pattern, hex(diff))


def test_case_list_covers_every_sort_and_cta_shape():
    cases = rr.kat_cases()
    colour, normal, wpc = set(), set(), {False: set(), True: set()}
    for _, a in cases:
        tw, th = a["tile"]
        qs = tw * th * 4 * a["samples"] + 4 * a["n_hitables"]
        assert qs < 1 << 22 and 4 * a["samples"] <= 16384 and a["max_bounces"] <= 254
        case = dict(samples=a["samples"], slot_bits=max(5, rr.bits_for(qs)), depth_bits=max(1, rr.bits_for(a["max_bounces"])))
        colour.add(case["slot_bits"] + case["depth_bits"])
        normal.add(case["slot_bits"] + 1)
        for mom in (False, True):
            wpc[mom].add(rr.expected_plan(case, mom)[1])
    assert colour == set(range(6, 31)) and normal == set(range(6, 24))
    assert {rr.sort_plan(k) for k in colour} >= {(1, 9), (2, 9), (3, 9), (4, 8), (3, 7), (4, 7)}
    assert wpc[False] == wpc[True] == {1, 2, 5, 8}


def test_cases_catch_an_unstable_sort_and_sample_order_sums():
    """a resolve that breaks ties in the wrong order, or sums in sample order, differs on the cases built for it"""
    unstable, sample_order = [], []
    for i, (cid, a) in enumerate(SMALL):
        case = rr.make_case(seed=1000 + rr.kat_cases().index((cid, a)), **a)
        ref = run(case)
        unstable.append((cid, not films_equal(run(case, stable=False), ref)))
        sample_order.append((cid, not films_equal(run(case, sample_order=True), ref)))
        if cid.endswith(("-equal", "-perm", "-max")):
            assert unstable[-1][1], cid
        # (chunks fall across 32-sample boundaries only above 32 spp)
        if cid.endswith(("-desc", "-perm", "-digit_low", "-digit_mid", "-digit_top")) or (cid.endswith("-chunk") and 4 * a["samples"] > 32):
            assert sample_order[-1][1], cid
    caught_u = {c for c, bad in unstable if bad}
    caught_s = {c for c, bad in sample_order if bad}
    assert len(caught_u) >= len(SMALL) // 2 and len(caught_s) >= len(SMALL) // 2
