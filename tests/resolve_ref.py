"""The film resolve (include/rayn_b200.h: rayn_b200_kat_resolve, rt_kernels.cuh: k_resolve) restated in numpy, and the path
records its known-answer tests feed it.  Shared by test_cpu_resolve.py and test_gpu_geometry.py.

Per pixel: the valid records in sample order, stably sorted by the depth-0 slot + 1 (normal and alpha) and by (depth, slot)
(colour and background); strictly sequential float32 sums from +0 in that order (np.add.accumulate, never the pairwise
np.sum), each divided by float(spp); alpha = count / spp.  The moments add ((0.2126 r + 0.7152 g) + 0.0722 b)^2 of the colour
and background records in the colour order.  Nothing here mirrors the kernel's radix sort, its digit widths or its
sortedness check: those are what the records are built to exercise."""
import numpy as np

F = np.float32
SENTINEL = F(-3.0e38)  # the planes' content before a resolve: it must survive wherever the resolve writes nothing
COUNTS = (0, 1, 31, 32, 33, 63, 64, 65)  # valid records per pixel, besides spp itself
PATTERNS = ("asc", "desc", "equal", "perm", "digit_low", "digit_mid", "digit_top", "max", "chunk")


def tile_grid(w, h, tw, th):
    return (w + w % tw) // tw, (h + h % th) // th  # film.rs:399-404


def tile_rect(w, h, tw, th, t):
    """(x0, y0, clipped width, clipped height) of tile t"""
    ntx, nty = tile_grid(w, h, tw, th)
    tx, ty = divmod(t, nty)
    x0, y0 = tx * tw, ty * th
    return x0, y0, min(x0 + tw, w) - x0, min(y0 + th, h) - y0


def sort_plan(key_bits):
    """(passes, digit bits) the radix sort makes for keys of key_bits significant bits (rt_kernels.cuh: warp_radix_sort)"""
    passes = (key_bits + 8) // 9
    return passes, -(-key_bits // passes)


def bits_for(v):
    """the least b with 2^b >= v + 1"""
    return int(v).bit_length()


def _seq_sum(vals):
    """[n_pix, n] float32 -> the strictly sequential sums from +0 along axis 1"""
    z = np.zeros((vals.shape[0], 1), np.float32)
    with np.errstate(all="ignore"):
        return np.add.accumulate(np.concatenate([z, vals], axis=1), axis=1, dtype=np.float32)[:, -1]


def _order(keys, valid, stable):
    """per row the sample indices of the valid entries by key, then the invalid ones; stable=False breaks ties in reverse
    sample order (a deliberately wrong resolve, for the sensitivity tests)"""
    k = np.where(valid, keys.astype(np.int64), np.int64(1) << 40)
    tie = np.arange(k.shape[1])
    return np.lexsort((np.broadcast_to(tie if stable else -tie, k.shape), k), axis=-1)


def resolve(case, planes, moments=None, stable=True, sample_order=False):
    """Writes the resolve of `case` (make_case) into planes (flat float32 arrays keyed color / alpha / background / normal)
    and moments ([2, W*H] or None), in place.  stable=False / sample_order=True: deliberately wrong variants."""
    w, h, (tw, th), spp = case["width"], case["height"], case["tile"], 4 * case["samples"]
    R = tw * th * spp
    div = F(spp)
    for k, t in enumerate(case["tile_ids"]):
        x0, y0, cw, ch = tile_rect(w, h, tw, th, t)
        npix = cw * ch
        g = k * R + np.arange(npix * spp).reshape(npix, spp)
        pl = np.arange(npix)
        xl, yl = pl // ch, pl % ch
        pix = (x0 + xl) + (y0 + yl) * w
        s0 = case["nrm0"][g, 3].view(np.uint32)
        term = case["term"][g]
        kind = term >> 30
        va, vb = s0 != 0, kind != 0
        keya = np.zeros_like(s0) if sample_order else s0
        keyb = np.zeros_like(term) if sample_order else term & np.uint32(0x3FFFFFFF)  # (depth, slot) order = depth << 22 | slot order
        oa, ob = _order(keya, va, stable), _order(keyb, vb, stable)
        take = lambda a, o: np.take_along_axis(a, o, axis=1)  # noqa: E731
        nrm = case["nrm0"][g][..., :3]
        rad = case["rad"][g][..., :3]
        va_o = take(va, oa)
        kind_o = take(kind, ob)
        for c in range(3):
            n_c = np.where(va_o, take(nrm[..., c], oa), F(0))
            r_c = take(rad[..., c], ob)
            with np.errstate(all="ignore"):
                planes["normal"][3 * pix + c] = _seq_sum(n_c) / div
                planes["color"][3 * pix + c] = _seq_sum(np.where(kind_o == 1, r_c, F(0))) / div
                planes["background"][3 * pix + c] = _seq_sum(np.where(kind_o == 2, r_c, F(0))) / div
        planes["alpha"][pix] = F(va.sum(axis=1)) / div
        if moments is not None:
            r = [take(rad[..., c], ob) for c in range(3)]
            with np.errstate(all="ignore"):
                lum = (F(0.2126) * r[0] + F(0.7152) * r[1]) + F(0.0722) * r[2]
                l2 = lum * lum
                moments[0][pix] = _seq_sum(np.where(kind_o == 1, l2, F(0))) / div
                moments[1][pix] = _seq_sum(np.where(kind_o == 2, l2, F(0))) / div


def fresh_planes(w, h):
    planes = {k: np.full((1 if k == "alpha" else 3) * w * h, SENTINEL, np.float32) for k in ("color", "alpha", "background", "normal")}
    return planes, np.full((2, w * h), SENTINEL, np.float32)


def _keys(rng, pattern, samples, lo, hi, key_bits, i_pix):
    """keys in [lo, hi] for the valid samples `samples` (ascending), in sample order, by pattern"""
    n = len(samples)
    if n == 0:
        return np.zeros(0, np.int64)
    if pattern == "asc":
        return np.sort(rng.integers(lo, hi + 1, n))
    if pattern == "desc":
        return np.sort(rng.integers(lo, hi + 1, n))[::-1]
    if pattern == "equal":
        return np.full(n, rng.integers(lo, hi + 1))
    if pattern == "max":  # the largest key of the order, alone or among the smallest
        return np.full(n, hi) if i_pix % 2 else rng.choice([lo, hi], n)
    if pattern == "chunk":  # ascending within every 32-sample chunk, each chunk's keys below the previous chunk's
        v = np.sort(rng.integers(lo, hi + 1, n))
        sizes = np.unique(samples // 32, return_counts=True)[1]
        out, end, pos = np.empty_like(v), n, 0
        for sz in sizes:
            out[pos:pos + sz] = v[end - sz:end]
            end -= sz
            pos += sz
        return out
    if pattern.startswith("digit"):  # keys that differ only in one digit of the radix sort
        passes, dbits = sort_plan(key_bits)
        shift = {"digit_low": 0, "digit_mid": dbits * (passes // 2), "digit_top": dbits * (passes - 1)}[pattern]
        base = int(rng.integers(lo, hi + 1))
        for _ in range(64):
            cand = (base & ~(((1 << dbits) - 1) << shift)) | (rng.integers(0, 1 << dbits, n) << shift)
            ok = (cand >= lo) & (cand <= hi)
            if ok.sum() > n // 2:
                return np.where(ok, cand, base)
        return np.full(n, base)
    return rng.integers(lo, hi + 1, n)  # perm


def _valid_samples(rng, pattern, n, spp):
    """which samples carry the n valid records; chunk: every 32-sample chunk ends in invalid lanes, so a key that falls
    across a chunk boundary is compared with a key several lanes back"""
    if pattern == "chunk" and n < spp:
        lanes = np.arange(spp)
        pref = lanes[(lanes % 32) < 24]
        rest = lanes[(lanes % 32) >= 24]
        pick = np.concatenate([pref, rest])[:n]
        return np.sort(pick)
    return np.sort(rng.choice(spp, n, replace=False))


def _payload(rng, n, specials):
    """float32 [n, 4] over many binades, so that every change of the summation order changes the sums"""
    v = (rng.standard_normal((n, 4)) * np.exp2(rng.integers(-6, 7, (n, 4)))).astype(np.float32)
    if specials:
        sp = np.array([np.nan, np.inf, -np.inf, -0.0, 1e-40, -1e-42, np.float32(2.0 ** -149), 3e38], np.float32)
        m = rng.random((n, 4)) < 0.05
        v[m] = rng.choice(sp, m.sum())
    return v


def make_case(width, height, tile, samples, max_bounces, n_hitables, tile_ids, pattern, seed, specials=False):
    """Path records (rayn_b200_kat_resolve's layout) for tiles tile_ids of a width x height film.  The i-th pixel (over the
    tiles) has COUNTS[i % 9] valid records (spp for the ninth), at most spp, in each order, keys by `pattern`.  Records of pixels outside a clipped
    tile are filled too (valid keys, NaN payloads): the resolve must never read them."""
    rng = np.random.default_rng(seed)
    tw, th = tile
    spp = 4 * samples
    R = tw * th * spp
    QS = R + 4 * n_hitables
    slot_bits = max(5, bits_for(QS))
    depth_bits = max(1, bits_for(max_bounces))
    n_paths = len(tile_ids) * R
    term = np.zeros(n_paths, np.uint32)
    nrm0 = np.zeros((n_paths, 4), np.float32)
    rad = np.zeros((n_paths, 4), np.float32)
    counts = list(COUNTS) + [spp]
    i_pix = 0  # pixels so far, over the tiles
    for k, t in enumerate(tile_ids):
        _, _, cw, ch = tile_rect(width, height, tw, th, t)
        used = cw * ch * spp
        junk = slice(k * R + used, (k + 1) * R)
        term[junk] = (1 << 30) | 5
        nrm0[junk] = np.nan
        nrm0[junk, 3] = np.array([1], np.uint32).view(np.float32)[0]
        rad[junk] = np.nan
        for p in range(cw * ch):
            g0 = k * R + p * spp
            n = min(counts[i_pix % len(counts)], spp)
            i_pix += 1
            # normal order: keys slot + 1 in [1, QS]
            sa = _valid_samples(rng, pattern, n, spp)
            ka = _keys(rng, pattern, sa, 1, QS, slot_bits + 1, p)
            nrm0[g0 + sa, 3] = ka.astype(np.uint32).view(np.float32)
            # colour order: packed key depth << slot_bits | slot with depth <= max_bounces; a slot >= QS becomes QS - 1, which
            # keeps the keys' order
            sb = _valid_samples(rng, pattern, n, spp)
            kb = _keys(rng, pattern, sb, 0, (max_bounces << slot_bits) | (QS - 1), slot_bits + depth_bits, p)
            depth, slot = kb >> slot_bits, np.minimum(kb & ((1 << slot_bits) - 1), QS - 1)
            kind = rng.choice([1, 2], n, p=[0.7, 0.3]).astype(np.uint32)
            term[g0 + sb] = (kind << 30) | (depth.astype(np.uint32) << 22) | slot.astype(np.uint32)
            nrm0[g0:g0 + spp, :3] = _payload(rng, spp, specials)[:, :3]
            rad[g0:g0 + spp] = _payload(rng, spp, specials)
    return dict(width=width, height=height, tile=tile, samples=samples, max_bounces=max_bounces, n_hitables=n_hitables,
                tile_ids=list(tile_ids), term=term, nrm0=nrm0, rad=rad, slot_bits=slot_bits, depth_bits=depth_bits)


def geometry(slot_bits, spp):
    """(tile_w, tile_h, n_hitables) whose shading-slot count QS = tile_w*tile_h*spp + 4*n_hitables needs exactly slot_bits
    bits (2^(slot_bits-1) <= QS < 2^slot_bits; 5 bits for any QS < 32), with the smallest tile; None if there is none"""
    lo, hi = (1 if slot_bits == 5 else 1 << (slot_bits - 1)), (1 << slot_bits) - 1
    area = max(1, lo // spp)
    for a in (area, area + 1):
        for n_hit in range(0, 17):
            qs = a * spp + 4 * n_hit
            if lo <= qs <= hi and qs < (1 << 22):
                # a tile that is not square and not a row: a x 1 for odd areas, else (a / 2) x 2 etc.
                tw = a
                for d in (3, 2):
                    if a % d == 0 and a > d:
                        tw = a // d
                        break
                return tw, a // tw, n_hit
    return None


def _case_args(slot_bits, max_bounces, spp, pattern, specials):
    tw, th, n_hit = geometry(slot_bits, spp)
    if tw * th * spp <= 4096:  # small tiles: a 2 x 2 grid whose last column and row are clipped tiles
        w, h = (2 * tw - tw // 2 if tw > 1 else 2), (2 * th - th // 2 if th > 1 else 2)
        ids = list(range(tile_grid(w, h, tw, th)[0] * tile_grid(w, h, tw, th)[1]))
    else:
        w, h, ids = tw, th, [0]
    return dict(width=w, height=h, tile=(tw, th), samples=spp // 4, max_bounces=max_bounces, n_hitables=n_hit, tile_ids=ids,
                pattern=pattern, specials=specials)


def _spp_for(slot_bits, i):
    """a sample count for the i-th case of slot_bits with a tile of at most 512 pixels: every warps-per-CTA plan (8, 5, 2, 1)
    recurs"""
    cands = [4, 12, 36, 68, 100, 260, 2048, 4000, 8192, 16384, 3000, 6000, 12000]
    paths = 1 << (slot_bits - 1)
    ok = [s for s in cands if s <= max(28, paths) and s * 512 >= paths]
    return ok[i % len(ok)]


def kat_cases():
    """(id, make_case kwargs) of the resolve known-answer tests: every slot_bits of the normal order (key_bits 6-23) and every
    key_bits 6-30 of the colour order, and every key pattern at one, two, three (9-bit digits) and four sort passes"""
    out = []
    for i, s in enumerate(range(5, 23)):  # depth_bits 1
        out.append((f"s{s}-d1", _case_args(s, 1, _spp_for(s, i), PATTERNS[i % len(PATTERNS)], i % 3 == 0)))
    for i, s in enumerate(range(16, 23)):  # depth_bits 8: colour key_bits 24-30
        out.append((f"s{s}-d8", _case_args(s, 254, _spp_for(s, i + 7), PATTERNS[(i + 4) % len(PATTERNS)], i % 2 == 0)))
    for s, mb, spp in ((5, 0, 16), (13, 31, 64), (18, 255 - 1, 4000), (22, 200, 16384)):  # colour key_bits 6, 18, 26, 30
        for j, p in enumerate(PATTERNS):
            out.append((f"s{s}-mb{mb}-{p}", _case_args(s, mb, spp, p, j % 2 == 1)))
    return out


def expected_plan(case, moments):
    """np, wpc, slot_bits, depth_bits of the resolve of a case (api.cu: resolve_plan, rt_kernels.cuh: resolve_smem_per_warp)"""
    spp = 4 * case["samples"]
    np_ = 32
    while np_ < spp:
        np_ *= 2
    per_warp = np_ * 8 + 512 * 4 + ((8 if moments else 6) * 33 + 2) * 4
    return np_, min(8, 200 * 1024 // per_warp), case["slot_bits"], case["depth_bits"]
