"""The persistent march kernels themselves - k_extend_march, k_shadow and k_normals - over given rays, segments and shading
bins, against the numpy statement of the reference's marches (tests/march_ref.py), bit for bit.

The hooks rayn_b200_kat_march_* run the render's own launch helpers (api.cu) on data laid out as a pass holds it.  Every
output word is compared: d_t.w and q_key of every path, vis words, nrm and trap_s, and the kernel's evaluation count, which
is the statement's less its dead evaluations (march_ref's docstring).  Paths and words the input does not name must come back
unchanged.  The cases reach every end kind and tie rule of the marches, per-tile live counts around the 64-slot warps and
128-ray batches, 1 to 3000 tiles, shuffled live lists, segment counts around the 128-segment batches, full and half (paired)
grids, and all six estimator specialisations."""

import numpy as np
import pytest

from rayn_b200 import _lib as L
from rayn_b200 import configs
from rayn_b200.film import Renderer
from rayn_b200.scene import Dielectric, HitableStore, OrbitTrapAlbedo, TracedSDF

import march_ref as mr
from helpers import assert_bit_equal, bits

pytestmark = pytest.mark.gpu
SENT_T, SENT_KEY = np.float32(-7.25), 77  # values of paths no tile lists


def world_of(kind="mandelbox", second=None):
    cam, world = configs.setup((64, 64), volume=False, fractal=kind)
    if second:
        _, w2 = configs.setup((64, 64), volume=False, fractal=second)
        hs = HitableStore()
        for i, h in enumerate(world.hitables.items):
            hs.push(h)
            if i == 1:
                hs.push(TracedSDF(w2.hitables.items[1].sdf, h.material))
        world.hitables = hs
    return cam, world


class Scene:
    """a context with one uploaded scene, its flattened descriptor and the oracle's estimator of each SDF"""

    def __init__(self, oracle, kind="mandelbox", flags=0, second=None, edit=None, trap=False):
        cam, world = world_of(kind, second)
        if trap:
            from test_cpu_trap import ALBEDO_HI, ALBEDO_LO, FRACTAL_MATERIAL, TRAP_HI, TRAP_LO
            mats = world.materials.items
            mats[FRACTAL_MATERIAL] = Dielectric(OrbitTrapAlbedo(TRAP_LO, TRAP_HI, ALBEDO_LO, ALBEDO_HI), mats[FRACTAL_MATERIAL].roughness)
            self.trap = (TRAP_LO, TRAP_HI, ALBEDO_LO, ALBEDO_HI)
        self.r = Renderer(0, flags=flags)
        desc, self.keep = world.flatten(cam)
        if edit:
            edit(desc)
        self.desc = desc
        self.r.upload_scene_desc(desc)
        if trap:
            self.r.set_albedo_traps(world.albedo_traps())
        self.sdf = [i for i in range(desc.n_hitables) if desc.hitables[i].kind != L.HITABLE_SPHERE]
        self.dist = {i: (lambda p, h=desc.hitables[i]: oracle.kat_sdf_dist(h, np.asarray(p, np.float32).reshape(-1, 3))) for i in self.sdf}
        self.S = np.float32(desc.consts.sdf_detail_scale)

    def close(self):
        self.r.close()


@pytest.fixture(scope="module")
def box(oracle):
    s = Scene(oracle)
    yield s
    s.close()


def layout(rays, n_live, R, seed):
    """tiles of R paths, tile t listing n_live[t] of them (a shuffled subset) -> (q_live [T, R], path index of each ray)"""
    rng = np.random.default_rng(seed)
    T = len(n_live)
    q_live = np.full((T, R), -1, np.int32)
    where = []
    for t, n in enumerate(n_live):
        ids = rng.permutation(R)[:n].astype(np.int32)
        q_live[t, :n] = ids
        where.append(t * R + ids)
    where = np.concatenate(where) if where else np.zeros(0, np.int64)
    assert where.size <= rays
    return q_live, where


def check_extend(sc, hk, depth, o, d, t_max, keys, n_live, R, spheres_first=False, paired=False, seed=0):
    n = int(np.sum(n_live))
    o, d, t_max, keys = o[:n], d[:n], t_max[:n], keys[:n]
    q_live, where = layout(n, n_live, R, seed)
    T = len(n_live)
    o_time = np.zeros((T, R, 4), np.float32)
    d_t = np.zeros((T, R, 4), np.float32)
    d_t[..., 3] = SENT_T
    q_key = np.full((T, R), SENT_KEY, np.int32)
    ot, dt, qk = o_time.reshape(-1, 4), d_t.reshape(-1, 4), q_key.reshape(-1)
    ot[where, :3], ot[where, 3] = o, 0.5
    dt[where, :3], dt[where, 3] = d, t_max
    qk[where] = keys
    thr = mr.make_thr(sc.desc.camera, depth)
    ref = mr.march_hit(sc.dist[hk], sc.S, sc.desc.consts.max_marches, o, d, t_max, thr)
    want_t, want_k = dt[:, 3].copy(), qk.copy()
    w = mr.write_rule(ref["t"], t_max, keys, hk, spheres_first)
    want_t[where[w]], want_k[where[w]] = ref["t"][w], hk
    before = d_t.copy()
    ev = sc.r.kat_march_extend(hk, depth, n_live, q_live, o_time, d_t, q_key, spheres_first, paired)
    assert_bit_equal(dt[:, 3], want_t, "d_t.w")
    assert (q_key.reshape(-1) == want_k).all(), "q_key"
    assert (bits(d_t[..., :3]) == bits(before[..., :3])).all(), "d_t.xyz must not change"
    assert ev == mr.kernel_evals(ref), (ev, mr.kernel_evals(ref), int(ref["evals"].sum()))
    return ref


def rays_for(sc, hk, depth, n, seed):
    c = mr.extend_cases(sc.dist[hk], sc.S, mr.make_thr(sc.desc.camera, depth), seed=seed, n=max(n, 300))
    reps = -(-n // len(c["t_max"]))
    o, d, t = (np.concatenate([c[k]] * reps)[:n] for k in ("o", "d", "t_max"))
    return o, d, t, c


# ---- extend --------------------------------------------------------------------------------------------------------------
R_GEOM = 200
GEOMS = {
    "live_edges": [0, 1, 63, 64, 65, 127, 128, 129, R_GEOM],
    "one_tile_under_a_warp": [40],
    "one_tile_full": [R_GEOM],
    "many_tiles": [17, 0, 129, 200, 5] * 30,
}


@pytest.mark.parametrize("paired", [False, True])
@pytest.mark.parametrize("geom", list(GEOMS))
def test_extend_geometries(box, geom, paired):
    n_live = np.array(GEOMS[geom], np.int32)
    o, d, t, _ = rays_for(box, 1, 0, int(n_live.sum()), seed=len(geom))
    keys = np.where(np.arange(len(t)) % 3 == 0, 4, -1).astype(np.int32)
    ref = check_extend(box, 1, 0, o, d, t, keys, n_live, R_GEOM, paired=paired, seed=3)
    if geom == "live_edges":
        assert {mr.END_HIT, mr.END_PAST, mr.END_NAN} <= set(ref["kind"].tolist())


def test_extend_thousands_of_tiles_and_many_waves(box):
    """3000 tiles of 24 paths, every slot refilled many times"""
    rng = np.random.default_rng(5)
    n_live = rng.integers(0, 25, 3000).astype(np.int32)
    o, d, t, _ = rays_for(box, 1, 2, int(n_live.sum()), seed=9)
    check_extend(box, 1, 2, o, d, t, np.full(len(t), -1, np.int32), n_live, 24, seed=4)


@pytest.mark.parametrize("spheres_first", [False, True])
def test_extend_write_rule_at_ties(box, spheres_first):
    """t < t_max writes hk; at t == t_max a later key loses to hk with spheres_first only, an earlier one never"""
    o, d, t, c = rays_for(box, 1, 0, 300, seed=21)
    g = c["groups"]
    sel = np.concatenate([g["fold_tie"], g["step_tie"], g["base"][:100]])
    o, d, t = c["o"][sel], c["d"][sel], c["t_max"][sel]
    keys = np.where(np.arange(len(t)) % 2 == 0, 0, 5).astype(np.int32)  # both sides of hk = 1
    ref = check_extend(box, 1, 0, o, d, t, keys, np.array([len(t)], np.int32), len(t), spheres_first=spheres_first, seed=2)
    tie = ref["t"] == t
    assert (tie & (keys > 1)).sum() >= 10 and (tie & (keys < 1)).sum() >= 10


@pytest.mark.parametrize("max_marches", [1, 2, 3, 256])
def test_extend_march_budgets(oracle, max_marches):
    def edit(desc):
        desc.consts.max_marches = max_marches
    sc = Scene(oracle, edit=edit)
    try:
        o, d, t, _ = rays_for(sc, 1, 0, 700, seed=max_marches)
        ref = check_extend(sc, 1, 0, o, d, t, np.full(700, -1, np.int32), np.array([300, 400], np.int32), 400)
        if max_marches < 256:
            assert mr.END_EXHAUSTED in set(ref["kind"].tolist())
    finally:
        sc.close()


def _ortho(desc):
    desc.camera.kind = L.CAMERA_ORTHOGRAPHIC


def _nan_scale(desc):
    desc.consts.sdf_detail_scale = float("nan")


def _generic(desc):
    desc.hitables[1].min_rad_sq = 1e-20  # outside the packed estimators' range: the generic Mandelbox


def _nine(desc):
    desc.hitables[1].iterations = 9


VARIANTS = [  # (id, kind, flags, edit, expected SDFV)
    ("box12_div3", "mandelbox", 0, None, 4), ("box12_fast", "mandelbox", L.FLAG_NO_DIV3, None, 1),
    ("boxN_div3", "mandelbox", 0, _nine, 5), ("boxN_fast", "mandelbox", L.FLAG_NO_DIV3, _nine, 2),
    ("generic", "mandelbox", 0, _generic, 0), ("bulb", "mandelbulb", 0, None, 3),
]


@pytest.mark.parametrize("vid,kind,flags,edit,want", VARIANTS, ids=[v[0] for v in VARIANTS])
def test_every_estimator_variant(oracle, vid, kind, flags, edit, want):
    """the six specialisations of the march kernels, each through extend (depth 0 and 3), shadow and normals"""
    sc = Scene(oracle, kind, flags, edit=edit)
    try:
        assert sc.r.sdf_variant(1) == want
        for depth in (0, 3):
            o, d, t, _ = rays_for(sc, 1, depth, 500, seed=depth)
            check_extend(sc, 1, depth, o, d, t, np.full(500, -1, np.int32), np.array([129, 371], np.int32), 371)
        check_shadow(sc, 0, n=400, seed=1)
        check_normals(sc, 0, 2, seed=1)
    finally:
        sc.close()


@pytest.mark.parametrize("edit", [_ortho, _nan_scale], ids=["orthographic", "nan_detail_scale"])
def test_extend_scene_constants(oracle, edit):
    sc = Scene(oracle, edit=edit)
    try:
        o, d, t, _ = rays_for(sc, 1, 0, 400, seed=8)
        ref = check_extend(sc, 1, 0, o, d, t, np.full(400, -1, np.int32), np.array([400], np.int32), 400)
        if edit is _nan_scale:
            assert not (ref["kind"] == mr.END_HIT).any()
        check_normals(sc, 0, 0, seed=2)
    finally:
        sc.close()


def test_extend_negative_estimates(oracle):
    """Mandelbulb rays that start inside the set, where the estimate is negative"""
    sc = Scene(oracle, "mandelbulb")
    try:
        rng = np.random.default_rng(3)
        o = (rng.uniform(-0.3, 0.3, (300, 3))).astype(np.float32)
        d = rng.normal(size=(300, 3))
        d = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
        assert (sc.dist[1](o) < 0).sum() > 50
        check_extend(sc, 1, 1, o, d, np.full(300, np.float32(200.0)), np.full(300, -1, np.int32), np.array([300], np.int32), 300)
    finally:
        sc.close()


def test_extend_hits_lie_in_the_float64_hit_band(box):
    """an independent float64 Mandelbox (test_cpu_oracle.mandelbox_ref) at the hit points: within the hit threshold, with a
    tolerance for the float32 rounding the chaotic folds amplify"""
    from test_cpu_oracle import mandelbox_ref
    o, d, t, _ = rays_for(box, 1, 2, 2000, seed=31)
    t = np.full(len(t), np.float32(200.0))
    ref = check_extend(box, 1, 2, o, d, t, np.full(len(t), -1, np.int32), np.array([1000, 1000], np.int32), 1000)
    k = ref["kind"] == mr.END_HIT
    p = o[k].astype(np.float64) + d[k].astype(np.float64) * ref["t"][k].astype(np.float64)[:, None]
    band = np.maximum(5e-5 * box.S, 0.05 * box.S * 0.0004 * ref["t"][k])
    de = np.abs(mandelbox_ref(p.astype(np.float32)))
    assert k.sum() > 500 and np.median(de / band) < 1.0 and np.quantile(de / band, 0.9) < 4.0, np.quantile(de / band, [0.5, 0.9])


# ---- shadow --------------------------------------------------------------------------------------------------------------
def check_shadow(sc, j, n, seed, owners=None, paired=False, n_vis=None):
    hk = sc.sdf[j]
    c = mr.shadow_cases(sc.dist[hk], sc.S, seed=seed)
    reps = -(-max(n, 1) // len(c["max_dist"]))
    st, dv, md = (np.concatenate([c[k]] * reps)[:n] for k in ("start", "dir", "max_dist"))
    rng = np.random.default_rng(seed)
    if owners is None:
        owners = rng.integers(0, max(n // 3, 1), n)  # several segments per owner, on random bits: repeats on one bit too
    bitn = rng.integers(0, 16, n)
    n_vis = n_vis or int(owners.max(initial=0)) + 5
    vis = rng.integers(0, 1 << 32, n_vis, dtype=np.uint64).astype(np.uint32)
    ref = mr.march_occluded(sc.dist[hk], sc.S, sc.desc.consts.max_vis_marches, st, dv, md)
    want = vis.copy()
    for g, b in zip(owners[ref["occluded"]], bitn[ref["occluded"]]):
        want[g] &= np.uint32(~(1 << int(b)) & 0xFFFFFFFF)
    seg_a = np.concatenate([st, md[:, None]], 1).astype(np.float32)
    seg_b = np.concatenate([dv, ((owners.astype(np.uint64) << 4) | bitn.astype(np.uint64)).astype(np.uint32).view(np.float32)[:, None]], 1)
    ev = sc.r.kat_march_shadow(j, seg_a, seg_b, vis, paired)
    assert (vis == want).all(), np.flatnonzero(vis != want)[:10]
    assert ev == mr.kernel_evals(ref), (ev, mr.kernel_evals(ref))
    return ref


@pytest.mark.parametrize("paired", [False, True])
@pytest.mark.parametrize("n_seg", [0, 1, 127, 128, 129, 5000])
def test_shadow_queue_lengths(box, n_seg, paired):
    ref = check_shadow(box, 0, n_seg, seed=n_seg, paired=paired)
    if n_seg >= 1000:
        assert {mr.END_HIT, mr.END_PAST, mr.END_NAN} <= set(ref["kind"].tolist())


@pytest.mark.parametrize("max_vis", [1, 2, 100])
def test_shadow_march_budgets(oracle, max_vis):
    def edit(desc):
        desc.consts.max_vis_marches = max_vis
    sc = Scene(oracle, edit=edit)
    try:
        ref = check_shadow(sc, 0, 1500, seed=max_vis)
        assert mr.END_HIT in set(ref["kind"].tolist())
    finally:
        sc.close()


def test_shadow_two_queues_in_one_scene(oracle):
    sc = Scene(oracle, second="mandelbulb")
    try:
        assert len(sc.sdf) == 2
        check_shadow(sc, 0, 700, seed=1)
        check_shadow(sc, 1, 700, seed=2)
    finally:
        sc.close()


def test_shadow_owner_limits(box):
    """owners 0 and 2^27 - 1, the largest a segment's packed owner word holds (a 512 MB vis array)"""
    owners = np.array([0, (1 << 27) - 1] * 100, np.int64)
    check_shadow(box, 0, 200, seed=4, owners=owners, n_vis=1 << 27)


# ---- normals -------------------------------------------------------------------------------------------------------------
def check_normals(sc, j, depth, seed, n_tiles=3, R=400):
    hk = sc.sdf[j]
    n_hit = sc.desc.n_hitables
    rng = np.random.default_rng(seed)
    thr = mr.make_thr(sc.desc.camera, depth)
    o, d = mr.random_rays(n_tiles * R, seed)
    hit = mr.march_hit(sc.dist[hk], sc.S, 256, o, d, np.full(len(o), np.float32(200.0)), thr)
    t = np.where(hit["kind"] == mr.END_HIT, hit["t"], np.float32(1.5)).astype(np.float32)
    t[::5] = np.float32(0.003)  # near the origin, where S threshold(t) is below 1e-4: the other branch of eps
    QS = R + 4 * n_hit
    bin_start = np.zeros((n_tiles, n_hit + 1), np.int32)
    q_shade = np.full((n_tiles, QS), -1, np.int32)
    for ts in range(n_tiles):
        n_bin = [0, 1, 300, 57][ts % 4] if ts else 0  # an empty bin, one lane, a bin across 128-slot blocks
        sizes = np.zeros(n_hit, np.int64)
        sizes[hk] = n_bin
        ids = rng.permutation(R)[:n_bin].astype(np.int32)
        padded = -(-sizes // 4) * 4
        bin_start[ts, 1:] = np.cumsum(padded)
        q_shade[ts, bin_start[ts, hk]:bin_start[ts, hk] + n_bin] = ids
    o_time = np.concatenate([o, np.zeros((len(o), 1), np.float32)], 1).reshape(n_tiles, R, 4)
    d_t = np.concatenate([d, t[:, None]], 1).reshape(n_tiles, R, 4).astype(np.float32)
    nrm = rng.standard_normal((n_tiles, R, 4)).astype(np.float32)
    trap = getattr(sc, "trap", None) is not None
    trap_s = rng.standard_normal((n_tiles, R)).astype(np.float32) if trap else None
    want_n, want_s = nrm.copy().reshape(-1, 4), None if trap_s is None else trap_s.copy().reshape(-1)
    ids = [q_shade[ts, bin_start[ts, hk]:bin_start[ts, hk + 1]] for ts in range(n_tiles)]
    g = np.concatenate([ts * R + q[q >= 0] for ts, q in enumerate(ids)])  # padding lanes (-1) name no path
    p, eps, nn = mr.shading_normal(sc.dist[hk], sc.S, o[g], d[g], t[g], thr)
    want_n[g, :3], want_n[g, 3] = nn, eps
    if trap:
        import trap_mirror as tm
        h = sc.desc.hitables[hk]
        if L.MULADD_FUSED:
            import mirrors
            tv = mirrors.kat_sdf_trap(h, p)
        else:
            tv = tm.sdf_trap(h, p)
        want_s[g] = tm.palette(sc.trap[0], sc.trap[1], sc.trap[2], sc.trap[3], tv)[0]
    ev = sc.r.kat_march_normals(j, depth, bin_start, q_shade, o_time, d_t, nrm, trap_s)
    assert_bit_equal(nrm.reshape(-1, 4), want_n, f"nrm depth {depth}")
    if trap:
        assert_bit_equal(trap_s.reshape(-1), want_s, "trap_s")
    assert ev == 4 * g.size
    return eps, nn, p


@pytest.mark.parametrize("depth", [0, 1, 8])
def test_normals_bins_and_eps(box, depth):
    eps, nn, p = check_normals(box, 0, depth, seed=depth, n_tiles=6)
    small = eps == np.float32(0.0001)
    if depth == 0:
        assert small.any() and (~small).any()  # both branches of eps = max(1e-4, S threshold(t))


def test_normals_trap_material(oracle):
    sc = Scene(oracle, trap=True)
    try:
        check_normals(sc, 0, 1, seed=5, n_tiles=4)
    finally:
        sc.close()


def test_normals_agree_with_float64_tetrahedral_estimate(box, oracle):
    """the same tetrahedral formula evaluated in float64 (distances from the oracle at the float32 sample points).  The float32
    sums lose about 8 ulp of the largest distance against |n|, and the normalisation a few ulp: the tolerance is that bound."""
    eps, nn, p = check_normals(box, 0, 1, seed=11, n_tiles=4)
    ds = [box.dist[1]((p + mr.TETRA[i][None, :] * eps[:, None]).astype(np.float32)).astype(np.float64) for i in range(4)]
    n64 = sum(mr.TETRA[i].astype(np.float64)[None, :] * ds[i][:, None] for i in range(4))
    mag = np.linalg.norm(n64, axis=1)
    bound = 8 * 2.0 ** -23 * np.max(np.abs(ds), axis=0) / mag + 4 * 2.0 ** -23
    assert (bound < 1e-5).sum() > 50  # well-conditioned points
    assert (np.abs(nn - n64 / mag[:, None]) <= 4 * bound[:, None]).all()


# ---- argument checks -----------------------------------------------------------------------------------------------------
def test_malformed_input_is_rejected_and_the_context_still_renders(box):
    r = box.r
    o, d, t, _ = rays_for(box, 1, 0, 8, seed=1)
    one = np.array([4], np.int32)

    def ext(hk=1, n_live=one, q=None, R=8, T=1):
        q = np.arange(R, dtype=np.int32)[None].repeat(T, 0) if q is None else q
        return r.kat_march_extend(hk, 0, n_live, q, np.zeros((T, R, 4), np.float32), np.zeros((T, R, 4), np.float32),
                                  np.zeros((T, R), np.int32))
    bad = [lambda: ext(q=np.array([[0, 1, 8, 2, 0, 0, 0, 0]], np.int32)),       # id >= R
           lambda: ext(n_live=np.array([9], np.int32)),                          # n_live > R
           lambda: ext(n_live=np.zeros(65536, np.int32), R=1, T=65536),          # more than 65535 tiles
           lambda: ext(hk=0)]                                                    # not an SDF
    seg_a = np.zeros((1, 4), np.float32)
    vis = np.zeros(4, np.uint32)
    for w in (np.uint32(4 << 4), np.uint32(1 << 31)):                             # owner >= n_vis; owner above 2^27 - 1
        bad.append(lambda w=w: r.kat_march_shadow(0, seg_a, np.array([[0, 0, 1, w.view(np.float32)]], np.float32), vis))
    bs = np.zeros((1, box.desc.n_hitables + 1), np.int32)
    bs[0, 2:] = 8
    bad.append(lambda: r.kat_march_normals(0, 0, np.where(bs > 0, 9, 0).astype(np.int32), np.zeros((1, 8), np.int32),  # bin past QS
                                           np.zeros((1, 8, 4), np.float32), np.zeros((1, 8, 4), np.float32), np.zeros((1, 8, 4), np.float32)))
    bad.append(lambda: r.kat_march_normals(0, 0, bs, np.full((1, 8), 8, np.int32), np.zeros((1, 8, 4), np.float32),  # path id >= R
                                           np.zeros((1, 8, 4), np.float32), np.zeros((1, 8, 4), np.float32)))
    for f in bad:
        with pytest.raises(RuntimeError, match="kat_march"):
            f()
    check_extend(box, 1, 0, o, d, t, np.full(8, -1, np.int32), one * 2, 8)
    from helpers import small_config
    c, inp = small_config(3, (16, 16), 1, 1)
    r.upload_scene(c["world"], c["camera"])
    g = r.render_host(inp, (16, 16), c["integrator"], configs.frame_time_range(1))
    assert np.isfinite(g["color"]).all()
    r.upload_scene_desc(box.desc)


@pytest.mark.skipif(L.MULADD_FUSED or L.LEGACY, reason="already inside a variant run")
def test_fused_mul_add_variant_passes_this_suite():
    from test_gpu_parity import _run_suite_variant
    assert " passed" in _run_suite_variant({"RAYN_MULADD_FUSED": "1"}, ["tests/test_gpu_march.py", "-k", "not variant_passes"])
