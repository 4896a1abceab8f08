"""The CPU oracle at the limits of include/rayn_b200.h (16 hitables, materials and lights), on scenes with exact ties, on
boundary sample tables and against the closed form of many-light direct illumination.  These are the oracle-side halves of
test_gpu_limits.py: the scenes must render (finite films) before a bit-exact comparison with the device means anything, and the
closed form checks the oracle itself, not only its agreement with the kernels."""
import numpy as np
import pytest

from rayn_b200 import _lib as L
from rayn_b200.film import FrameInputs

import limits_scenes as S
from helpers import CH, assert_bit_equal, small_config


def _assert_sane(o, what):
    for ch in CH:
        assert np.isfinite(o[ch]).all(), f"{what}: non-finite {ch}"
    assert (o["color"] >= 0).all() and (o["background"] >= 0).all(), what
    assert o["alpha"].min() >= 0 and o["alpha"].max() <= 1.0, what


@pytest.mark.parametrize("shape", ["A", "B", "B16", "C"])
def test_limit_scenes_use_every_slot(shape):
    cam, world = S.SHAPES[shape]((32, 24), True)
    desc, _ = world.flatten(cam)
    assert desc.n_hitables == desc.n_materials == desc.n_lights == L.RAYN_MAX_HITABLES == L.RAYN_MAX_MATERIALS == L.RAYN_MAX_LIGHTS
    assert sorted(h.material for h in world.hitables.items) == list(range(S.N))  # each hitable has its own material
    assert {desc.materials[m].kind for m in range(S.N)} == {L.MATERIAL_LAMBERTIAN, L.MATERIAL_DIELECTRIC, L.MATERIAL_SKY,
                                                            L.MATERIAL_EMISSIVE}
    kinds = [desc.hitables[i].kind for i in range(S.N)]
    if shape == "A":
        assert kinds == [L.HITABLE_SPHERE] * 8 + [L.HITABLE_MANDELBOX] + [L.HITABLE_SPHERE] * 7
    elif shape == "C":
        assert kinds == [L.HITABLE_SPHERE] * S.N and all(np.any(desc.hitables[i].center_velocity[:]) for i in range(1, S.N))
    else:
        assert {L.HITABLE_MANDELBOX, L.HITABLE_MANDELBULB} <= set(kinds) and kinds.count(L.HITABLE_SPHERE) == (shape == "B")


@pytest.mark.parametrize("shape", ["A", "B", "B16", "C"])
@pytest.mark.parametrize("volume", [False, True])
def test_oracle_renders_limit_scenes(oracle, shape, volume):
    cam, world = S.SHAPES[shape]((32, 24), volume)
    integ, inp = S.inputs((32, 24), 1, 3)
    o, info = oracle.render(world, cam, inp, (8, 8), integ, S.TR)
    _assert_sane(o, f"shape {shape}")
    assert o["color"].sum() > 0 and o["alpha"].sum() > 0 and o["background"].sum() > 0
    assert info["shadow_rays"] > 0 and info["extend_rays"] >= 32 * 24 * 4


@pytest.mark.parametrize("shape", ["A", "B"])
def test_trap_oracles_render_every_trap_material(shape):
    import mirrors
    cam, world = S.SHAPES[shape]((32, 24), True, traps=True)
    traps = world.albedo_traps()
    assert [t.material for t in traps] == S.TRAPPABLE and traps[-1].material == S.N - 1
    integ, inp = S.inputs((32, 24), 1, 3)
    o, _ = mirrors.render(world, cam, inp, (8, 8), integ, S.TR)
    _assert_sane(o, f"trap shape {shape}")
    plain, _ = mirrors.render(world, cam, inp, (8, 8), integ, S.TR, traps=[])
    assert not np.array_equal(o["color"], plain["color"])  # the traps show
    alb, _ = mirrors.render_albedo(world, cam, inp, (8, 8), integ, S.TR)
    assert np.isfinite(alb).all() and alb.max() > 0


def sphere_closest_hit_f64(world, o, d, t_max=200.0):
    """float64 restatement of sphere.rs:48-72 folded over the hitables in order, first index wins (hitable.rs:170-210).
    -> (t, object, gap, cond): gap = relative distance between the two nearest roots of all spheres, where a ray whose
    discriminant is within float32 rounding of 0 (float32 may decide hit or miss either way) counts as a double root;
    cond = the relative condition of the hit's t (|b| + (b^2 + |oc|^2 + r^2) / sqrt(disc)) / t: float32 rounding moves t by
    about cond * 2^-24 relative, which is large for tangent rays and for roots that cancel (an origin on the surface)"""
    o, d = np.asarray(o, np.float64), np.asarray(d, np.float64)
    cands, conds, roots = [], [], []
    for h in world.hitables.items:
        oc = o - np.asarray(h.center, np.float64)
        b = np.sum(oc * d, axis=1)
        r2 = float(h.radius) ** 2
        oc2 = np.sum(oc * oc, axis=1)
        disc = b * b - (oc2 - r2)
        undecided = np.abs(disc) <= 16 * 2.0 ** -24 * (b * b + oc2 + r2)
        sq = np.sqrt(np.maximum(disc, 0.0))
        t = np.full(len(o), np.inf)
        for r in (-b + sq, -b - sq):  # the smaller valid root wins
            ok = (r > 1e-4) & (r <= t_max)
            t = np.where((disc > 0) & ok & (r < t), r, t)
            roots.append(np.where(undecided & (-b > 1e-4), -b, np.where((disc > 0) & ok, r, np.inf)))
        cands.append(t)
        conds.append((np.abs(b) + (b * b + oc2 + r2) / np.sqrt(np.maximum(disc, 1e-300))) / np.maximum(t, 1e-30))
    cands, conds = np.stack(cands), np.stack(conds)
    obj = np.argmin(cands, axis=0)
    t = cands[obj, np.arange(len(o))]
    srt = np.sort(np.stack(roots), axis=0)
    gap = (srt[1] - srt[0]) / np.maximum(srt[0], 1e-30)
    return np.where(np.isfinite(t), t, t_max), np.where(np.isfinite(t), obj, -1), gap, conds[obj, np.arange(len(o))]


def check_sphere_closest_hit(t, obj, world, o, d):
    rt, robj, gap, cond = sphere_closest_hit_f64(world, o, d)
    clear = (gap > 1e-4) | ~np.isfinite(gap)
    assert clear.mean() > 0.99 and len(np.unique(robj[clear & (robj >= 0)])) == S.N
    assert np.array_equal(obj[clear], robj[clear]), f"{np.count_nonzero(obj[clear] != robj[clear])} rays hit another object"
    hit = (robj >= 0) & clear & (cond * 2.0 ** -24 < 2e-6)  # away from tangent rays and cancelling roots
    assert hit.mean() > 0.8
    assert np.allclose(t[hit], rt[hit], rtol=1e-5, atol=0), np.abs(t[hit] / rt[hit] - 1).max()
    assert (t[robj < 0] == 200.0).all()


def sphere_rays(n=40_000, seed=8):
    """rays from a shell around the 16-sphere scene aimed at its spheres, plus rays from inside the scene"""
    from helpers import random_rays
    o, d = random_rays(n, seed, origin_radius=4.5, spread=0.9)
    o[: n // 4] *= np.float32(0.1)  # inside: some start within a sphere, some between them
    return o, d


def test_oracle_closest_hit_matches_float64_sphere_roots(oracle):
    cam, world = S.spheres_only()
    desc, _ = world.flatten(cam)
    o, d = sphere_rays()
    t, obj = oracle.kat_closest_hit(desc, 0, o, d)
    check_sphere_closest_hit(t, obj, world, o, d)


@pytest.mark.parametrize("kind", ["spheres_before", "spheres_after", "spheres_across", "boxes_adjacent", "boxes_separated"])
def test_oracle_first_copy_wins_exact_ties(oracle, kind):
    """the later of two identical hitables is never hit: re-materialing it changes no plane"""
    from rayn_b200 import Emissive, Srgb
    integ, inp = S.inputs((32, 32), 1, 3)
    cam, world, later = S.tie_scene(kind, (32, 32))
    o, _ = oracle.render(world, cam, inp, (16, 16), integ, S.TR)
    cam2, world2, _ = S.tie_scene(kind, (32, 32), second_material=Emissive.new_splat(Srgb(9.0, 0.1, 0.1)))
    o2, _ = oracle.render(world2, cam2, inp, (16, 16), integ, S.TR)
    for ch in CH:
        assert_bit_equal(o2[ch], o[ch], f"{kind} {ch}")
    # and the duplicate is really visible: with the FIRST copy's material changed the film changes
    first = world.hitables.items[later - (2 if kind in ("spheres_across", "boxes_separated") else 1)]
    world.materials.items[first.material] = Emissive.new_splat(Srgb(9.0, 0.1, 0.1))
    o3, _ = oracle.render(world, cam, inp, (16, 16), integ, S.TR)
    assert not np.array_equal(o3["background"], o["background"])


BOUNDARY_CONFIGS = [1, 3, 4]
SCRAMBLES = [None, 0.0, S.ONE_MINUS]


@pytest.mark.parametrize("n", BOUNDARY_CONFIGS)
@pytest.mark.parametrize("scramble", SCRAMBLES)
def test_oracle_stays_finite_on_boundary_tables(oracle, n, scramble):
    c, inp = small_config(n, (32, 32), 2, 4)
    S.boundary_tables(inp, S.boundary_values(c["world"].materials.items), 10 + n, scramble=scramble)
    o, _ = oracle.render(c["world"], c["camera"], inp, (16, 16), c["integrator"], S.TR)
    _assert_sane(o, f"cfg{n} scramble {scramble}")


@pytest.mark.parametrize("shape", ["A", "B"])
@pytest.mark.parametrize("scramble", SCRAMBLES)
def test_oracle_stays_finite_on_boundary_tables_at_the_limits(oracle, shape, scramble):
    cam, world = S.SHAPES[shape]((32, 24), True)
    integ, inp = S.inputs((32, 24), 1, 3)
    S.boundary_tables(inp, S.boundary_values(world.materials.items), 30, scramble=scramble)
    o, _ = oracle.render(world, cam, inp, (8, 8), integ, S.TR)
    _assert_sane(o, f"shape {shape} scramble {scramble}")


FAMILIES = list(S.set_families(S.inputs((8, 8), 1, 4)[0]))


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("scramble", S.EXTREME_TABLE_VALUES, ids=["zero", "one_minus"])
def test_one_family_reads_only_extreme_values(family, scramble):
    """what the path reads is fract(table + scramble): with the constant scramble plane every read of the family's sets is
    exactly 0 or 1 - 2^-24 (both appear), and every other set keeps its R_d values"""
    c, inp = small_config(4, (32, 32), 2, 4)
    ref = FrameInputs(32, 32, 2, c["integrator"])
    S.extreme_family_tables(inp, family, c["integrator"], scramble, 20)
    assert (inp.scramble == np.float32(scramble)).all()
    sets_1d, sets_2d = S.set_families(c["integrator"])[family]
    spp = inp.spp

    def read(table):  # dm::fract(table + scramble) in float32
        x = table + np.float32(scramble)
        return x - np.trunc(x)
    t1 = inp.samples_1d.reshape(-1, spp)
    t2 = inp.samples_2d.reshape(-1, 2 * spp)
    got = np.concatenate([read(t1[s]) for s in sets_1d] + [read(t2[s]) for s in sets_2d])
    assert set(np.unique(got).tolist()) == {0.0, float(S.ONE_MINUS)}
    other_1d = [s for s in range(inp.sets_1d) if s not in sets_1d]
    other_2d = [s for s in range(inp.sets_2d) if s not in sets_2d]
    assert np.array_equal(t1[other_1d], ref.samples_1d.reshape(-1, spp)[other_1d])
    assert np.array_equal(t2[other_2d], ref.samples_2d.reshape(-1, 2 * spp)[other_2d])


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("scramble", S.EXTREME_TABLE_VALUES, ids=["zero", "one_minus"])
def test_oracle_stays_finite_with_one_family_at_its_extremes(oracle, family, scramble):
    for n in (3, 4):
        c, inp = small_config(n, (32, 32), 2, 4)
        S.extreme_family_tables(inp, family, c["integrator"], scramble, 20 + n)
        o, _ = oracle.render(c["world"], c["camera"], inp, (16, 16), c["integrator"], S.TR)
        _assert_sane(o, f"cfg{n} family {family} scramble {scramble}")


def test_boundary_values_and_set_families():
    v = S.boundary_values()
    assert v.dtype == np.float32 and v.min() == 0.0 and v.max() == S.ONE_MINUS
    for x in (np.float32(2.0 ** -24), np.float32(0.5), np.float32(0.04), np.float32(0.05), np.float32(15) / np.float32(16),
              np.nextafter(np.float32(1) / np.float32(16), np.float32(0))):
        assert x in v
    integ, inp = S.inputs((8, 8), 1, 4)
    fam = S.set_families(integ)
    used_1d = sorted(s for f in fam.values() for s in f[0])
    used_2d = sorted(s for f in fam.values() for s in f[1])
    # every 1-D set and every 2-D set the path reads belongs to a family (the integrator requests twice the 2-D sets it reads,
    # film.rs:432 / integrator.rs: 12 + 8 vm per depth, of which the first half are read as pairs)
    assert sorted(set(used_1d)) == list(range(inp.sets_1d))
    assert sorted(set(used_2d)) == list(range(2 + (integ.max_bounces + 1) * (6 + 4 * integ.volume_marches)))
    assert used_2d[-1] < inp.sets_2d


K_FRAMES, CF_SAMPLES = 64, 16


def closed_form_films(render):
    """K_FRAMES colour planes of the closed-form scene through render(world, cam, inputs, integrator), and the expectation.
    Each frame gets its own seeded uniform scramble plane: the SmallRng plane does not depend on the frame, and the R_d set s
    of frame f + 1 is set s + 1 of frame f, so frames that differ only in their number are not independent estimates.  With
    a fresh plane each frame is an independent Cranley-Patterson rotation of its tables, an unbiased estimate of the pixel,
    and the spread between frames is a true standard error."""
    cam, world = S.closed_form_scene()
    films = []
    for k in range(K_FRAMES):
        integ, inp = S.inputs(S.CF_RES, CF_SAMPLES, 0, frame=1 + k)
        inp.scramble[:] = np.random.default_rng(100 + k).random(inp.scramble.size, dtype=np.float32)
        films.append(render(world, cam, inp, integ)["color"])
    return films, S.closed_form_film(world, cam, inp.fis)


def test_many_light_direct_illumination_matches_closed_form(oracle):
    """16 lights, NEE only: the oracle's K-frame mean lies within 5 standard errors of (albedo / pi) sum_j E_j in every pixel,
    and the film-wide mean within 3"""
    films, expected = closed_form_films(lambda w, c, inp, integ: oracle.render(w, c, inp, (8, 8), integ, S.TR)[0])
    assert all(np.isfinite(f).all() and (f > 0).all() for f in films)  # every camera ray hits the lit sphere
    z_px, z_all = S.closed_form_check(films, expected)
    assert z_px < 5 and z_all < 3, (z_px, z_all)
