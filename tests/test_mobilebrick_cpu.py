"""The MobileBrick evaluation's CPU restatement (oracle/mobilebrick_oracle.py) and its host-side inputs: the random
stream against the C++ standard and an independent MT19937, the round-based Poisson-disk elimination against Open3D's
sequential heap loop, the uniform sampler's counts, the no-triangle fallback, the DOUBT points' sensitivity, and the
synthetic scan builder reaching the cases the GPU tests rely on."""
from fractions import Fraction

import numpy as np
import pytest

from oracle import mobilebrick_oracle as mo
from tests import mobilebrick_cases as mc


# ------------------------------------------------------------------------------------------------------------ stream
def _mt19937_python(seed, n):
    """MT19937 from its definition (Matsumoto and Nishimura 1998), init_genrand seeding."""
    mt = [0] * 624
    mt[0] = seed & 0xFFFFFFFF
    for i in range(1, 624):
        mt[i] = (1812433253 * (mt[i - 1] ^ (mt[i - 1] >> 30)) + i) & 0xFFFFFFFF
    idx, out = 624, []
    for _ in range(n):
        if idx >= 624:
            for i in range(624):
                y = (mt[i] & 0x80000000) | (mt[(i + 1) % 624] & 0x7FFFFFFF)
                mt[i] = mt[(i + 397) % 624] ^ (y >> 1) ^ (0x9908B0DF if y & 1 else 0)
            idx = 0
        y = mt[idx]
        idx += 1
        y ^= y >> 11
        y ^= (y << 7) & 0x9D2C5680
        y ^= (y << 15) & 0xEFC60000
        y ^= y >> 18
        out.append(y)
    return out


def test_stream_matches_the_standard():
    assert int(mo.mt19937_outputs(5489, 10000)[-1]) == 4123659995  # [rand.predef]: the 10000th output of mt19937


@pytest.mark.parametrize("seed", [0, 1, 5489, 2 ** 32 - 1])
def test_stream_matches_python_mt19937(seed):
    assert mo.mt19937_outputs(seed, 1000).tolist() == _mt19937_python(seed, 1000)


def test_stream_skip_and_object():
    from gs2mesh_b200.mobilebrick import Mt19937Stream

    s = Mt19937Stream(3)
    a = s.uniform(5)
    b = s.uniform(7)
    assert s.drawn == 24
    np.testing.assert_array_equal(np.concatenate([a, b]), mo.canonical(mo.mt19937_outputs(3, 24)))
    o = mo.Stream(3)
    np.testing.assert_array_equal(np.concatenate([o.uniform(5), o.uniform(7)]), np.concatenate([a, b]))


def test_canonical_matches_fraction():
    rng = np.random.default_rng(0)
    u = np.concatenate([rng.integers(0, 2 ** 32, (2000, 2), dtype=np.uint64),
                        np.array([[0, 0], [2 ** 32 - 1, 2 ** 32 - 1], [2 ** 32 - 1, 0], [0, 2 ** 32 - 1], [1, 0]],
                                 np.uint64)])
    got = mo.canonical(u.reshape(-1))
    for (u0, u1), g in zip(u.tolist(), got.tolist()):
        s = float(Fraction(u0) + Fraction(u1) * 2 ** 32)  # the double sum, correctly rounded once
        r = float(Fraction(s) / 2 ** 64)  # an exact power-of-two scaling
        if r >= 1.0:
            r = float(np.nextafter(1.0, 0.0))
        assert g == r
    assert got[-4] == np.nextafter(1.0, 0.0)  # (2^32-1)(1 + 2^32) rounds to 2^64: clamped below 1


# ------------------------------------------------------------------------------------------------------ elimination
CLOUDS = mc.elimination_clouds()


@pytest.mark.parametrize("chunk", range(4))
def test_rounds_keep_the_heap_set(chunk):
    """The round-based restatement (DESIGN section 7e) keeps exactly the set Open3D's heap loop keeps, and every removal
    key it gives equals the heap's key for the points the heap deletes."""
    names = sorted(CLOUDS)[chunk::4]
    for name in names:
        p, N, r_max, r_min = CLOUDS[name]
        nbr, d2 = mo.neighbour_lists(p, r_max)
        term = mo.weight_term(d2, r_min, r_max)
        kept_h, key_h, order = mo.eliminate_heap(nbr, term, N)
        kept_r, key_r, rnd, rounds = mo.eliminate_rounds(nbr, term, N)
        assert np.array_equal(kept_h, kept_r), name
        gone = np.asarray(order, np.int64)
        assert np.array_equal(key_h[gone], key_r[gone]), name
        # the heap's removal keys strictly decrease
        k = list(zip(key_h[gone].tolist(), gone.tolist()))
        assert all(a > b for a, b in zip(k, k[1:])), name
        assert len(kept_r) == min(N, len(p)) and rounds >= 1


def test_elimination_clouds_reach_their_edges():
    assert len([k for k in CLOUDS if k.startswith("random_")]) >= 200
    p, N, r_max, r_min = CLOUDS["at_r_max"]
    nbr, d2 = mo.neighbour_lists(p, r_max)
    d = p[:, None, :] - p[None, :, :]
    full = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
    assert (full == r_max * r_max).sum() > 0 and not (d2[nbr >= 0] >= r_max * r_max).any()  # at r_max: excluded
    p, N, r_max, r_min = CLOUDS["r_min_clamp"]
    nbr, d2 = mo.neighbour_lists(p, r_max)
    assert (np.sqrt(d2[nbr >= 0]) < r_min).all()
    p, N, r_max, r_min = CLOUDS["isolated"]
    nbr, d2 = mo.neighbour_lists(p, r_max)
    assert ((nbr >= 0).sum(1) == 0).sum() == 10
    dup = [k for k in CLOUDS if k.startswith("random_") and int(k[-3:]) % 5 == 3]
    assert any((mo.neighbour_lists(CLOUDS[k][0], CLOUDS[k][2])[1][mo.neighbour_lists(CLOUDS[k][0], CLOUDS[k][2])[0] >= 0]
                == 0).any() for k in dup)
    p, N, r_max, r_min = CLOUDS["gradient_chain"]
    nbr, d2 = mo.neighbour_lists(p, r_max)
    assert mo.eliminate_rounds(nbr, mo.weight_term(d2, r_min, r_max), N)[3] > 50  # many rounds


# ------------------------------------------------------------------------------------------------- uniform sampling
def test_uniform_counts_on_half_and_zero_area():
    v, t = mc.half_round_mesh()
    areas = mo.triangle_areas(v, t)
    assert areas[2] == 0.0
    S = mo.surface_area(areas)
    b = mo.sample_bounds(areas, S, 10)
    np.testing.assert_array_equal(np.diff(b), [3, 2, 0, 3, 2])  # 2.5 -> 3 and 7.5 -> 8 (half away from zero)
    pts, _, _ = mo.sample_uniform(v, t, 10, mo.Stream(0).uniform(20))
    assert pts.shape == (10, 3) and np.isfinite(pts).all()


def test_uniform_errors():
    with pytest.raises(ValueError, match="Input mesh has no triangles."):
        mo.sample_uniform(np.zeros((3, 3)), np.zeros((0, 3), np.int64), 5, np.zeros(10))
    with pytest.raises(ValueError, match="Invalid surface area"):
        mo.sample_uniform(np.zeros((3, 3)), np.array([[0, 1, 2]]), 5, np.zeros(10))


# ------------------------------------------------------------------------------------------------------- the pipeline
def test_scan_builder_reaches_the_gpu_cases(tmp_path):
    gt_dir, pred, exp, info = mc.write_scan(str(tmp_path))
    gv, gt, pv, pt, pc, m = mc.load_scan(gt_dir, pred)
    assert pc is not None and np.array_equal(np.rint(pc * 255), np.rint(info["colors"] * 255))
    out, (v, t, c, n), fitness = mo.evaluate_single(gv, gt, pv, pt, m, seed=0, number_of_points=500, pred_colors=pc)
    assert fitness > 0.99  # the transform branch
    assert 0 < len(v) < len(pv) and 0 < len(t) < len(pt)  # the crop removes vertices and triangles, some remain
    used = np.zeros(len(v), bool)
    used[t.reshape(-1)] = True
    assert not used.all()  # unreferenced vertices stay
    assert c is not None and len(c) == len(v) and len(out) == 7 and all(np.isfinite(out))


def test_fallback_without_triangles(tmp_path):
    gt_dir, pred, exp, _ = mc.write_scan(str(tmp_path), nx=6, ny=6, no_triangles=True)
    gv, gt, pv, pt, pc, m = mc.load_scan(gt_dir, pred)
    out, (v, t, c, n), _ = mo.evaluate_single(gv, gt, pv, pt, m, seed=3, number_of_points=500, pred_colors=pc)
    assert len(t) == 0 and len(v) > 0
    assert (n == 0).all()  # no triangle: zero normals
    assert len(out) == 7


def test_doubt_sensitivity():
    """The DOUBT points of DESIGN section 7e quantified on a 500 000-sample mesh (100 000 kept): std::pow instead of the
    squarings, and a shuffled order inside equal-distance runs of the neighbour lists.  Reports how many kept points
    change."""
    v, t = mc.grid_mesh(300, 300, seed=5)
    N = 100000
    pts, _, S = mo.sample_uniform(v, t, 5 * N, mo.Stream(0).uniform(10 * N))
    r_max, r_min = mo.poisson_radii(S, N, 5 * N)
    nbr, d2 = mo.neighbour_lists(pts, r_max)
    base = mo.eliminate_rounds(nbr, mo.weight_term(d2, r_min, r_max), N)
    powk = mo.eliminate_rounds(nbr, mo.weight_term(d2, r_min, r_max, exact_pow=True), N)
    nbr_s, d2_s = mo.neighbour_lists(pts, r_max, tie_shuffle_seed=1)
    tie = mo.eliminate_rounds(nbr_s, mo.weight_term(d2_s, r_min, r_max), N)
    ch_pow = len(np.setdiff1d(base[0], powk[0]))
    ch_tie = len(np.setdiff1d(base[0], tie[0]))
    print(f"\nDOUBT sensitivity (500000 samples, 100000 kept): std::pow changes {ch_pow} kept points, tie order "
          f"{ch_tie}; rounds {base[3]}, neighbours per point {float((nbr >= 0).sum(1).mean()):.1f}")
    assert ch_pow <= N // 100 and ch_tie <= N // 100
