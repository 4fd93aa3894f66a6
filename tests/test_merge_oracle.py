"""The host restatement of the multi-GPU merge (tests/merge_oracle.py) on hand-made cases, without a GPU: the signs of
zero sums, the 3-rank candidate set, the colour rules and the drop counts."""
import numpy as np

from tests.merge_oracle import _rn32_exact, candidates, check_rank, merge_oracle

F32 = np.float32


def _unit(t, w, col=None):
    tw = np.zeros((4096, 2), F32)
    tw[:, 0], tw[:, 1] = t, w
    c = None
    if col is not None:
        c = np.zeros((4096, 4), F32)
        c[:] = col
        c[tw[:, 1] == 0] = 0
    return tw, c


def test_negative_zero_tsdf_held_by_one_rank_becomes_positive():
    """-0 * w travels as -0; the other rank's zero payload is +0, and -0 + +0 = +0 (the GPU's add, not Python's 0 + ...)."""
    k = (0, 0, 0)
    out = merge_oracle([{k: _unit(-0.0, 3)}, {}], None, 4)
    tw = out[0].merged[k][0][0]
    assert not np.signbit(tw[:, 0]).any() and (tw[:, 1] == 3).all()
    both = merge_oracle([{k: _unit(-0.0, 3)}, {k: _unit(-0.0, 1)}], None, 4)[1].merged[k][0][0]
    assert np.signbit(both[:, 0]).all() and (both[:, 1] == 4).all()


def test_colour_rules():
    """Colour sums only where w != 0, the fourth channel summed as it is, colour 0 where the summed weight is 0."""
    k = (1, 2, 3)
    a = _unit(0.5, 2, (10.0, 20.0, 30.0, 0.25))
    b = _unit(-0.5, 0, (0, 0, 0, 0))
    tw, col = merge_oracle([{k: a}, {k: b}], 0, 4)[0].merged[k]
    assert (tw[0][:, 0] == F32(0.5)).all() and (col[0][:, :3] == F32([10, 20, 30])).all() and (col[0][:, 3] == F32(0.25)).all()
    tw, col = merge_oracle([{k: _unit(0, 0, (0, 0, 0, 0))}, {}], 0, 4)[0].merged[k]
    assert (tw == 0).all() and not np.signbit(tw).any() and (col == 0).all()


def test_three_rank_candidates_cover_every_order_and_one_rounding():
    rng = np.random.default_rng(0)
    a, b, c = (rng.uniform(-1, 1, 10000).astype(F32) * F32(2.0) ** rng.integers(-140, 30, 10000).astype(F32) for _ in range(3))
    cand = candidates([a, b, c])
    for s in ((a + b) + c, (a + c) + b, (b + c) + a):
        assert (cand == s[None]).any(0).all()
    exact = _rn32_exact((a, b, c))
    from fractions import Fraction

    for i in range(0, 10000, 97):  # spot checks against exact rationals
        e = Fraction(float(a[i])) + Fraction(float(b[i])) + Fraction(float(c[i]))
        g = exact[i]
        for n in (np.nextafter(g, F32(-np.inf)), np.nextafter(g, F32(np.inf))):
            assert abs(Fraction(float(g)) - e) <= abs(Fraction(float(n)) - e)


def test_drop_counts_and_check_rank():
    """2 ranks: drops = keys named but dead here + lacking keys beyond the free slots; the rank must open exactly the free
    slots' worth, and a brick outside the canonical order keeps its own bits."""
    own = {(i, 0, 0): _unit(0.25, 1) for i in (0, 1, 2)}
    other = {(i, 0, 0): _unit(0.5, 1) for i in (1, 3, 4, 5)}
    exp = merge_oracle([own, other], None, 4, dead=[{(5, 0, 0)}, set()])
    e0, e1 = exp[0], exp[1]
    assert e0.lacking == [(3, 0, 0), (4, 0, 0)] and e0.opened == 1 and e0.drops == (2, 2)
    assert e1.lacking == [(0, 0, 0), (2, 0, 0)] and e1.opened == 0 and e1.drops == (2, 2)
    got = {k: (e0.merged[k][0][0], None) for k in [*own, (3, 0, 0)]}
    check_rank(e0, got, 2, set(got))
    for bad in (dict(drops=1), dict(extra=(4, 0, 0))):
        g = dict(got)
        if "extra" in bad:
            g[bad["extra"]] = e0.merged[bad["extra"]][0][0], None
        try:
            check_rank(e0, g, bad.get("drops", 2), set(g))
        except AssertionError:
            continue
        raise AssertionError(f"{bad} passed")
    # bricks the canonical rank did not store keep rank 1's own bits
    got1 = {k: (e1.merged[k][0][0], None) if k in got else other[k] for k in other}
    check_rank(e1, got1, 2, set(got))
