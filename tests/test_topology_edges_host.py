"""The restatement's narrow phase (tests/topology_oracle.py) against the exact integer intersection of
tests/topology_edge_cases.py on lattice soups and crafted branch families, its coplanar projection on normals that tie,
its epsilon clamp, and the grid cases' stated levels and registrations against the numpy port of the grid rule."""
import numpy as np
import pytest

from tests import topology_edge_cases as ec
from tests import topology_oracle as to


def _classes(P, Q):
    """(robust class, exact verdict, restatement verdict) per pair."""
    return ec.robust_class(P, Q), ec.exact_tri_tri(P, Q), to.tri_tri(np.asarray(P, np.float64), np.asarray(Q, np.float64))


def test_exact_tri_tri_known_answers():
    floor = np.array([[0, 0, 0], [4, 0, 0], [0, 4, 0]])
    cases = [
        ([[1, 1, 0], [2, 1, 3], [1, 2, 3]], True, ec.CONTACT),     # corner on the face
        ([[1, 1, -1], [2, 1, 3], [1, 2, 3]], True, ec.CROSSING),
        ([[1, 1, 1], [2, 1, 3], [1, 2, 3]], False, ec.SEPARATED),
        ([[4, 4, 0], [8, 4, 0], [4, 8, 0]], False, ec.SEPARATED),  # coplanar, apart
        ([[2, 2, 0], [6, 2, 0], [2, 6, 0]], True, ec.CONTACT),     # coplanar, corner on the long edge
        ([[1, 1, 0], [3, 1, 0], [1, 3, 0]], True, ec.CROSSING),    # coplanar, overlapping
        ([[0, 0, 0], [4, 0, 0], [0, 4, 0]], True, ec.CROSSING),    # the same triangle
        ([[-1, 2, 0], [5, 2, 0], [2, 2, 5]], True, ec.CONTACT),    # an edge in the plane across the face
        ([[5, 0, 0], [6, 0, 0], [5, 0, 3]], False, ec.SEPARATED),  # an edge on the line of an edge, past its end
        ([[4, 0, 0], [6, 0, 0], [5, 0, 3]], True, ec.CONTACT),     # ... touching its end
    ]
    P = np.repeat(floor[None], len(cases), axis=0)
    Q = np.array([c[0] for c in cases])
    assert ec.exact_tri_tri(P, Q).tolist() == [c[1] for c in cases]
    assert ec.exact_tri_tri(Q, P).tolist() == [c[1] for c in cases]
    assert ec.robust_class(P, Q).tolist() == [c[2] for c in cases]


@pytest.mark.parametrize("seed", range(2))
def test_lattice_soups_equal_the_exact_intersection(seed, capsys):
    """Every separated and crossing pair of a lattice soup: the restatement's pair list equals the exact verdict."""
    T = ec.lattice_soup(seed)
    i, j = ec.box_pairs(T)
    cls = ec.robust_class(T[i], T[j])
    exact = ec.exact_tri_tri(T[i], T[j])
    got = ec.pair_flags(to.self_intersecting_triangles(*ec.soup_mesh(T)), i, j, len(T))
    counts = np.bincount(cls, minlength=3)
    with capsys.disabled():
        print(f"\nlattice soup {seed}: separated {counts[0]}, crossing {counts[1]}, contact {counts[2]} "
              f"(restatement true on {got[cls == ec.CONTACT].sum()} contacts)")
    assert counts.min() >= 1000
    robust = cls != ec.CONTACT
    assert (got[robust] == exact[robust]).all()
    assert (exact[cls == ec.CROSSING]).all() and not exact[cls == ec.SEPARATED].any()


@pytest.mark.parametrize("name", sorted(ec.FAMILIES))
def test_branch_families(name):
    """Each family as built is a contact; pushed in it crosses (or, beside P, touches) and pushed apart it is
    separated; the restatement equals the exact verdict on every robust pair."""
    P, Q = ec.branch_family_pairs()[name]
    cls, exact, got = _classes(P, Q)
    k = len(P) // 3
    built, pushed_in, pushed_apart = cls[:k], cls[k:2 * k], cls[2 * k:]
    if name == "edge_in_plane_beside":
        assert (built == ec.SEPARATED).all() and (pushed_in == ec.CONTACT).all()
    else:
        assert (built == ec.CONTACT).all() and (pushed_in == ec.CROSSING).all()
    assert (pushed_apart == ec.SEPARATED).all()
    robust = cls != ec.CONTACT
    assert (got[robust] == exact[robust]).all()


def test_tie_families_hit_the_tie_branches(monkeypatch):
    """Coplanar pairs in planes whose normalised normals tie: the ties hold in the restatement's arithmetic, every
    pair reaches the coplanar test with the tie, Moeller's rule picks the projection of TIE_AXES, and the verdict equals
    the exact one on every robust pair."""
    seen = []
    monkeypatch.setattr(to, "coplanar_axes_hook", lambda A, i0, i1: seen.append((A.copy(), i0.copy(), i1.copy())))
    hits = {}
    for (tie, name), (P, Q) in ec.tie_family_pairs().items():
        assert ec.ties(P, Q, tie).all()
        seen.clear()
        cls, exact, got = _classes(P, Q)
        robust = cls != ec.CONTACT
        assert (got[robust] == exact[robust]).all(), (tie, name)
        A = np.concatenate([s[0] for s in seen])
        axes = np.stack([np.concatenate([s[1] for s in seen]), np.concatenate([s[2] for s in seen])], axis=1)
        nz = [k for k in range(3) if tie[k]]
        tied = (A[:, nz] == A[:, nz[:1]]).all(axis=1) & (A.max(axis=1) == A[:, nz[0]])
        assert len(A) == len(P) and tied.all(), (tie, name)  # every pair is coplanar and tied
        assert (axes == ec.TIE_AXES[tie]).all(), (tie, name)
        hits[tie] = hits.get(tie, 0) + len(A)
        if name != "cyclic":
            assert set(cls.tolist()) >= ({ec.CROSSING} if name in ("overlap", "q_in_p", "p_in_q") else {ec.SEPARATED})
    print("tie branch hits:", hits)
    assert set(hits) == set(ec.TIE_AXES) and min(hits.values()) >= 100


def test_epsilon_pairs_flip_at_the_clamp():
    """A corner 0.9e-6 from the other plane (normalised) is clamped onto it and the pair touches; at 1.1e-6 the pair is
    rejected.  Both signs."""
    rows = ec.epsilon_pairs()
    got = [bool(to.tri_tri(P[None], Q[None])[0]) for P, Q, _ in rows]
    dists = [d for _, _, d in rows]
    assert [abs(d) < 1e-6 for d in dists] == [True, False, True, False]
    assert got == [True, False, True, False]
    # through the mesh path: the boxes overlap, so the pair reaches the narrow phase
    assert [len(to.self_intersecting_triangles(*ec.soup_mesh(np.stack([P, Q])))) for P, Q, _ in rows] == [1, 0, 1, 0]


@pytest.mark.parametrize("L", [0, 1, 5, 10, 15, 19, 20, 21])
def test_level_cases_reach_their_level(L):
    T, level, regs, crossing = ec.level_case(L)
    v, t = ec.soup_mesh(T)
    assert ec.grid_level(v, t) == (level, regs)
    o, e = ec.grid_extent(v, t)
    assert o.tolist() == [0, 0, 0] and e == 1.0
    assert ec.cell_of(1.0, 0.0, 1.0, L) == 2 ** (20 - L) if L < 21 else ec.cell_of(1.0, 0.0, 1.0, L) == 0
    pairs = {tuple(p) for p in to.self_intersecting_triangles(v, t).tolist()}
    assert set(crossing) <= pairs


@pytest.mark.parametrize("over", [False, True])
def test_threshold_case(over):
    T, level, regs = ec.threshold_case(over=over)
    v, t = ec.soup_mesh(T)
    assert ec.grid_level(v, t) == (level, regs)
    o, e = ec.grid_extent(v, t)
    p = v[t]
    lo, hi = p.min(axis=1), p.max(axis=1)
    at_L = np.prod(ec.cell_of(hi, o, e, 10) - ec.cell_of(lo, o, e, 10) + 1, axis=1).sum()
    assert at_L == 4 * len(T) + over


def test_boundary_and_flat_cases():
    T, level, regs = ec.boundary_case()
    v, t = ec.soup_mesh(T)
    assert ec.grid_level(v, t) == (level, regs)
    o, e = ec.grid_extent(v, t)
    assert o.tolist() == [0, 0, 0] and e == 8.0
    cell = 2.0 ** (level - 20) * e
    assert (np.mod(T, cell) == 0).all()  # every corner, so every box face and intersection corner, on a cell face
    for axes in (1, 2, 3):
        T, level, regs = ec.flat_case(axes)
        assert ec.grid_level(*ec.soup_mesh(T)) == (level, regs), axes
    assert ec.grid_extent(*ec.soup_mesh(ec.flat_case(3)[0]))[1] == 1.0
