"""The mesh-quality oracle (oracle/eval_oracle.py) against the reference's own formulation: the literal per-triangle
np.mgrid sampler of eval.py, hand-computed sample counts, and sklearn's kd_tree for distances and radius neighbours."""
import numpy as np
import pytest

from oracle import eval_oracle as eo


def _sample_literal(vertices, triangles, thresh):
    """eval.py:48-71 as written there: one np.mgrid per triangle."""
    tri_vert = vertices[triangles]
    v1 = tri_vert[:, 1] - tri_vert[:, 0]
    v2 = tri_vert[:, 2] - tri_vert[:, 0]
    l1 = np.linalg.norm(v1, axis=-1, keepdims=True)
    l2 = np.linalg.norm(v2, axis=-1, keepdims=True)
    area2 = np.linalg.norm(np.cross(v1, v2), axis=-1, keepdims=True)
    nz = (area2 > 0)[:, 0]
    l1, l2, area2, v1, v2, tri_vert = [arr[nz] for arr in [l1, l2, area2, v1, v2, tri_vert]]
    thr = thresh * np.sqrt(l1 * l2 / area2)
    n1 = np.floor(l1 / thr)
    n2 = np.floor(l2 / thr)
    pts = []
    for i in range(len(n1)):
        c = np.mgrid[:n1[i, 0] + 1, :n2[i, 0] + 1]
        c += 0.5
        c[0] /= max(n1[i, 0], 1e-7)
        c[1] /= max(n2[i, 0], 1e-7)
        c = np.transpose(c, (1, 2, 0))
        k = c[c.sum(axis=-1) < 1]
        pts.append(v1[i:i + 1] * k[:, :1] + v2[i:i + 1] * k[:, 1:] + tri_vert[i:i + 1, 0])
    return np.concatenate([vertices] + pts, axis=0)


def _random_mesh(seed, nv=300, nt=500):
    rng = np.random.default_rng(seed)
    v = rng.uniform(-3, 3, size=(nv, 3))
    t = rng.integers(0, nv, size=(nt, 3))
    t[:10, 2] = t[:10, 1]  # zero-area triangles
    return v, t


@pytest.mark.parametrize("thresh", [0.2, 0.5, 1.3])
def test_sampling_equals_literal_mgrid_loop(thresh):
    v, t = _random_mesh(int(thresh * 10))
    got = eo.sample_mesh(v, t, thresh)
    ref = _sample_literal(v, t, thresh)
    assert got.shape == ref.shape and got.shape[0] > len(v)
    assert np.array_equal(got.view(np.uint64), ref.view(np.uint64))


def test_sampling_known_counts():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0],          # right triangle
                  [0.1, 0, 0], [0, 10, 0],                   # with vertex 0: l1 < thr, n1 = 0
                  [10, 0, 0], [10, 0.01, 0],                 # sliver
                  [2, 0, 0]], dtype=np.float64)              # collinear with 0 and 1: zero area
    t = np.array([[0, 1, 2], [0, 3, 4], [0, 5, 6], [0, 1, 7]])
    # right triangle, thresh 0.25: thr = 0.25, n1 = n2 = 4, k = (i+.5)/4 is exact -> i + j <= 2: 6 points
    # n1 = 0: k0 = 0.5/1e-7 -> no point; sliver: n1 = n2 = 1, k0 + k1 = 1 at best -> no point; zero area: dropped
    assert eo.sample_counts(v, t, 0.25).tolist() == [6, 0, 0, 0]
    pts = eo.sample_mesh(v, t[:1], 0.25)[len(v):]
    assert np.array_equal(pts[:, :2], np.array([[.125, .125], [.125, .375], [.125, .625], [.375, .125], [.375, .375],
                                                [.625, .125]]))


def test_nearest_equals_sklearn_kd_tree():
    skln = pytest.importorskip("sklearn.neighbors")
    rng = np.random.default_rng(3)
    ref = rng.uniform(-1, 1, size=(20000, 3))
    q = np.concatenate([rng.uniform(-1.2, 1.2, size=(5000, 3)), ref[:100]])  # exact hits included
    dist, idx = eo.nearest(q, ref)
    nn = skln.NearestNeighbors(n_neighbors=1, algorithm="kd_tree").fit(ref)
    sd, si = nn.kneighbors(q, n_neighbors=1, return_distance=True)
    assert np.array_equal(dist.view(np.uint64), sd[:, 0].view(np.uint64))
    same = idx == si[:, 0]
    assert np.array_equal(dist[~same], eo.distance(q[~same], ref[si[~same, 0]]))  # an index differs only on a tie


def test_radius_downsample_equals_sklearn_loop():
    """Pins the neighbour rule: sklearn's radius_neighbors(return_distance=False) is inclusive on the reduced distance."""
    skln = pytest.importorskip("sklearn.neighbors")
    rng = np.random.default_rng(5)
    thresh = 0.2
    p = rng.uniform(0, 3, size=(3000, 3))
    p = np.concatenate([p, p[:200]])  # duplicates
    axis = np.zeros((300, 3))
    axis[np.arange(300), rng.integers(0, 3, 300)] = thresh * rng.choice([-1.0, 1.0], 300)
    p = np.concatenate([p, p[200:500] + axis])  # points at exactly thresh along an axis (as far as the sum rounds)
    p = p[rng.permutation(len(p))]
    nn = skln.NearestNeighbors(n_neighbors=1, radius=thresh, algorithm="kd_tree").fit(p)
    rnn = nn.radius_neighbors(p, radius=thresh, return_distance=False)
    mask = np.ones(len(p), dtype=np.bool_)
    for curr, idxs in enumerate(rnn):
        if mask[curr]:
            mask[idxs] = 0
            mask[curr] = 1
    got = eo.radius_downsample(p, thresh)
    assert np.array_equal(got, mask)
    assert 0 < got.sum() < len(p)


def test_precision_recall_f1_keys_and_values():
    rng = np.random.default_rng(7)
    a = rng.uniform(0, 1, size=(2000, 3))
    b = a + rng.normal(scale=0.01, size=a.shape)
    out = eo.precision_recall_f1(a, b, 0.02)
    assert set(out) == {"pred_gt", "accuracy", "gt_pred", "recall", "chamfer", "F1"}
    assert 0 < out["accuracy"] <= 1 and 0 < out["recall"] <= 1
    assert out["chamfer"] == out["pred_gt"] + out["gt_pred"]


def test_radius_rule_on_pairs_that_separate_the_two_rules():
    """Pairs whose squared distance rounds above fl(r*r) while its root rounds to r: `sum <= r*r` excludes them,
    `sqrt(sum) <= r` includes them.  sklearn's radius_neighbors (return_distance=False) and the oracle must exclude them."""
    skln = pytest.importorskip("sklearn.neighbors")
    r = 0.35
    rng = np.random.default_rng(0)
    g = np.arange(16) * 2.0 + 1.0
    a = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)  # pair k = (a_k, a_k + d_k), 2 apart
    d = rng.normal(size=a.shape)
    d = d / np.linalg.norm(d, axis=1, keepdims=True) * r
    b = a + d
    dd = b - a
    s = (dd[:, 0] * dd[:, 0] + dd[:, 1] * dd[:, 1]) + dd[:, 2] * dd[:, 2]
    sep = np.nonzero((s > r * r) & (np.sqrt(s) <= r))[0][:40]
    inc = np.nonzero(s <= r * r)[0][:40]
    assert len(sep) >= 10 and len(inc) == 40
    k = np.concatenate([sep, inc])
    p = np.empty((2 * len(k), 3))
    p[0::2], p[1::2] = a[k], b[k]
    dd = p[1::2] - p[0::2]
    s = (dd[:, 0] * dd[:, 0] + dd[:, 1] * dd[:, 1]) + dd[:, 2] * dd[:, 2]
    sq_rule, sqrt_rule = s <= r * r, np.sqrt(s) <= r
    assert (sq_rule != sqrt_rule).sum() == len(sep)  # the cloud does separate the two rules
    nn = skln.NearestNeighbors(n_neighbors=1, radius=r, algorithm="kd_tree").fit(p)
    rnn = nn.radius_neighbors(p[0::2], radius=r, return_distance=False)
    sk_pair = np.array([2 * k + 1 in set(ix.tolist()) for k, ix in enumerate(rnn)])
    assert np.array_equal(sk_pair, sq_rule)
    assert np.array_equal(eo.radius_downsample(p, r)[1::2], ~sq_rule)
