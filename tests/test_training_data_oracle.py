"""CPU: the training-pair contract (oracle/pairs_np.py) against the reference's own tools, at the strict radius
boundary, for the sampler and the rotation; and the argument checks of d3feat_b200/training_data.py, which refuse bad
arguments before anything reaches the library (a stub whose every symbol raises)."""
import numpy as np
import pytest
import torch

from oracle import pairs_np as op


def _rng_pose(rng):
    from scipy.spatial.transform import Rotation
    T = np.eye(4)
    T[:3, :3] = Rotation.random(random_state=rng.integers(1 << 31)).as_matrix()
    T[:3, 3] = rng.normal(size=3) * 0.3
    return T


def _clouds(rng, na=700, nb=600):
    a = (rng.random((na, 3)) * 2.0).astype(np.float32)
    b = (rng.random((nb, 3)) * 2.0).astype(np.float32)
    return np.concatenate([a, b]), [na, nb]


def test_radius_mode_is_query_ball_point():
    from scipy.spatial import cKDTree
    rng = np.random.default_rng(0)
    pts, lens = _clouds(rng)
    T = _rng_pose(rng)
    tau = 0.08
    got = op.correspondences(pts, lens, [[0, 1]], T[None], tau, "radius", exhaustive=True)
    a = pts[:lens[0]].astype(np.float64)
    q = a @ T[:3, :3].T + T[:3, 3]
    lists = cKDTree(pts[lens[0]:].astype(np.float64)).query_ball_point(q, tau)
    ref = [(i, j) for i, l in enumerate(lists) for j in sorted(l)]
    assert [tuple(r) for r in got["rows"]] == ref
    assert got["count"][0] == len(ref) and got["overlap"][0] == len(ref) / lens[0]


def test_nearest_mode_is_bfmatcher_below_tau():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(1)
    pts, lens = _clouds(rng, 800, 900)
    T = _rng_pose(rng)
    tau = 0.05
    got = op.correspondences(pts, lens, [[0, 1]], T[None], tau, "nearest", exhaustive=True)
    a = pts[:lens[0]].astype(np.float64)
    q = (a @ T[:3, :3].T + T[:3, 3]).astype(np.float32)
    m = cv2.BFMatcher(cv2.NORM_L2).match(q, pts[lens[0]:])
    ref = sorted((x.queryIdx, x.trainIdx) for x in m if x.distance < tau)
    assert [tuple(r) for r in got["rows"]] == ref
    np.testing.assert_equal(got["overlap"], [len(ref) / lens[0]])


def test_tree_candidates_equal_the_exhaustive_search():
    rng = np.random.default_rng(2)
    pts, lens = _clouds(rng)
    T = np.stack([_rng_pose(rng), np.eye(4)])
    for mode in op.MODES:
        e = op.correspondences(pts, lens, [[0, 1], [1, 0]], T, 0.07, mode, exhaustive=True)
        t = op.correspondences(pts, lens, [[0, 1], [1, 0]], T, 0.07, mode, exhaustive=False)
        for key in e:
            np.testing.assert_array_equal(e[key], t[key])


def test_strict_boundary_on_a_lattice_and_one_ulp_either_side():
    """d^2 equal to tau^2 exactly is dropped; 1 ulp inside is kept, 1 ulp outside dropped. A non-strict test or an fp32
    distance would decide differently."""
    g = np.arange(4, dtype=np.float32) * 0.25
    lat = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    pts = np.concatenate([lat, lat])
    n = len(lat)
    got = op.correspondences(pts, [n, n], [[0, 1]], np.eye(4)[None], 0.25, "radius", exhaustive=True)
    d2 = ((lat[:, None, :].astype(np.float64) - lat[None]) ** 2).sum(-1)
    assert len(got["rows"]) == int((d2 < 0.0625).sum()) == n          # only the point itself: neighbours sit at tau
    assert int((d2 <= 0.0625).sum()) > n                                # a non-strict test would keep them
    y = np.float32(0.3)                 # d^2 = y^2 is exact in fp64
    pair = np.array([[0, 0, 0], [y, 0, 0]], np.float32)

    def kept(tau):
        r = op.correspondences(pair, [1, 1], [[0, 1]], np.eye(4)[None], tau, "radius", exhaustive=True)
        return len(r["rows"]) == 1
    up, down = np.nextafter(float(y), 1.0), np.nextafter(float(y), 0.0)
    assert not kept(float(y)) and kept(up) and not kept(down)
    # tau 1 fp64 ulp above y rounds to y in fp32: an fp32 test would drop the row the contract keeps
    assert np.float32(up) == y and not np.float32(y) * np.float32(y) < np.float32(up) * np.float32(up)


def test_nonfinite_and_out_of_range_pairs_match_nothing():
    pts = np.array([[np.nan, 0, 0], [0, 0, 0], [0, 0, 0]], np.float32)
    r = op.correspondences(pts, [2, 1], [[0, 1], [0, 5], [-1, 0]], np.eye(4)[None].repeat(3, 0), 0.1, "radius")
    assert [tuple(x) for x in r["rows"]] == [(1, 0)]
    np.testing.assert_array_equal(r["count"], [1, 0, 0])


def _table(counts):
    off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    rows = np.stack([np.arange(off[-1]), np.arange(off[-1]) + 7], 1).astype(np.int32)
    return off, rows


def test_sampler_without_replacement_and_validity():
    off, rows = _table([0, 5, 40, 2000, 30])
    anc, pos, valid = op.sample(off, rows, [100] * 5, 32, False, 32, seed=9)
    np.testing.assert_array_equal(valid, [False, False, True, True, False])   # n = 0, n < k, ok, ok, n < min_count
    for p in range(5):
        if valid[p]:
            assert len(set(anc[p].tolist())) == 32
            assert ((anc[p] >= off[p]) & (anc[p] < off[p + 1])).all()
            np.testing.assert_array_equal(pos[p], anc[p] + 7 + 100)
        else:
            assert (anc[p] == -1).all() and (pos[p] == -1).all()
    _, _, v = op.sample(off, rows, [0] * 5, 32, False, 1000, seed=9)
    np.testing.assert_array_equal(v, [False, False, False, True, False])
    # the without-replacement order is by (key, candidate): a random order, not ascending
    assert not (np.diff(anc[3]) > 0).all()


def test_sampler_with_replacement_is_roughly_uniform():
    off, rows = _table([10])
    hits = np.zeros(10)
    for seed in range(200):
        anc, _, valid = op.sample(off, rows, [0], 50, True, 0, seed)
        assert valid[0]
        hits += np.bincount(anc[0], minlength=10)
    expect = 200 * 50 / 10
    assert np.abs(hits - expect).max() < 5 * np.sqrt(expect)
    _, _, v = op.sample(*_table([0]), [0], 4, True, 0, 1)
    assert not v[0]


def test_counters_are_distinct_across_slots_and_pairs():
    z = [op.draw(3, p, i, s) for p in range(3) for i in range(4) for s in range(15)]
    assert len(set(int(x) for x in z)) == len(z)


@pytest.mark.parametrize("axis", [0, 1, 2])
def test_rotation_restates_rotate_and_is_proper(axis):
    for theta in np.linspace(0, 2 * np.pi, 17):
        R = op.rotation(theta, axis)
        c, s = np.float32(np.cos(theta)), np.float32(np.sin(theta))
        full = np.array([[c, -s, -s], [s, c, -s], [s, s, c]], np.float32)
        keep = [i for i in range(3) if i != axis]
        np.testing.assert_array_equal(R[np.ix_(keep, keep)], full[np.ix_(keep, keep)])
        assert R[axis, axis] == 1 and (R[axis, keep] == 0).all() and (R[keep, axis] == 0).all()
        R64 = R.astype(np.float64)
        assert np.abs(R64 @ R64.T - np.eye(3)).max() < 1e-6
        assert abs(np.linalg.det(R64) - 1) < 1e-6


def test_augmentation_draws():
    pts = np.random.default_rng(0).random((30, 3)).astype(np.float32)
    a = op.augment(pts, [10, 20], [[0, 1]], np.eye(4)[None], 5, 0.01, 1, (0.8, 1.2), 2.0)
    assert 0.8 <= a["scale"][0] < 1.2 and (np.abs(a["shift"]) <= 2).all()
    np.testing.assert_array_equal(a["lengths"], [[10, 20]])
    np.testing.assert_array_equal(a["backup_points"], pts)
    noise = a["points"] - pts          # not the same chain, but every point moves
    assert (np.abs(noise).sum(1) > 0).all()
    b = op.augment(pts, [10, 20], [[0, 1]], np.eye(4)[None], 5, 0.0, 3)
    for side in range(2):
        for r in range(3):
            assert b["R"][side, r][r, r] == 1
    np.testing.assert_array_equal(b["scale"], [1.0])
    np.testing.assert_array_equal(b["shift"], np.zeros((2, 3)))


# ---------------------------------------------------------------------------------------------------- arguments

class _Stub:
    def __getattr__(self, name):
        raise AssertionError("%s reached the library" % name)


@pytest.fixture
def stub(monkeypatch):
    from d3feat_b200 import _lib
    monkeypatch.setattr(_lib, "_lib", _Stub())
    monkeypatch.setattr(_lib, "DEVICE_TYPE", "cpu")


def _good():
    return dict(points=torch.zeros((8, 3)), lengths=torch.tensor([4, 4], dtype=torch.int32),
                pairs=torch.tensor([[0, 1]], dtype=torch.int32), trans=torch.eye(4, dtype=torch.float64)[None])


BAD = [("points", torch.zeros((8, 3), dtype=torch.float64)), ("points", torch.zeros((8, 4))),
       ("points", torch.zeros((8, 3), device="meta")), ("lengths", torch.tensor([4, 4])),
       ("pairs", torch.tensor([[0, 1]])), ("pairs", torch.zeros((1, 3), dtype=torch.int32)),
       ("trans", torch.eye(4)[None]), ("trans", torch.eye(4, dtype=torch.float64)[None].repeat(2, 1, 1)),
       ("lengths", torch.zeros((0,), dtype=torch.int32))]


@pytest.mark.parametrize("key,value", BAD)
def test_bad_tensors_raise_before_any_launch(stub, key, value):
    from d3feat_b200 import training_data as td
    a = _good()
    a[key] = value
    with pytest.raises(ValueError):
        td.correspondences(a["points"], a["lengths"], a["pairs"], a["trans"], 0.1, "radius")
    with pytest.raises(ValueError):
        td.augment(a["points"], a["lengths"], a["pairs"], a["trans"], seed=0, noise=0.01)


def test_bad_options_raise_before_any_launch(stub):
    from d3feat_b200 import synth, training_data as td
    a = _good()
    args = (a["points"], a["lengths"], a["pairs"], a["trans"])
    for d, m in ((0.0, "radius"), (float("nan"), "radius"), (0.1, "ball")):
        with pytest.raises(ValueError):
            td.correspondences(*args, d, m)
    for kw in (dict(noise=-1.0), dict(noise=0.01, num_axis=2), dict(noise=0.01, scale=(0.8, 1.2)),
               dict(noise=0.01, scale=(1.2, 0.8), shift_range=2.0), dict(noise=0.01, seed=-1),
               dict(noise=0.01, capacity=-1)):
        kw = dict(dict(seed=0), **kw)
        with pytest.raises(ValueError):
            td.augment(*args, **kw)
    corr = td.Correspondences(torch.tensor([0, 3]), torch.zeros((3, 2), dtype=torch.int32), None, None)
    lens = torch.tensor([4], dtype=torch.int32)
    for kw in (dict(k=0), dict(replace=1), dict(min_count=-1), dict(seed=1 << 64),
               dict(anchor_lengths=torch.tensor([4]))):
        full = dict(dict(k=4, replace=True, min_count=0, seed=0, anchor_lengths=lens), **kw)
        with pytest.raises(ValueError):
            td.sample_correspondences(corr, **full)
    with pytest.raises(ValueError):
        td.sample_correspondences(corr._replace(offset=torch.tensor([0, 3], dtype=torch.int32)), 4, True, 0, 0, lens)
    with pytest.raises(ValueError):
        td.training_pairs(*args, synth.Config(keypts_num=4), "eth", 0)


def test_training_kitti_config():
    from d3feat_b200 import training as T
    assert T.TRAINING_KITTI["keypts_num"] == 1024 and T.TRAINING_KITTI["safe_radius"] == 1.0
    assert T.TRAINING_KITTI["first_subsampling_dl"] == 0.30
    assert T.TRAINING_3DMATCH["keypts_num"] == 256
