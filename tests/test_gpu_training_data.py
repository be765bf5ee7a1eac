"""GPU: training pairs (d3feat_b200/training_data.py, csrc/correspond.cu) bit for bit against oracle/pairs_np.py.

  * correspondences in both modes on random and lattice clouds, identity and random transforms, scenes far off the
    origin inside the grid bound (outside it: ValueError), empty and one-point clouds, a pair naming one cloud twice or
    a cloud out of range, P = 256, a lidar pair at tau = 0.45 and a 16-fragment all-pairs table at tau = 0.03;
  * sampling with and without replacement; the augmentation's parameters and points (given the GPU's own R, which is
    also compared where fp32 rounding of cos / sin is not ambiguous);
  * the same bits from two runs and from two streams; sampling plus augmentation captured and replayed in a CUDA graph;
  * end to end: training_pairs -> training.forward -> d3feat_loss on a room pair and a lidar pair.
"""
import numpy as np
import pytest
import torch

from oracle import pairs_np as op

pytestmark = pytest.mark.gpu


def _pose(rng, shift=0.3):
    from scipy.spatial.transform import Rotation
    T = np.eye(4)
    T[:3, :3] = Rotation.random(random_state=int(rng.integers(1 << 31))).as_matrix()
    T[:3, 3] = rng.normal(size=3) * shift
    return T


def _dev(dev, pts, lens, pairs, trans):
    return (torch.as_tensor(np.ascontiguousarray(pts, np.float32)).to(dev),
            torch.as_tensor(np.asarray(lens, np.int32)).to(dev),
            torch.as_tensor(np.asarray(pairs, np.int32).reshape(-1, 2)).to(dev),
            torch.as_tensor(np.asarray(trans, np.float64).reshape(-1, 4, 4)).to(dev))


def _check_corr(dev, pts, lens, pairs, trans, tau, mode, exhaustive=None):
    from d3feat_b200 import training_data as td
    got = td.correspondences(*_dev(dev, pts, lens, pairs, trans), tau, mode)
    ref = op.correspondences(pts, lens, pairs, trans, tau, mode, exhaustive=exhaustive)
    for key in ("offset", "rows", "count", "overlap"):
        g = getattr(got, key).cpu().numpy()
        assert g.dtype == ref[key].dtype and g.shape == ref[key].shape, key
        np.testing.assert_array_equal(g, ref[key], err_msg=key)
    return got, ref


def _random_case(rng, n=(900, 700, 1), scale=1.5):
    return np.concatenate([(rng.random((m, 3)) * scale).astype(np.float32) for m in n]), list(n)


def _lattice(offset=0.0):
    g = np.arange(8, dtype=np.float32) * np.float32(0.05)
    lat = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3) + np.float32(offset)
    return np.concatenate([lat, lat]).astype(np.float32), [len(lat), len(lat)]


CASES = ["random_identity", "random_pose", "lattice", "far", "empty_and_one", "same_cloud_and_out_of_range"]


@pytest.mark.parametrize("mode", op.MODES)
@pytest.mark.parametrize("case", CASES)
def test_correspondences(cuda, case, mode):
    rng = np.random.default_rng(CASES.index(case))
    if case.startswith("random"):
        pts, lens = _random_case(rng)
        pairs = [[0, 1], [1, 0], [2, 1]]
        T = [np.eye(4) if case.endswith("identity") else _pose(rng) for _ in pairs]
        tau = 0.07
    elif case == "lattice":
        pts, lens = _lattice()
        pairs, T, tau = [[0, 1]], [np.eye(4)], 0.05           # neighbours at d^2 == tau^2 exactly
    elif case == "far":
        pts, lens = _random_case(rng, (600, 500))
        pts = (pts + np.float32(40.0)).astype(np.float32)    # within 1024 cells of 0.07 * 1.001 of the origin
        pairs, T, tau = [[0, 1], [1, 0]], [_pose(rng, 0.1), np.eye(4)], 0.07
    elif case == "empty_and_one":
        pts, lens = _random_case(rng, (0, 1, 300, 0))
        pairs = [[0, 2], [1, 2], [2, 1], [2, 0], [2, 3], [1, 1]]
        T, tau = [np.eye(4)] * len(pairs), 2.0
    else:
        pts, lens = _random_case(rng, (500, 400))
        pairs = [[0, 0], [1, 1], [0, 2], [-1, 1], [1, 0]]
        T, tau = [_pose(rng, 0.05) for _ in pairs], 0.06
    _check_corr(cuda, pts, lens, pairs, T, tau, mode, exhaustive=True)


def test_far_scene_outside_the_bound_is_refused(cuda):
    from d3feat_b200 import training_data as td
    pts, lens = _random_case(np.random.default_rng(0), (100, 100))
    pts = (pts + np.float32(200.0)).astype(np.float32)
    with pytest.raises(ValueError):
        td.correspondences(*_dev(cuda, pts, lens, [[0, 1]], np.eye(4)[None]), 0.07, "radius")


@pytest.mark.parametrize("mode", op.MODES)
def test_256_pairs(cuda, mode):
    rng = np.random.default_rng(7)
    pts, lens = _random_case(rng, tuple(int(x) for x in rng.integers(0, 200, 40)))
    pairs = rng.integers(0, 40, (256, 2))
    T = [_pose(rng, 0.05) for _ in range(256)]
    _check_corr(cuda, pts, lens, pairs, T, 0.1, mode, exhaustive=True)


def test_lidar_pair_and_all_pairs_table(cuda):
    from d3feat_b200 import synth
    rng = np.random.default_rng(11)
    a = synth.lidar_scan(0, 16000)
    T = _pose(rng, 1.0)
    b = ((a.astype(np.float64) @ T[:3, :3].T + T[:3, 3]) + rng.normal(size=a.shape) * 0.05).astype(np.float32)
    got, ref = _check_corr(cuda, np.concatenate([a, b]), [len(a), len(b)], [[0, 1]], T[None], 0.45, "radius",
                           exhaustive=False)
    assert ref["count"][0] > 1024
    frags = [synth.room_fragment(s, 4000) for s in range(16)]
    pairs = [[i, j] for i in range(16) for j in range(i + 1, 16)]
    got, ref = _check_corr(cuda, np.concatenate(frags), [len(f) for f in frags], pairs, [np.eye(4)] * len(pairs), 0.03,
                           "nearest", exhaustive=False)
    assert len(pairs) == 120


def _table(dev, rng, P=6):
    counts = [0, 3, 50, 2000, 1500, 10][:P]
    offset = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    rows = np.stack([rng.integers(0, 5000, offset[-1]), rng.integers(0, 5000, offset[-1])], 1).astype(np.int32)
    anchor = rng.integers(0, 9000, P).astype(np.int32)
    from d3feat_b200 import training_data as td
    corr = td.Correspondences(torch.as_tensor(offset).to(dev), torch.as_tensor(rows).to(dev), None, None)
    return corr, offset, rows, anchor


@pytest.mark.parametrize("replace", [True, False])
def test_sampling(cuda, replace):
    from d3feat_b200 import training_data as td
    rng = np.random.default_rng(3)
    corr, offset, rows, anchor = _table(cuda, rng)
    for k, min_count, seed in ((16, 0, 0), (64, 20, 5), (1024, 1024, (1 << 64) - 1)):
        s = td.sample_correspondences(corr, k, replace, min_count, seed, torch.as_tensor(anchor).to(cuda))
        ra, rp, rv = op.sample(offset, rows, anchor, k, replace, min_count, seed)
        np.testing.assert_array_equal(s.anc.cpu().numpy(), ra)
        np.testing.assert_array_equal(s.pos.cpu().numpy(), rp)
        np.testing.assert_array_equal(s.valid.cpu().numpy(), rv)


def _aug_case(rng):
    pts, lens = _random_case(rng, (700, 0, 1, 900))
    pairs = [[0, 3], [3, 0], [1, 2], [2, 2], [0, 9]]
    return pts, lens, pairs, [_pose(rng) for _ in pairs]


@pytest.mark.parametrize("kitti,num_axis", [(False, 1), (True, 1), (False, 3)])
def test_augmentation(cuda, kitti, num_axis):
    from d3feat_b200 import training_data as td
    rng = np.random.default_rng(4)
    pts, lens, pairs, T = _aug_case(rng)
    kw = dict(scale=(0.8, 1.2), shift_range=2.0) if kitti else {}
    seed = 1234567
    a = td.augment(*_dev(cuda, pts, lens, pairs, T), seed=seed, noise=0.01, num_axis=num_axis, **kw)
    R = a.R.cpu().numpy()
    ref = op.augment(pts, lens, pairs, T, seed, 0.01, num_axis, R=R, **kw)
    for key, got in (("points", a.points), ("backup_points", a.backup_points), ("lengths", a.lengths),
                     ("row_offset", a.row_offset), ("scale", a.scale), ("shift", a.shift)):
        np.testing.assert_array_equal(got.cpu().numpy(), ref[key], err_msg=key)
    clear = ~ref["ambiguous"]
    np.testing.assert_array_equal(R[clear], ref["R"][clear])
    assert clear.sum() >= len(clear) - 1


def test_same_bits_across_runs_and_streams(cuda):
    from d3feat_b200 import training_data as td
    rng = np.random.default_rng(5)
    pts, lens, pairs, T = _aug_case(rng)
    args = _dev(cuda, pts, lens, pairs, T)

    def run():
        c = td.correspondences(*args, 0.2, "radius")
        s = td.sample_correspondences(c, 32, False, 1, 9, args[1][args[2][:, 0].long().clamp(0, 3)].contiguous())
        a = td.augment(*args, seed=9, noise=0.01, scale=(0.8, 1.2), shift_range=2.0)
        return [t.cpu() for t in (c.offset, c.rows, s.anc, s.pos, s.valid, a.points, a.backup_points, a.R)]

    first = run()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        second = run()
    torch.cuda.synchronize()
    for x, y, z in zip(first, run(), second):
        assert torch.equal(x, y) and torch.equal(x, z)


def test_sampling_and_augmentation_in_a_cuda_graph(cuda):
    from d3feat_b200 import training_data as td
    rng = np.random.default_rng(6)
    pts, lens, pairs, T = _aug_case(rng)
    args = _dev(cuda, pts, lens, pairs, T)
    corr = td.correspondences(*args, 0.2, "radius")
    anchor = torch.tensor([700, 900, 0, 1, 0], dtype=torch.int32, device=cuda)
    cap = 4000
    seed = 77

    def step():
        s = td.sample_correspondences(corr, 32, False, 1, seed, anchor)
        a = td.augment(*args, seed=seed, noise=0.01, scale=(0.8, 1.2), shift_range=2.0, capacity=cap)
        return s, a

    eager = step()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        s, a = step()
    g.replay()
    torch.cuda.synchronize()
    n = int(eager[1].row_offset[-1])
    for x, y in ((eager[0].anc, s.anc), (eager[0].pos, s.pos), (eager[0].valid, s.valid)):
        assert torch.equal(x, y)
    assert torch.equal(eager[1].points[:n], a.points[:n]) and torch.equal(eager[1].backup_points[:n],
                                                                         a.backup_points[:n])


def _room_pair():
    from d3feat_b200 import synth
    a = synth.room_fragment(0, 3000)
    T = np.eye(4)
    th = 0.4
    T[:3, :3] = [[np.cos(th), -np.sin(th), 0], [np.sin(th), np.cos(th), 0], [0, 0, 1]]
    T[:3, 3] = [0.3, -0.2, 0.1]
    b = (a.astype(np.float64) @ T[:3, :3].T + T[:3, 3]).astype(np.float32)
    return np.concatenate([a, b]), [len(a), len(b)], T


def _lidar_pair():
    from d3feat_b200 import synth
    a = synth.lidar_scan(1, 12000)
    T = np.eye(4)
    th = 0.1
    T[:3, :3] = [[np.cos(th), -np.sin(th), 0], [np.sin(th), np.cos(th), 0], [0, 0, 1]]
    T[:3, 3] = [2.0, 0.5, 0.0]
    b = (a.astype(np.float64) @ T[:3, :3].T + T[:3, 3]).astype(np.float32)
    return np.concatenate([a, b]), [len(a), len(b)], T


@pytest.mark.parametrize("dataset", ["3dmatch", "kitti"])
def test_end_to_end_step(cuda, dataset):
    from d3feat_b200 import synth, training as T, training_data as td
    from d3feat_b200.encoder import KPFCNN
    from d3feat_b200.variables import ParamStore, use_params
    kitti = dataset == "kitti"
    cfg = synth.Config(**(T.TRAINING_KITTI if kitti else T.TRAINING_3DMATCH))
    pts, lens, M = _lidar_pair() if kitti else _room_pair()
    tp = td.training_pairs(*_dev(cuda, pts, lens, [[0, 1]], M[None]), cfg, dataset, seed=3)
    assert bool(tp.valid[0])
    p_pts, p_lens, anc, pos, backup = tp.pair(0)
    tau = 1.5 * cfg.first_subsampling_dl if kitti else cfg.first_subsampling_dl
    d = (backup[anc.long()].double() - backup[pos.long()].double()).norm(dim=1)
    assert float(d.max()) < tau * (1 + 1e-6)
    store = ParamStore(synth.make_params(cfg, seed=0), cuda)
    enc = KPFCNN(cfg, store, [34] * 5, device=cuda)
    inputs = enc.build_inputs(p_pts, p_lens)
    T.trainable(store)
    with use_params(store):
        desc, scores = T.forward(inputs, cfg)
        loss, _, _, acc, _, _ = T.d3feat_loss(desc, scores, anc, pos, backup, cfg)
    loss.backward()
    assert torch.isfinite(loss).item() and float(acc) != -1.0
