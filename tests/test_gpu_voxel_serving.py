"""GraphPipeline(..., voxel_size=v): raw scans in, the serving loop's results out, bit for bit equal to the same
pipeline without voxel_size fed the C port's voxelised clouds (oracle/voxel_oracle.c) with the same capacities and
bbox -- level counts, descriptors, scores, keypoints, matches, RANSAC and ICP poses and the evaluation, over several
steps including one in which every length is 0."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

LIMITS = [35, 33, 34, 36, 30]
V = 0.03


def t(a, dev):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def rigid(rng, deg=3.0, shift=0.2):
    from scipy.spatial.transform import Rotation
    T = np.eye(4)
    T[:3, :3] = Rotation.from_rotvec(np.deg2rad(deg) * rng.normal(size=3) / np.sqrt(3)).as_matrix()
    T[:3, 3] = rng.uniform(-shift, shift, 3)
    return T


def raw_batch(rng, seed, n_raw):
    """Three raw scans of one room: the scan and two moved partial copies, with their truth (source onto target)."""
    from d3feat_b200 import synth
    from d3feat_b200.evaluation import GroundTruth
    base = synth.raw_room_scan(seed, n_raw, box=2.0)
    clouds, poses = [base], []
    for keep in (0.9, 0.8):
        T = rigid(rng)
        proj = base @ rng.normal(size=3)
        part = base[proj <= np.quantile(proj, keep)]
        clouds.append((part @ T[:3, :3].T + T[:3, 3]).astype(np.float32))
        poses.append(T)
    G = np.stack([poses[0], poses[1], poses[1] @ np.linalg.inv(poses[0])])
    return (np.concatenate(clouds, 0), np.array([len(c) for c in clouds], np.int32),
            GroundTruth(G, None, np.array([1, 1, 1], np.int32)))


def snapshot(res, counts):
    """Every tensor of a step's result as host arrays (level-0 rows past the count are undefined: cut there)."""
    n = counts.cpu().numpy()
    out = {"counts": n}
    out["descriptors"] = res.descriptors[:n[0]].cpu().numpy()
    out["scores"] = res.scores[:n[0]].cpu().numpy()
    for name in ("keypoints", "matches", "registration", "refinement", "evaluation"):
        part = getattr(res, name)
        for f in part._fields:
            x = getattr(part, f)
            if x is not None and hasattr(x, "cpu"):
                out[name + "." + f] = x.cpu().numpy()
    return out


def same_bits(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def test_raw_scans_in_equal_voxelised_clouds_in(cuda):
    from d3feat_b200 import synth
    from d3feat_b200.encoder import EvaluatedDetections, GraphPipeline, KPFCNN
    from oracle.voxel_native import port_voxel_down_sample
    cfg = synth.Config(architecture=synth.ARCH_3DMATCH)
    enc = KPFCNN(cfg, synth.make_params(cfg, 5), LIMITS, device=cuda)
    rng = np.random.default_rng(3)
    batches = [raw_batch(rng, 20 + i, n) for i, n in enumerate([90000, 80000, 90000, 70000])]
    empty = batches[1]
    batches.insert(2, (empty[0][:1000], np.zeros(3, np.int32), empty[2]))   # every length 0 (rows of no cloud)
    pairs = [(0, 1), (0, 2), (1, 2)]
    opts = dict(decoder=True, keypoints=250, match_pairs=pairs,
                register=dict(distance=0.1, edge_ratio=0.5, ransac_n=4, max_iterations=2000, max_validation=200),
                icp=dict(distance=0.1), evaluate=dict(repeat_levels=[4, 16, 64, 250], rte_max=0.5, rre_max_deg=10.0))
    raw = GraphPipeline.for_batch(enc, t(batches[0][0], cuda), t(batches[0][1], cuda), slack=1.5, voxel_size=V, **opts)
    assert raw.voxel[0].capacity % 256 == 0 and raw.voxel[0].capacity >= 1.5 * len(batches[0][0])
    vox = GraphPipeline(enc, raw.caps, 3, raw.bbox, **opts)
    ported = [port_voxel_down_sample(p, l, V) for p, l, _ in batches]

    def run(pipe, feed):
        pipe.prime(t(feed[0][0], cuda), t(feed[0][1], cuda), truth=batches[0][2])
        steps = []
        for i in range(len(feed)):
            nxt = feed[i + 1] if i + 1 < len(feed) else None
            res, counts = (pipe.step(t(nxt[0], cuda), t(nxt[1], cuda), next_truth=batches[i + 1][2]) if nxt
                           else pipe.step())
            assert isinstance(res, EvaluatedDetections)
            steps.append(snapshot(res, counts))
        pipe.check()
        return steps

    got = run(raw, [(p, l) for p, l, _ in batches])
    want = run(vox, ported)
    assert raw.kernels_per_step > vox.kernels_per_step
    for i, (g, w) in enumerate(zip(got, want)):
        assert g["counts"][0] == len(ported[i][0]), i
        assert set(g) == set(w)
        bad = [k for k in g if not same_bits(g[k], w[k])]
        assert bad == [], (i, bad)
    assert got[2]["counts"][0] == 0
    assert got[0]["counts"][0] > 10000
    assert same_bits(raw.evaluation_totals(), vox.evaluation_totals())
