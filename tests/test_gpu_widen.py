"""GPU parity for the rows SURVEY.md §8(f) marks "next": the detection score that is dumped next to the descriptors,
neighbourhood calibration, and the deformable KITTI-shaped configuration at its full size (BASELINE.json configs[2]).

Tolerances as in test_gpu_kpconv.py: 1e-4 max-norm relative on fp32 features, exact on integers; the detection scores
also element by element against float64 (tests/_oracle.py).
"""
import numpy as np
import pytest
import torch

from oracle import native as on
from oracle import kpconv_np as ok

from _oracle import TOL, assert_close

pytestmark = pytest.mark.gpu

RTOL = 1e-4


def t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def rel_err(a, b):
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-30)


SCORE_KINDS = ("plain", "steep", "negative_max", "cancelling", "max_near_minus_eps", "all_zero")


def score_case(seed, lengths, D, H):
    """Features [N, D], level-0 style neighbours [N, H] (shadow index N) and lengths for the detection scores. Cloud b
    is of kind SCORE_KINDS[b % 6] (clouds of fewer than two rows stay plain):
      plain               normal features, 10 % zero rows (a neighbour that does not vote)
      steep               as plain, plus rows holding the cloud maximum in channel 0 whose other neighbours hold
                          -(2..50) x that maximum there: d = f - mean from ~3 to past 20 (both softplus branches)
      negative_max        every feature negative, so the cloud scale is negative
      cancelling          as plain, plus rows whose channels cancel to an exactly zero sum in the kernel's
                          warp-shuffle order and in numpy's pairwise order (D = 32 or 64; x[c + 8] = -x[c])
      max_near_minus_eps  every feature negative with maximum ~ -1.05e-6: M + 1e-6 cancels to ~5e-8
      all_zero            every feature zero (scale 1e6, score 0)
    Neighbours: the row itself first, then random rows of its own cloud, 20 % shadow padding."""
    rng = np.random.default_rng(seed)
    lengths = np.asarray(lengths, np.int32)
    N = int(lengths.sum())
    start = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    x = rng.normal(size=(N, D)).astype(np.float32)
    x[rng.uniform(size=N) < 0.1] = 0.0
    nbr = np.full((N, H), N, np.int32)
    for b, n in enumerate(lengths):
        a, e = start[b], start[b + 1]
        if n and H:
            nbr[a:e] = rng.integers(a, e, (n, H))
            nbr[a:e][rng.uniform(size=(n, H)) < 0.2] = N
            nbr[a:e, 0] = np.arange(a, e)
        kind = SCORE_KINDS[b % len(SCORE_KINDS)] if n >= 2 else "plain"
        xb = x[a:e]
        if kind == "steep" and H >= 2:
            M = xb.max()
            for r in rng.choice(n, min(n, 8), replace=False):
                others = nbr[a + r, 1:]
                others = others[(others < N) & (others != a + r)]
                x[others, 0] = -rng.uniform(2, 50) * M
            for r in rng.choice(n, min(n, 8), replace=False):
                x[a + r, 0] = M
        elif kind == "negative_max":
            xb[:] = -np.abs(xb) - 0.25
        elif kind == "cancelling" and D in (32, 64):
            lo = np.arange(D)[(np.arange(D) & 8) == 0]
            sel = rng.uniform(size=n) < 0.2
            xb[np.ix_(sel, lo + 8)] = -xb[np.ix_(sel, lo)]
        elif kind == "max_near_minus_eps":
            xb[:] = -(np.abs(xb) + 1.05) * np.float32(1e-6)
        elif kind == "all_zero":
            xb[:] = 0.0
    return x, nbr, lengths


SCORE_CASES = {
    # the three earlier (lengths, D) inputs, under the ids they have always had
    "lengths0-32": ([1500, 1300], 32, 30), "lengths1-32": ([700, 1, 900], 32, 30), "lengths2-48": ([1200], 48, 30),
    # many clouds, with empty and one-point clouds at the start, in the middle and at the end
    "B17": ([0, 1, 300, 0, 0, 1, 250, 400, 1, 0, 350, 200, 1, 300, 280, 1, 0], 32, 24),
    "B33": ([1, 0] + [37 * (i % 7) + (i % 3) for i in range(29)] + [0, 1], 32, 20),
    "B300": ([(0, 1, 2, 17, 40, 5, 23)[i % 7] for i in range(300)], 32, 12),
    # lane tails and several channels per lane
    "D1": ([600, 0, 500, 400, 300, 350, 250], 1, 16),
    "D31": ([600, 1, 500, 400, 300, 350, 250], 31, 16),
    "D33": ([600, 500, 1, 400, 300, 350, 250], 33, 16),
    "D64": ([600, 500, 450, 400, 300, 350, 250], 64, 16),
    "H0": ([600, 500, 450, 400, 300, 350], 32, 0),
    "H1": ([600, 500, 450, 400, 300, 350], 32, 1),
}


@pytest.mark.parametrize("case", sorted(SCORE_CASES))
def test_detection_scores_match_restatement(cuda, case):
    """models/D3Feat.py:67-115 against the float64 restatement, element by element (tests/_oracle.py): zero rows
    (count_nonzero), negative values, shadow neighbours, and the clouds of score_case."""
    from d3feat_b200 import network_blocks as nb
    lengths, D, H = SCORE_CASES[case]
    x, idx, lengths = score_case(sum(map(ord, case)), lengths, D, H)
    N = x.shape[0]
    ref, mag, alt = ok.detection_scores(x.astype(np.float64), idx, lengths, magnitude=True)
    out = nb.detection_scores(t(x, cuda), t(idx, cuda), t(lengths, cuda)).cpu().numpy()
    assert out.shape == (N, 1)
    assert rel_err(out, ref) < RTOL
    assert_close(out, ref, mag, TOL, "detection_scores %s" % case, alt=alt)


def test_descriptors_and_scores_end_to_end(cuda):
    """Two stacked fragments (anchor || positive, the reference's batch) through pyramid + encoder + decoder +
    detection branch, vs the float64 restatement on the same pyramid."""
    from d3feat_b200 import synth
    from d3feat_b200.encoder import KPFCNN
    cfg = synth.Config()
    clouds = [synth.room_fragment(50, 5000), synth.room_fragment(51, 4500)]
    P = np.concatenate(clouds, 0)
    L = np.array([c.shape[0] for c in clouds], np.int32)
    params = synth.make_params(cfg, 3)
    out = KPFCNN(cfg, params, [35, 33, 34, 36, 30], device=cuda)(P, L)
    inputs = {k: [x.cpu().numpy() for x in v] for k, v in out["inputs"].items() if k != "features"}
    inputs["features"] = np.ones((P.shape[0], 1), np.float32)
    orc = ok.EncoderOracle(cfg, params, np.float64)
    d_ref, s_ref = orc.decoder(inputs, orc.encoder(inputs), return_scores=True)
    assert np.abs(out["descriptors"].cpu().numpy() - d_ref).max() < RTOL
    s = out["scores"].cpu().numpy()
    assert s.shape == (P.shape[0], 1) and np.isfinite(s).all()
    assert rel_err(s, s_ref) < RTOL


def test_calibrate_neighbors_matches_oracle_counts(cuda):
    """datasets/common.py:572-673: the 80th-percentile column caps from the histogram of conv-neighbour counts --
    integer result, must equal the same statistic computed from the oracle's neighbour matrices."""
    from d3feat_b200 import synth
    from d3feat_b200 import pyramid as pyr
    cfg = synth.Config(architecture=synth.ARCH_ENCODER)
    clouds = [synth.room_fragment(60 + i, 4000) for i in range(3)]
    got = pyr.calibrate_neighbors(cfg, clouds, keep_ratio=0.8, device=cuda)
    levels = pyr._level_radii(cfg)
    hist_n = int(np.ceil(4 / 3 * np.pi * (cfg.density_parameter + 1) ** 3))
    hists = np.zeros((len(levels), hist_n), np.int64)
    for c in clouds:
        p, b = np.asarray(c, np.float32), np.array([c.shape[0]], np.int32)
        for li, lv in enumerate(levels):
            nbm = on.port_batch_neighbors(p, p, b, b, lv["conv_r"])
            counts = np.sum(nbm < p.shape[0], axis=1)
            hists[li] += np.bincount(counts, minlength=hist_n)[:hist_n]
            if lv["dl"] is None:
                break
            p, b = on.port_batch_subsampling(p, b, lv["dl"])
    cumsum = np.cumsum(hists.T, axis=0)
    want = [int(v) for v in np.sum(cumsum < (0.8 * cumsum[hist_n - 1, :]), axis=0)]
    assert got == want
    assert all(5 < v < hist_n for v in got)


def test_config3_full_size_deformable(cuda, monkeypatch):
    """BASELINE.json configs[2]: one 120k-point KITTI-shaped scan through the deformable architecture. Too large for
    the numpy restatement, so the check is the size-independent one: the wgmma 3xTF32 path and the independent
    CUDA-core fp32 path (each pinned to the restatement at small sizes) agree to 1e-4 on every level, the pyramid
    is well-formed, and a second run is bit-identical (no atomics on float data)."""
    from d3feat_b200 import synth
    from d3feat_b200 import convolution_ops as co
    from d3feat_b200.encoder import KPFCNN
    # a 64-beam scan voxelised at the KITTI setting (0.3 m) keeps ~20k points; the 120k-point level 0 that
    # configs[2] names is reached with a denser azimuth sampling and a 4 cm first voxel
    cfg = synth.Config(architecture=synth.ARCH_KITTI_DEFORM, first_subsampling_dl=0.04, first_features_dim=32)
    cloud = synth.lidar_scan(1, 120000, dl=0.04)
    L = np.array([cloud.shape[0]], np.int32)
    assert cloud.shape[0] == 120000
    params = synth.make_params(cfg, 1)
    enc = KPFCNN(cfg, params, [40, 40, 40, 60, 40], device=cuda)
    monkeypatch.setattr(co, "USE_TENSOR_CORES", True)
    out_tc = enc(cloud, L)
    F_tc = [f.cpu().numpy() for f in out_tc["F"]]
    F_tc2 = [f.cpu().numpy() for f in enc(cloud, L)["F"]]
    monkeypatch.setattr(co, "USE_TENSOR_CORES", False)
    F_cc = [f.cpu().numpy() for f in enc(cloud, L)["F"]]
    sizes = [int(p.shape[0]) for p in out_tc["inputs"]["points"]]
    assert sizes[0] == cloud.shape[0] and all(a > b > 0 for a, b in zip(sizes, sizes[1:]))
    for l, nbm in enumerate(out_tc["inputs"]["neighbors"]):
        nbm = nbm.cpu().numpy()
        assert nbm.min() >= 0 and nbm.max() <= sizes[l]
        assert (nbm[:, 0] == np.arange(sizes[l])).all()         # a point is its own nearest neighbour
    for l, (a, b, c) in enumerate(zip(F_tc, F_cc, F_tc2)):
        assert np.isfinite(a).all() and a.shape[0] == sizes[l]
        assert rel_err(a, b) < RTOL, "level %d" % l
        assert np.array_equal(a.view(np.uint32), c.view(np.uint32)), "level %d not reproducible" % l


def test_released_weights_on_real_scan(cuda):
    """First four blocks of the RELEASED 3DMatch model (trained weights, BN statistics and kernel points read from the
    reference's snapshot by tf_checkpoint.py -> tests/golden/released_3dmatch_head.npz) on a crop of the reference's
    real demo scan, two stacked clouds: GPU vs the float64 restatement."""
    import os
    from d3feat_b200 import synth
    from d3feat_b200.encoder import KPFCNN
    gold = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    z = np.load(os.path.join(gold, "released_3dmatch_head.npz"))
    params = {k.replace("|", "/"): z[k] for k in z.files}
    scan = np.load(os.path.join(gold, "subsampling_demo.npz"))
    P, L = on.port_batch_subsampling(scan["points"], scan["lengths"], 0.03)
    assert P.shape[0] > 1000
    cfg = synth.Config(architecture=["simple", "resnetb", "resnetb_strided", "resnetb"])
    limits = [38, 36]
    out = KPFCNN(cfg, params, limits, device=cuda)(P, L)
    inputs = {k: [x.cpu().numpy() for x in v] for k, v in out["inputs"].items() if k != "features"}
    inputs["features"] = np.ones((P.shape[0], 1), np.float32)
    F_ref, trace = ok.EncoderOracle(cfg, params, np.float64).encoder(inputs, return_all=True)
    assert len(out["F"]) == len(F_ref) == 2
    assert [f.shape[1] for f in F_ref] == [128, 256]
    for l, (a, b) in enumerate(zip(out["F"], F_ref)):
        assert np.abs(b).max() > 1e-3                       # trained weights produce a live signal
        assert rel_err(a.cpu().numpy(), b) < RTOL, "level %d" % l


def test_batch_pipeline_matches_single_shot(cuda):
    """BatchPipeline (pyramid(i+1) || encoder(i), ring of pre-allocated pyramid slots): seven batches of varying size
    through a 3-slot ring give bit-identical features to the one-batch-at-a-time path."""
    from d3feat_b200 import synth
    from d3feat_b200.encoder import KPFCNN, BatchPipeline
    cfg = synth.Config(architecture=synth.ARCH_ENCODER)
    params = synth.make_params(cfg, 5)
    enc = KPFCNN(cfg, params, [35, 33, 34, 36, 30], device=cuda)
    batches = []
    for i, n in enumerate([5000, 5000, 3500, 6500, 5000, 4000, 5000]):
        clouds = [synth.room_fragment(70 + 2 * i, n), synth.room_fragment(71 + 2 * i, n - 500)]
        batches.append((np.concatenate(clouds, 0), np.array([c.shape[0] for c in clouds], np.int32)))
    want = [enc(P, L, decoder=False)["F"][-1].cpu().numpy() for P, L in batches]
    pipe = BatchPipeline(enc, decoder=False)
    pipe.prime(*batches[0])
    got = []
    for i in range(len(batches)):
        nxt = batches[i + 1] if i + 1 < len(batches) else (None, None)
        res = pipe.step(nxt[0], nxt[1])
        got.append(res)                       # keep device tensors alive; read back after the drain
    pipe.drain()
    for i, (a, b) in enumerate(zip(got, want)):
        a = a.cpu().numpy()
        assert a.shape == b.shape, i
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), "batch %d" % i
