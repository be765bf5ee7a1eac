"""CPU: the random-keypoint contract (oracle/keypoints_np.py), the refusals of sample_keypoints and of
GraphPipeline(..., sweep=...), and evaluation.sweep_summary against totals of oracle/evaluate_np.py.

The sampler is checked against a plain-integer restatement of its formula, for the prefix property that lets the
random arm of a sweep use the first c slots of one draw, for the count rules (empty, one-point and cut clouds, rows of
no cloud), and by a chi-square test of uniformity on a large draw. Every refusal runs with the library replaced by a
stub whose every symbol raises, so a check that came too late would fail here rather than reach a GPU."""
import numpy as np
import pytest

from oracle import evaluate_np, keypoints_np

M64 = (1 << 64) - 1
GOLDEN = 0x9E3779B97F4A7C15


def splitmix64_int(z):
    z &= M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def slot_row(seed, b, j, s, n):
    """The contract for one slot in Python integers: s + (((z >> 32) * n) >> 32)."""
    z = splitmix64_int(seed + (((b << 32) | j) * GOLDEN))
    return s + (((z >> 32) * n) >> 32)


# ---- 1. the sampler ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("seed", [0, 1, 12345, M64])
def test_sampler_equals_the_formula(seed):
    lens = [7, 0, 1, 300, 2, 5]
    n = sum(lens)
    idx, cnt = keypoints_np.sample_keypoints(lens, 9, seed, n)
    start = np.concatenate([[0], np.cumsum(lens)])
    for b, L in enumerate(lens):
        want = [slot_row(seed, b, j, int(start[b]), L) if L else -1 for j in range(9)]
        assert idx[b].tolist() == want, b
        assert cnt[b] == (9 if L else 0)


def test_prefix_of_a_draw_is_the_smaller_draw():
    rng = np.random.default_rng(3)
    lens = rng.integers(0, 400, 64)
    lens[::9] = 0
    lens[1::13] = 1
    n = int(lens.sum())
    big, cnt_big = keypoints_np.sample_keypoints(lens, 5000, 77, n)
    for c in (2500, 1000, 500, 250, 1):
        small, cnt = keypoints_np.sample_keypoints(lens, c, 77, n)
        assert np.array_equal(small, big[:, :c]), c
        assert np.array_equal(cnt, np.minimum(cnt_big, c)), c
    other, _ = keypoints_np.sample_keypoints(lens, 5000, 78, n)
    assert not np.array_equal(other, big)


def test_count_rules_and_rows_of_no_cloud():
    """Empty clouds: count 0 and index -1. One-point clouds: every slot is that row. A cloud reaching past n is cut
    there, and one starting at or past n is empty. Rows past the last cloud are never drawn."""
    lens = np.array([0, 1, 50, 0, 1, 40, 30], np.int64)
    start = np.concatenate([[0], np.cumsum(lens)])
    k = 700
    for n in (int(start[-1]) + 25, int(start[-1]), int(start[5]) + 10, int(start[5])):
        idx, cnt = keypoints_np.sample_keypoints(lens, k, 5, n)
        for b in range(len(lens)):
            lo, hi = min(start[b], n), min(start[b + 1], n)
            if hi == lo:
                assert cnt[b] == 0 and (idx[b] == -1).all(), (n, b)
                continue
            assert cnt[b] == k
            assert ((idx[b] >= lo) & (idx[b] < hi)).all(), (n, b)
            if hi - lo == 1:
                assert (idx[b] == lo).all()
            else:
                assert len(np.unique(idx[b])) > 1            # with replacement, but not constant
        assert (idx < min(int(start[-1]), n)).all()


def test_draws_are_uniform_and_with_replacement():
    """One cloud of 97 rows, 194 000 draws (2000 expected per row): chi-square with 96 degrees of freedom. The draws
    are fixed by the seed, so this is a fixed check, not a flaky one; p > 1e-3 for a uniform sampler."""
    from scipy import stats
    n, k = 97, 194_000
    idx, cnt = keypoints_np.sample_keypoints([n], k, 2024, n)
    hist = np.bincount(idx[0], minlength=n)
    chi2, p = stats.chisquare(hist)
    assert cnt[0] == k and hist.min() > 0
    assert p > 1e-3, (chi2, p)
    # consecutive slots are independent draws: (slot 2i, slot 2i + 1) is uniform over the n * n cells
    pairs = idx[0][0::2] * n + idx[0][1::2]
    chi2, p = stats.chisquare(np.bincount(pairs, minlength=n * n))
    assert p > 1e-3, (chi2, p)


def test_gather_pads_with_zeros():
    rows = np.arange(12, dtype=np.float32).reshape(4, 3)
    got = keypoints_np.gather(np.array([[3, -1], [0, 0]]), rows)
    assert np.array_equal(got, np.array([[[9, 10, 11], [0, 0, 0]], [[0, 1, 2], [0, 1, 2]]], np.float32))


# ---- 2. refusals before the library -----------------------------------------------------------------------------------

@pytest.fixture
def no_library(monkeypatch):
    """The library replaced by a stub that raises on any use, and the ops told their device type is "cpu"."""
    from d3feat_b200 import _lib

    def refuse(*a, **k):
        raise AssertionError("the library was reached")
    monkeypatch.setattr(_lib, "lib", refuse)
    monkeypatch.setattr(_lib, "DEVICE_TYPE", "cpu")


@pytest.mark.parametrize("B,k,seed,match", [
    (0, 5, 0, "B=0"), (1025, 5, 0, "B=1025"), (3, 0, 0, "k=0"), (3, -2, 0, "k=-2"),
    (1024, 2 ** 21, 0, "within int32"), (2, 5, -1, "seed"), (2, 5, 1 << 64, "seed")])
def test_sample_keypoints_refusals(no_library, B, k, seed, match):
    import torch
    from d3feat_b200.keypoints import sample_keypoints
    with pytest.raises(ValueError, match=match):
        sample_keypoints(torch.ones(B, dtype=torch.int32), k, seed, points=torch.zeros((B, 3)))


@pytest.mark.parametrize("what", ["points", "descriptors", "scores", "rows"])
def test_sample_keypoints_refuses_bad_tensors(no_library, what):
    import torch
    from d3feat_b200.keypoints import sample_keypoints
    args = dict(points=torch.zeros((6, 3)), descriptors=torch.zeros((6, 4)), scores=torch.zeros((6, 1)),
                rows=torch.tensor([6], dtype=torch.int32))
    bad = dict(points=torch.zeros((6, 2)), descriptors=torch.zeros((5, 4)), scores=torch.zeros((6, 2)),
               rows=torch.tensor([6, 6], dtype=torch.int32))
    args[what] = bad[what]
    with pytest.raises(ValueError, match=what):
        sample_keypoints(torch.tensor([3, 3], dtype=torch.int32), 4, **args)
    args[what] = bad[what].to(torch.float64 if what != "rows" else torch.int64)
    with pytest.raises(ValueError, match=what):
        sample_keypoints(torch.tensor([3, 3], dtype=torch.int32), 4, **args)


BAD_SWEEPS = [
    ([(0, 1)], 64, dict(counts=(64, 32)), "needs match_pairs", dict(match_pairs=None)),
    ([(0, 1)], 64, [64, 32], "must be a dict", {}),
    ([(0, 1)], 64, dict(arms=("score",)), "must be a dict", {}),
    ([(0, 1)], 64, dict(counts=(64,), other=1), "must be a dict", {}),
    ([(0, 1)], 64, dict(counts=()), "non-empty sequence", {}),
    ([(0, 1)], 64, dict(counts=5), "non-empty sequence", {}),
    ([(0, 1)], 64, dict(counts=(64, 32.0)), "non-empty sequence", {}),
    ([(0, 1)], 64, dict(counts=(64, True)), "non-empty sequence", {}),
    ([(0, 1)], 64, dict(counts=(32, 64)), "descend strictly", {}),
    ([(0, 1)], 64, dict(counts=(64, 64)), "descend strictly", {}),
    ([(0, 1)], 64, dict(counts=(65, 32)), "descend strictly", {}),
    ([(0, 1)], 64, dict(counts=(64, 0)), "descend strictly", {}),
    ([(0, 1)], 64, dict(counts=(64,), arms=()), "arms", {}),
    ([(0, 1)], 64, dict(counts=(64,), arms=("score", "score")), "arms", {}),
    ([(0, 1)], 64, dict(counts=(64,), arms=("pred",)), "arms", {}),
    ([(0, 1)], 64, dict(counts=(64,), arms=None), "arms", {}),
    ([(0, 1)], 64, dict(counts=(64,), seed=-1), "seed", {}),
    ([(0, 1)], 64, dict(counts=(64,), seed=1 << 64), "seed", {}),
    ([(0, 1)], 64, dict(counts=(64,), seed=1.5), "seed", {}),
    # the repeatability levels are checked against the smallest count
    ([(0, 1)], 64, dict(counts=(64, 16)), "repeat_levels", dict(evaluate=dict(repeat_levels=[4, 32]))),
]


@pytest.mark.parametrize("pairs,k,sweep,match,extra", BAD_SWEEPS)
def test_sweep_option_refusals(no_library, pairs, k, sweep, match, extra):
    """Every bad sweep is a ValueError at construction, before the encoder, the device or the library is touched
    (the encoder here is a bare object)."""
    from d3feat_b200.encoder import GraphPipeline
    kw = dict(decoder=True, keypoints=k, match_pairs=pairs, sweep=sweep)
    kw.update(extra)
    with pytest.raises(ValueError, match=match):
        GraphPipeline(object(), [100, 50, 25, 12, 6], 2, np.zeros(6, np.float32), **kw)


def test_sweep_options_accepted():
    from d3feat_b200.encoder import check_sweep
    assert check_sweep(dict(counts=[5000, 2500, 1000, 500, 250]), 5000) == (
        (5000, 2500, 1000, 500, 250), ("score", "random"), 0)
    assert check_sweep(dict(counts=(np.int64(8),), arms=["random"], seed=M64), 8) == ((8,), ("random",), M64)
    assert check_sweep(dict(counts=(6, 2), arms="score", seed=np.uint64(3)), 8) == ((6, 2), ("score",), 3)


# ---- 3. sweep_summary -------------------------------------------------------------------------------------------------

def test_sweep_summary_is_summary_of_each_row():
    """Totals of evaluate_np for every (arm, count) of a 2 x 3 sweep, stacked as GraphPipeline.evaluation_totals()
    returns them: each row of sweep_summary is summary() of its totals, and its headline numbers are those of the
    per-pair metrics."""
    from d3feat_b200.evaluation import summary, sweep_summary
    from test_gpu_evaluation import OPTS, info_matrices, make_case
    arms, counts, levels = ("score", "random"), (40, 20, 10), (4, 8)
    pairs = [(a, b) for a in range(4) for b in range(a + 1, 4)]
    P = len(pairs)
    rng = np.random.default_rng(8)
    info = info_matrices(P)
    totals = np.zeros((len(arms), len(counts), 4 + len(levels) + 7 * 2))
    per_pair = {}
    for i, arm in enumerate(arms):
        for j, c in enumerate(counts):
            pts, cnt, matches, n_m, G, poses = make_case(rng, c, rng.integers(0, c + 1, 4), pairs, poison=0.0)
            flags = rng.choice([0, 1, 3], P).astype(np.int32)
            out = evaluate_np.evaluate(pts, cnt, matches, n_m, pairs, G, info, flags, poses, levels=levels, **OPTS)
            totals[i, j] = out["totals"]
            per_pair[(arm, c)] = out
    rows = sweep_summary(totals, arms, counts, levels, ("ransac", "icp"))
    assert [(r["arm"], r["count"]) for r in rows] == [(a, c) for a in arms for c in counts]
    for r in rows:
        i, j = arms.index(r["arm"]), counts.index(r["count"])
        want = summary(totals[i, j], levels, ("ransac", "icp"))
        got = {f: v for f, v in r.items() if f not in ("arm", "count")}
        assert repr(got) == repr(want)           # NaN (an empty divisor) prints the same on both sides
        out = per_pair[(r["arm"], r["count"])]
        valid = out["valid"].astype(bool)
        assert r["n_pairs"] == valid.sum() and r["fmr_hits"] == out["fmr_hit"].sum()
        if valid.any():
            assert r["fmr"] == out["fmr_hit"].sum() / valid.sum()
            assert np.isclose(r["repeatability"][8], out["repeatability"][valid, 1].sum() / valid.sum())
        assert r["ransac"]["successes"] == out["success"][0].sum()
        assert r["icp"]["recall_hits"] == out["recall_hit"][1].sum()
    with pytest.raises(ValueError, match="sweep_summary"):
        sweep_summary(totals[:, :2], arms, counts, levels, ("ransac", "icp"))
    with pytest.raises(ValueError, match="summary"):
        sweep_summary(totals, arms, counts, levels, ("ransac",))
