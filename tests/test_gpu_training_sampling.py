"""GPU: keypoint sampling of training pairs (training_data.sample_correspondences: sample_keys_kernel, the radix sort of
csrc/sort.cu and sample_pick_kernel in csrc/correspond.cu) bit for bit against oracle/pairs_np.sample, at training
scale and at the edges of the sort.

Without replacement, candidate c of pair p gets the key (p << 32) | (32-bit draw); rows that belong to no pair get
pair P and draw ~0, so they sort last. The keys go through a stable LSD radix sort over sort_bits(P) = 32 +
bit_length(P) bits, 8 per pass, and pair p takes the first k entries of its run. The cases:

  * sort widths: P = 255 (40 bits, 5 passes), 256 (41 bits, 6 passes) and 65536 (49 bits, 7 passes), small counts
    with runs of empty pairs and trailing rows of no pair. The 7-pass case stands in for P = 2^24, the most pairs the
    counters allow (57 bits, 8 passes), which is beyond the oracle's per-pair loop;
  * tied draws: two pairs of 300 000 candidates whose 32-bit draws collide, sampled whole (k = n) and 1024 at a time;
  * a training-size table: millions of candidates over 120 pairs, 0 to 10^6 per pair, k = 64 with replacement and
    1024 without, k and min_count exactly at a pair's count and one above it, seeds 0 and 2^64 - 1;
  * tables that do not start at 0 (offset[a:b+1] of the training-size table over its full rows) or end before M;
  * M = 0, and P = 1;
  * the tables correspondences builds for KITTI and 3DMatch pairs, and training_pairs on a 120-pair 3DMatch batch
    against oracle correspondences -> augment -> sample;
  * the same bits from two runs, a side stream and a CUDA graph replay of the training-size table.

tests/test_training_sampling_oracle.py shows on the CPU that these cases catch a sort one bit too narrow, an unstable
order of tied draws, positions read from offset[p] rather than offset[p] - offset[0], and rows of no pair sorted first.
"""
import functools
from collections import namedtuple

import numpy as np
import pytest
import torch

from oracle import pairs_np as op

pytestmark = pytest.mark.gpu

SEED_MAX = (1 << 64) - 1

Case = namedtuple("Case", "offset rows anchor calls")
Case.__doc__ = """A sampling table: offset [P+1] int64, rows [M,2] int32, anchor [P] int32 (the anchor's length), and
    calls, the (k, replace, min_count, seed) it is sampled with."""


def sort_bits(P):
    """Key bits of the sampler's sort: the 32-bit draw under pair ids 0 .. P (P: rows of no pair)."""
    return 32 + int(P).bit_length()


def sort_passes(P):
    return -(-sort_bits(P) // 8)


def tied_draws(seed, p, n):
    """How many of pair p's n candidates share their 32-bit draw with an earlier candidate."""
    key = op.draw(seed, p, np.arange(n), op.SLOT_KEY) >> np.uint64(32)
    return n - len(np.unique(key))


def _table(counts, seed, *, extra=0):
    """offset of `counts` from 0, then `extra` trailing rows of no pair. The anchor row is the row's own index, so a
    candidate taken from the wrong place shows; the positive row is random."""
    rng = np.random.default_rng(seed)
    offset = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    M = int(offset[-1]) + extra
    rows = np.stack([np.arange(M), rng.integers(0, 1 << 20, M)], 1).astype(np.int32)
    anchor = rng.integers(0, 1 << 20, len(counts)).astype(np.int32)
    return offset, rows, anchor


def _small_counts(P, seed, hi, empty_runs):
    counts = np.random.default_rng(seed).integers(1, hi, P)
    for a, b in empty_runs:
        counts[a:b] = 0
    return counts


def _sort_width(P, empty_runs):
    counts = _small_counts(P, P, 12 if P < 1024 else 7, empty_runs)
    offset, rows, anchor = _table(counts, P, extra=37)
    return Case(offset, rows, anchor, [(4, False, 0, 11), (4, True, 0, SEED_MAX)])


TIES_N, TIES_SEED = 300_000, 0

# the training-size table: 120 pairs (a 16-fragment scene's all-pairs table) of up to 60 000 candidates, one of 10^6,
# a run of empty pairs, and pairs at the k and min_count boundaries of LARGE_CALLS
LARGE_COUNTS = {0: 0, 3: 0, 7: 1_000_000, 20: 1023, 21: 1024, 50: 0, 51: 0, 52: 0, 60: 5000, 61: 5001, 90: 1, 119: 0}
LARGE_CALLS = [(64, True, 5001, 0),               # count 5001 valid, 5000 (one below min_count) not
               (64, True, 0, SEED_MAX),
               (1024, False, 1, 0),               # count 1024 valid, 1023 (k one above it) not
               (1024, False, 5001, SEED_MAX)]
SLICE = (5, 100)                                  # offset[a:b+1], over the full rows


@functools.lru_cache(maxsize=None)
def large_table():
    counts = np.random.default_rng(120).integers(0, 60_000, 120)
    for p, n in LARGE_COUNTS.items():
        counts[p] = n
    return _table(counts, 120)


def _build(name):
    if name == "P255":
        return _sort_width(255, [(10, 20), (100, 131), (200, 203)])
    if name == "P256":
        return _sort_width(256, [(0, 1), (10, 20), (100, 131), (254, 256)])
    if name == "P65536":
        return _sort_width(65536, [(1000, 3000), (40000, 40100), (65530, 65535)])
    if name == "ties":
        offset, rows, anchor = _table([TIES_N, TIES_N], 2)
        return Case(offset, rows, anchor, [(TIES_N, False, 0, TIES_SEED), (1024, False, 1024, TIES_SEED)])
    if name == "large":
        return Case(*large_table(), LARGE_CALLS)
    if name in ("slice", "tail"):
        offset, rows, anchor = large_table()
        a, b = SLICE if name == "slice" else (0, SLICE[1])
        return Case(offset[a:b + 1], rows, anchor[a:b], [(1024, False, 1, 3), (64, True, 0, 3)])
    if name == "empty":
        return Case(np.zeros(4, np.int64), np.zeros((0, 2), np.int32), np.array([5, 0, 9], np.int32),
                    [(1, False, 0, 0), (8, True, 0, 0)])
    if name == "one_pair":
        offset, rows, anchor = _table([5000], 1)
        return Case(offset, rows, anchor, [(5000, False, 0, 1), (5001, False, 0, 1), (1024, False, 1024, 2),
                                           (64, True, 5000, 3), (64, True, 5001, 3)])
    raise KeyError(name)


CASES = ["P255", "P256", "P65536", "ties", "large", "slice", "tail", "empty", "one_pair"]


@functools.lru_cache(maxsize=None)
def case(name):
    return _build(name)


def _corr(dev, offset, rows):
    from d3feat_b200 import training_data as td
    return td.Correspondences(torch.as_tensor(offset).to(dev), torch.as_tensor(rows).to(dev), None, None)


def _check(dev, c, what):
    from d3feat_b200 import training_data as td
    corr = _corr(dev, c.offset, c.rows)
    anchor = torch.as_tensor(c.anchor).to(dev)
    for call in c.calls:
        s = td.sample_correspondences(corr, *call, anchor)
        ra, rp, rv = op.sample(c.offset, c.rows, c.anchor, *call)
        msg = "%s k=%d replace=%s min_count=%d seed=%d" % ((what,) + call)
        np.testing.assert_array_equal(s.valid.cpu().numpy(), rv, err_msg=msg + ": valid")
        np.testing.assert_array_equal(s.anc.cpu().numpy(), ra, err_msg=msg + ": anc")
        np.testing.assert_array_equal(s.pos.cpu().numpy(), rp, err_msg=msg + ": pos")


@pytest.mark.parametrize("name,passes", [("P255", 5), ("P256", 6), ("P65536", 7)])
def test_sort_widths(cuda, name, passes):
    c = case(name)
    assert sort_passes(len(c.offset) - 1) == passes
    assert int(c.offset[-1]) < len(c.rows)                  # rows of no pair: pair P must sort after pair 0
    _check(cuda, c, name)


def test_tied_draws_keep_candidate_order(cuda):
    c = case("ties")
    assert tied_draws(TIES_SEED, 0, TIES_N) > 0 and tied_draws(TIES_SEED, 1, TIES_N) > 0
    _check(cuda, c, "ties")


def test_training_size_table(cuda):
    c = case("large")
    assert len(c.offset) == 121 and int(c.offset[-1]) > 3_000_000
    _check(cuda, c, "large")


@pytest.mark.parametrize("name", ["slice", "tail"])
def test_tables_that_do_not_span_the_rows(cuda, name):
    """offset[a:b+1] of the training-size table over all its rows: rows before offset[0] and from offset[P] on belong
    to no pair ("slice"); offset[:b+1] leaves only trailing rows of no pair ("tail")."""
    c = case(name)
    assert (int(c.offset[0]) > 0) == (name == "slice") and int(c.offset[-1]) < len(c.rows)
    _check(cuda, c, name)


@pytest.mark.parametrize("name", ["empty", "one_pair"])
def test_degenerate_tables(cuda, name):
    from d3feat_b200 import training_data as td
    c = case(name)
    _check(cuda, c, name)
    if name == "empty":
        s = td.sample_correspondences(_corr(cuda, c.offset, c.rows), 8, False, 0, 0, torch.as_tensor(c.anchor).to(cuda))
        assert not s.valid.any() and (s.anc == -1).all() and (s.pos == -1).all()


def _lidar_table():
    from d3feat_b200 import synth
    from test_gpu_training_data import _pose
    rng = np.random.default_rng(11)
    a = synth.lidar_scan(0, 16000)
    T = _pose(rng, 1.0)
    b = ((a.astype(np.float64) @ T[:3, :3].T + T[:3, 3]) + rng.normal(size=a.shape) * 0.05).astype(np.float32)
    return np.concatenate([a, b]), [len(a), len(b)], [[0, 1]], T[None]


def _room_batch():
    from d3feat_b200 import synth
    frags = [synth.room_fragment(s, 4000) for s in range(16)]
    pairs = [[i, j] for i in range(16) for j in range(i + 1, 16)]
    return np.concatenate(frags), [len(f) for f in frags], pairs, np.stack([np.eye(4)] * len(pairs))


@pytest.mark.parametrize("dataset", ["kitti", "3dmatch"])
def test_tables_from_correspondences(cuda, dataset):
    """The tables correspondences builds, sampled at keypts_num as training_pairs samples them."""
    from d3feat_b200 import synth, training as T, training_data as td
    from test_gpu_training_data import _dev
    kitti = dataset == "kitti"
    cfg = synth.Config(**(T.TRAINING_KITTI if kitti else T.TRAINING_3DMATCH))
    pts, lens, pairs, trans = _lidar_table() if kitti else _room_batch()
    args = _dev(cuda, pts, lens, pairs, trans)
    dl = cfg.first_subsampling_dl
    corr = td.correspondences(*args, 1.5 * dl if kitti else dl, "radius" if kitti else "nearest")
    offset, rows = corr.offset.cpu().numpy(), corr.rows.cpu().numpy()
    anchor = np.asarray(lens, np.int32)[np.asarray(pairs)[:, 0]]
    call = (cfg.keypts_num, not kitti, 1024 if kitti else 0, 8)
    s = td.sample_correspondences(corr, *call, torch.as_tensor(anchor).to(cuda))
    ra, rp, rv = op.sample(offset, rows, anchor, *call)
    assert rv.any()
    np.testing.assert_array_equal(s.valid.cpu().numpy(), rv)
    np.testing.assert_array_equal(s.anc.cpu().numpy(), ra)
    np.testing.assert_array_equal(s.pos.cpu().numpy(), rp)


def test_training_pairs_against_the_oracle_chain(cuda):
    """training_pairs on a 120-pair 3DMatch batch equals oracle correspondences -> augment (given the GPU's own R) ->
    sample."""
    from d3feat_b200 import synth, training as T, training_data as td
    from test_gpu_training_data import _dev
    cfg = synth.Config(**T.TRAINING_3DMATCH)
    pts, lens, pairs, trans = _room_batch()
    args = _dev(cuda, pts, lens, pairs, trans)
    seed = 21
    aug = td.AUGMENT_3DMATCH
    tp = td.training_pairs(*args, cfg, "3dmatch", seed)
    R = td.augment(*args, seed=seed, noise=aug["augment_noise"], num_axis=aug["augment_rotation"]).R.cpu().numpy()
    corr = op.correspondences(pts, lens, pairs, trans, cfg.first_subsampling_dl, "nearest", exhaustive=False)
    a = op.augment(pts, lens, pairs, trans, seed, aug["augment_noise"], aug["augment_rotation"], R=R)
    anc, pos, valid = op.sample(corr["offset"], corr["rows"], a["lengths"][:, 0], cfg.keypts_num, True, 0, seed)
    assert len(pairs) == 120 and valid.any() and not valid.all()
    for key, got, want in (("points", tp.points, a["points"]), ("lengths", tp.lengths, a["lengths"]),
                           ("row_offset", tp.row_offset, a["row_offset"]),
                           ("backup_points", tp.backup_points, a["backup_points"]),
                           ("anc_inds", tp.anc_inds, anc), ("pos_inds", tp.pos_inds, pos), ("valid", tp.valid, valid),
                           ("count", tp.count, corr["count"])):
        np.testing.assert_array_equal(got.cpu().numpy(), want, err_msg=key)


@pytest.mark.parametrize("replace", [False, True])
def test_same_bits_from_runs_streams_and_graph_replay(cuda, replace):
    """The training-size table at full size: two runs, a side stream and a CUDA graph replay give the same bits."""
    from d3feat_b200 import training_data as td
    c = case("large")
    corr = _corr(cuda, c.offset, c.rows)
    anchor = torch.as_tensor(c.anchor).to(cuda)
    k, seed = (64 if replace else 1024), 5

    def run():
        s = td.sample_correspondences(corr, k, replace, 1, seed, anchor)
        return s.anc, s.pos, s.valid

    first = run()
    second = run()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        third = run()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        graphed = run()
    for t in graphed:
        t.fill_(7)
    g.replay()
    torch.cuda.synchronize()
    assert bool(first[2].any()) and not bool(first[2].all())
    for other in (second, third, graphed):
        for x, y in zip(first, other):
            assert torch.equal(x, y)
