"""Batches of up to 1024 clouds (the library's kMaxBatch) through the half of the pipeline that assigns every row to its
cloud: grid subsampling, the radius searches and the input pyramid (exact form, static form, and replayed by
GraphPipeline), bit for bit against the exhaustive C restatement (oracle/native.py port_*).

The batches are built so that a row assigned to the wrong cloud changes the result:
* every cloud is a crop or a random subset of ONE 1.5 m room scene, so neighbouring clouds overlap in space and a query
  searched in the wrong cloud finds neighbours there instead of none;
* some clouds are exact copies of earlier ones, so a support leaking in from another cloud shows up as a wrong index at
  an equal d2;
* some clouds are cut from a lattice of spacing 1/32 (exact in float32), whose exact d2 ties force the exact sorts;
* cloud sizes are 0, 1, 2, 31, 32, 33 and a few hundred (a warp's 32 rows span several clouds), with runs of empty
  clouds at the start, in the middle and at the end, and batches where every cloud but one is empty;
* B runs over both sides of the query kernels' ballot thresholds (16 and 32 clouds) up to 1024.
tests/test_oracle_sensitivity.py shows that emulated batch-assignment bugs change the oracle's result on these batches.

Rows past the last cloud (lengths summing to less than the row count) belong to no cloud: they are not subsampled, no
query finds them, and as queries they get count 0 and a row of padding. Lengths summing past the row count cut the
last cloud there.
"""
import functools

import numpy as np
import pytest
import torch

from oracle import kpconv_np as ok
from oracle import native as on

pytestmark = pytest.mark.gpu

R = 0.075                                    # level-0 conv radius of the standard configuration
DL = 0.06                                    # its first subsampling
CAP = 12                                     # capped fill: fewer columns than most dense rows have
LIMITS = [24, 20, 18, 16, 14]
SENTINEL = np.int32(0x7FBADBAD)
SCENE_POINTS = 7500                          # synth.room_fragment: a 3 m * sqrt(7500 / 30000) = 1.5 m box
SIZES = [0, 1, 2, 31, 32, 33, 300, 0, 0, 1, 120, 33, 2, 450, 31, 0, 64, 200]
CASES = ["B1", "B2", "B16", "B17", "B32", "B33", "B300", "B1024", "B33_lone", "B1024_lone"]


# ---- batches ----------------------------------------------------------------------------------------------------------

@functools.lru_cache(maxsize=None)
def scene():
    """The room every cloud is cut from, and a lattice slab of spacing 1/32 over the same floor."""
    from d3feat_b200 import synth
    room = synth.room_fragment(77, SCENE_POINTS)
    lo = np.floor(room.min(0) * 32) / 32
    ijk = np.stack(np.meshgrid(np.arange(48), np.arange(48), np.arange(6), indexing="ij"), -1).reshape(-1, 3)
    lattice = (lo + ijk / 32.0).astype(np.float32)            # multiples of 1/32: exact, so d2 ties are exact
    return room, lattice


def lengths_for(B, variant=0):
    """Cloud sizes of a batch: SIZES cycled, runs of empty clouds at the start, in the middle and at the end;
    variant 4 leaves one cloud of 300 points among empty ones."""
    if B == 1:
        return np.array([300], np.int32)
    if B == 2:
        return np.array([33, 300], np.int32)
    if variant == 4:
        L = np.zeros(B, np.int32)
        L[(2 * B) // 3] = 300
        return L
    L = np.array([SIZES[(b + 5 * variant) % len(SIZES)] for b in range(B)], np.int32)
    L[variant:variant + 3] = 0
    L[B // 2 - 1:B // 2 + 2] = 0
    L[-3:] = 0
    return L


def make_batch(lengths, seed):
    """Stacked points for the given cloud sizes: crops and random subsets of the scene, lattice cuts, and exact copies
    of earlier clouds of the same size."""
    rng = np.random.default_rng(seed)
    room, lattice = scene()
    clouds, first_of_size = [], {}
    for b, n in enumerate(int(x) for x in lengths):
        kind = b % 4
        if n == 0:
            c = np.zeros((0, 3), np.float32)
        elif kind == 3 and n in first_of_size:
            c = first_of_size[n].copy()                        # same rows, same order
        elif kind in (1, 2):
            src = lattice if kind == 1 else room
            centre = room[rng.integers(len(room))]
            near = np.argsort(((src - centre) ** 2).sum(1), kind="stable")[:n]
            c = src[rng.permutation(near)]
        else:
            c = room[rng.choice(len(room), n, replace=False)]
        first_of_size.setdefault(n, c)
        clouds.append(c)
    return np.ascontiguousarray(np.concatenate(clouds, 0), np.float32)


@functools.lru_cache(maxsize=None)
def batch(case, variant=0):
    B = int(case.split("_")[0][1:])
    L = lengths_for(B, 4 if case.endswith("lone") else variant)
    return make_batch(L, seed=B * 10 + variant), L


@functools.lru_cache(maxsize=None)
def tail_batch(B, excess):
    """Lengths summing to N + excess. excess < 0: the -excess rows past the last cloud are copies of the last cloud's
    rows (a leak into it shows at equal d2); excess > 0: the last cloud is cut at N."""
    L = lengths_for(B)
    L[-1] = 120
    P = make_batch(L, seed=1000 + B)
    if excess < 0:
        P = np.concatenate([P, P[len(P) - 120:][np.arange(-excess) % 120]], 0)
    elif excess > 0:
        P = P[:len(P) - excess]
    return np.ascontiguousarray(P), L


def clip_lengths(L, n):
    """Lengths cut at n rows: what the rows that belong to a cloud are."""
    start = np.minimum(np.concatenate([[0], np.cumsum(L)]), n)
    return np.diff(start).astype(np.int32)


# ---- oracle -----------------------------------------------------------------------------------------------------------

def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def widen(a, cols, pad):
    """Rows cut or padded to `cols` columns."""
    if a.shape[1] >= cols:
        return a[:, :cols]
    return np.concatenate([a, np.full((a.shape[0], cols - a.shape[1]), pad, np.int32)], 1)


def oracle_neighbors(q, qb, s, sb, r):
    """(rows, counts) of the search over the rows that belong to a cloud. Rows are padded with len(s), as the batch op
    pads; queries of no cloud get count 0 and a row of padding."""
    nq, ns = int(min(qb.sum(), len(q))), int(min(sb.sum(), len(s)))
    rows, cnt = on.port_batch_neighbors(q[:nq], s[:ns], clip_lengths(qb, len(q)), clip_lengths(sb, len(s)), r,
                                        pad_value=len(s), return_counts=True)
    rows = np.concatenate([rows, np.full((len(q) - nq, rows.shape[1]), len(s), np.int32)], 0)
    return rows, np.concatenate([cnt, np.zeros(len(q) - nq, np.int32)])


def oracle_subsampling(P, L, dl):
    n = int(min(L.sum(), len(P)))
    return on.port_batch_subsampling(P[:n], clip_lengths(L, len(P)), dl)


def search_args(P, L, kind):
    """(queries, q_lengths, supports, s_lengths, radius) of the conv, pool and upsample searches of one level."""
    if kind == "conv":
        return P, L, P, L, R
    sp, sb = oracle_subsampling(P, L, DL)
    if kind == "pool":
        return sp, sb, P, L, R
    return P, L, sp, sb, 2 * R


@functools.lru_cache(maxsize=None)
def oracle_case_neighbors(case, kind):
    P, L = batch(case)
    q, qb, s, sb, r = search_args(P, L, kind)
    return oracle_neighbors(q, qb, s, sb, r)


def oracle_pyramid(config, P, L):
    n = int(min(L.sum(), len(P)))
    return ok.descriptor_input_pyramid(config, P[:n], clip_lengths(L, len(P)), LIMITS, on.port_batch_neighbors,
                                       on.port_batch_subsampling)


def expected_pyramid(ref, n0):
    """What the pyramid must hold for a level-0 count n0 (n0 >= the rows that belong to a cloud): the oracle's levels,
    with level-0 rows of no cloud padded, every matrix `limit` wide and padded with its supports' count."""
    sizes = [n0] + [p.shape[0] for p in ref["points"][1:]]
    ref_sizes = [p.shape[0] for p in ref["points"]]

    def rows(a, sup, n_rows, lim):
        a = widen(np.where(a == ref_sizes[sup], sizes[sup], a), lim, sizes[sup])
        return np.concatenate([a, np.full((n_rows - a.shape[0], lim), sizes[sup], np.int32)], 0)

    L = len(sizes)
    exp = dict(sizes=sizes, points=ref["points"], lengths=ref["lengths"], neighbors=[], pools=[], upsamples=[])
    for l in range(L):
        exp["neighbors"].append(rows(ref["neighbors"][l], l, sizes[l], LIMITS[l]))
        if l + 1 < L:
            exp["pools"].append(rows(ref["pools"][l], l, sizes[l + 1], LIMITS[l]))
            exp["upsamples"].append(rows(ref["upsamples"][l], l + 1, sizes[l], LIMITS[l]))
    return exp


def assert_pyramid_rows(got, exp, what):
    """got: per-level numpy arrays cut to the level counts (points, lengths, neighbors, pools, upsamples)."""
    for l in range(len(exp["sizes"])):
        if l > 0:
            assert np.array_equal(bits(got["points"][l]), bits(exp["points"][l])), "%s: points level %d" % (what, l)
            assert np.array_equal(got["lengths"][l], exp["lengths"][l]), "%s: lengths level %d" % (what, l)
        for key in ("neighbors", "pools", "upsamples"):
            if l < len(exp[key]):
                a, b = got[key][l], exp[key][l]
                assert a.shape == b.shape and np.array_equal(a, b), "%s: %s level %d" % (what, key, l)


# ---- device helpers ---------------------------------------------------------------------------------------------------

def t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def poisoned(a, n):
    """a with every row >= n replaced by NaN (even rows) / 1e30 (odd rows)."""
    a = np.array(a, np.float32, copy=True)
    a[n::2] = np.nan
    a[n + 1::2] = 1e30
    return a


@pytest.fixture(scope="module")
def enc(cuda):
    from d3feat_b200 import synth
    from d3feat_b200.encoder import KPFCNN
    cfg = synth.Config(architecture=synth.ARCH_ENCODER)
    return KPFCNN(cfg, synth.make_params(cfg, 0), LIMITS, device=cuda)


def scene_bbox(*clouds, margin=0.05):
    P = np.concatenate(clouds, 0)
    lo, hi = P.min(0), P.max(0)
    ext = hi - lo
    return np.concatenate([lo - margin * ext, hi + margin * ext]).astype(np.float32)


def static_pyramid(enc, P, L, n0, caps, bbox):
    """The static form on buffers whose level-0 rows at or past n0 are poisoned and whose outputs hold a sentinel."""
    from d3feat_b200 import pyramid as pyr
    dev = enc.device
    buf = pyr.PyramidBuffers(enc.config, LIMITS, caps, len(L), dev, bbox=bbox)
    pts0 = np.zeros((buf.caps[0], 3), np.float32)
    pts0[:n0] = P[:n0]
    buf.points0.copy_(t(poisoned(pts0, n0), dev))
    buf.lengths0.copy_(t(L, dev))
    buf.n0.fill_(n0)
    for x in buf.pts[1:] + buf.len[1:] + buf.nb + buf.pool + buf.up:
        if x is not None:
            x.view(torch.int32).fill_(int(SENTINEL))
    st = enc.build_inputs_static(buf)
    torch.cuda.synchronize()
    return buf, st


def read_slot(buf, counts):
    """Per-level numpy rows of a static pyramid's buffers, cut to the level counts."""
    L = len(buf.caps)
    got = dict(points=[None], lengths=[None], neighbors=[], pools=[], upsamples=[])
    for l in range(L):
        n = counts[l]
        if l > 0:
            got["points"].append(buf.pts[l][:n].cpu().numpy())
            got["lengths"].append(buf.len[l].cpu().numpy())
        got["neighbors"].append(buf.nb[l][:n].cpu().numpy())
        if l + 1 < L:
            got["pools"].append(buf.pool[l][:counts[l + 1]].cpu().numpy())
            got["upsamples"].append(buf.up[l][:n].cpu().numpy())
    return got


def assert_tails_untouched(buf, counts):
    L = len(buf.caps)
    for l in range(L):
        tails = [("neighbors", buf.nb[l], counts[l])]
        if l > 0:
            tails.append(("points", buf.pts[l], counts[l]))
        if l + 1 < L:
            tails += [("pools", buf.pool[l], counts[l + 1]), ("upsamples", buf.up[l], counts[l])]
        for what, x, n in tails:
            tail = x[n:].contiguous().view(torch.int32).cpu().numpy()
            assert np.all(tail == SENTINEL), "%s level %d: %d rows past the count written" % (
                what, l, int((tail != SENTINEL).any(-1).sum()))


def check_static(enc, P, L, n0, ref, what):
    from d3feat_b200 import pyramid as pyr
    exp = expected_pyramid(ref, n0)
    buf, st = static_pyramid(enc, P, L, n0, pyr.bucket_capacities(exp["sizes"]), scene_bbox(P[:n0]))
    counts = st["counts"][:5].cpu().tolist()
    assert counts == exp["sizes"], what
    assert int(st["status"].item()) == 0, what
    assert_pyramid_rows(read_slot(buf, counts), exp, what)
    assert_tails_untouched(buf, counts)


# ---- grid subsampling -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dl", [DL, 2 * DL])
@pytest.mark.parametrize("case", CASES)
def test_grid_subsampling_matches_oracle(cuda, case, dl):
    from d3feat_b200 import tf_custom_ops as ops
    P, L = batch(case)
    sp, sb = ops.batch_grid_subsampling(t(P, cuda), t(L, cuda), dl)
    rp, rb = oracle_subsampling(P, L, dl)
    assert np.array_equal(sb.cpu().numpy(), rb)
    assert np.array_equal(bits(sp.cpu().numpy()), bits(rp))


def test_grid_subsampling_features_and_classes_per_cloud(cuda):
    """B = 33 through the cpp_wrappers signature: barycenters, feature means and the largest label of every cell equal
    the oracle run on each cloud alone."""
    from d3feat_b200 import tf_custom_ops as ops
    P, L = batch("B33")
    rng = np.random.default_rng(33)
    F = rng.normal(size=(len(P), 5)).astype(np.float32)
    C = rng.integers(0, 7, (len(P), 2)).astype(np.int32)
    p, b, f, c = ops._subsample(t(P, cuda), t(L, cuda), DL, features=t(F, cuda), classes=t(C, cuda))
    p, b, f, c = p.cpu().numpy(), b.cpu().numpy(), f.cpu().numpy(), c.cpu().numpy()
    i = o = 0
    for cloud, (n, m) in enumerate(zip(L, b)):
        if n == 0:
            assert m == 0, cloud
            continue
        rp, rf, rc = on.port_grid_subsample(P[i:i + n], F[i:i + n], C[i:i + n], sampleDl=DL)
        assert m == len(rp), cloud
        assert np.array_equal(bits(p[o:o + m]), bits(rp)), cloud
        assert np.array_equal(bits(f[o:o + m]), bits(rf)), cloud
        assert np.array_equal(c[o:o + m], rc), cloud
        i, o = i + n, o + m
    assert o == len(p)


# ---- radius neighbours ------------------------------------------------------------------------------------------------

def check_search(q, qb, s, sb, r, ref, cnt, dev):
    """Both forms: the count pass (every count, and the maximum as the exact width) + fill, and capped fills."""
    from d3feat_b200 import tf_custom_ops as ops
    tq, tqb = t(q, dev), t(qb, dev)
    grid = ops.NeighborGrid(t(s, dev), t(sb, dev), r)
    counts, mx = grid.count(tq, tqb)
    assert int(mx.item()) == ref.shape[1]
    assert np.array_equal(counts.cpu().numpy(), cnt)
    assert np.array_equal(grid.fill(tq, tqb, ref.shape[1], len(s)).cpu().numpy(), ref)
    for cols in (CAP, ref.shape[1] + 5):
        assert np.array_equal(grid.fill(tq, tqb, cols, len(s)).cpu().numpy(), widen(ref, cols, len(s))), cols


@pytest.mark.parametrize("halfwarp", ["1", "0"])
@pytest.mark.parametrize("kind", ["conv", "pool", "up"])
@pytest.mark.parametrize("case", CASES)
def test_radius_neighbors_match_oracle(cuda, monkeypatch, case, kind, halfwarp):
    """Conv (queries = supports, r), pool (queries = the subsampled points, r) and upsample (the reverse, 2r), through
    the two-queries-per-warp fill (the default) and the one-query-per-warp fill (D3F_NB_HALFWARP=0)."""
    monkeypatch.setenv("D3F_NB_HALFWARP", halfwarp)
    P, L = batch(case)
    q, qb, s, sb, r = search_args(P, L, kind)
    ref, cnt = oracle_case_neighbors(case, kind)
    check_search(q, qb, s, sb, r, ref, cnt, cuda)


# ---- the input pyramid ------------------------------------------------------------------------------------------------

PYRAMID_CASES = ["B17", "B33", "B300", "B1024"]


@pytest.mark.parametrize("case", PYRAMID_CASES)
def test_exact_pyramid_matches_oracle(enc, case):
    from test_gpu_real_configs import assert_pyramid_equal
    P, L = batch(case)
    inputs = enc.build_inputs(P, L)
    got = {k: [x.cpu().numpy() for x in inputs[k]] for k in ("points", "lengths", "neighbors", "pools", "upsamples")}
    assert_pyramid_equal(got, oracle_pyramid(enc.config, P, L), 5)


@pytest.mark.parametrize("case", PYRAMID_CASES)
def test_static_pyramid_matches_oracle(enc, case):
    """Capacities from bucket_capacities, level-0 rows past n0 poisoned, outputs pre-filled with a sentinel: the counts
    and every row below them equal the oracle, no row at or past a count is written, and no status bit is set."""
    P, L = batch(case)
    check_static(enc, P, L, len(P), oracle_pyramid(enc.config, P, L), case)


def test_graph_pipeline_replays_the_pyramid_exactly(enc, cuda):
    """Five B = 33 batches with different empty and one-point patterns through one captured bucket: after every step
    the pyramid slot the batch used equals the oracle pyramid bit for bit (the captured pyramid replayed with new
    lengths), and the encoder output equals the exact path within 2e-5."""
    from d3feat_b200 import pyramid as pyr
    from d3feat_b200.encoder import GraphPipeline
    from test_gpu_real_configs import rel_err
    batches = [batch("B33", v) for v in range(5)]
    assert len({tuple(L) for _, L in batches}) == 5
    exps = [expected_pyramid(oracle_pyramid(enc.config, P, L), len(P)) for P, L in batches]
    sizes = np.max([e["sizes"] for e in exps], 0).tolist()
    want = [enc(P, L, decoder=False)["F"][-1].cpu().numpy() for P, L in batches]
    pipe = GraphPipeline(enc, pyr.bucket_capacities(sizes), 33, scene_bbox(*[P for P, _ in batches]))
    pipe.prime(t(batches[0][0], cuda), t(batches[0][1], cuda))
    for i, exp in enumerate(exps):
        k = pipe.pending
        nxt = batches[i + 1] if i + 1 < len(batches) else None
        res, counts = pipe.step(t(nxt[0], cuda), t(nxt[1], cuda)) if nxt else pipe.step()
        torch.cuda.synchronize()
        counts = counts[:5].cpu().tolist()
        assert counts == exp["sizes"], i
        assert_pyramid_rows(read_slot(pipe.slots[k], counts), exp, "batch %d" % i)
        n = counts[4]
        assert n == want[i].shape[0]
        assert rel_err(res[:n].cpu().numpy(), want[i]) < 2e-5, i
    pipe.check()


# ---- rows past the last cloud -----------------------------------------------------------------------------------------

# Lengths summing to N - 37, N and N + 37 rows. Short of N: the clouds equal the oracle on the rows that belong to a
# cloud, no row finds a support of no cloud, and a query of no cloud has count 0 and a row of padding. Past N: the last
# cloud is cut at N.
TAILS = [(B, excess) for B in (17, 33) for excess in (-37, 0, 37)]
TAIL_IDS = ["B%d_sum_N%+d" % c for c in TAILS]


@pytest.mark.parametrize("B,excess", TAILS, ids=TAIL_IDS)
def test_rows_past_the_last_cloud_subsampling(cuda, B, excess):
    from d3feat_b200 import tf_custom_ops as ops
    P, L = tail_batch(B, excess)
    assert int(L.sum()) == len(P) + excess
    sp, sb = ops.batch_grid_subsampling(t(P, cuda), t(L, cuda), DL)
    rp, rb = oracle_subsampling(P, L, DL)
    assert np.array_equal(sb.cpu().numpy(), rb)
    assert np.array_equal(bits(sp.cpu().numpy()), bits(rp))


@pytest.mark.parametrize("halfwarp", ["1", "0"])
@pytest.mark.parametrize("kind", ["conv", "pool", "up"])
@pytest.mark.parametrize("B,excess", TAILS, ids=TAIL_IDS)
def test_rows_past_the_last_cloud_neighbors(cuda, monkeypatch, B, excess, kind, halfwarp):
    monkeypatch.setenv("D3F_NB_HALFWARP", halfwarp)
    P, L = tail_batch(B, excess)
    q, qb, s, sb, r = search_args(P, L, kind)
    ref, cnt = oracle_neighbors(q, qb, s, sb, r)
    if excess < 0 and kind != "pool":                      # the queries of no cloud
        assert (ref[len(P) + excess:] == len(s)).all() and not cnt[len(P) + excess:].any()
    check_search(q, qb, s, sb, r, ref, cnt, cuda)


@pytest.mark.parametrize("B,excess", TAILS, ids=TAIL_IDS)
def test_rows_past_the_last_cloud_static_pyramid(enc, B, excess):
    """n0 = N level-0 rows with lengths summing to n0 - 37, n0 and n0 + 37."""
    P, L = tail_batch(B, excess)
    check_static(enc, P, L, len(P), oracle_pyramid(enc.config, P, L), "B%d excess %+d" % (B, excess))


# ---- scene bounds -----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("how", ["translated", "oversized"])
def test_scene_bounds(enc, cuda, how):
    """One cloud moved 40 m out of the bucket's bbox, or scaled to 60 times the bbox's extent. The bbox only bounds the
    width of the subsampling's sort key (cell keys are relative to each cloud's own origin) and the neighbour grid
    clamps coordinates into its edge cells (which only adds candidates), so a moved cloud stays exact and is not
    flagged. An oversized cloud overflows the sort key: status bit 0 in the static form, an error in the exact form."""
    from d3feat_b200 import _lib, pyramid as pyr
    P, L = batch("B33")
    bbox = scene_bbox(P)
    b = int(np.argmax(L == 300))
    s0 = int(L[:b].sum())
    Q = P.copy()
    seg = Q[s0:s0 + 300]
    if how == "translated":
        Q[s0:s0 + 300] = seg + np.float32([40.0, 0.0, -25.0])
    else:
        c = seg.mean(0)
        Q[s0:s0 + 300] = c + (seg - c) * np.float32(60.0)
    ref = oracle_pyramid(enc.config, Q, L)
    exp = expected_pyramid(ref, len(Q))
    caps = pyr.bucket_capacities(exp["sizes"])
    buf, st = static_pyramid(enc, Q, L, len(Q), caps, bbox)
    status = int(st["status"].item())
    if how == "translated":
        assert status == 0
        counts = st["counts"][:5].cpu().tolist()
        assert counts == exp["sizes"]
        assert_pyramid_rows(read_slot(buf, counts), exp, how)
        inputs = enc.build_inputs(Q, L, bbox=bbox)
        got = {k: [x.cpu().numpy() for x in inputs[k]] for k in ("points", "lengths", "neighbors", "pools", "upsamples")}
        assert_pyramid_rows(got, exp, how + " exact form")
    else:
        assert status & 1, status
        with pytest.raises(_lib.D3FError, match="wider than the supplied bbox"):
            enc.build_inputs(Q, L, bbox=bbox)
