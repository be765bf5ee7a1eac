"""GPU: grid subsampling, the radius search and the input pyramid on cell-aligned lattices and clouds far from the origin
(tests/_grid_edge_cases.py), bit for bit against the reference cores (oracle/_ref) and the C port (oracle/d3f_oracle.c).
The reference is compared where it is defined: not on empty clouds for the subsampling, not across an empty cloud for
the search (tests/test_grid_edge_oracle.py); the port everywhere, in the library's own row order.

The data is where fp32 cell arithmetic is on a knife edge: minima one ulp below a multiple of dl (the origin rounds
above the minimum, keys go negative and wrap, ix = -1 aliases into the row below), lattices on and one ulp off the cell
boundaries, offsets up to 10^5 m and millimetre clouds, supports on the search grid's cell boundaries, pairs at fp32
d2 = r2 and one ulp either side, and the longest search-grid axis the library accepts (nbgrid.cuh: kMaxScanAxisCells).
The pyramid, the serving loop and one encoder run see far-offset and aligned clouds; the encoder's KPConv inputs
there are fp32 differences s - q, which this data keeps exact, so the float64 restatement still applies element by
element."""
import numpy as np
import pytest
import torch

import _grid_edge_cases as gc
from oracle import native as on
from test_grid_edge_oracle import canonical, clouds
from test_gpu_many_clouds import (LIMITS, assert_pyramid_rows, check_static, expected_pyramid, oracle_pyramid,
                                  read_slot, scene_bbox)

pytestmark = pytest.mark.gpu

SUB = gc.subsampling_cases()
SEARCH = gc.search_cases()
CAP = 12                                     # capped fill: fewer columns than the dense rows have


def t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def widen(a, cols, pad):
    if a.shape[1] >= cols:
        return a[:, :cols]
    return np.concatenate([a, np.full((a.shape[0], cols - a.shape[1]), pad, np.int32)], 1)


# ---- grid subsampling -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("case", SUB, ids=[c[0] for c in SUB])
def test_tf_batch_subsampling(cuda, case):
    from d3feat_b200 import _lib, tf_custom_ops as ops
    name, P, L, dl, _ = case
    L = np.asarray(L, np.int32)
    if name.startswith("batch"):
        # clouds 2 x 10^5 m apart: the batch's bbox asks for a sort key wider than 62 bits, which is refused. Cell
        # keys are relative to each cloud's own origin, so the widest cloud's extent is all the key width needs.
        with pytest.raises(_lib.D3FError, match="sort key"):
            ops.tf_batch_subsampling(t(P, cuda), t(L, cuda), dl)
        ext = np.max([c.max(0) - c.min(0) for c in clouds(P, L) if len(c)], 0)
        sp, sl = ops.batch_grid_subsampling(t(P, cuda), t(L, cuda), dl, bbox=np.concatenate([0 * ext, ext]))
    else:
        sp, sl = ops.tf_batch_subsampling(t(P, cuda), t(L, cuda), dl)
    sp, sl = sp.cpu().numpy(), sl.cpu().numpy()
    pp, pl = on.port_batch_subsampling(P, L, dl)
    assert np.array_equal(sl, pl), name
    assert np.array_equal(bits(sp), bits(pp)), name
    if on.have_ref():
        keep = [c for c in clouds(P, L) if len(c)]
        rp, rl = on.ref_batch_subsampling(np.concatenate(keep, 0), [len(c) for c in keep], dl)
        assert np.array_equal(rl, sl[L > 0]), name
        for a, b in zip(clouds(rp, rl), clouds(sp, sl[L > 0])):
            assert np.array_equal(canonical(a), canonical(b)), name


@pytest.mark.parametrize("case", SUB, ids=[c[0] for c in SUB])
def test_cpp_subsampling_with_features_and_classes(cuda, case):
    from d3feat_b200 import cpp_subsampling
    name, P, L, dl, _ = case
    for b, c in enumerate(clouds(P, L)):
        if len(c) == 0:
            continue
        F, C = gc.features_and_classes(len(c), b)
        got = cpp_subsampling.compute(c, features=F, classes=C, sampleDl=dl)
        want = on.port_grid_subsample(c, F, C, sampleDl=dl)
        for g, w in zip(got, want):
            assert g.shape == w.shape and np.array_equal(g.view(np.uint32), w.view(np.uint32)), (name, b)
        if on.have_ref():
            assert np.array_equal(canonical(*got), canonical(*on.ref_grid_subsample(c, F, C, sampleDl=dl))), (name, b)


# ---- radius search ----------------------------------------------------------------------------------------------------

def check_search(dev, q, ql, s, sl, r, what):
    """tf_batch_neighbors (count pass + fill), every count, and capped fills, against the port; the rows against the
    reference where it is defined."""
    from d3feat_b200 import tf_custom_ops as ops
    ql, sl = np.asarray(ql, np.int32), np.asarray(sl, np.int32)
    want, cnt = on.port_batch_neighbors(q, s, ql, sl, r, return_counts=True)
    tq, ts, tql, tsl = t(q, dev), t(s, dev), t(ql, dev), t(sl, dev)
    got = ops.tf_batch_neighbors(tq, ts, tql, tsl, r).cpu().numpy()
    assert got.shape == want.shape and np.array_equal(got, want), what
    counts, mx = ops.NeighborGrid(ts, tsl, r).count(tq, tql)
    assert np.array_equal(counts.cpu().numpy(), cnt) and int(mx.item()) == want.shape[1], what
    for cols in (CAP, want.shape[1] + 3):
        capped = ops.batch_ordered_neighbors(tq, ts, tql, tsl, r, max_cols=cols).cpu().numpy()
        assert np.array_equal(capped, widen(want, cols, len(s))), (what, cols)
    if on.have_ref():
        keep = ql > 0
        assert np.array_equal(keep, sl > 0)
        ref, _ = on.canonicalize_neighbors(on.ref_batch_neighbors(q, s, ql[keep], sl[keep], r), q, s, len(s))
        assert np.array_equal(ref, want), what


@pytest.mark.parametrize("halfwarp", ["1", "0"])
@pytest.mark.parametrize("case", SEARCH, ids=[c[0] for c in SEARCH])
def test_tf_batch_neighbors(cuda, monkeypatch, case, halfwarp):
    """Both query kernels: two queries per warp (the default) and one (D3F_NB_HALFWARP=0)."""
    monkeypatch.setenv("D3F_NB_HALFWARP", halfwarp)
    name, q, ql, s, sl, r, _ = case
    check_search(cuda, q, ql, s, sl, r, name)


@pytest.mark.parametrize("halfwarp", ["1", "0"])
@pytest.mark.parametrize("r,offset", [(0.075, 0.0), (0.075, 1e4), (0.75, -1e3)])
def test_longest_accepted_axis_stays_exact(cuda, monkeypatch, r, offset, halfwarp):
    """A 4096-cell axis (the longest the search accepts): rows on the boundaries of its last cells and partners 0.999 r
    away across them. The first axis past it is refused before any launch."""
    from d3feat_b200 import _lib, tf_custom_ops as ops
    monkeypatch.setenv("D3F_NB_HALFWARP", halfwarp)
    p = gc.long_axis_cloud(r, np.random.default_rng(5), offset=offset)
    assert gc.grid_axis_cells(p[:, 0].min(), p[:, 0].max(), r) == gc.MAX_SCAN_AXIS_CELLS
    check_search(cuda, p, [len(p)], p, [len(p)], r, "long axis r=%g" % r)
    c = float(np.float32(np.float32(r) * np.float32(1.001)))
    longer = np.concatenate([p, [[p[:, 0].min() + c * (gc.MAX_SCAN_AXIS_CELLS - 0.5), 0.25, -0.5]]]).astype(np.float32)
    assert gc.grid_axis_cells(longer[:, 0].min(), longer[:, 0].max(), r) == gc.MAX_SCAN_AXIS_CELLS + 1
    with pytest.raises(_lib.D3FError, match="too large"):
        ops.tf_batch_neighbors(t(longer, cuda), t(longer, cuda), t(np.int32([len(longer)]), cuda),
                               t(np.int32([len(longer)]), cuda), r)


# ---- the input pyramid, the serving loop and the encoder --------------------------------------------------------------

@pytest.fixture(scope="module")
def enc(cuda):
    from d3feat_b200 import synth
    from d3feat_b200.encoder import KPFCNN
    cfg = synth.Config(architecture=synth.ARCH_ENCODER)
    return KPFCNN(cfg, synth.make_params(cfg, 0), LIMITS, device=cuda)


def far_batch(offset, seed):
    """Two room fragments and a cloud whose minimum is one ulp below a multiple of 0.06 (the first pooling's dl),
    around `offset`, with an empty and a one-point cloud."""
    from d3feat_b200 import synth
    rng = np.random.default_rng(seed)
    aligned, _ = gc.aligned_cloud(0.06, offset, -1, rng, n_random=200)
    lo = aligned.min(0).astype(np.float64)
    rooms = [(synth.room_fragment(seed + k, n) - synth.room_fragment(seed + k, n).min(0) + lo + 0.4 * k)
             .astype(np.float32) for k, n in ((1, 1500), (2, 900))]
    parts = [rooms[0], np.zeros((0, 3), np.float32), aligned, lo[None].astype(np.float32), rooms[1]]
    return np.ascontiguousarray(np.concatenate(parts, 0)), np.array([len(x) for x in parts], np.int32)


FAR_BATCHES = [(0.0, 1), (123.0, 2), (1e4, 3), (-98765.0, 4)]


@pytest.mark.parametrize("offset,seed", FAR_BATCHES, ids=["off%g" % o for o, _ in FAR_BATCHES])
def test_exact_and_static_pyramid(enc, offset, seed):
    from test_gpu_real_configs import assert_pyramid_equal
    P, L = far_batch(offset, seed)
    if offset >= 0:       # the aligned cloud's origin rounds above its minimum at the first pooling
        assert "wrapped" in gc.conditions(clouds(P, L)[2], 0.06)
    ref = oracle_pyramid(enc.config, P, L)
    inputs = enc.build_inputs(P, L)
    got = {k: [x.cpu().numpy() for x in inputs[k]] for k in ("points", "lengths", "neighbors", "pools", "upsamples")}
    assert_pyramid_equal(got, ref, 5)
    check_static(enc, P, L, len(P), ref, "offset %g" % offset)


def test_graph_pipeline_far_from_the_origin(enc, cuda):
    """Two batches around 10^4 m through one captured bucket whose scene box is there: each step's pyramid slot equals
    the oracle bit for bit, and the encoder output the exact path within 2e-5."""
    from d3feat_b200 import pyramid as pyr
    from d3feat_b200.encoder import GraphPipeline
    from test_gpu_real_configs import rel_err
    batches = [far_batch(1e4, 3), far_batch(1e4, 7)]
    exps = [expected_pyramid(oracle_pyramid(enc.config, P, L), len(P)) for P, L in batches]
    sizes = np.max([e["sizes"] for e in exps], 0).tolist()
    want = [enc(P, L, decoder=False)["F"][-1].cpu().numpy() for P, L in batches]
    box = scene_bbox(*[P for P, _ in batches])
    assert box.min() > 9e3
    pipe = GraphPipeline(enc, pyr.bucket_capacities(sizes), len(batches[0][1]), box)
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


def test_encoder_far_from_the_origin(enc):
    """A batch around 10^4 m through the encoder: every KPConv's fp32 differences s - q are exact (same binade), and
    every traced op equals the float64 restatement element by element (tests/_oracle.assert_close)."""
    from _trace import check_sampled_rows, record_ops
    P, L = far_batch(1e4, 11)
    with record_ops() as tr:
        enc(P, L, decoder=False)
        torch.cuda.synchronize()
    n_kp = 0
    for r in tr.records:
        if r["op"] != "kpconv":
            continue
        q, s, idx = (r[k].cpu().numpy() for k in ("q", "s", "idx"))
        valid = idx < len(s)
        sq = s[np.where(valid, idx, 0)]
        d32 = (sq - q[:, None, :]).astype(np.float32)
        d64 = sq.astype(np.float64) - q[:, None, :].astype(np.float64)
        assert np.array_equal(d32[valid].astype(np.float64), d64[valid]), "inexact s - q"
        n_kp += 1
    assert n_kp > 0
    check_sampled_rows(tr, 256, np.random.default_rng(9), 1e-4, what="encoder at 1e4 m")
