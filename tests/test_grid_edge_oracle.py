"""CPU: grid subsampling and the radius search on cell-aligned lattices and clouds far from the origin
(tests/_grid_edge_cases.py), in three restatements that must agree bit for bit -- the compiled reference cores
(cpp_wrappers and the TF batch ops), the C port (oracle/d3f_oracle.c) and a plain-Python dict loop below -- and the
proof that the data tells the contract from its plausible mistakes: every emulated arithmetic slip changes the result
of some case. Last, the search grid's completeness bound (nbgrid.cuh: kMaxScanAxisCells): the longest grid axis the
library accepts, and the first one past it refused before any launch."""
import ctypes
import math

import numpy as np
import pytest

import _grid_edge_cases as gc
from oracle import native as on

f32 = np.float32
SUB = gc.subsampling_cases()
SEARCH = gc.search_cases()


def clouds(points, lengths):
    start = np.concatenate([[0], np.cumsum(lengths)]).astype(int)
    return [points[start[b]:start[b + 1]] for b in range(len(lengths))]


def bits(a):
    return np.ascontiguousarray(a, f32).view(np.uint32)


def canonical(*cols):
    """Rows of the column blocks (points, features, classes) sorted by their bit patterns, for comparing outputs whose
    row order is an implementation artefact (the reference's unordered_map)."""
    rows = np.concatenate([np.ascontiguousarray(c).reshape(len(c), -1).view(np.uint32) for c in cols], 1)
    return rows[np.lexsort(rows.T[::-1])] if len(rows) else rows


def dict_grid_subsample(points, dl, features=None, classes=None, bug=None):
    """One cloud in the reference's arithmetic, one fp32 rounding per operation, cells in a dict keyed by the 64-bit
    key and emitted in ascending key. `bug` replaces one step by a plausible mistake:
      reciprocal     index = floor(fl(x - ox) * fl(1 / dl)) instead of / dl
      origin_fp64    origin floor(mn / dl) * dl evaluated in fp64 (then stored as float)
      fma            index = floor(fma(x, inv, -fl(ox * inv)))  ((x - ox) * inv expanded and contracted)
      clamp          negative keys clamped to 0 instead of wrapping mod 2^64
      divide         barycenter sum / count instead of sum * (float)(1.0 / count)"""
    p = np.asarray(points, f32)
    d = f32(dl)
    inv = f32(1) / d
    mn, mx = p.min(0), p.max(0)
    if bug == "origin_fp64":
        org = np.array([f32(math.floor(float(m) / float(d)) * float(d)) for m in mn], f32)
    else:
        org = np.floor(mn * inv) * d

    def index(v):
        v = np.asarray(v, f32)
        if bug == "reciprocal":
            return np.floor((v - org) * inv).astype(np.int64)
        if bug == "fma":
            c = (org * inv).astype(f32)
            return np.floor((v.astype(np.float64) * float(inv) - c.astype(np.float64)).astype(f32)).astype(np.int64)
        return np.floor((v - org) / d).astype(np.int64)

    NX, NY = (int(x) + 1 for x in index(mx)[:2])
    cells = {}
    for i, ijk in enumerate(index(p).tolist()):
        k = ijk[0] + NX * ijk[1] + NX * NY * ijk[2]
        k = max(k, 0) if bug == "clamp" else k % 2 ** 64
        c = cells.setdefault(k, dict(s=[f32(0)] * 3, n=0, f=None, l=None))
        c["s"] = [c["s"][a] + p[i, a] for a in range(3)]
        c["n"] += 1
        if features is not None:
            c["f"] = features[i].copy() if c["f"] is None else (c["f"] + features[i]).astype(f32)
        if classes is not None:
            c["l"] = classes[i].copy() if c["l"] is None else np.maximum(c["l"], classes[i])
    out_p, out_f, out_l = [], [], []
    for k in sorted(cells):
        c = cells[k]
        if bug == "divide":
            out_p.append([s / f32(c["n"]) for s in c["s"]])
        else:
            r = f32(1.0 / c["n"])
            out_p.append([s * r for s in c["s"]])
        if features is not None:
            out_f.append((c["f"] / f32(c["n"])).astype(f32))
        if classes is not None:
            out_l.append(c["l"])
    out = [np.array(out_p, f32).reshape(-1, 3)]
    if features is not None:
        out.append(np.array(out_f, f32).reshape(-1, features.shape[1]))
    if classes is not None:
        out.append(np.array(out_l, np.int32).reshape(-1, classes.shape[1]))
    return out


def port(c, dl, features=None, classes=None):
    if len(c) == 0:
        return [np.zeros((0, 3), f32)]
    out = on.port_grid_subsample(c, features, classes, sampleDl=dl)
    return list(out) if isinstance(out, tuple) else [out]


def same(a, b):
    return len(a) == len(b) and all(x.shape == y.shape and np.array_equal(x.view(np.uint32), y.view(np.uint32))
                                    for x, y in zip(a, b))


ref = pytest.mark.skipif(not on.have_ref(), reason="reference cores not built (oracle/_ref)")


# ---- the cases reach the edges they were built for --------------------------------------------------------------------

@pytest.mark.parametrize("case", SUB, ids=[c[0] for c in SUB])
def test_subsampling_case_reaches_its_edges(case):
    name, points, lengths, dl, expect = case
    got = set()
    for c in clouds(points, lengths):
        got |= gc.conditions(c, dl)
    assert expect <= got, (name, expect - got)


def test_subsampling_cases_cover_every_edge():
    """Origin above the minimum, a wrapped key and an aliased row, in single clouds and batches, near the origin, far
    from it (10^5 m) and in millimetres; batches with empty and one-point clouds."""
    built = {n for n, *_, e in SUB if {"origin_above", "wrapped", "aliased"} <= e}
    for name in ("aligned-1-dl0.03-off0", "aligned-1-dl0.06-off100000", "aligned-1-dl0.3-off10000",
                 "mm-aligned-1-dl30-off123000", "batch-dl0.03", "batch-dl0.3"):
        assert name in built, name
    for name, _, lengths, *_ in SUB:
        if name.startswith("batch"):
            assert 0 in lengths and 1 in lengths


@pytest.mark.parametrize("case", SEARCH, ids=[c[0] for c in SEARCH])
def test_search_case_reaches_its_edges(case):
    name, q, ql, s, sl, r, expect = case
    assert expect <= gc.search_conditions(q, ql, s, sl, r), name


# ---- three restatements agree -----------------------------------------------------------------------------------------

@pytest.mark.parametrize("case", SUB, ids=[c[0] for c in SUB])
def test_dict_restatement_equals_the_port(case):
    name, points, lengths, dl, _ = case
    for b, c in enumerate(clouds(points, lengths)):
        if len(c) == 0:
            continue
        F, C = gc.features_and_classes(len(c), b)
        assert same(dict_grid_subsample(c, dl, F, C), port(c, dl, F, C)), (name, b)


@ref
@pytest.mark.parametrize("case", SUB, ids=[c[0] for c in SUB])
def test_port_equals_the_reference_cores(case):
    """cpp_wrappers (points, features, classes) and the TF ops (one cloud, and the batch op) against the port, rows
    compared in a canonical order. The reference cores are not defined on an empty cloud: those are left out of the
    batch op's input, and their count is checked to be 0 in the port."""
    name, points, lengths, dl, _ = case
    keep = []
    for b, c in enumerate(clouds(points, lengths)):
        if len(c) == 0:
            continue
        keep.append(c)
        F, C = gc.features_and_classes(len(c), b)
        want = port(c, dl, F, C)
        got = on.ref_grid_subsample(c, F, C, sampleDl=dl)
        assert np.array_equal(canonical(*got), canonical(*want)), (name, b, "cpp_wrappers")
        assert np.array_equal(canonical(on.ref_grid_subsampling_tf(c, dl)), canonical(want[0])), (name, b, "tf")
    pts, lens = np.concatenate(keep, 0), [len(c) for c in keep]
    rp, rl = on.ref_batch_subsampling(pts, lens, dl)
    pp, pl = on.port_batch_subsampling(points, lengths, dl)
    assert np.array_equal(rl, pl[np.asarray(lengths) > 0]) and not pl[np.asarray(lengths) == 0].any(), name
    for a, b in zip(clouds(rp, rl), clouds(pp, pl[np.asarray(lengths) > 0])):
        assert np.array_equal(canonical(a), canonical(b)), (name, "tf batch")


@ref
@pytest.mark.parametrize("case", SEARCH, ids=[c[0] for c in SEARCH])
def test_search_port_equals_the_reference(case):
    """The TF batch search (nanoflann) against the port, every row in the canonical (d2, index) order. The reference
    is not defined across an empty cloud (it finds nothing for the clouds after one), so empty clouds are left out of
    its input; that changes no row index."""
    name, q, ql, s, sl, r, _ = case
    ql, sl = np.asarray(ql), np.asarray(sl)
    assert np.array_equal(ql == 0, sl == 0)
    ql, sl = ql[ql > 0], sl[sl > 0]
    want = on.port_batch_neighbors(q, s, ql, sl, r)
    got, _ = on.canonicalize_neighbors(on.ref_batch_neighbors(q, s, ql, sl, r), q, s, len(s))
    assert got.shape == want.shape and np.array_equal(got, want), name


# ---- sensitivity: the data catches every plausible slip ---------------------------------------------------------------

SUB_BUGS = ["reciprocal", "origin_fp64", "fma", "clamp", "divide"]


@pytest.mark.parametrize("bug", SUB_BUGS)
def test_subsampling_cases_catch_a_wrong_step(bug):
    caught = []
    for name, points, lengths, dl, expect in SUB:
        for c in clouds(points, lengths):
            if len(c) and not same(dict_grid_subsample(c, dl, bug=bug), port(c, dl)):
                caught.append(name)
                break
    assert caught, "no case changes under %s" % bug
    if bug in ("origin_fp64", "clamp"):        # only the clouds whose origin rounds above the minimum can tell
        assert any(n.startswith(("aligned-1", "mm-aligned-1", "batch")) for n in caught), caught


def search_hits(q, ql, s, sl, r, bug=None):
    """Per query, the sorted support indices with d2 < r2 -- or, under `bug`, d2 with FMA ('fma') or d2 <= r2
    ('le')."""
    r2 = f32(f32(r) * f32(r))
    qs, ss = np.cumsum([0] + list(ql)), np.cumsum([0] + list(sl))
    out = []
    for b in range(len(ql)):
        qq, sv = q[qs[b]:qs[b + 1], None, :], s[None, ss[b]:ss[b + 1], :]
        if bug == "fma":       # r = dx*dx; r = fma(dy, dy, r); r = fma(dz, dz, r)
            d = (qq - sv).astype(f32).astype(np.float64)
            d2 = (d[..., 0] * d[..., 0]).astype(f32)
            d2 = (d[..., 1] * d[..., 1] + d2.astype(np.float64)).astype(f32)
            d2 = (d[..., 2] * d[..., 2] + d2.astype(np.float64)).astype(f32)
        else:
            d2 = gc.sqdist(qq, sv)
        hit = d2 <= r2 if bug == "le" else d2 < r2
        out += [tuple(ss[b] + np.flatnonzero(h)) for h in hit]
    return out


@pytest.mark.parametrize("bug", ["fma", "le"])
def test_search_cases_catch_a_wrong_distance_test(bug):
    caught = [name for name, q, ql, s, sl, r, _ in SEARCH if name.startswith("pairs")
              and search_hits(q, ql, s, sl, r, bug) != search_hits(q, ql, s, sl, r)]
    assert caught, "no pair case changes under %s" % bug


def test_search_hits_restate_the_port():
    """search_hits (the contract the bugs are measured against) is the port's hit set."""
    for name, q, ql, s, sl, r, _ in SEARCH:
        if name.startswith("pairs"):
            rows, cnt = on.port_batch_neighbors(q, s, ql, sl, r, return_counts=True)
            want = [tuple(sorted(row[:n])) for row, n in zip(rows.tolist(), cnt)]
            assert search_hits(q, ql, s, sl, r) == want, name


# ---- the search grid's completeness bound -----------------------------------------------------------------------------

@pytest.fixture(scope="module")
def abi():
    from d3feat_b200 import _lib, build
    build.build()
    return _lib.lib()


def axis_bbox(cells, r, offset=0.0):
    """A thin bbox whose x axis has exactly `cells` search-grid cells."""
    c = float(f32(f32(r) * f32(1.001)))
    lo = f32(offset)
    hi = f32(float(lo) + (cells - 1.5) * c)
    assert gc.grid_axis_cells(lo, hi, r) == cells
    return (ctypes.c_float * 6)(float(lo), 0.0, 0.0, float(hi), 0.1, 0.1)


@pytest.mark.parametrize("r", [0.075, 0.15625, 0.75])
def test_the_longest_complete_axis_is_accepted_and_the_next_refused(abi, r):
    """4096 cells on one axis (about 307 m at r = 0.075) get a workspace; 4097 get none, and every entry point refuses
    them with an invalid-argument error before any CUDA call (the fake pointers are never dereferenced)."""
    fake = ctypes.c_void_p(256)
    ok = axis_bbox(gc.MAX_SCAN_AXIS_CELLS, r, 1e4)
    past = axis_bbox(gc.MAX_SCAN_AXIS_CELLS + 1, r, 1e4)
    assert abi.d3f_radius_neighbors_workspace_bytes(1000, 2, r, ok) > 0
    assert abi.d3f_radius_neighbors_workspace_bytes(1000, 2, r, past) == 0
    calls = [
        lambda: abi.d3f_radius_neighbors_build(fake, fake, 2, 1000, r, past, fake, 1 << 40, None),
        lambda: abi.d3f_radius_neighbors_count(fake, fake, 1000, fake, fake, 2, 1000, r, past, fake, fake, fake, None),
        lambda: abi.d3f_radius_neighbors_fill(fake, fake, 1000, fake, fake, 2, 1000, r, past, fake, 8, 1000, fake,
                                              None),
    ]
    for call in calls:
        assert call() == -1
        assert b"axis longer than 4096 cells" in abi.d3f_last_error()


def test_long_axis_case_is_the_longest_accepted_axis():
    for r in (0.075, 0.75):
        p = gc.long_axis_cloud(r, np.random.default_rng(0))
        assert gc.grid_axis_cells(p[:, 0].min(), p[:, 0].max(), r) == gc.MAX_SCAN_AXIS_CELLS
        assert "on_boundary" in gc.search_conditions(p, [len(p)], p, [len(p)], r)
