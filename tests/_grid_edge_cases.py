"""Inputs of the grid subsampling and radius search edge tests (shared by the CPU oracle test and the GPU tests).

Both ops decide their result with fp32 cell arithmetic, which is only on a knife edge where points lie on or within an
ulp of a cell boundary, or where the ulp of the coordinates is large (far from the origin). Every case here is fp32
points built from exact fp64 values, so that the edge is hit on purpose:

Grid subsampling (dl as the float32 the ops take, grid_subsampling.cpp of the reference):
  origin  ox = fl(floor(fl(mn * fl(1 / dl))) * dl)      index  floor(fl(fl(x - ox) / dl))
  key     ix + NX * iy + NX * NY * iz  (size_t: a negative index wraps mod 2^64)
* lattices at exact multiples of dl, and the same lattices moved by +-1 ulp;
* clouds whose bbox minimum sits on, one ulp below and one ulp above a multiple of dl. One ulp below, the origin
  rounds ABOVE the minimum: the rows on the minimum get index -1, their key is negative (it wraps to the top of the
  64-bit range in the reference) and ix = -1 aliases into row iy - 1. `geometry` computes all three, and the cases
  built for them say so in `expect` (the tests assert it). Only positive minima can do this: for a negative minimum
  with these voxel sizes fl(mn * fl(1 / dl)) never rounds to the integer that would put the origin above it;
* the same clouds at offsets 10^2 .. 10^5 m either side of the origin, and scaled x1000 with dl x1000 (millimetres);
* batches in which every cloud has its own offset and alignment, with empty and one-point clouds among them;
* random clouds at the same offsets (several points per cell: the barycenter arithmetic).

Radius search (cell edge c = fl(r * 1.001f), index floor(fl(fl(v - mn) * fl(1 / c))), hit iff fp32 d2 < fl(r * r)):
* supports on the search grid's cell boundaries mn + k c and one ulp either side, mn being the supports' bbox minimum;
* pairs whose fp32 d2 is exactly r^2, one ulp below and one ulp above it;
* a long thin box with the largest axis the search accepts (kMaxScanAxisCells in nbgrid.cuh), boundary rows at the
  far end of it.
The radii are the level radii of the reference voxel sizes 0.03, 0.0625 and 0.3 (2.5 dl 2^l).
"""
import numpy as np

f32 = np.float32

DLS = (0.03, 0.06, 0.0625, 0.3)
REF_DLS = (0.03, 0.0625, 0.3)                 # first subsampling of 3DMatch, ETH and KITTI
OFFSETS = (0.0, -7.0, 123.0, 4321.0, -98765.0)
FAR = (1e2, -1e2, 1e3, -1e3, 1e4, -1e4, 1e5, -1e5)
MAX_SCAN_AXIS_CELLS = 4096                    # nbgrid.cuh: kMaxScanAxisCells


def ulps(a, n):
    """a moved by n fp32 ulps (n < 0: down)."""
    a = np.asarray(a, f32)
    for _ in range(abs(int(n))):
        a = np.nextafter(a, f32(np.inf) if n > 0 else f32(-np.inf))
    return a


def jitter(a, rng):
    """Every coordinate moved one ulp up or down at random."""
    a = np.asarray(a, f32)
    return np.nextafter(a, np.where(rng.random(a.shape) < 0.5, f32(-np.inf), f32(np.inf))).astype(f32)


# ---- grid subsampling -------------------------------------------------------------------------------------------------

def geometry(points, dl):
    """The reference's fp32 cell arithmetic on ONE cloud: dict(mn, origin, NX, NY, idx[n, 3], key[n]) with the signed
    key (the reference's size_t key is key mod 2^64)."""
    p = np.asarray(points, f32)
    d = f32(dl)
    inv = f32(1) / d
    mn, mx = p.min(0), p.max(0)
    org = (np.floor(mn * inv) * d).astype(f32)
    NX = int(np.floor((mx[0] - org[0]) / d)) + 1
    NY = int(np.floor((mx[1] - org[1]) / d)) + 1
    idx = np.floor((p - org) / d).astype(np.int64)
    key = idx[:, 0] + NX * idx[:, 1] + NX * NY * idx[:, 2]
    return dict(mn=mn, origin=org, NX=NX, NY=NY, idx=idx, key=key)


def conditions(points, dl):
    """Which knife edges a cloud reaches: origin above the minimum, a wrapped (negative) key, two different cells
    sharing one key (ix = -1 aliasing into the row below)."""
    out = set()
    if len(points) == 0:
        return out
    g = geometry(points, dl)
    if (g["origin"] > g["mn"]).any():
        out.add("origin_above")
    if (g["key"] < 0).any():
        out.add("wrapped")
    cells = {}
    for k, c in zip(g["key"].tolist(), map(tuple, g["idx"].tolist())):
        cells.setdefault(k, set()).add(c)
    if any(len(v) > 1 for v in cells.values()):
        out.add("aliased")
    return out


def multiple(dl, k, scale=1.0):
    """fl32(k * dl) in the op's arithmetic: k times the float32 dl (exact in fp64), rounded once."""
    return f32(k * float(f32(dl * scale)))


def _origin_above(m, dl):
    d = f32(dl)
    return f32(np.floor(f32(m) * (f32(1) / d)) * d) > m


def aligned_min(dl, offset, variant, axis, scale=1.0):
    """(value, origin_above): one coordinate of a bbox minimum near offset * scale, a multiple of dl (variant 0), one
    ulp below (-1) or above (+1). For variant -1 the first of 2000 multiples (away from zero) whose origin rounds above
    the minimum is taken where there is one."""
    d = float(f32(dl * scale))
    k0 = int(np.floor(offset * scale / d)) + 3 * axis
    if variant == -1:
        for k in (range(max(k0, 1), max(k0, 1) + 2000) if offset >= 0 else range(k0, k0 - 2000, -1)):
            m = ulps(multiple(dl, k, scale), -1)
            if _origin_above(m, dl * scale):
                return m, True
    m = ulps(multiple(dl, k0, scale), variant)
    return m, bool(_origin_above(m, dl * scale))


def aligned_cloud(dl, offset, variant, rng, scale=1.0, shape=(7, 6, 4), n_random=150):
    """(points, expect): a lattice of spacing dl from an aligned minimum (every axis) plus random rows inside it;
    expect = all three knife edges where the origin rounds above the minimum on every axis."""
    d = float(f32(dl * scale))
    mins = [aligned_min(dl, offset, variant, a, scale) for a in range(3)]
    mn = np.array([m for m, _ in mins], np.float64)
    ijk = np.stack(np.meshgrid(*[np.arange(n) for n in shape], indexing="ij"), -1).reshape(-1, 3)
    lat = (mn + ijk * d).astype(f32)
    lat[0] = mn.astype(f32)                     # the minimum itself is a row
    extra = (mn + rng.uniform(0.0, 1.0, (n_random, 3)) * (np.array(shape) - 1) * d).astype(f32)
    pts = np.concatenate([lat, extra], 0)
    expect = {"origin_above", "wrapped", "aliased"} if all(a for _, a in mins) else set()
    return np.ascontiguousarray(pts[rng.permutation(len(pts))]), expect


def lattice(dl, offset, rng, jittered=False, shape=(20, 20, 5)):
    ijk = np.stack(np.meshgrid(*[np.arange(n) for n in shape], indexing="ij"), -1).reshape(-1, 3)
    p = (float(f32(offset)) + ijk * float(f32(dl))).astype(f32)
    return jitter(p, rng) if jittered else p


def random_cloud(offset, rng, n=1500, extent=0.5):
    return (float(f32(offset)) + rng.uniform(0.0, extent, (n, 3))).astype(f32)


def subsampling_cases():
    """[(name, points, lengths, dl, expect)]: one cloud per case except the batches; `expect` = the conditions
    (see `conditions`) some cloud of the case is built to reach."""
    rng = np.random.default_rng(2024)
    out = []
    for dl in DLS:
        for off in OFFSETS:
            for jit in (False, True):
                p = lattice(dl, off, rng, jit)
                out.append(("lattice%s-dl%g-off%g" % ("-jit" if jit else "", dl, off), p, [len(p)], dl, set()))
        for off in (0.0, 123.0, 4321.0) + FAR:
            for variant in (-1, 0, 1):
                p, want = aligned_cloud(dl, off, variant, rng)
                out.append(("aligned%+d-dl%g-off%g" % (variant, dl, off), p, [len(p)], dl, want))
        for off in OFFSETS + FAR:
            p = random_cloud(off, rng)
            out.append(("random-dl%g-off%g" % (dl, off), p, [len(p)], dl, set()))
    for dl in REF_DLS:
        for off in (0.0, -7.0, 123.0, 1e2, 1e3):
            for variant in (-1, 0, 1):
                p, want = aligned_cloud(dl, off, variant, rng, scale=1000.0)
                out.append(("mm-aligned%+d-dl%g-off%g" % (variant, dl * 1000, off * 1000), p, [len(p)], dl * 1000.0,
                            want))
    for dl in DLS:
        out.append(batch_case(dl, rng))
    return out


def batch_case(dl, rng):
    """Ten clouds, each with its own offset and alignment, with empty and one-point clouds among them."""
    plan = [(123.0, -1), None, (4321.0, 0), (-98765.0, 1), "one", (1e5, -1), (-7.0, -1), None, (0.0, 1), "one",
            (1e4, -1), None]
    clouds, want = [], set()
    for item in plan:
        if item is None:
            clouds.append(np.zeros((0, 3), f32))
        elif item == "one":
            clouds.append(np.array([[aligned_min(dl, 55.0, -1, a)[0] for a in range(3)]], f32))
        else:
            p, w = aligned_cloud(dl, item[0], item[1], rng, n_random=60)
            clouds.append(p)
            want |= w
    p = np.ascontiguousarray(np.concatenate(clouds, 0))
    return ("batch-dl%g" % dl, p, [len(c) for c in clouds], dl, want)


def features_and_classes(n, seed):
    rng = np.random.default_rng(seed)
    return (rng.normal(size=(n, 4)).astype(f32) * f32(3.0), rng.integers(-3, 9, (n, 2)).astype(np.int32))


# ---- radius search ----------------------------------------------------------------------------------------------------

def level_radii(dl, levels=3):
    return [float(f32(2.5 * dl * 2 ** l)) for l in range(levels)]


RADII = [r for dl in REF_DLS for r in level_radii(dl)]


def search_grid(bbox_min, r):
    """(mn, c, inv) of the search grid: cell edge fl(r * 1.001f), inv = fl(1 / c)."""
    c = f32(f32(r) * f32(1.001))
    return np.asarray(bbox_min, f32), c, f32(1) / c


def cell_position(v, mn, inv):
    """fl(fl(v - mn) * inv): the cell coordinate before the floor."""
    return ((np.asarray(v, f32) - mn) * inv).astype(f32)


def sqdist(q, s):
    d = (np.asarray(q, f32) - np.asarray(s, f32)).astype(f32)
    r = (d[..., 0] * d[..., 0]).astype(f32)
    r = (r + (d[..., 1] * d[..., 1]).astype(f32)).astype(f32)
    return (r + (d[..., 2] * d[..., 2]).astype(f32)).astype(f32)


def boundary_values(mn, c, ks, shifts=(-1, 0, 1)):
    """fl32(mn + k c) and `shifts` ulps either side, for every k."""
    base = (np.float64(mn) + np.asarray(ks, np.float64) * np.float64(c)).astype(f32)
    return np.concatenate([ulps(base, s) for s in shifts])


def boundary_cloud(offset, r, rng, n_cells=24, cube=4):
    """Rows on the cell boundaries of the grid of their own bbox: every axis walks the boundaries of n_cells cells,
    the other two coordinates are boundary values too; plus a dense cube of all boundary triples of `cube` cells (rows
    with many neighbours and exact d2 ties). The first row pins the bbox minimum."""
    mn = np.full(3, f32(offset), f32)
    _, c, _ = search_grid(mn, r)
    vals = boundary_values(mn[0], c, np.arange(1, n_cells + 1))
    walk = np.stack([vals, rng.permutation(vals), rng.permutation(vals)], 1)
    cv = boundary_values(mn[0], c, np.arange(2, 2 + cube))
    dense = np.stack(np.meshgrid(cv, cv, cv, indexing="ij"), -1).reshape(-1, 3)
    pts = np.concatenate([mn[None], walk, dense], 0).astype(f32)
    return np.ascontiguousarray(pts[np.concatenate([[0], 1 + rng.permutation(len(pts) - 1)])])


def d2_pairs(r, unit, n_each=3):
    """[((dx, dy, dz), kind)]: differences whose fp32 d2 is fl(r*r) ('eq'), one ulp below ('below') and one ulp above
    ('above'), all exact multiples of `unit`, the largest ulp of the coordinates (so fl(q - s) is exact). dx and dy run
    over a range, dz is solved for each target and its neighbours tried."""
    r32 = f32(r)
    r2 = f32(r32 * r32)
    n0 = float(r32) / unit
    nx = np.arange(int(0.55 * n0), int(0.55 * n0) + 400, dtype=np.float64)
    dx = (nx[:, None] * unit).astype(f32)
    dy = (nx[None, :] * unit).astype(f32)
    a = ((dx * dx).astype(f32) + (dy * dy).astype(f32)).astype(f32)
    out = []
    for kind, v in (("eq", r2), ("below", ulps(r2, -1)), ("above", ulps(r2, 1))):
        nz0 = np.round(np.sqrt(np.maximum(float(v) - a.astype(np.float64), 0.0)) / unit)
        hits = []
        for dn in (-1, 0, 1):
            dz = ((nz0 + dn) * unit).astype(f32)
            d2 = (a + (dz * dz).astype(f32)).astype(f32)
            for i, j in np.argwhere(d2 == v):
                hits.append((float(dx[i, 0]), float(dy[0, j]), float(dz[i, j])))
        assert len(hits) >= n_each, "no pair with d2 %s r2 for r=%g, unit %g" % (kind, r, unit)
        out += [(hits[i], kind) for i in np.linspace(0, len(hits) - 1, n_each).astype(int)]
    return out


def pair_cloud(offset, r):
    """(queries, supports): isolated pairs 4 r apart along z, query = support + a difference of `d2_pairs`."""
    unit = float(np.spacing(f32(abs(offset) + 2.0 + 40.0 * r)))
    base = np.round((offset + 1.0) / unit) * unit
    step = np.ceil(4 * r / unit) * unit
    q, s = [], []
    for i, (d, _) in enumerate(d2_pairs(r, unit)):
        sp = np.array([base, base, base + i * step], np.float64)
        s.append(sp)
        q.append(sp + np.array(d, np.float64))
    q, s = np.array(q), np.array(s)
    assert np.array_equal(q.astype(f32), q) and np.array_equal(s.astype(f32), s)   # exact: fl(q - s) = q - s
    return q.astype(f32), s.astype(f32)


def search_cases():
    """[(name, queries, q_lengths, supports, s_lengths, radius, expect)], expect from {'on_boundary', 'd2_eq',
    'd2_below', 'd2_above'}."""
    rng = np.random.default_rng(77)
    out = []
    for r in RADII:
        for off in (0.0, 123.0, 4321.0, -98765.0, 1e5):
            p = boundary_cloud(off, r, rng)
            n = len(p)
            two = np.concatenate([p, jitter(p, rng)], 0)
            out.append(("boundary-r%g-off%g" % (r, off), two, [n, 0, n], two, [n, 0, n], r, {"on_boundary"}))
        for off in (0.0, -7.0, 100.0):
            q, s = pair_cloud(off, r)
            out.append(("pairs-r%g-off%g" % (r, off), q, [len(q)], s, [len(s)], r, {"d2_eq", "d2_below", "d2_above"}))
            both = np.concatenate([q, s], 0)
            out.append(("pairs-conv-r%g-off%g" % (r, off), both, [len(both)], both, [len(both)], r,
                        {"d2_eq", "d2_below", "d2_above"}))
    return out


def search_conditions(q, ql, s, sl, r):
    """Which edges a search case reaches: a support on a cell boundary (one fp32 ulp up or down moves the coordinate
    into another cell) and query/support pairs of one cloud at fp32 d2 == r2, one ulp below and one ulp above."""
    q, s = np.asarray(q, f32), np.asarray(s, f32)
    out = set()
    if len(s):
        mn, _, inv = search_grid(s.min(0), r)
        cell = np.floor(cell_position(s, mn, inv))
        for n in (-1, 1):
            if ((np.floor(cell_position(ulps(s, n), mn, inv)) != cell) & (cell > 0)).any():
                out.add("on_boundary")
    r2 = f32(f32(r) * f32(r))
    qs, ss = np.cumsum([0] + list(ql)), np.cumsum([0] + list(sl))
    for b in range(len(ql)):
        d2 = sqdist(q[qs[b]:qs[b + 1], None, :], s[None, ss[b]:ss[b + 1], :])
        for kind, v in (("d2_eq", r2), ("d2_below", ulps(r2, -1)), ("d2_above", ulps(r2, 1))):
            if (d2 == v).any():
                out.add(kind)
    return out


def long_axis_cloud(r, rng, cells=MAX_SCAN_AXIS_CELLS, offset=0.0):
    """A thin box whose x axis has exactly `cells` search-grid cells (n = floor(ext / c) + 2, nbgrid.cuh: make_grid),
    with rows on the boundaries of the last 40 cells, one ulp either side, and pairs at d2 just below r2 straddling
    them."""
    mn = np.array([offset, 0.25, -0.5], f32)
    _, c, _ = search_grid(mn, r)
    ks = np.arange(cells - 42, cells - 2)
    xs = boundary_values(mn[0], c, ks)
    yz = np.array([0.25, -0.5], np.float64)
    rows = [mn[None].astype(np.float64)]
    rows.append(np.stack([xs, np.full(len(xs), yz[0] + 0.3 * c), np.full(len(xs), yz[1] + 0.2 * c)], 1))
    # partners at x - 0.999 r and x + 0.999 r: inside r, on the far side of the neighbouring cell boundary
    part = np.asarray(xs[::3], np.float64)
    for sgn in (-1.0, 1.0):
        rows.append(np.stack([part + sgn * 0.999 * float(f32(r)), np.full(len(part), yz[0] + 0.3 * c),
                              np.full(len(part), yz[1] + 0.2 * c)], 1))
    pts = np.concatenate(rows, 0).astype(f32)
    ext = float(pts[:, 0].max()) - float(pts[:, 0].min())
    hi = mn.astype(np.float64) + float(c) * (cells - 2) + float(c) * 0.5     # last axis cell of the box
    pts = np.concatenate([pts, np.array([[hi[0], yz[0], yz[1]]], f32)], 0)
    return np.ascontiguousarray(pts[np.concatenate([[0], 1 + rng.permutation(len(pts) - 1)])])


def grid_axis_cells(lo, hi, r):
    """Cells of one axis of the search grid over [lo, hi] (nbgrid.cuh: make_grid, in its own arithmetic)."""
    c = f32(f32(r) * f32(1.001))
    ext = float(f32(hi)) - float(f32(lo))
    return int(np.floor(ext / float(c)) + 2.0)
