"""Point-to-point ICP on the GPU (d3f_icp_pairs, registration.icp_pairs, GraphPipeline(..., icp=...)) against the
numpy restatement oracle/icp_np.py.

Every comparison is exact: pose, fitness and inlier_rmse as int64 bit patterns, n_correspondences and iterations as
integers. The contract is fp64 without FMA in a fixed blocked order, so a contracted multiply-add, a different
reduction order or a different nearest row shows up in the bits."""
import numpy as np
import pytest

from oracle import icp_np

FIELDS = ("pose", "fitness", "inlier_rmse", "n_correspondences", "iterations")


def t(a, dev):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def mismatches(got, want):
    bad = []
    for f in FIELDS:
        g, w = np.asarray(got[f]), np.asarray(want[f])
        if g.dtype == np.float64:
            g, w = g.view(np.int64), w.view(np.int64)
        if g.shape != w.shape or not np.array_equal(g, w):
            bad.append(f)
    return bad


def as_numpy(ref):
    return {f: getattr(ref, f).cpu().numpy() for f in FIELDS}


def rotation(axis, deg):
    axis = np.asarray(axis, float)
    axis = axis / np.linalg.norm(axis)
    th = np.deg2rad(deg)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K


def rigid(R, tr):
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, tr
    return T


def perturbed(rng, T, deg=2.0, shift=0.03):
    d = rng.normal(size=3)
    return rigid(rotation(rng.normal(size=3), deg), shift * d / np.linalg.norm(d)) @ T


def moved_copy(rng, pts, keep=0.8, noise=0.002, deg=10.0):
    """A rigid copy of the part of `pts` below a random plane (fraction `keep`), with noise: (copy, true pose)."""
    T = rigid(rotation(rng.normal(size=3), deg), rng.uniform(-0.2, 0.2, 3))
    d = rng.normal(size=3)
    proj = pts @ d
    part = pts[proj <= np.quantile(proj, keep)] if len(pts) else pts
    out = part @ T[:3, :3].T + T[:3, 3] + rng.normal(scale=noise, size=part.shape)
    return out.astype(np.float32), T


def bbox_of(pts, margin=0.05):
    lo, hi = pts.min(0), pts.max(0)
    ext = np.maximum(hi - lo, 1e-3)
    return np.concatenate([lo - margin * ext, hi + margin * ext]).astype(np.float32)


def icp_raw(dev, points, lengths, pairs, init, bbox, *, distance, max_iterations=30, relative_fitness=1e-6,
            relative_rmse=1e-6, rows=None):
    """The entry point itself, on outputs filled with sentinels: every element must be written."""
    import torch
    from d3feat_b200 import _lib
    lib = _lib.lib()
    points = np.asarray(points, np.float32).reshape(-1, 3)
    N, B, P = points.shape[0], len(lengths), len(pairs)
    tp, tl, tq, ti = (t(a, dev) for a in (points, np.asarray(lengths, np.int32), np.asarray(pairs, np.int32),
                                           np.asarray(init, np.float64)))
    tr = None if rows is None else t(np.array([rows], np.int32), dev)
    pose = torch.full((P, 4, 4), 7.0, dtype=torch.float64, device=dev)
    fit, rmse = (torch.full((P,), 7.0, dtype=torch.float64, device=dev) for _ in range(2))
    nc, it = (torch.full((P,), 7, dtype=torch.int32, device=dev) for _ in range(2))
    bb = np.ascontiguousarray(bbox, np.float32)
    bbp = bb.ctypes.data_as(_lib.C.c_void_p)
    ws = _lib.workspace(lib.d3f_icp_pairs_workspace_bytes(N, B, P, distance, bbp), dev)
    _lib.check(lib.d3f_icp_pairs(_lib.ptr(tp), _lib.ptr(tl), B, N, _lib.ptr(tr), bbp, _lib.ptr(tq), P, _lib.ptr(ti),
                                 distance, max_iterations, relative_fitness, relative_rmse, _lib.ptr(pose),
                                 _lib.ptr(fit), _lib.ptr(rmse), _lib.ptr(nc), _lib.ptr(it), _lib.ptr(ws), ws.numel(),
                                 _lib.stream()),
               "d3f_icp_pairs")
    return dict(pose=pose.cpu().numpy(), fitness=fit.cpu().numpy(), inlier_rmse=rmse.cpu().numpy(),
                n_correspondences=nc.cpu().numpy(), iterations=it.cpu().numpy())


def check(dev, points, lengths, pairs, init, bbox, **kw):
    got = icp_raw(dev, points, lengths, pairs, init, bbox, **kw)
    want = icp_np.icp(points, lengths, pairs, init, **kw)
    assert mismatches(got, want) == []
    return want


# ---- 1. cloud sizes 0 .. 30000, inits near / far / identity, I in {0, 1, 30, 200} -------------------------------

def mixed_batch(seed):
    """Clouds of 30000, 5000, 0, 1, 2, 3 and 100 points with moved partial copies, and pairs between them."""
    from d3feat_b200 import synth
    rng = np.random.default_rng(seed)
    big = synth.room_fragment(seed, 30000)
    mid = synth.room_fragment(seed + 1, 5000)
    big2, Tb = moved_copy(rng, big)
    mid2, Tm = moved_copy(rng, mid)
    clouds = [big, big2, mid, mid2, np.zeros((0, 3), np.float32), mid[:1], mid[:2], mid[:3], mid[100:200]]
    far = rigid(rotation([0, 0, 1], 90), [1.0, 0.5, 0.0]) @ Tm
    pairs = [(0, 1, perturbed(rng, Tb)), (1, 0, np.linalg.inv(perturbed(rng, Tb))), (2, 3, perturbed(rng, Tm)),
             (2, 3, np.eye(4)), (2, 3, far), (4, 1, Tb), (0, 4, Tb), (5, 3, Tm), (6, 3, Tm), (7, 3, Tm),
             (8, 3, perturbed(rng, Tm)), (3, 8, np.linalg.inv(Tm)), (3, 2, np.linalg.inv(perturbed(rng, Tm, 1, 0.01)))]
    pts = np.concatenate(clouds).astype(np.float32)
    return pts, [len(c) for c in clouds], [p[:2] for p in pairs], np.stack([p[2] for p in pairs])


@pytest.mark.gpu
@pytest.mark.parametrize("I", [0, 1, 30, 200])
def test_icp_pairs_against_oracle(cuda, I):
    pts, lens, pairs, init = mixed_batch(40 + I)
    want = check(cuda, pts, lens, pairs, init, bbox_of(pts), distance=0.05, max_iterations=I)
    if I >= 30:
        assert want["iterations"][0] > 1 and want["fitness"][0] > 0.5
        assert (want["iterations"][5:7] == 0).all() and (want["n_correspondences"][5:7] == 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("thresholds,expect", [(0.0, "all"), (1e9, "one")])
def test_icp_pairs_thresholds(cuda, thresholds, expect):
    """Thresholds 0 never stop a pair early; huge thresholds stop every pair after its first update."""
    pts, lens, pairs, init = mixed_batch(7)
    keep = [2, 3, 4, 10, 11, 12]
    pairs, init = [pairs[i] for i in keep], init[keep]
    want = check(cuda, pts, lens, pairs, init, bbox_of(pts), distance=0.05, max_iterations=12,
                 relative_fitness=thresholds, relative_rmse=thresholds)
    live = want["n_correspondences"] >= 3
    assert live.any()
    assert (want["iterations"][live] == (12 if expect == "all" else 1)).all()


# ---- 2. lattices: equidistant targets (the tie rule) and targets exactly at the distance (the strict rule) ----------

def lattice_pair(h=0.25):
    """Source and target on one lattice of spacing h (exact in fp32). Unshifted, the source rows at x = 0 have their
    nearest target exactly at h, and rows moved by h / 2 along x or along x and y are equidistant from two or four
    targets (exact d^2 ties)."""
    g = np.stack(np.meshgrid(*[np.arange(6) * h] * 3, indexing="ij"), -1).reshape(-1, 3)
    src = np.concatenate([g, g[:40] + [h / 2, 0, 0], g[60:80] + [h / 2, h / 2, 0]]).astype(np.float32)
    tgt = (g + [h, 0, 0]).astype(np.float32)
    return src, tgt


@pytest.mark.gpu
@pytest.mark.parametrize("distance,shift,I", [(0.25, 0.0, 0), (0.25, 0.0, 3), (0.2, 0.25, 3), (0.25, 0.125, 5)])
def test_icp_pairs_lattice_ties_and_strict_distance(cuda, distance, shift, I):
    src, tgt = lattice_pair()
    pts = np.concatenate([src, tgt])
    init = rigid(np.eye(3), [shift, 0, 0])[None]
    check(cuda, pts, [len(src), len(tgt)], [(0, 1)], init, bbox_of(pts), distance=distance, max_iterations=I)


# ---- 3. NaN init, clouds outside host_bbox, pairs naming clouds outside [0, B) ------------------------------------

@pytest.mark.gpu
def test_icp_pairs_nan_init_outside_bbox_and_bad_pair_ids(cuda):
    from d3feat_b200 import synth
    rng = np.random.default_rng(3)
    a = synth.room_fragment(3, 3000)
    b, T = moved_copy(rng, a)
    box = bbox_of(np.concatenate([a, b]))
    far_a, far_b = a + np.float32(40.0), b + np.float32(40.0)          # 40 m outside the bbox
    pts = np.concatenate([a, b, far_a, far_b])
    shift = rigid(np.eye(3), [40.0, 40.0, 40.0])
    far_init = shift @ perturbed(rng, T) @ np.linalg.inv(shift)      # the same perturbation, about the moved cloud
    nan = np.full((4, 4), np.nan)
    pairs = [(0, 1), (2, 3), (0, 1), (-1, 1), (0, 4), (4, 0), (1 << 30, 0)]
    init = np.stack([perturbed(rng, T), far_init, nan, T, T, T, T])
    lens = [len(a), len(b), len(far_a), len(far_b)]
    want = check(cuda, pts, lens, pairs, init, box, distance=0.05, max_iterations=30)
    assert want["fitness"][1] > 0.5 and want["iterations"][1] > 1
    for p in range(2, 7):
        assert want["iterations"][p] == 0 and want["n_correspondences"][p] == 0, p


# ---- 4. up to 1024 clouds, lengths summing short of the row count, NaN garbage past it ----------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("B", [33, 1024])
def test_icp_pairs_many_clouds_and_row_counts(cuda, B):
    rng = np.random.default_rng(B)
    clouds, pairs, init = [], [], []
    for i in range(B // 2):
        n = int(rng.integers(0, 70))
        src = rng.uniform(0, 1, (n, 3)).astype(np.float32)
        tgt, T = moved_copy(rng, src, keep=0.9, noise=0.001, deg=5)
        clouds += [src, tgt]
        pairs.append((2 * i, 2 * i + 1))
        init.append(perturbed(rng, T, 1, 0.01))
    if B % 2:
        clouds.append(rng.uniform(0, 1, (5, 3)).astype(np.float32))
    pairs += [(0, B - 1), (B - 1, 1), (B, 0), (-1, 2)]
    init += [np.eye(4)] * 4
    lens = [len(c) for c in clouds]
    real = np.concatenate(clouds)
    extra = rng.uniform(0, 1, (37, 3)).astype(np.float32)                 # rows of no cloud, before the row count
    rows = len(real) + len(extra)
    box = bbox_of(np.concatenate([real, extra]))
    outs = []
    for garbage in (np.nan, 0.5):
        pts = np.concatenate([real, extra, np.full((300, 3), garbage, np.float32)])
        got = icp_raw(cuda, pts, lens, pairs, np.stack(init), box, distance=0.1, max_iterations=20, rows=rows)
        outs.append(got)
    assert mismatches(outs[0], outs[1]) == []
    want = icp_np.icp(np.concatenate([real, extra]), lens, pairs, np.stack(init), distance=0.1, max_iterations=20)
    assert mismatches(outs[0], want) == []
    # the last cloud cut by the row count: lengths summing past it
    cut = len(real) - 7
    got = icp_raw(cuda, np.concatenate([real, np.full((50, 3), np.nan, np.float32)]), lens, pairs, np.stack(init), box,
                  distance=0.1, max_iterations=20, rows=cut)
    want = icp_np.icp(real, lens, pairs, np.stack(init), distance=0.1, max_iterations=20, rows=cut)
    assert mismatches(got, want) == []


# ---- 5. registration.icp_pairs (KITTI-like scan pair) and a captured graph -------------------------------------------

@pytest.mark.gpu
def test_icp_pairs_python_api_and_cuda_graph(cuda):
    import torch
    from d3feat_b200 import synth
    from d3feat_b200.registration import icp_pairs
    rng = np.random.default_rng(9)
    a = synth.lidar_scan(2, 16000, dl=0.30)
    b, T = moved_copy(rng, a, keep=0.9, noise=0.01, deg=3)
    pts = np.concatenate([a, b])
    lens = np.array([len(a), len(b)], np.int32)
    init = perturbed(rng, T)[None]
    box = bbox_of(pts)
    want = icp_np.icp(pts, lens, [(0, 1)], init, distance=0.2, max_iterations=200)
    assert want["fitness"][0] > 0.5
    tp, tl, ti = t(pts, cuda), t(lens, cuda), t(init, cuda)
    assert mismatches(as_numpy(icp_pairs(tp, tl, [(0, 1)], ti, distance=0.2, max_iterations=200, bbox=box)), want) == []
    assert mismatches(as_numpy(icp_pairs(tp, tl, [(0, 1)], init, distance=0.2, max_iterations=200)),
                      icp_np.icp(pts, lens, [(0, 1)], init, distance=0.2, max_iterations=200)) == []
    with pytest.raises(ValueError, match="outside"):
        icp_pairs(tp, tl, [(0, 2)], init, distance=0.2)
    # a graph captured once and replayed on inputs rewritten in place
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    pairs = t(np.array([[0, 1], [1, 0]], np.int32), cuda)
    init2 = t(np.stack([init[0], np.linalg.inv(init[0])]), cuda)
    with torch.cuda.stream(s):
        icp_pairs(tp, tl, pairs, init2, distance=0.2, max_iterations=40, bbox=box)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ref = icp_pairs(tp, tl, pairs, init2, distance=0.2, max_iterations=40, bbox=box)
    for trial in range(2):
        b2, T2 = moved_copy(rng, a, keep=0.85, noise=0.01, deg=3)
        pts2 = np.concatenate([a, b2[:len(b)], np.zeros((max(0, len(b) - len(b2)), 3), np.float32)])
        lens2 = np.array([len(a), min(len(b), len(b2))], np.int32)
        i2 = np.stack([perturbed(rng, T2), np.linalg.inv(perturbed(rng, T2))])
        tp.copy_(t(pts2, cuda))
        tl.copy_(t(lens2, cuda))
        init2.copy_(t(i2, cuda))
        g.replay()
        torch.cuda.synchronize()
        want = icp_np.icp(pts2, lens2, [(0, 1), (1, 0)], i2, distance=0.2, max_iterations=40)
        assert mismatches(as_numpy(ref), want) == [], trial


# ---- 6. GraphPipeline(..., register={}, icp=...) -------------------------------------------------------------------

LIMITS = [35, 33, 34, 36, 30]


@pytest.mark.gpu
def test_graph_pipeline_icp(cuda):
    """Five batches of three clouds through one captured bucket. Each step's refinement equals an eager icp_pairs on
    that step's level-0 clouds from the step's own RANSAC poses, and the oracle."""
    import torch
    from d3feat_b200 import synth
    from d3feat_b200.encoder import KPFCNN, GraphPipeline, RefinedDetections
    from d3feat_b200.registration import icp_pairs
    cfg = synth.Config(architecture=synth.ARCH_3DMATCH)
    enc = KPFCNN(cfg, synth.make_params(cfg, 5), LIMITS, device=cuda)
    rng = np.random.default_rng(12)
    batches = []
    for i, n in enumerate([9000, 8500, 9000, 7000, 8800]):
        base = synth.room_fragment(300 + i, n)
        c1, _ = moved_copy(rng, base, keep=0.9, deg=3)
        c2, _ = moved_copy(rng, base, keep=0.8, deg=3)
        clouds = [base, c1, c2]
        batches.append((np.concatenate(clouds, 0), np.array([c.shape[0] for c in clouds], np.int32)))
    pairs = [(i, j) for i in range(3) for j in range(i + 1, 3)]
    reg = dict(distance=0.5, edge_ratio=0.5, ransac_n=4, max_iterations=2000, max_validation=200)
    opts = dict(distance=0.3, max_iterations=30)
    pipe = GraphPipeline.for_batch(enc, t(batches[0][0], cuda), t(batches[0][1], cuda), slack=1.2, decoder=True,
                                   keypoints=250, match_pairs=pairs, register=reg, icp=opts)
    pipe.prime(t(batches[0][0], cuda), t(batches[0][1], cuda))
    got = []
    for i in range(len(batches)):
        nxt = batches[i + 1] if i + 1 < len(batches) else None
        res, _ = pipe.step(t(nxt[0], cuda), t(nxt[1], cuda)) if nxt else pipe.step()
        assert isinstance(res, RefinedDetections)
        got.append((res.registration.pose.clone(), as_numpy(res.refinement)))
    pipe.check()
    for i, (pose, ref) in enumerate(got):
        pts, lens = batches[i]
        eager = icp_pairs(t(pts, cuda), t(lens, cuda), pairs, pose, bbox=pipe.bbox, **opts)
        assert mismatches(ref, as_numpy(eager)) == [], i
        want = icp_np.icp(pts, lens, pairs, pose.cpu().numpy(), **opts)
        assert mismatches(ref, want) == [], i
        assert (ref["iterations"] >= 1).any(), i
    torch.cuda.synchronize()
