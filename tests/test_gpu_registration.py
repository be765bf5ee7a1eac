"""RANSAC registration on the GPU (d3f_register_pairs, registration.register_pairs,
GraphPipeline(..., register=...)) against the numpy restatement oracle/register_np.py.

Every comparison is exact: the pose is compared as int64 bit patterns, and n_inliers, hypothesis and n_validated as
integers. The contract is fp64 without FMA in a fixed order, so a contracted multiply-add, a different Jacobi order
or a different reduction order shows up in the pose bits."""
import ctypes as C

import numpy as np
import pytest

from oracle import register_np

KMAX_BATCH = 1024
FIELDS = ("pose", "n_inliers", "hypothesis", "n_validated")
SMALL = dict(max_iterations=2000, max_validation=200)


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


def options(**kw):
    o = dict(distance=0.05, ransac_n=3, edge_ratio=0.9, max_iterations=50000, max_validation=1000, seed=0)
    o.update(kw)
    return o


def register_raw(dev, points, count, corr, n_corr, pairs, **kw):
    """The entry point itself, on outputs filled with sentinels: every element must be written."""
    import torch
    from d3feat_b200 import _lib
    o = options(**kw)
    lib = _lib.lib()
    B, k, _ = points.shape
    P, L, _ = corr.shape
    tp, tc, tr, tn, tq = (t(np.asarray(a), dev) for a in (
        np.asarray(points, np.float32), np.asarray(count, np.int32), np.asarray(corr, np.int32),
        np.asarray(n_corr, np.int32), np.asarray(pairs, np.int32)))
    pose = torch.full((P, 4, 4), 7.0, dtype=torch.float64, device=dev)
    ints = [torch.full((P,), 7, dtype=torch.int32, device=dev) for _ in range(3)]
    ws = _lib.workspace(lib.d3f_register_pairs_workspace_bytes(L, P, o["max_iterations"], o["max_validation"]), dev)
    _lib.check(lib.d3f_register_pairs(_lib.ptr(tp), _lib.ptr(tc), B, k, _lib.ptr(tr), _lib.ptr(tn), L, _lib.ptr(tq), P,
                                      o["ransac_n"], o["max_iterations"], o["max_validation"], o["distance"],
                                      o["edge_ratio"], o["seed"], _lib.ptr(pose), *[_lib.ptr(x) for x in ints],
                                      _lib.ptr(ws), ws.numel(), _lib.stream()),
               "d3f_register_pairs")
    return dict(zip(FIELDS, [pose.cpu().numpy()] + [x.cpu().numpy() for x in ints]))


def check(dev, points, count, corr, n_corr, pairs, **kw):
    got = register_raw(dev, points, count, corr, n_corr, pairs, **kw)
    want = register_np.register(points, count, corr, n_corr, pairs, **options(**kw))
    assert mismatches(got, want) == []
    return want


def rotation(rng):
    q = rng.normal(size=4)
    w, x, y, z = q / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def scene(rng, B, k, extent=1.0):
    """B rigidly moved copies of one cloud: slot j of every cloud is the same point. Returns points [B,k,3], poses."""
    base = rng.uniform(-extent, extent, (k, 3))
    poses = [(rotation(rng), rng.uniform(-extent, extent, 3)) for _ in range(B)]
    return np.stack([base @ R.T + tr for R, tr in poses]).astype(np.float32), poses


def rows(rng, L, n_s, n_t, outliers):
    """L correspondence rows between clouds with n_s / n_t real slots: (j, j), or a random target slot for a fraction
    `outliers` of them."""
    src = rng.integers(0, max(1, min(n_s, n_t)), L)
    tgt = src.copy()
    bad = rng.random(L) < outliers
    tgt[bad] = rng.integers(0, max(1, n_t), int(bad.sum()))
    return np.stack([src, tgt], 1).astype(np.int32)


def true_pose(poses, a, b):
    (Ra, ta), (Rb, tb) = poses[a], poses[b]
    R = Rb @ Ra.T
    return R, tb - R @ ta


# ---- 1. correspondence counts x outlier fractions, n = 3 and 4, several seeds --------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("n,seed", [(3, 0), (3, 977), (4, 1), (4, 2 ** 64 - 5)])
def test_register_pairs_against_oracle(cuda, n, seed):
    rng = np.random.default_rng(n * 31 + seed % 1000)
    B, k, L = 4, 250, 5000
    points, poses = scene(rng, B, k)
    counts = np.full(B, k, np.int32)
    pairs, corr, n_corr = [], [], []
    for nc in (0, 1, 2, 3, 4, 250, 5000):
        for out in (0.0, 0.5, 0.95, 1.0):
            a, b = rng.choice(B, 2, replace=False)
            pairs.append((a, b))
            corr.append(rows(rng, L, k, k, out))
            n_corr.append(nc)
    pairs, corr, n_corr = np.array(pairs, np.int32), np.stack(corr), np.array(n_corr, np.int32)
    want = check(cuda, points, counts, corr, n_corr, pairs, ransac_n=n, seed=seed, **SMALL)
    assert (want["n_validated"] == SMALL["max_validation"]).any(), "some pair should reach V early"
    assert ((want["n_validated"] > 0) & (want["n_validated"] < SMALL["max_validation"])).any() or n == 4
    clean = (n_corr >= 250) & (np.array([0.0, 0.5, 0.95, 1.0] * 7) == 0)
    for p in np.nonzero(clean)[0]:
        R, tr = true_pose(poses, *pairs[p])
        assert np.abs(want["pose"][p, :3, :3] - R).max() < 1e-5 and want["n_inliers"][p] == n_corr[p]


@pytest.mark.gpu
def test_register_pairs_default_iterations(cuda):
    """The 3DMatch evaluation's parameters (50000, 1000) on pairs that reach V early and pairs that never do."""
    rng = np.random.default_rng(50)
    B, k = 3, 250
    points, _ = scene(rng, B, k)
    pairs = np.array([(0, 1), (1, 2), (2, 0)], np.int32)
    corr = np.stack([rows(rng, k, k, k, out) for out in (0.3, 0.9, 1.0)])
    want = check(cuda, points, np.full(B, k), corr, np.full(3, k), pairs)
    assert want["n_validated"][0] == 1000 and want["n_validated"][2] < 1000


# ---- 2. degenerate geometry ----------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("case", ["duplicates", "collinear", "nan_point", "far"])
def test_register_pairs_degenerate_points(cuda, case):
    rng = np.random.default_rng({"duplicates": 1, "collinear": 2, "nan_point": 3, "far": 4}[case])
    B, k = 2, 250
    points, _ = scene(rng, B, k, extent=1e4 if case == "far" else 1.0)
    if case == "duplicates":           # every point five times over: repeated rows and zero-length edges
        points[:, 50:] = np.tile(points[:, :50], (1, 4, 1))
    elif case == "collinear":          # points on one line: the covariance has rank one
        s = rng.uniform(-1, 1, k)
        points[0] = np.stack([s, 2 * s, -s], 1)
        points[1] = np.stack([-s, s + 1, 3 * s], 1)
    elif case == "nan_point":
        points[0, 17] = np.nan
    corr = np.stack([rows(rng, k, k, k, 0.5), rows(rng, k, k, k, 0.2)])
    corr[:, :40, 0] = 17                # the NaN point's slot, in many rows
    corr[:, :40, 1] = 17
    dist = 50.0 if case == "far" else 0.05
    for n in (3, 4):
        check(cuda, points, [k, k], corr, [k, k], [(0, 1), (1, 0)], ransac_n=n, distance=dist, **SMALL)


# ---- 3. padding poisoned with NaN, bad rows and cloud ids, counts and n_corr out of range -------------------------

@pytest.mark.gpu
def test_register_pairs_padding_bad_rows_and_pair_ids(cuda):
    rng = np.random.default_rng(9)
    B, k, L = 5, 200, 300
    points, _ = scene(rng, B, k)
    count = np.array([k + 5, 120, -3, k, 60], np.int32)
    for b, c in enumerate(np.clip(count, 0, k)):
        points[b, c:] = np.nan
    pairs, corr, n_corr = [], [], []

    def add(a, b, nc, fix=None):
        ns, nt = (int(np.clip(count[x], 0, k)) if 0 <= x < B else 1 for x in (a, b))
        c = rows(rng, L, ns, nt, 0.4)
        real = min(max(nc, 0), L)
        c[real:] = rng.integers(k, 2 * k, (L - real, 2))    # unread garbage
        if fix:
            fix(c)
        pairs.append((a, b))
        corr.append(c)
        n_corr.append(nc)

    add(0, 1, 250)
    add(1, 3, L + 40)                                   # n_corr above L: clamped
    add(3, 0, -5)                                       # below 0: nothing
    add(0, 2, 100)                                      # an empty cloud: every real row is bad
    add(0, 1, 200, lambda c: c.__setitem__((150, 1), 120))     # a target slot at the count
    add(1, 0, 200, lambda c: c.__setitem__((199, 0), -1))      # a negative source slot
    add(1, 0, 200, lambda c: c.__setitem__((200, 0), 5000))    # past n_c: never read
    add(-1, 1, 100)
    add(1, B, 100)
    add(4, 3, 60)
    pairs, corr, n_corr = np.array(pairs, np.int32), np.stack(corr), np.array(n_corr, np.int32)
    want = check(cuda, points, count, corr, n_corr, pairs, **SMALL)
    assert (want["hypothesis"][[2, 3, 4, 5, 7, 8]] == -1).all()
    assert want["hypothesis"][[0, 1, 6, 9]].min() >= 0


# ---- 4. many clouds and pairs --------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_register_pairs_many_clouds_and_pairs(cuda):
    rng = np.random.default_rng(5)
    B, k, L, P = KMAX_BATCH, 24, 24, 4096
    points, _ = scene(rng, B, k)
    count = rng.integers(-2, k + 3, B).astype(np.int32)
    pairs = rng.integers(0, B, (P, 2)).astype(np.int32)
    pairs[::97, 0] = -1
    pairs[::89, 1] = B
    corr = np.stack([rows(rng, L, k, k, 0.3) for _ in range(P)])
    n_corr = rng.integers(0, L + 1, P).astype(np.int32)
    check(cuda, points, count, corr, n_corr, pairs, max_iterations=64, max_validation=16, distance=0.1)


# ---- 5. captured in a CUDA graph, inputs rewritten in place -----------------------------------------------------

@pytest.mark.gpu
def test_register_pairs_in_a_cuda_graph(cuda):
    import torch
    from d3feat_b200 import _lib
    from d3feat_b200.keypoints import KeypointSet
    from d3feat_b200.matching import Matches
    from d3feat_b200.registration import register_pairs
    rng = np.random.default_rng(6)
    B, k = 4, 250
    pairs = np.array([(0, 1), (1, 2), (3, 0), (2, 2)], np.int32)
    P = len(pairs)

    def inputs():
        pts, _ = scene(rng, B, k)
        cnt = rng.integers(k - 60, k + 2, B).astype(np.int32)
        nn = np.full((P, k), -1, np.int32)
        for p, (a, b) in enumerate(pairs):
            ns, nt = min(cnt[a], k), min(cnt[b], k)
            nn[p, :ns] = np.where(rng.random(ns) < 0.5, np.arange(ns) % nt, rng.integers(0, nt, ns))
        return pts, cnt, nn

    pts, cnt, nn = inputs()
    tp, tc, tn = t(pts, cuda), t(cnt, cuda), t(nn, cuda)
    kp = KeypointSet(None, tc, tp, None, None)
    z = torch.zeros((P, k), dtype=torch.int32, device=cuda)
    m = Matches(tn, z.float(), z, z.float(), torch.zeros((P, k, 2), dtype=torch.int32, device=cuda), z[:, 0])
    tq = t(pairs, cuda)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        register_pairs(kp, m, tq, **SMALL)          # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    n0 = _lib.launch_count()
    with torch.cuda.graph(g):
        reg = register_pairs(kp, m, tq, **SMALL)
    assert _lib.launch_count() > n0
    for r in range(3):
        pts, cnt, nn = inputs()
        tp.copy_(t(pts, cuda))
        tc.copy_(t(cnt, cuda))
        tn.copy_(t(nn, cuda))
        g.replay()
        torch.cuda.synchronize()
        corr = np.stack([np.broadcast_to(np.arange(k, dtype=np.int32), (P, k)), nn], 2)
        want = register_np.register(pts, cnt, corr, (nn >= 0).sum(1), pairs, **options(**SMALL))
        got = dict(zip(FIELDS, [x.cpu().numpy() for x in (reg.pose, reg.n_inliers, reg.hypothesis, reg.n_validated)]))
        assert mismatches(got, want) == [], r
        assert np.array_equal(reg.n_correspondences.cpu().numpy(), (nn >= 0).sum(1)), r


# ---- 6. register_pairs on real matches: one-way (Open3D) and mutual ----------------------------------------------

def oracle_from_matches(kp, m, pairs, mutual, **kw):
    nn = m.nn_st.cpu().numpy()
    P, k = nn.shape
    if mutual:
        corr, n_corr = m.matches.cpu().numpy(), m.n_matches.cpu().numpy()
    else:
        corr, n_corr = np.stack([np.broadcast_to(np.arange(k, dtype=np.int32), (P, k)), nn], 2), (nn >= 0).sum(1)
    return register_np.register(kp.points.cpu().numpy(), kp.count.cpu().numpy(), corr, n_corr, pairs,
                                **options(**kw)), n_corr


def as_numpy(reg):
    return dict(zip(FIELDS, [x.cpu().numpy() for x in (reg.pose, reg.n_inliers, reg.hypothesis, reg.n_validated)]))


@pytest.mark.gpu
@pytest.mark.parametrize("mutual", [False, True])
def test_register_pairs_on_descriptor_matches(cuda, mutual):
    from d3feat_b200.keypoints import KeypointSet
    from d3feat_b200.matching import match_keypoints
    from d3feat_b200.registration import register_pairs
    rng = np.random.default_rng(21)
    B, k, D = 4, 250, 32
    points, poses = scene(rng, B, k)
    base = rng.normal(size=(k, D))
    desc = base[None] + rng.normal(scale=0.6, size=(B, k, D))
    desc = (desc / np.linalg.norm(desc, axis=-1, keepdims=True)).astype(np.float32)
    count = np.array([k, 230, k, 190], np.int32)
    kp = KeypointSet(None, t(count, cuda), t(points, cuda), t(desc, cuda), None)
    pairs = [(i, j) for i in range(B) for j in range(i + 1, B)]
    m = match_keypoints(kp, pairs)
    reg = register_pairs(kp, m, pairs, mutual=mutual, **SMALL)
    want, n_corr = oracle_from_matches(kp, m, pairs, mutual, **SMALL)
    assert mismatches(as_numpy(reg), want) == []
    assert np.array_equal(reg.n_correspondences.cpu().numpy(), n_corr)
    for p, (a, b) in enumerate(pairs):
        R, _ = true_pose(poses, a, b)
        assert np.abs(want["pose"][p, :3, :3] - R).max() < 1e-3, p


# ---- 7. GraphPipeline(..., match_pairs=every i < j, register={...}) ----------------------------------------------

LIMITS = [35, 33, 34, 36, 30]


@pytest.mark.gpu
def test_graph_pipeline_register(cuda):
    """Five batches of three clouds through one captured bucket. The registration equals an eager register_pairs of
    the graph's own keypoints and matches, and the oracle applied to them."""
    import torch
    from d3feat_b200 import synth
    from d3feat_b200.encoder import KPFCNN, GraphPipeline, RegisteredDetections
    from d3feat_b200.keypoints import KeypointSet
    from d3feat_b200.matching import Matches
    from d3feat_b200.registration import register_pairs
    cfg = synth.Config(architecture=synth.ARCH_3DMATCH)
    enc = KPFCNN(cfg, synth.make_params(cfg, 5), LIMITS, device=cuda)
    batches = []
    for i, n in enumerate([9000, 8500, 9000, 7000, 8800]):
        clouds = [synth.room_fragment(300 + 3 * i + c, n - 400 * c) for c in range(3)]
        batches.append((np.concatenate(clouds, 0), np.array([c.shape[0] for c in clouds], np.int32)))
    pairs = [(i, j) for i in range(3) for j in range(i + 1, 3)]
    # the synthetic weights give uninformative descriptors: loose checkers so that hypotheses validate
    opts = dict(distance=0.5, edge_ratio=0.5, ransac_n=4, **SMALL)
    pipe = GraphPipeline.for_batch(enc, t(batches[0][0], cuda), t(batches[0][1], cuda), slack=1.2, decoder=True,
                                   keypoints=250, match_pairs=pairs, register=opts)
    pipe.prime(t(batches[0][0], cuda), t(batches[0][1], cuda))
    got = []
    for i in range(len(batches)):
        nxt = batches[i + 1] if i + 1 < len(batches) else None
        res, _ = pipe.step(t(nxt[0], cuda), t(nxt[1], cuda)) if nxt else pipe.step()
        assert isinstance(res, RegisteredDetections)
        got.append((KeypointSet(*[None if x is None else x.clone() for x in res.keypoints]),
                    Matches(*[x.clone() for x in res.matches]), as_numpy(res.registration)))
    pipe.check()
    for i, (kp, m, reg) in enumerate(got):
        want, _ = oracle_from_matches(kp, m, pairs, False, **opts)
        assert mismatches(reg, want) == [], i
        assert (want["hypothesis"] >= 0).any(), i
        assert mismatches(as_numpy(register_pairs(kp, m, pairs, **opts)), reg) == [], i
    torch.cuda.synchronize()


# ---- CPU: argument validation, pipeline arguments, the oracle itself -------------------------------------------

def test_register_pairs_invalid_arguments_without_a_gpu():
    from d3feat_b200 import build
    from d3feat_b200._lib import SYMBOLS
    lib = C.CDLL(build.build())
    lib.d3f_last_error.restype = C.c_char_p
    for name in ("d3f_register_pairs_workspace_bytes", "d3f_register_pairs"):
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = [(r, a) for n, r, a in SYMBOLS if n == name][0]
    fake = C.c_void_p(256)          # never dereferenced: validation fails first
    ws_ok = lib.d3f_register_pairs_workspace_bytes(250, 6, 50000, 1000)
    assert ws_ok >= 6 * (50000 // 8 + 16 * 1000)
    assert lib.d3f_register_pairs_workspace_bytes(0, 6, 50000, 1000) == 0
    assert lib.d3f_register_pairs_workspace_bytes(250, 6, 50000, 50001) == 0
    assert lib.d3f_register_pairs_workspace_bytes(65536, 65536, 10, 10) == 0

    def call(B=4, k=250, L=250, P=6, n=3, T=50000, V=1000, tau=0.05, ratio=0.9, ws=ws_ok, null=None):
        p = [None if i == null else fake for i in range(10)]
        return lib.d3f_register_pairs(p[0], p[1], B, k, p[2], p[3], L, p[4], P, n, T, V, tau, ratio, 0, *p[5:9],
                                      p[9], ws, None)

    cases = [(dict(B=0), b"B=0"), (dict(B=KMAX_BATCH + 1), b"B=1025"), (dict(k=0), b"k=0"), (dict(L=0), b"L=0"),
             (dict(P=0), b"P=0"), (dict(n=2), b"ransac_n=2"), (dict(n=9), b"ransac_n=9"), (dict(T=0), b"max_iter"),
             (dict(T=(1 << 24) + 1), b"max_iter"), (dict(V=0), b"max_validation"),
             (dict(V=50001), b"max_validation"), (dict(tau=0.0), b"distance"), (dict(tau=-1.0), b"distance"),
             (dict(tau=float("inf")), b"distance"), (dict(tau=float("nan")), b"distance"),
             (dict(ratio=0.0), b"edge_ratio"), (dict(ratio=1.5), b"edge_ratio"),
             (dict(ratio=float("nan")), b"edge_ratio"), (dict(L=65536, P=65536, T=10, V=10), b"exceeds int32"),
             (dict(P=4096, T=1 << 20, V=10), b"exceeds int32"), (dict(B=1024, k=1 << 20), b"exceeds int32")]
    cases += [(dict(null=i), b"null pointer") for i in range(10)]
    for kw, msg in cases:
        assert call(**kw) == -1, kw
        assert msg in lib.d3f_last_error(), (kw, lib.d3f_last_error())
    assert call(ws=ws_ok - 1) == -4
    assert b"workspace" in lib.d3f_last_error()


def test_graph_pipeline_register_checked_first():
    """register without match_pairs, unknown keys and out-of-range values are refused before the pipeline touches the
    encoder or the device."""
    from d3feat_b200.encoder import GraphPipeline
    bbox = np.zeros(6, np.float32)
    with pytest.raises(ValueError, match="needs match_pairs"):
        GraphPipeline(None, [1024] * 5, 2, bbox, decoder=True, keypoints=250, register={})
    for bad in ({"ransac": 3}, [("ransac_n", 3)], {"ransac_n": 2}, {"ransac_n": 9}, {"ransac_n": 3.0},
                {"max_iterations": 0}, {"max_iterations": (1 << 24) + 1}, {"max_validation": 0},
                {"max_iterations": 10, "max_validation": 11}, {"distance": 0}, {"distance": float("nan")},
                {"edge_ratio": 0}, {"edge_ratio": 1.01}, {"seed": -1}, {"seed": 1 << 64}, {"mutual": 1}):
        with pytest.raises(ValueError, match="GraphPipeline"):
            GraphPipeline(None, [1024] * 5, 2, bbox, decoder=True, keypoints=250, match_pairs=[(0, 1)], register=bad)


def kabsch(s, tt):
    cs, ct = s.mean(0), tt.mean(0)
    U, _, Vt = np.linalg.svd((s - cs).T @ (tt - ct))
    d = np.sign(np.linalg.det(Vt.T @ U.T))
    R = Vt.T @ np.diag([1.0, 1.0, d]) @ U.T
    return R, ct - R @ cs


def oracle_pose(s, tt):
    """register_np's Horn solve on one set of rows (s, tt: [m,3] float64)."""
    rows_ = [([np.array([x]) for x in s[i]], [np.array([x]) for x in tt[i]], None) for i in range(len(s))]
    R, tr = register_np.horn(rows_, np.array([float(len(s))]))
    return np.array([[R[i][j][0] for j in range(3)] for i in range(3)]), np.array([x[0] for x in tr])


def test_oracle_pose_agrees_with_svd_kabsch():
    rng = np.random.default_rng(31)
    for trial in range(200):
        m = int(rng.integers(3, 40))
        s = rng.uniform(-1, 1, (m, 3)).astype(np.float32).astype(np.float64)
        R0 = rotation(rng)
        tt = (s @ R0.T + rng.uniform(-2, 2, 3) + rng.normal(scale=0.01, size=(m, 3))).astype(np.float32)
        R, tr = oracle_pose(s, tt.astype(np.float64))
        Rk, tk = kabsch(s, tt.astype(np.float64))
        assert np.abs(R - Rk).max() < 1e-12 and np.abs(tr - tk).max() < 1e-12, trial
        assert abs(np.linalg.det(R) - 1) < 1e-12


def test_oracle_recovers_a_known_transform_with_60_percent_outliers():
    rng = np.random.default_rng(32)
    B, k = 2, 250
    points, poses = scene(rng, B, k)
    src = rng.permutation(k)
    tgt = src.copy()
    bad = rng.random(k) < 0.6
    tgt[bad] = rng.integers(0, k, int(bad.sum()))
    inl = src == tgt
    corr = np.stack([src, tgt], 1)[None].astype(np.int32)
    want = register_np.register(points, [k, k], corr, [k], [(0, 1)], distance=0.01, **SMALL)
    assert want["n_inliers"][0] == inl.sum()
    s, tt = points[0, src[inl]].astype(np.float64), points[1, tgt[inl]].astype(np.float64)
    Rk, tk = kabsch(s, tt)
    assert np.abs(want["pose"][0, :3, :3] - Rk).max() < 1e-12 and np.abs(want["pose"][0, :3, 3] - tk).max() < 1e-12
    R, tr = true_pose(poses, 0, 1)      # the points themselves are rounded to fp32
    assert np.abs(want["pose"][0, :3, :3] - R).max() < 1e-5 and np.abs(want["pose"][0, :3, 3] - tr).max() < 1e-5


def _pick_best_ties_to_larger_h(cnt, sums, hs):
    return int(np.lexsort((-hs, sums, -cnt))[0])


def _last_validated(hs, V):
    return hs[-V:]


def _no_refit(R, t, rows_, m):
    return R, t


def best_residuals(points, corr, want, tau):
    """d^2 of every row under the pose of the best hypothesis (before the refit)."""
    L = corr.shape[1]
    rows_ = register_np._Rows(points, corr, np.array([(0, 1)]), np.array([L]), [0])
    one = np.zeros(1, np.int64)
    _, R, tr = register_np.hypotheses(rows_, one, want["hypothesis"].astype(np.int64), one, np.array([L]), 3,
                                      tau * tau, 0.9, 0)
    return np.array([register_np.residual2(R, tr, *rows_.at(np.array([r])))[0] for r in range(L)])


def threshold_on_a_row(points, corr, kw):
    """A distance at which a row of the best hypothesis has d^2 == distance^2 exactly. Candidates are the rows closest
    to the distance whose d^2 is the square of its rounded square root; the one kept must still be a row of the best
    hypothesis found at that distance."""
    args = (points, [points.shape[1]] * 2, corr, [corr.shape[1]], [(0, 1)])
    d2 = best_residuals(points, corr, register_np.register(*args, **kw), kw["distance"])
    for r in np.argsort(np.abs(d2 - kw["distance"] ** 2)):
        tau = float(np.sqrt(d2[r]))
        if not np.isfinite(tau) or tau * tau != d2[r]:
            continue
        want = register_np.register(*args, **dict(kw, distance=tau))
        if (best_residuals(points, corr, want, tau) == tau * tau).any():
            return tau
    raise AssertionError("no row lies exactly on a usable distance")


@pytest.mark.parametrize("bug", ["ties_to_larger_h", "inlier_le", "validations_out_of_order", "no_edge_check",
                                 "no_refit"])
def test_oracle_rejects_emulated_bugs(monkeypatch, bug):
    rng = np.random.default_rng(33)
    k = 64
    points, _ = scene(rng, 2, k)
    corr = rows(rng, k, k, k, 0.5)[None]
    kw = dict(distance=0.05, max_iterations=400, max_validation=20)
    if bug == "ties_to_larger_h":
        # three rows: every validated hypothesis is a permutation of the same three, so scores tie exactly
        corr, kw = np.array([[[0, 0], [1, 1], [2, 2]]], np.int32), dict(distance=0.05, max_iterations=50,
                                                                         max_validation=20)
    elif bug == "inlier_le":           # noisy inliers: residuals spread up to the distance
        points[1] += rng.normal(scale=0.015, size=points[1].shape).astype(np.float32)
        kw["distance"] = threshold_on_a_row(points, corr, kw)
    elif bug == "no_edge_check":
        kw = dict(distance=1.5, max_iterations=400, max_validation=400)
    elif bug == "validations_out_of_order":
        kw = dict(distance=0.05, max_iterations=400, max_validation=3)
    args = (points, [k, k], corr, [corr.shape[1]], [(0, 1)])
    want = register_np.register(*args, **kw)
    assert want["hypothesis"][0] >= 0
    name, fn = {"ties_to_larger_h": ("pick_best", _pick_best_ties_to_larger_h),
                "inlier_le": ("is_inlier", lambda d2, tau2: d2 <= tau2),
                "validations_out_of_order": ("first_validated", _last_validated),
                "no_edge_check": ("edge_ok", lambda S, T, ratio: np.ones(S[0][0].shape, bool)),
                "no_refit": ("refit", _no_refit)}[bug]
    monkeypatch.setattr(register_np, name, fn)
    got = register_np.register(*args, **kw)
    assert mismatches(got, want), bug
