"""ICP contract (oracle/icp_np.py) on the CPU: agreement with an independent float64 ICP, recovery of a known pose, the
emulated bugs it rejects, and the argument checks of registration.icp_pairs, GraphPipeline(icp=...) and
d3f_icp_pairs that run before any device work."""
import ctypes as C

import numpy as np
import pytest

from oracle import icp_np

FIELDS = ("pose", "fitness", "inlier_rmse", "n_correspondences", "iterations")


def mismatches(got, want):
    bad = []
    for f in FIELDS:
        g, w = np.asarray(got[f]), np.asarray(want[f])
        if g.dtype == np.float64:
            g, w = g.view(np.int64), w.view(np.int64)
        if g.shape != w.shape or not np.array_equal(g, w):
            bad.append(f)
    return bad


def rotation(axis, deg):
    axis = np.asarray(axis, float)
    axis = axis / np.linalg.norm(axis)
    th = np.deg2rad(deg)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K


def rigid(R, t):
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    return T


def partial_pair(rng, n, noise=0.0):
    """(source, target, true pose): the source's first n points (a unit cube) appear in the target moved by the true
    pose, plus noise; n/3 source-only points sit 3 m along +x and n/3 target-only points 3 m along -x, further than
    any distance used here, so the overlap is partial."""
    A = rng.uniform(0, 1, (n, 3))
    src = np.concatenate([A, rng.uniform(0, 1, (n // 3, 3)) + [3, 0, 0]]).astype(np.float32)
    T = rigid(rotation(rng.normal(size=3), 20), rng.uniform(-0.5, 0.5, 3))
    moved = A @ T[:3, :3].T + T[:3, 3] + rng.normal(scale=noise, size=A.shape)
    tgt = np.concatenate([moved, rng.uniform(0, 1, (n // 3, 3)) + [-3, 0, 0]]).astype(np.float32)
    return src, tgt, T


def perturbed(rng, T, deg=2.0, shift=0.03):
    d = rng.normal(size=3)
    return rigid(rotation(rng.normal(size=3), deg), shift * d / np.linalg.norm(d)) @ T


def kabsch(s, tt):
    cs, ct = s.mean(0), tt.mean(0)
    U, _, Vt = np.linalg.svd((s - cs).T @ (tt - ct))
    d = np.sign(np.linalg.det(Vt.T @ U.T))
    R = Vt.T @ np.diag([1.0, 1.0, d]) @ U.T
    return R, ct - R @ cs


def reference_icp(src, tgt, init, tau, I, rf, rr):
    """An independent float64 point-to-point ICP: scipy cKDTree nearest within tau, SVD Kabsch, Open3D's stopping
    rule. Returns (pose, fitness, rmse, n, iterations)."""
    from scipy.spatial import cKDTree
    src, tgt = src.astype(np.float64), tgt.astype(np.float64)
    tree = cKDTree(tgt)

    def evaluate(T):
        q = src @ T[:3, :3].T + T[:3, 3]
        d, j = tree.query(q, k=1, distance_upper_bound=tau)
        use = d < tau
        n = int(use.sum())
        return q, j, use, n, n / len(src), (np.sqrt(np.sum(d[use] ** 2) / n) if n else 0.0)

    T = init.copy()
    q, j, use, n, fit, rmse = evaluate(T)
    it = 0
    for _ in range(I):
        if n < 3:
            break
        T = rigid(*kabsch(q[use], tgt[j[use]])) @ T
        it += 1
        prev = (fit, rmse)
        q, j, use, n, fit, rmse = evaluate(T)
        if abs(fit - prev[0]) < rf and abs(rmse - prev[1]) < rr:
            break
    return T, fit, rmse, n, it


def stacked(*clouds):
    return np.concatenate(clouds).astype(np.float32), np.array([len(c) for c in clouds], np.int32)


@pytest.mark.parametrize("seed,noise,I", [(1, 0.0, 30), (2, 0.005, 30), (3, 0.01, 5), (4, 0.005, 0)])
def test_oracle_agrees_with_an_independent_float64_icp(seed, noise, I):
    rng = np.random.default_rng(seed)
    src, tgt, T = partial_pair(rng, 1200, noise)
    init = perturbed(rng, T)
    pts, lens = stacked(src, tgt)
    want = icp_np.icp(pts, lens, [(0, 1)], init[None], distance=0.1, max_iterations=I)
    Tr, fit, rmse, n, it = reference_icp(src, tgt, init, 0.1, I, 1e-6, 1e-6)
    assert want["iterations"][0] == it and want["n_correspondences"][0] == n
    assert np.abs(want["pose"][0] - Tr).max() < 1e-9
    assert abs(want["fitness"][0] - fit) < 1e-12 and abs(want["inlier_rmse"][0] - rmse) < 1e-9


def test_oracle_recovers_a_known_pose_on_noise_free_partial_overlap():
    rng = np.random.default_rng(5)
    for trial in range(3):
        src, tgt, T = partial_pair(rng, 1500)
        pts, lens = stacked(src, tgt)
        want = icp_np.icp(pts, lens, [(0, 1)], perturbed(rng, T)[None], distance=0.1, max_iterations=100)
        assert np.abs(want["pose"][0] - T).max() < 1e-5, trial
        assert want["n_correspondences"][0] == 1500 and want["fitness"][0] == 0.75, trial
        assert want["iterations"][0] < 100, trial


def test_oracle_invalid_pairs_and_row_counts():
    """Pairs naming a cloud outside [0, B) or an empty cloud keep init; rows past the row count belong to no cloud."""
    rng = np.random.default_rng(6)
    src, tgt, T = partial_pair(rng, 300)
    pts, lens = stacked(src, tgt)
    init = np.stack([perturbed(rng, T)] * 5)
    init[4] = np.nan
    lens3 = np.append(lens, 0)
    out = icp_np.icp(pts, lens3, [(0, 1), (-1, 1), (0, 3), (2, 1), (0, 1)], init, distance=0.1)
    for p in (1, 2, 3, 4):
        assert np.array_equal(out["pose"][p].view(np.int64), init[p].view(np.int64)), p
        assert out["iterations"][p] == 0 and out["n_correspondences"][p] == 0, p
        assert out["fitness"][p] == 0 and out["inlier_rmse"][p] == 0, p
    assert out["iterations"][0] > 0
    # the same pair with the target cut short by the row count equals it with the target's length cut short
    cut = len(src) + 100
    a = icp_np.icp(pts, lens, [(0, 1)], init[:1], distance=0.1, rows=cut)
    b = icp_np.icp(pts[:cut], [len(src), 100], [(0, 1)], init[:1], distance=0.1)
    assert mismatches(a, b) == []


def lattice_pair(h=0.25):
    """Source and target on one lattice of spacing h (exact in fp32): every target row at exactly h = distance from a
    source row, and source rows halfway between two target rows (equidistant, exact d^2)."""
    g = np.stack(np.meshgrid(*[np.arange(6) * h] * 3, indexing="ij"), -1).reshape(-1, 3)
    src = np.concatenate([g, g[:40] + [h / 2, 0, 0]]).astype(np.float32)
    tgt = (g + [h, 0, 0]).astype(np.float32)
    return src, tgt


def _nearest_ties_to_larger_row(qi, row, d2):
    order = np.lexsort((-row, d2, qi))
    first = np.ones(len(order), bool)
    first[1:] = qi[order][1:] != qi[order][:-1]
    return order[first]


def _sequential_sum(x, use):
    total = np.zeros(x.shape[0])
    for i in np.nonzero(use)[0]:
        total = total + x[:, i]
    return total


def _in_place(s, R, t, U, q_prev):
    return icp_np.transform(U[0], U[1], q_prev)


def _relative_change(fit, prev_fit, rmse, prev_rmse, relative_fitness, relative_rmse):
    return abs(fit - prev_fit) < relative_fitness * abs(prev_fit) and abs(rmse - prev_rmse) < relative_rmse * abs(prev_rmse)


@pytest.mark.parametrize("bug", ["inlier_le", "ties_to_larger_row", "sequential_sum", "in_place_transform",
                                 "relative_convergence"])
def test_oracle_rejects_emulated_bugs(monkeypatch, bug):
    rng = np.random.default_rng(7)
    if bug in ("inlier_le", "ties_to_larger_row"):
        src, tgt = lattice_pair()
        h = 0.25
        kw = dict(distance=h if bug == "inlier_le" else 0.2, max_iterations=0 if bug == "inlier_le" else 3)
        init = np.eye(4)[None]
        if bug == "ties_to_larger_row":
            init = rigid(np.eye(3), [h, 0, 0])[None]      # every lattice row lands on a target; the extra rows tie
    else:
        src, tgt, T = partial_pair(rng, 1500, 0.01)
        init = perturbed(rng, T)[None]
        kw = dict(distance=0.1, max_iterations=30)
        if bug == "relative_convergence":
            kw.update(relative_fitness=1e-3, relative_rmse=1e-3)    # absolute: 3 updates, relative: 4
    pts, lens = stacked(src, tgt)
    want = icp_np.icp(pts, lens, [(0, 1)], init, **kw)
    name, fn = {"inlier_le": ("corresponds", lambda d2, tau2: d2 <= tau2),
                "ties_to_larger_row": ("pick_nearest", _nearest_ties_to_larger_row),
                "sequential_sum": ("blocked_sum", _sequential_sum),
                "in_place_transform": ("next_queries", _in_place),
                "relative_convergence": ("converged", _relative_change)}[bug]
    monkeypatch.setattr(icp_np, name, fn)
    got = icp_np.icp(pts, lens, [(0, 1)], init, **kw)
    assert mismatches(got, want), bug


# ---- argument checks before any device work -----------------------------------------------------------------

def test_icp_options_checked():
    from d3feat_b200.registration import check_icp_options
    assert check_icp_options(0.2, 200) == (0.2, 200, 1e-6, 1e-6)
    for bad in (dict(distance=None), dict(distance=0), dict(distance=-1), dict(distance=float("inf")),
                dict(distance=float("nan")), dict(distance=0.1, max_iterations=-1),
                dict(distance=0.1, max_iterations=1025), dict(distance=0.1, max_iterations=2.0),
                dict(distance=0.1, max_iterations=True), dict(distance=0.1, relative_fitness=-1e-9),
                dict(distance=0.1, relative_rmse=float("nan")), dict(distance=0.1, relative_fitness="x")):
        with pytest.raises(ValueError, match="icp_pairs"):
            check_icp_options(**bad)


def test_graph_pipeline_icp_checked_first():
    from d3feat_b200.encoder import GraphPipeline
    bbox = np.zeros(6, np.float32)
    with pytest.raises(ValueError, match="needs register"):
        GraphPipeline(None, [1024] * 5, 2, bbox, decoder=True, keypoints=250, match_pairs=[(0, 1)],
                      icp=dict(distance=0.05))
    for bad in ({}, {"max_iterations": 30}, {"distance": 0.05, "max_iter": 3}, [("distance", 0.05)],
                {"distance": 0}, {"distance": 0.05, "max_iterations": 2000}, {"distance": 0.05, "relative_rmse": -1}):
        with pytest.raises(ValueError, match="GraphPipeline"):
            GraphPipeline(None, [1024] * 5, 2, bbox, decoder=True, keypoints=250, match_pairs=[(0, 1)], register={},
                          icp=bad)


def test_icp_pairs_invalid_arguments_without_a_gpu():
    from d3feat_b200 import build
    from d3feat_b200._lib import SYMBOLS
    lib = C.CDLL(build.build())
    lib.d3f_last_error.restype = C.c_char_p
    for name in ("d3f_icp_pairs_workspace_bytes", "d3f_icp_pairs"):
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = [(r, a) for n, r, a in SYMBOLS if n == name][0]
    box = (C.c_float * 6)(-1, -1, -1, 2, 2, 2)
    far = (C.c_float * 6)(-1, -1, -1, 60, 2, 2)
    huge = (C.c_float * 6)(-1, -1, -1, 2000, 2000, 2000)
    fake = C.c_void_p(256)          # never dereferenced: validation fails first
    ws_ok = lib.d3f_icp_pairs_workspace_bytes(60000, 2, 1, 0.05, box)
    assert ws_ok >= 60000 * 4 + 4 * 61 ** 3
    assert lib.d3f_icp_pairs_workspace_bytes(60000, 0, 1, 0.05, box) == 0
    assert lib.d3f_icp_pairs_workspace_bytes(60000, 2, 0, 0.05, box) == 0
    assert lib.d3f_icp_pairs_workspace_bytes(60000, 2, 1, 0.0, box) == 0
    assert lib.d3f_icp_pairs_workspace_bytes(60000, 2, 1, 0.05, None) == 0
    assert lib.d3f_icp_pairs_workspace_bytes(60000, 2, 1, 0.05, far) == 0       # 60 m = 1199 cells from the origin
    assert lib.d3f_icp_pairs_workspace_bytes(60000, 2, 1, 0.05, huge) == 0      # beyond the grid-cell cap
    assert lib.d3f_icp_pairs_workspace_bytes(1 << 30, 2, 64, 0.05, box) == 0     # P * N beyond int32

    def call(B=2, N=60000, P=1, tau=0.05, I=30, rf=1e-6, rr=1e-6, bb=box, ws=ws_ok, null=None):
        p = [None if i == null else fake for i in range(10)]
        return lib.d3f_icp_pairs(p[0], p[1], B, N, None, bb, p[2], P, p[3], tau, I, rf, rr, *p[4:9], p[9], ws, None)

    cases = [(dict(B=0), b"B=0"), (dict(B=1025), b"B=1025"), (dict(N=-1), b"N=-1"), (dict(P=0), b"P=0"),
             (dict(I=-1), b"max_iterations"), (dict(I=1025), b"max_iterations"), (dict(tau=0.0), b"distance"),
             (dict(tau=-1.0), b"distance"), (dict(tau=float("inf")), b"distance"), (dict(tau=float("nan")), b"distance"),
             (dict(rf=-1e-9), b"relative_fitness"), (dict(rr=float("nan")), b"relative_rmse"),
             (dict(rf=float("inf")), b"relative_fitness"), (dict(bb=None), b"null pointer"),
             (dict(bb=huge), b"cells"), (dict(bb=far), b"1024 cells"),
             (dict(N=1 << 30, P=64), b"exceeds int32")]
    cases += [(dict(null=i), b"null pointer") for i in range(10)]
    for kw, msg in cases:
        assert call(**kw) == -1, kw
        assert msg in lib.d3f_last_error(), (kw, lib.d3f_last_error())
    assert call(ws=ws_ok - 1) == -4
    assert b"workspace" in lib.d3f_last_error()
