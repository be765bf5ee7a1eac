"""The ops and the network from several host threads and CUDA streams at once (include/d3feat_b200.h: no global
mutable state, re-entrant across host threads and streams; INTEGRATION.md section 5: one stream per thread).

Every op is deterministic (no float atomics), so the criterion is bitwise equality with the same calls made serially
on one stream, and that serial run is itself checked against the float64 restatement.

  A  parameter scopes and stores are per thread; the folded batch norm follows in-place statistics updates (CPU)
  B  d3f_last_error() names the failure of the calling thread (CPU, built library)
  C  a cache entry (packed weights, folded pair, folded batch norm) made on a busy stream, read at once on another
  D  two models in two threads; a replaying GraphPipeline next to an eager model
  E  every op family from a pool of four threads, each on its own stream; per-thread launch counts
  F  the KPConv chunk pipeline's auxiliary stream: two threads, a thread that exits with work pending, graph capture
  G  a GraphPipeline whose level-0 KPConvs take several chunks (20 x 30 000 points)

Rules for the threaded tests: threads start on a barrier, are joined with a timeout and their exceptions are raised
in the main thread; tests/_trace.record_ops swaps module attributes and is only used single-threaded.
"""
import json
import os
import random
import subprocess
import sys
import tempfile
import threading

import numpy as np
import pytest
import torch

from _oracle import TOL, assert_close, epilogue as epi_ref, gemm_mag, kpconv_ref
from _trace import check_sampled_rows, record_ops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RTOL = 1e-4
SLEEP_CYCLES = 400_000_000        # torch.cuda._sleep: a bounded spin of ~0.25 s that keeps a stream busy


def run_threads(fns, timeout=600):
    """Run fns[i](barrier) in one thread each; every thread waits on `barrier` before its work. Returns the results;
    re-raises the first exception of any thread."""
    barrier = threading.Barrier(len(fns))
    res, err = [None] * len(fns), [None] * len(fns)

    def body(i):
        try:
            barrier.wait(timeout)
            res[i] = fns[i](barrier)
        except BaseException as e:          # noqa: BLE001 -- re-raised in the main thread
            err[i] = e
            barrier.abort()

    ths = [threading.Thread(target=body, args=(i,), daemon=True) for i in range(len(fns))]
    for th in ths:
        th.start()
    for th in ths:
        th.join(timeout)
    assert not any(th.is_alive() for th in ths), "a thread did not finish within %d s" % timeout
    for e in err:
        if e is not None and not isinstance(e, threading.BrokenBarrierError):
            raise e
    for e in err:
        if e is not None:
            raise e
    return res


def t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def flat(x):
    """Every tensor of a (nested) result, in a fixed order; None skipped."""
    if x is None:
        return []
    if torch.is_tensor(x):
        return [x]
    if isinstance(x, dict):
        return [v for k in sorted(x) for v in flat(x[k])]
    if isinstance(x, (list, tuple)):
        return [v for e in x for v in flat(e)]
    return []


def first_difference(a, b, what):
    """None when a and b are bitwise equal tensor lists (NaN == NaN), else a message."""
    fa, fb = flat(a), flat(b)
    if len(fa) != len(fb):
        return "%s: %d vs %d tensors" % (what, len(fa), len(fb))
    for i, (x, y) in enumerate(zip(fa, fb)):
        if x.shape != y.shape or x.dtype != y.dtype:
            return "%s: tensor %d %s %s vs %s %s" % (what, i, tuple(x.shape), x.dtype, tuple(y.shape), y.dtype)
        if x.is_floating_point():
            same = torch.equal(x.view(torch.int32 if x.element_size() == 4 else torch.int64),
                               y.view(torch.int32 if y.element_size() == 4 else torch.int64)) if x.numel() else True
        else:
            same = torch.equal(x, y)
        if not same:
            return "%s: tensor %d %s differs" % (what, i, tuple(x.shape))
    return None


def clone_all(x):
    return [v.clone() for v in flat(x)]


# ---------------------------------------------------------------------------------------------------------------------
#  A. parameter scopes are per thread (CPU)
# ---------------------------------------------------------------------------------------------------------------------

def _bn_params(rng, scope, C):
    pre = scope + "/batch_normalization/"
    return {pre + "gamma": rng.uniform(0.5, 1.5, C), pre + "beta": rng.normal(size=C),
            pre + "moving_mean": rng.normal(size=C), pre + "moving_variance": rng.uniform(0.5, 2.0, C)}


@pytest.mark.parametrize("holder", [0, 1])
def test_parameter_scope_and_store_are_per_thread(holder):
    from d3feat_b200 import variables as V
    rng = np.random.default_rng(0)
    stores = [V.ParamStore(_bn_params(rng, "layer_0/simple_0", 8), "cpu"),
              V.ParamStore(_bn_params(rng, "x", 8), "cpu")]
    seen = {}

    def holding(barrier):
        with V.use_params(stores[0]), V.variable_scope("layer_0/simple_0"):
            barrier.wait(60)        # 1: the other thread looks while these scopes are open
            barrier.wait(60)        # 2: the other thread's own scopes are open now
            seen["holder"] = (V.current_store(), V.current_scope(), V.scoped("weights"))
            barrier.wait(60)        # 3
        return V.current_store(), V.current_scope()

    def other(barrier):
        barrier.wait(60)
        seen["other_before"] = (V.current_store(), V.current_scope())
        with V.use_params(stores[1]), V.variable_scope("x"), V.variable_scope("y"):
            seen["other_inside"] = (V.current_store(), V.current_scope())
            barrier.wait(60)
            barrier.wait(60)
        return V.current_store(), V.current_scope()

    fns = [holding, other] if holder == 0 else [other, holding]
    res = run_threads(fns, timeout=120)
    assert seen["other_before"] == (None, "")
    assert seen["other_inside"][0] is stores[1] and seen["other_inside"][1] == "x/y"
    assert seen["holder"][0] is stores[0]
    assert seen["holder"][1:] == ("layer_0/simple_0", "layer_0/simple_0/weights")
    assert res == [(None, ""), (None, "")]
    assert V.current_store() is None and V.current_scope() == ""      # the main thread saw none of it


def test_bn_affine_follows_statistics_updates():
    """The folded scale / shift is recomputed when a BN tensor is updated in place or replaced."""
    from d3feat_b200.variables import ParamStore
    rng = np.random.default_rng(1)
    p = {k: v.astype(np.float32) for k, v in _bn_params(rng, "s", 16).items()}
    store = ParamStore(p, "cpu")

    def fold(q):
        g, b, m, v = (np.asarray(q["s/batch_normalization/" + k], np.float64)
                      for k in ("gamma", "beta", "moving_mean", "moving_variance"))
        sc = g / np.sqrt(v + 1e-6)
        return sc.astype(np.float32), (b - m * sc).astype(np.float32)

    def check(q):
        scale, shift = store.bn_affine("s")
        want = fold(q)
        assert np.array_equal(scale.numpy(), want[0]) and np.array_equal(shift.numpy(), want[1])

    check(p)
    assert store.bn_affine("s")[0] is store.bn_affine("s")[0]          # cached while nothing changes
    store.t["s/batch_normalization/moving_variance"].mul_(3.0)          # in place
    p["s/batch_normalization/moving_variance"] = store.t["s/batch_normalization/moving_variance"].numpy().copy()
    check(p)
    newbeta = rng.normal(size=16).astype(np.float32)                    # replaced by a new tensor
    store.t["s/batch_normalization/beta"] = torch.from_numpy(newbeta)
    p["s/batch_normalization/beta"] = newbeta
    check(p)


# ---------------------------------------------------------------------------------------------------------------------
#  B. per-thread error state of the C library (CPU, built library)
# ---------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def built():
    from d3feat_b200 import build, _lib
    build.build()
    return _lib.lib()


def test_last_error_is_per_thread(built):
    """Two threads fail different argument checks at the same time; each reads its own message."""
    lib = built

    def unary(barrier):
        bad = 0
        for _ in range(3000):
            rc = lib.d3f_unary_forward(None, None, None, -1, 4, 4, None, None, None, None, -1.0, None, None, None)
            msg = lib.d3f_last_error()
            bad += rc != -1 or b"bad shape" not in msg or b"Unknown" in msg
        return bad

    def kpconv(barrier):
        bad = 0
        for _ in range(3000):
            rc = lib.d3f_kpconv_forward(None, None, None, None, None, None, None, None, 0, 0, 0, 15, 1, 1, 1.0, 7, 0, 1,
                                        None, None, None, -1.0, None, None, 0, None, None, None)
            msg = lib.d3f_last_error()
            bad += rc != -1 or b"Unknown influence" not in msg or b"bad shape" in msg
        return bad

    assert run_threads([unary, kpconv, unary, kpconv], timeout=120) == [0, 0, 0, 0]


# ---------------------------------------------------------------------------------------------------------------------
#  C. cache publication across streams (GPU)
# ---------------------------------------------------------------------------------------------------------------------

def _poisoned_stream(dev):
    """A fresh stream whose allocator pool holds two small-pool segments filled with NaN: every small allocation made
    on it (a packed image, a folded weight, a BN fold) starts as NaN, so an image read before its producer ran cannot
    pass by luck. A large free block serves the workspaces, so no call on it waits in cudaMalloc."""
    s = torch.cuda.Stream(device=dev)
    with torch.cuda.stream(s):
        blocks = [torch.full((131072,), float("nan"), device=dev) for _ in range(8)]     # 8 x 512 KB = 2 segments
        blocks.append(torch.empty((64 << 20,), dtype=torch.uint8, device=dev))          # workspaces: no cudaMalloc
    s.synchronize()
    del blocks
    return s


def _busy_then(a, b, fn, warm):
    """fn() on stream a behind ~0.25 s of spinning (the first use of a fresh cache entry), then at once on b. warm()
    makes the same call with another cache entry first, so that every kernel is loaded: a module loaded lazily on
    first launch could wait for the spinning stream and hide the race."""
    warm()
    torch.cuda.synchronize()
    with torch.cuda.stream(a):
        torch.cuda._sleep(SLEEP_CYCLES)
        out_a = fn()
    with torch.cuda.stream(b):
        out_b = fn()
    torch.cuda.synchronize()
    return out_a, out_b


def _hit_returns_without_waiting(a, fn):
    """A cache hit enqueued behind the spin returns to the host while a is still busy: no host synchronisation."""
    torch.cuda.synchronize()
    with torch.cuda.stream(a):
        torch.cuda._sleep(SLEEP_CYCLES)
        out = fn()
        busy = not a.query()
    torch.cuda.synchronize()
    assert busy, "a cache hit waited for the stream"
    return out


@pytest.mark.gpu
def test_unary_and_kpconv_packed_weight_published_complete(cuda):
    from d3feat_b200 import convolution_ops as co
    from test_gpu_kpconv import make_case
    rng = np.random.default_rng(20)
    x = rng.normal(size=(2000, 64)).astype(np.float32)
    w = (rng.normal(size=(64, 96)) * 0.2).astype(np.float32)
    xt, wt = t(x, cuda), t(w, cuda)                    # fresh weight tensor: no cache entry yet
    b = _poisoned_stream(cuda)             # its pool is filled too: no cudaMalloc between the two calls
    ya, yb = _busy_then(_poisoned_stream(cuda), b, lambda: co.unary_convolution(xt, wt),
                        lambda: co.unary_convolution(xt, wt.clone()))
    ref, mag = x.astype(np.float64) @ w.astype(np.float64), gemm_mag(x, w)
    assert_close(ya.cpu().numpy(), ref, mag, TOL, "unary on the producing stream")
    assert_close(yb.cpu().numpy(), ref, mag, TOL, "unary on another stream")
    yc = _hit_returns_without_waiting(_poisoned_stream(cuda), lambda: co.unary_convolution(xt, wt))
    assert torch.equal(yc, ya)

    q, s, idx, f, Kp, W = make_case(rng, 1500, 1500, 30, 32, 32, extent=0.08)
    args = [t(v, cuda) for v in (q, s, idx, f, Kp, W)]
    ka, kb = _busy_then(_poisoned_stream(cuda), _poisoned_stream(cuda),
                        lambda: co.KPConv_ops(*args, 0.08, "linear", "sum"),
                        lambda: co.KPConv_ops(*args[:5], args[5].clone(), 0.08, "linear", "sum"))
    ref, mag, alt = kpconv_ref(q, s, idx, f, Kp, W, 0.08)
    assert_close(ka.cpu().numpy(), ref, mag, TOL, "kpconv on the producing stream", alt=alt)
    assert_close(kb.cpu().numpy(), ref, mag, TOL, "kpconv on another stream", alt=alt)
    kc = _hit_returns_without_waiting(_poisoned_stream(cuda), lambda: co.KPConv_ops(*args, 0.08, "linear", "sum"))
    assert torch.equal(kc, ka)


def _pair_ref(x1, w1, a1, x2, w2, a2, alpha):
    y1, m1 = epi_ref(x1.astype(np.float64) @ w1, gemm_mag(x1, w1), a1[0], a1[1])
    y2, m2 = epi_ref(x2.astype(np.float64) @ w2, gemm_mag(x2, w2), a2[0], a2[1])
    return epi_ref(y1 + y2, m1 + m2, alpha=alpha)


@pytest.mark.gpu
def test_pair_fold_published_complete_and_keyed_on_all_six_tensors(cuda):
    from d3feat_b200 import convolution_ops as co
    rng = np.random.default_rng(21)
    N, C1, C2, Cout = 1800, 64, 32, 64
    x1 = rng.normal(size=(N, C1)).astype(np.float32)
    x2 = rng.normal(size=(N, C2)).astype(np.float32)
    w1 = (rng.normal(size=(C1, Cout)) * 0.2).astype(np.float32)
    w2 = (rng.normal(size=(C2, Cout)) * 0.2).astype(np.float32)

    def affine():
        return rng.uniform(0.5, 1.5, Cout).astype(np.float32), rng.normal(size=Cout).astype(np.float32)

    a1, a2 = affine(), affine()
    X1, X2, W1, W2 = (t(v, cuda) for v in (x1, x2, w1, w2))
    A1, A2 = tuple(t(v, cuda) for v in a1), tuple(t(v, cuda) for v in a2)
    call = lambda: co.unary_pair_convolution(X1, W1, A1, X2, W2, A2, 0.2)       # noqa: E731
    ya, yb = _busy_then(_poisoned_stream(cuda), _poisoned_stream(cuda), call,
                        lambda: co.unary_pair_convolution(X1, W1.clone(), A1, X2, W2.clone(), A2, 0.2))
    ref, mag = _pair_ref(x1, w1, a1, x2, w2, a2, 0.2)
    assert_close(ya.cpu().numpy(), ref, mag, TOL, "pair on the producing stream")
    assert_close(yb.cpu().numpy(), ref, mag, TOL, "pair on another stream")
    assert torch.equal(_hit_returns_without_waiting(_poisoned_stream(cuda), call), ya)
    # same weights, a new affine with other values (new tensors, all at version 0): the new fold, output and shift
    for _ in range(2):
        n1, n2 = affine(), affine()
        B1, B2 = tuple(t(v, cuda) for v in n1), tuple(t(v, cuda) for v in n2)
        y = co.unary_pair_convolution(X1, W1, B1, X2, W2, B2, 0.2)
        ref, mag = _pair_ref(x1, w1, n1, x2, w2, n2, 0.2)
        assert_close(y.cpu().numpy(), ref, mag, TOL, "pair with a new affine")
    # and an in-place update of one shift
    A2[1].add_(1.0)
    y = co.unary_pair_convolution(X1, W1, A1, X2, W2, A2, 0.2)
    ref, mag = _pair_ref(x1, w1, a1, x2, w2, (a2[0], a2[1] + np.float32(1.0)), 0.2)
    assert_close(y.cpu().numpy(), ref, mag, TOL, "pair after an in-place shift update")


@pytest.mark.gpu
def test_batch_norm_fold_published_complete(cuda):
    from d3feat_b200 import network_blocks as nb
    from d3feat_b200.variables import ParamStore, use_params, variable_scope
    rng = np.random.default_rng(22)
    C = 128
    p = _bn_params(rng, "s", C)
    store = ParamStore(p, cuda)
    x = rng.normal(size=(3000, C)).astype(np.float32)
    X = t(x, cuda)

    def call(st=store):
        with use_params(st), variable_scope("s"):
            return nb.batch_norm(X, True, 0.99, False)

    ya, yb = _busy_then(_poisoned_stream(cuda), _poisoned_stream(cuda), call, lambda: call(ParamStore(p, cuda)))
    g, be, m, v = (np.asarray(p["s/batch_normalization/" + k], np.float64)
                   for k in ("gamma", "beta", "moving_mean", "moving_variance"))
    sc = g / np.sqrt(v + 1e-6)
    ref = x.astype(np.float64) * sc + (be - m * sc)
    mag = np.abs(x.astype(np.float64) * sc) + np.abs(be - m * sc)
    assert_close(ya.cpu().numpy(), ref, mag, TOL, "batch norm on the producing stream")
    assert_close(yb.cpu().numpy(), ref, mag, TOL, "batch norm on another stream")
    assert torch.equal(_hit_returns_without_waiting(_poisoned_stream(cuda), call), ya)


# ---------------------------------------------------------------------------------------------------------------------
#  E. every op family from a thread pool (GPU)
# ---------------------------------------------------------------------------------------------------------------------

def _rotation(rng, deg):
    a = rng.normal(size=3)
    a /= np.linalg.norm(a)
    th = np.deg2rad(deg)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K


def _op_table(cuda, seed, w_shared):
    """name -> zero-argument call of one op on inputs seeded by `seed` (device tensors made here, on the default
    stream), and the numpy inputs of the ops checked against float64."""
    from d3feat_b200 import convolution_ops as co, network_blocks as nb, synth, tf_custom_ops as ops
    from d3feat_b200.evaluation import GroundTruth, evaluate_pairs
    from d3feat_b200.keypoints import select_keypoints
    from d3feat_b200.matching import match_keypoints
    from d3feat_b200.registration import icp_pairs, register_pairs
    from test_gpu_kpconv import make_case
    rng = np.random.default_rng(100 + seed)
    n = 2500
    src = synth.room_fragment(200 + seed, n)
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = _rotation(rng, 10.0), rng.normal(size=3) * 0.1
    tgt = (src.astype(np.float64) @ T[:3, :3].T + T[:3, 3] + rng.normal(size=src.shape) * 0.002).astype(np.float32)
    P, L = t(np.concatenate([src, tgt]), cuda), t(np.array([n, n], np.int32), cuda)
    d = rng.normal(size=(n, 32))
    D = np.concatenate([d, d + rng.normal(size=d.shape) * 0.05])
    D = t((D / np.linalg.norm(D, axis=1, keepdims=True)).astype(np.float32), cuda)
    scores = t(rng.uniform(0, 1, (2 * n, 1)).astype(np.float32), cuda)
    pairs = t(np.array([[0, 1]], np.int32), cuda)
    truth = GroundTruth(t(T[None], cuda), None, t(np.array([1], np.int32), cuda))
    nbr = ops.batch_ordered_neighbors(P, P, L, L, 0.075, max_cols=30)

    kp_cases = {}
    for Cin in (32, 64):
        q, s, idx, f, Kp, W = make_case(rng, 1500, 1500, 30, Cin, Cin, extent=0.08)
        kp_cases[Cin] = (q, s, idx, f, Kp, W)
    q, s, idx, f, Kp, W = make_case(rng, 1200, 1200, 30, 32, 32, extent=0.08)
    off = (rng.normal(size=(1200, 15, 3)) * 0.02).astype(np.float32)
    kp_cases["deform"] = (q, s, idx, f, Kp, W, off)
    x = rng.normal(size=(3000, 64)).astype(np.float32)
    w_own = (rng.normal(size=(64, 128)) * 0.2).astype(np.float32)
    x2 = rng.normal(size=(3000, 32)).astype(np.float32)
    w1, w2 = ((rng.normal(size=(c, 64)) * 0.2).astype(np.float32) for c in (64, 32))
    aff = [tuple(t(v, cuda) for v in (rng.uniform(0.5, 1.5, 64).astype(np.float32),
                                      rng.normal(size=64).astype(np.float32))) for _ in range(2)]
    feats = rng.normal(size=(2 * n, 32)).astype(np.float32)
    inds = rng.integers(0, 2 * n + 1, (n, 17)).astype(np.int32)

    dv = {k: [t(a, cuda) for a in v] for k, v in kp_cases.items()}
    X, Wown, X2, W1, W2 = (t(a, cuda) for a in (x, w_own, x2, w1, w2))
    F, I = t(feats, cuda), t(inds, cuda)
    kp = select_keypoints(scores, L, 64, points=P, descriptors=D)
    m = match_keypoints(kp, pairs)
    reg = register_pairs(kp, m, pairs, max_iterations=2000)
    ref = icp_pairs(P, L, pairs, reg.pose, distance=0.05, max_iterations=10)
    calls = {
        "grid_subsampling": lambda: ops.batch_grid_subsampling(P, L, 0.06),
        "ordered_neighbors": lambda: ops.batch_ordered_neighbors(P, P, L, L, 0.075),
        "kpconv_cin32": lambda: co.KPConv_ops(*dv[32], 0.08, "linear", "sum"),
        "kpconv_cin64": lambda: co.KPConv_ops(*dv[64], 0.08, "linear", "sum"),
        "kpconv_deform": lambda: co.KPConv_deform_ops(*dv["deform"][:5], dv["deform"][6], None, dv["deform"][5], 0.08,
                                                      "linear", "sum"),
        "unary_shared_weight": lambda: co.unary_convolution(X, w_shared),
        "unary_own_weight": lambda: co.unary_convolution(X, Wown),
        "unary_pair": lambda: co.unary_pair_convolution(X, W1, aff[0], X2, W2, aff[1], 0.2),
        "ind_max_pool": lambda: nb.ind_max_pool(F, I),
        "closest_pool": lambda: nb.closest_pool(F, I),
        "detection_scores": lambda: nb.detection_scores(F, nbr, L),
        "select_keypoints": lambda: select_keypoints(scores, L, 64, points=P, descriptors=D),
        "match_keypoints": lambda: match_keypoints(kp, pairs),
        "register_pairs": lambda: register_pairs(kp, m, pairs, max_iterations=2000),
        "icp_pairs": lambda: icp_pairs(P, L, pairs, reg.pose, distance=0.05, max_iterations=10),
        "evaluate_pairs": lambda: evaluate_pairs(kp, m, pairs, truth, reg, ref),
    }
    host = dict(kp=kp_cases, x=x, w_own=w_own, x2=x2, w1=w1, w2=w2,
                aff=[tuple(v.cpu().numpy() for v in a) for a in aff])
    return calls, host


@pytest.mark.gpu
def test_every_op_family_from_a_thread_pool(cuda):
    from d3feat_b200 import _lib
    rng = np.random.default_rng(30)
    w_shared_np = (rng.normal(size=(64, 128)) * 0.2).astype(np.float32)
    w_shared = t(w_shared_np, cuda)
    n_threads, rounds = 4, 3
    tables = [_op_table(cuda, i, w_shared) for i in range(n_threads)]
    orders = []
    for i in range(n_threads):
        names = sorted(tables[i][0]) * rounds
        random.Random(i).shuffle(names)
        orders.append(names)
    torch.cuda.synchronize()

    def serial(i):
        n0 = _lib.launch_count()
        outs = [clone_all(tables[i][0][name]()) for name in orders[i]]
        torch.cuda.synchronize()
        return outs, _lib.launch_count() - n0

    for i in range(n_threads):
        serial(i)                              # warm-up: packed images, folds, kernel attributes
    want = [serial(i) for i in range(n_threads)]

    # the serial run vs float64 (thread 0's inputs; every thread runs the same ops on other seeds)
    first = {name: want[0][0][orders[0].index(name)] for name in tables[0][0]}
    h = tables[0][1]
    for Cin in (32, 64):
        q, s, idx, f, Kp, W = h["kp"][Cin]
        ref, mag, alt = kpconv_ref(q, s, idx, f, Kp, W, 0.08)
        assert_close(first["kpconv_cin%d" % Cin][0].cpu().numpy(), ref, mag, TOL, "pool kpconv cin%d" % Cin, alt=alt)
    q, s, idx, f, Kp, W, off = h["kp"]["deform"]
    ref, mag, alt = kpconv_ref(q, s, idx, f, Kp, W, 0.08, offsets=off, deform=True)
    assert_close(first["kpconv_deform"][0].cpu().numpy(), ref, mag, TOL, "pool kpconv deform", alt=alt)
    for name, w in (("unary_shared_weight", w_shared_np), ("unary_own_weight", h["w_own"])):
        assert_close(first[name][0].cpu().numpy(), h["x"].astype(np.float64) @ w, gemm_mag(h["x"], w), TOL, name)
    ref, mag = _pair_ref(h["x"], h["w1"], h["aff"][0], h["x2"], h["w2"], h["aff"][1], 0.2)
    assert_close(first["unary_pair"][0].cpu().numpy(), ref, mag, TOL, "pool unary pair")

    def worker(i):
        def run(barrier):
            s = torch.cuda.Stream(device=cuda)
            bad = []
            with torch.cuda.stream(s):
                n0 = _lib.launch_count()
                outs = [clone_all(tables[i][0][name]()) for name in orders[i]]
                launches = _lib.launch_count() - n0
                s.synchronize()
                for k, (name, o) in enumerate(zip(orders[i], outs)):
                    msg = first_difference(o, want[i][0][k], "thread %d call %d %s" % (i, k, name))
                    if msg:
                        bad.append(msg)
            return bad, launches
        return run

    res = run_threads([worker(i) for i in range(n_threads)])
    for i, (bad, launches) in enumerate(res):
        assert not bad, bad[:5]
        assert launches == want[i][1], "thread %d: %d launches, %d serially" % (i, launches, want[i][1])


# ---------------------------------------------------------------------------------------------------------------------
#  D. two models in two threads (GPU)
# ---------------------------------------------------------------------------------------------------------------------

LIMITS = [35, 33, 34, 36, 30]
PAIRS = [(0, 1)]
REGISTER = dict(max_iterations=500, max_validation=500)


def _model_batches(seed):
    from d3feat_b200 import synth
    out = []
    for b in range(3):
        clouds = [synth.room_fragment(300 + 10 * seed + 2 * b + j, 6000 - 300 * j) for j in range(2)]
        out.append((np.concatenate(clouds, 0), np.array([c.shape[0] for c in clouds], np.int32)))
    return out


def _serve(enc, P, L):
    from d3feat_b200.matching import match_keypoints
    from d3feat_b200.registration import register_pairs
    out = enc(P, L, num_keypoints=64)
    m = match_keypoints(out["keypoints"], PAIRS)
    reg = register_pairs(out["keypoints"], m, PAIRS, **REGISTER)
    return [out["F"], out["descriptors"], out["scores"], out["keypoints"], m, reg]


@pytest.fixture(scope="module")
def two_models(cuda):
    from d3feat_b200 import synth
    from d3feat_b200.encoder import KPFCNN
    cfg = synth.Config(architecture=synth.ARCH_3DMATCH)
    encs = [KPFCNN(cfg, synth.make_params(cfg, seed), LIMITS, device=cuda) for seed in (1, 2)]
    batches = [_model_batches(seed) for seed in (1, 2)]
    want = []
    for m, (enc, bs) in enumerate(zip(encs, batches)):
        with record_ops() as tr:
            first = _serve(enc, *bs[0])
            torch.cuda.synchronize()
        check_sampled_rows(tr, 300, np.random.default_rng(m), RTOL, min_kpconv=10, what="model %d" % (m + 1))
        want.append([clone_all(first)] + [clone_all(_serve(enc, *b)) for b in bs[1:]])
        # deterministic: a second serial pass gives the same bits
        assert first_difference(clone_all(_serve(enc, *bs[0])), want[m][0], "model %d repeat" % (m + 1)) is None
    torch.cuda.synchronize()
    return cfg, encs, batches, want


def _eager_worker(cuda, enc, batches, want, iters, tag):
    def run(barrier):
        s = torch.cuda.Stream(device=cuda)
        bad = []
        with torch.cuda.stream(s):
            for it in range(iters):
                b = it % len(batches)
                got = clone_all(_serve(enc, *batches[b]))
                s.synchronize()
                msg = first_difference(got, want[b], "%s iteration %d batch %d" % (tag, it, b))
                if msg:
                    bad.append(msg)
        return bad
    return run


@pytest.mark.gpu
def test_two_models_in_two_threads(cuda, two_models):
    cfg, encs, batches, want = two_models
    res = run_threads([_eager_worker(cuda, encs[m], batches[m], want[m], 20, "model %d" % (m + 1)) for m in (0, 1)])
    assert res == [[], []], [r[:3] for r in res]


@pytest.mark.gpu
def test_replaying_graph_pipeline_next_to_an_eager_model(cuda, two_models):
    """Model 1's GraphPipeline, stepped past its first DEPTH steps (every slot captured, single-threaded), replays in
    one thread while model 2 runs eagerly in another; the pipeline's results equal its single-threaded replays."""
    from d3feat_b200.encoder import GraphPipeline
    cfg, encs, batches, want = two_models
    bs = [(t(P, cuda), t(L, cuda)) for P, L in batches[0]]
    pipe = GraphPipeline.for_batch(encs[0], *bs[0], decoder=True, keypoints=64, match_pairs=PAIRS, register=REGISTER)

    def result(res, counts):
        n0 = int(counts[0].item())
        return [res.descriptors[:n0].clone(), res.scores[:n0].clone()] + clone_all(res[2:]) + [counts.clone()]

    steps = 3 * pipe.DEPTH
    pipe.prime(*bs[0])
    serial = []
    for i in range(steps):
        serial.append(result(*pipe.step(*bs[(i + 1) % 3])))
    torch.cuda.synchronize()
    for i in range(3, steps):
        assert first_difference(serial[i], serial[i % 3], "serial replay %d" % i) is None

    def replaying(barrier):
        s = torch.cuda.Stream(device=cuda)
        bad = []
        with torch.cuda.stream(s):
            for i in range(steps, steps + 20):
                got = result(*pipe.step(*bs[(i + 1) % 3]))
                msg = first_difference(got, serial[i % 3], "graph step %d" % i)
                if msg:
                    bad.append(msg)
            pipe.drain()
        return bad

    res = run_threads([replaying, _eager_worker(cuda, encs[1], batches[1], want[1], 20, "model 2")])
    pipe.check()
    assert res == [[], []], [r[:3] for r in res]


# ---------------------------------------------------------------------------------------------------------------------
#  F. the chunk pipeline's auxiliary stream (GPU, child process: D3F_KPCONV_CHUNK is read once per process)
# ---------------------------------------------------------------------------------------------------------------------

CHUNK = 1024

CHUNK_DRIVER = r"""
import json, sys, threading
import numpy as np
import torch
sys.path.insert(0, sys.argv[1])
from d3feat_b200 import convolution_ops as co, _lib
d = sys.argv[2]
dev = torch.device("cuda", 0)
z = {c: dict(np.load("%s/in_%s.npz" % (d, c))) for c in ("rigid", "deform")}
T = {c: {k: torch.from_numpy(v).to(dev) for k, v in z[c].items()} for c in z}

def call(c, f=None):
    a = T[c]
    f = a["f"] if f is None else f
    if c == "rigid":
        return co.KPConv_ops(a["q"], a["s"], a["idx"], f, a["Kp"], a["W"], 0.06, "linear", "sum")
    return co.KPConv_deform_ops(a["q"], a["s"], a["idx"], f, a["Kp"], a["off"], None, a["W"], 0.06, "linear", "sum")

def same(x, y):
    return torch.equal(x.view(torch.int32), y.view(torch.int32))

def threads(fns):
    b = threading.Barrier(len(fns))
    res, err = [None] * len(fns), [None] * len(fns)
    def body(i):
        try:
            b.wait(60)
            res[i] = fns[i]()
        except BaseException as e:
            err[i] = e
            b.abort()
    ths = [threading.Thread(target=body, args=(i,), daemon=True) for i in range(len(fns))]
    [th.start() for th in ths]
    [th.join(300) for th in ths]
    assert not any(th.is_alive() for th in ths), "thread timeout"
    for e in err:
        if e is not None:
            raise e
    return res

fsets = [T["rigid"]["f%d" % k] for k in range(3)]
serial = {"rigid": call("rigid"), "deform": call("deform")}
for k in range(3):
    serial["set%d" % k] = call("rigid", fsets[k])
torch.cuda.synchronize()
report = {}

# two threads, each on its own stream, multi-chunk rigid and deformable KPConvs at once
def worker(order):
    def run():
        s = torch.cuda.Stream(device=dev)
        bad = []
        with torch.cuda.stream(s):
            for r in range(3):
                outs = [(c, call(c)) for c in order]
                s.synchronize()
                bad += ["%s round %d" % (c, r) for c, o in outs if not same(o, serial[c])]
        return bad
    return run
report["two_threads"] = sum(threads([worker(["rigid", "deform"]), worker(["deform", "rigid"])]), [])

# a thread enqueues one call and exits at once: its auxiliary stream and events go with work pending
s_exit = torch.cuda.Stream(device=dev)
held = {}
def enqueue_and_exit():
    with torch.cuda.stream(s_exit):
        torch.cuda._sleep(100000000)
        held["out"] = call("deform")
threads([enqueue_and_exit])
s_exit.synchronize()
report["thread_exit"] = [] if same(held["out"], serial["deform"]) else ["deform after thread exit"]

def replay_sets(g, f_static, out):
    bad = []
    for k in range(3):
        f_static.copy_(fsets[k])
        g.replay()
        torch.cuda.synchronize()
        if not same(out, serial["set%d" % k]):
            bad.append("replay set %d" % k)
    return bad

# capture in a thread whose auxiliary stream exists (warmed up eagerly first)
def capture(warm):
    def run():
        f_static = fsets[0].clone()
        if warm:
            call("rigid", f_static)
            torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        try:
            with torch.cuda.graph(g):
                out = call("rigid", f_static)
        except _lib.D3FError as e:
            return ("refused", str(e))
        return ("captured", replay_sets(g, f_static, out))
    return run
report["capture_warm"] = threads([capture(True)])[0]
report["capture_cold"] = threads([capture(False)])[0]
for k, v in serial.items():
    np.save("%s/serial_%s.npy" % (d, k), v.cpu().numpy())
json.dump(report, open(d + "/report.json", "w"))
"""


@pytest.mark.gpu
def test_kpconv_chunk_pipeline_from_threads_and_graphs(cuda):
    from test_gpu_kpconv import make_case
    rng = np.random.default_rng(40)
    with tempfile.TemporaryDirectory() as d:
        data = {}
        for c, n, Cin in (("rigid", 3500, 32), ("deform", 3300, 64)):
            assert -(-n // CHUNK) >= 3 and n % CHUNK != 0
            q, s, idx, f, Kp, W = make_case(rng, n, n, 36, Cin, 32, extent=0.06)
            f[::5] = -np.abs(f[::5])
            z = dict(q=q, s=s, idx=idx, f=f, Kp=Kp, W=W)
            if c == "deform":
                z["off"] = (rng.normal(size=(n, 15, 3)) * 0.02).astype(np.float32)
            else:
                for k in range(3):
                    z["f%d" % k] = rng.normal(size=f.shape).astype(np.float32)
            np.savez(os.path.join(d, "in_%s.npz" % c), **z)
            data[c] = z
        env = dict(os.environ, D3F_KPCONV_CHUNK=str(CHUNK))
        r = subprocess.run([sys.executable, "-c", CHUNK_DRIVER, ROOT, d], env=env, capture_output=True, text=True,
                           timeout=900)
        assert r.returncode == 0, r.stderr[-4000:]
        rep = json.load(open(os.path.join(d, "report.json")))
        out = {k: np.load(os.path.join(d, "serial_%s.npy" % k)) for k in ("rigid", "deform", "set0", "set1", "set2")}
    assert rep["two_threads"] == [] and rep["thread_exit"] == [], rep
    assert rep["capture_warm"] == ["captured", []], rep
    kind, detail = rep["capture_cold"]
    if kind == "refused":
        assert "warm" in detail.lower(), detail
    else:
        assert detail == [], rep
    z = data["rigid"]
    for name, f in (("rigid", z["f"]), ("set0", z["f0"]), ("set1", z["f1"]), ("set2", z["f2"])):
        ref, mag, alt = kpconv_ref(z["q"], z["s"], z["idx"], f, z["Kp"], z["W"], 0.06)
        assert_close(out[name], ref, mag, TOL, "chunked %s" % name, alt=alt)
    z = data["deform"]
    ref, mag, alt = kpconv_ref(z["q"], z["s"], z["idx"], z["f"], z["Kp"], z["W"], 0.06, offsets=z["off"], deform=True)
    assert_close(out["deform"], ref, mag, TOL, "chunked deform", alt=alt)


# ---------------------------------------------------------------------------------------------------------------------
#  G. a GraphPipeline whose level-0 KPConvs take several chunks (GPU, no environment override)
# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_graph_pipeline_with_chunked_level0(cuda):
    """20 x 30 000-point fragments = 600 000 level-0 rows; one chunk holds 279 552 rows of a Cin = 32 layer
    (chunk_queries(15, 32)), so level 0 runs three chunks on the auxiliary stream inside the captured graphs."""
    from d3feat_b200 import pyramid as pyr, synth
    from d3feat_b200.encoder import GraphPipeline, KPFCNN
    cfg = synth.Config(architecture=synth.ARCH_ENCODER)
    enc = KPFCNN(cfg, synth.make_params(cfg, seed=0), [40] * 5, device=cuda)
    batches = []
    for b in range(3):
        clouds = [synth.room_fragment(20 * b + j, 30000) for j in range(20)]
        batches.append((t(np.concatenate(clouds, 0), cuda), t(np.full(20, 30000, np.int32), cuda)))
    pipe = GraphPipeline.for_batch(enc, *batches[0], decoder=False, encoder_streams=2)
    assert pipe.caps[0] > 279552 * 2

    def eager_static(P, L, trace=False):
        buf = pyr.PyramidBuffers(cfg, enc.limits, pipe.caps, pipe.n_clouds, cuda, bbox=pipe.bbox)
        n0 = int(P.shape[0])
        buf.points0[:n0].copy_(P)
        buf.lengths0.copy_(L)
        buf.n0.fill_(n0)
        inputs = enc.build_inputs_static(buf)
        if trace:
            with record_ops() as tr:
                F = enc.encode(inputs)
                torch.cuda.synchronize()
        else:
            F = enc.encode(inputs)
        counts = inputs["counts"][:5].cpu().tolist()
        assert int(inputs["status"].item()) == 0
        return F[-1][:counts[4]].clone(), counts, (tr if trace else None)

    e0, c0, tr = eager_static(*batches[0], trace=True)
    assert c0[0] == 600000
    rep = check_sampled_rows(tr, 2000, np.random.default_rng(3), RTOL, min_kpconv=10, what="600k static")
    assert sum(1 for r in rep if r[0] in ("unary", "unary_pair")) >= 18
    del tr
    eager = [(e0, c0)] + [eager_static(*b)[:2] for b in batches[1:]]
    pipe.prime(*batches[0])
    got = []
    for i in range(3):
        res, cnt = pipe.step(*batches[i + 1]) if i < 2 else pipe.step()
        got.append((res.clone(), cnt[:5].cpu().tolist()))
    pipe.check()
    for i, ((res, cnt), (want, wc)) in enumerate(zip(got, eager)):
        assert cnt == wc, i
        assert torch.equal(res[:wc[4]], want), "graph step %d" % i
