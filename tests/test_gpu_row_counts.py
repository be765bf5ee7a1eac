"""The device row-count contract of every row-wise entry point (include/d3feat_b200.h, "Device-side row counts"): with
capacity-sized buffers and the actual count n in device memory, rows below n equal the float64 restatement on the
unpadded inputs, and rows at or beyond n are neither read nor written.

Every input row past the count holds NaN / 1e30, every index row past the count holds in-range but wrong indices (real
support rows), and the output is pre-filled with a sentinel bit pattern, so a kernel that reads past its count gives
a wrong value (never an out-of-bounds access) and one that writes past it leaves a changed sentinel. A negative count
means zero rows (dyn_rows clamps it). Called through the raw C ABI so that the output buffer is the caller's.
"""
import numpy as np
import pytest
import torch

from oracle import kpconv_np as ok
from oracle import native as on

from _oracle import TOL, assert_close, epilogue, gemm_mag, kpconv_ref

pytestmark = pytest.mark.gpu

CAP = 300
COUNTS = [0, 1, CAP // 2 + 3, CAP, -5]
SENTINEL = np.int32(0x7FBADBAD)         # a NaN payload no kernel produces


def t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def P(x):
    from d3feat_b200 import _lib
    return _lib.ptr(x)


def poisoned(a, n):
    """a with every row >= n replaced by NaN (even rows) / 1e30 (odd rows)."""
    a = np.array(a, np.float32, copy=True)
    a[n::2] = np.nan
    a[n + 1::2] = 1e30
    return a


def wrong_indices(idx, n, rng):
    idx = np.array(idx, np.int32, copy=True)
    idx[n:] = rng.integers(0, max(n, 1), idx[n:].shape)
    return idx


def sentinel_out(rows, cols, dev):
    return torch.full((rows, cols), int(SENTINEL), dtype=torch.int32, device=dev).view(torch.float32)


def check_tail(out, n, what):
    tail = out[n:].cpu().view(torch.int32).numpy()
    assert np.all(tail == SENTINEL), "%s: %d rows past the count were written" % (what, int((tail != SENTINEL).any(-1).sum()))


class Keep:
    """Device pointers of arrays / tensors that stay alive until the test ends (a temporary would be freed, and its
    memory handed to the next argument, before the asynchronous kernel reads it)."""

    def __init__(self, dev):
        self.dev, self.held = dev, []

    def __call__(self, a):
        if a is None:
            return None
        x = a if torch.is_tensor(a) else t(a, self.dev)
        self.held.append(x)
        return P(x)


def dev_count(n, dev):
    return torch.tensor([n], dtype=torch.int32, device=dev)


def call(rc, what):
    from d3feat_b200 import _lib
    _lib.check(rc, what)


# ---- GEMMs ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("path", ["tc", "gemm_f32"])
@pytest.mark.parametrize("n", COUNTS)
def test_unary_forward_row_count(cuda, n, path):
    from d3feat_b200 import _lib, convolution_ops as co
    D = Keep(cuda)
    L, m = _lib.lib(), max(n, 0)
    rng = np.random.default_rng(n + 7)
    Cin, Cout = 64, 48
    x = rng.normal(size=(CAP, Cin)).astype(np.float32)
    w = (rng.normal(size=(Cin, Cout)) * 0.2).astype(np.float32)
    res = rng.normal(size=(CAP, Cout)).astype(np.float32)
    scale = rng.uniform(0.5, 1.5, Cout).astype(np.float32)
    shift = rng.normal(size=Cout).astype(np.float32)
    wt = t(w, cuda)
    wp = co.packed_weight(wt) if path == "tc" else None
    out = sentinel_out(CAP, Cout, cuda)
    call(L.d3f_unary_forward(D(poisoned(x, m)), P(wt), P(wp), CAP, Cin, Cout, D(scale),
                             D(shift), None, D(poisoned(res, m)), 0.2, P(out), _lib.stream(),
                             D(dev_count(n, cuda))), "d3f_unary_forward")
    torch.cuda.synchronize()
    ref, mag = epilogue(x[:m].astype(np.float64) @ w, gemm_mag(x[:m], w), scale, shift, residual=res[:m], alpha=0.2)
    assert_close(out[:m].cpu().numpy(), ref, mag, TOL, "unary %s n=%d" % (path, n))
    check_tail(out, m, "unary")


@pytest.mark.parametrize("n", COUNTS)
def test_unary_pair_forward_row_count(cuda, n):
    from d3feat_b200 import _lib
    D = Keep(cuda)
    L, m = _lib.lib(), max(n, 0)
    rng = np.random.default_rng(n + 11)
    C1, C2, Cout = 32, 36, 64
    x1 = rng.normal(size=(CAP, C1)).astype(np.float32)
    x2 = rng.normal(size=(CAP, C2)).astype(np.float32)
    w = (rng.normal(size=(C1 + C2, Cout)) * 0.2).astype(np.float32)       # the folded [w1 * s1 ; w2 * s2]
    shift = rng.normal(size=Cout).astype(np.float32)
    packed = torch.empty((L.d3f_packed_weight_floats(C1 + C2, Cout),), dtype=torch.float32, device=cuda)
    call(L.d3f_pack_weight(D(w), C1 + C2, Cout, P(packed), _lib.stream()), "d3f_pack_weight")
    out = sentinel_out(CAP, Cout, cuda)
    call(L.d3f_unary_pair_forward(D(poisoned(x1, m)), C1, D(poisoned(x2, m)), C2, P(packed), CAP,
                                  Cout, D(shift), 0.2, P(out), _lib.stream(), D(dev_count(n, cuda))),
         "d3f_unary_pair_forward")
    torch.cuda.synchronize()
    xx = np.concatenate([x1[:m], x2[:m]], 1)
    ref, mag = epilogue(xx.astype(np.float64) @ w, gemm_mag(xx, w), shift=None, bias=shift, alpha=0.2)
    assert_close(out[:m].cpu().numpy(), ref, mag, TOL, "unary_pair n=%d" % n)
    check_tail(out, m, "unary_pair")


# ---- KPConv -----------------------------------------------------------------------------------------------------------

KP_FAMILIES = {
    "cin1": dict(Cin=1, Cout=64), "fast4": dict(Cin=32, Cout=32), "mma8": dict(Cin=64, Cout=32, infl="gaussian"),
    "splitk": dict(Cin=64, Cout=64), "v2": dict(Cin=96, Cout=32), "generic": dict(Cin=5, Cout=32),
    "anyk": dict(Cin=32, Cout=32, K=7), "deform_mma4": dict(Cin=32, Cout=32, deform=True),
    "fused": dict(Cin=32, Cout=32, cap=4000, env={"D3F_FUSED_KPCONV": "1"}),
}


@pytest.mark.parametrize("n", COUNTS)
@pytest.mark.parametrize("fam", sorted(KP_FAMILIES))
def test_kpconv_row_count(cuda, monkeypatch, fam, n):
    from d3feat_b200 import _lib, convolution_ops as co
    D = Keep(cuda)
    spec = dict(K=15, infl="linear", deform=False, cap=CAP, env={})
    spec.update(KP_FAMILIES[fam])
    for k, v in spec["env"].items():
        monkeypatch.setenv(k, v)
    L, cap, K, Cin, Cout = _lib.lib(), spec["cap"], spec["K"], spec["Cin"], spec["Cout"]
    if n == CAP:
        n = cap
    elif n == CAP // 2 + 3:
        n = cap // 2 + 3
    m = max(n, 0)
    rng = np.random.default_rng(cap + m + Cin)
    extent, H = 0.08, 30
    s = rng.uniform(0, 1, (cap, 3)).astype(np.float32)
    f = rng.normal(size=(cap, Cin)).astype(np.float32)
    if Cin > 1:
        f[::5] = -np.abs(f[::5])
    idx = np.full((cap, H), m, np.int32)                            # shadow index = the actual support count
    if m:
        nb = on.port_batch_neighbors(s[:m], s[:m], [m], [m], 2.5 * extent, max_cols=H)
        idx[:m, :nb.shape[1]] = nb
    idx = wrong_indices(idx, m, rng)
    Kp = np.concatenate([np.zeros((1, 3)), rng.normal(size=(K - 1, 3))], 0)
    Kp[1:] *= 1.5 * extent / np.linalg.norm(Kp[1:], axis=1, keepdims=True)
    Kp = Kp.astype(np.float32)
    W = (rng.normal(size=(K, Cin, Cout)) * np.sqrt(2.0 / Cout)).astype(np.float32)
    scale = rng.uniform(0.5, 1.5, Cout).astype(np.float32)
    shift = rng.normal(size=Cout).astype(np.float32)
    order = np.arange(cap, dtype=np.int32)
    order[:m] = rng.permutation(m)                                  # first n slots: a permutation of [0, n)
    use_order = fam not in ("fused",)
    Wt = t(W, cuda)
    wp = co.packed_weight(Wt)
    ws = _lib.workspace(L.d3f_kpconv_workspace_bytes(cap, cap, H, K, Cin, Cout), cuda)
    out = sentinel_out(cap, Cout, cuda)
    cnt = dev_count(n, cuda)
    q_d, s_d = t(poisoned(s, m), cuda), t(poisoned(s, m), cuda)
    f_d, idx_d = t(poisoned(f, m), cuda), t(idx, cuda)
    ord_d = t(order, cuda) if use_order else None
    off = mod = None
    if spec["deform"]:
        off = (rng.normal(size=(cap, K, 3)) * 0.02).astype(np.float32)
        mod = rng.uniform(0.5, 1.5, (cap, K)).astype(np.float32)
        call(L.d3f_kpconv_deform_forward(P(q_d), P(s_d), P(idx_d), P(f_d), D(Kp), D(poisoned(off, m)),
                                         D(poisoned(mod, m)), P(Wt), P(wp), P(ord_d), cap, cap, H, K, Cin,
                                         Cout, extent, 1, 0, D(scale), D(shift), None, 0.2, P(out),
                                         P(ws), ws.numel(), _lib.stream(), P(cnt), P(cnt)), "d3f_kpconv_deform_forward")
    else:
        infl = {"linear": 1, "gaussian": 2}[spec["infl"]]
        call(L.d3f_kpconv_forward(P(q_d), P(s_d), P(idx_d), P(f_d), D(Kp), P(Wt), P(wp), P(ord_d), cap, cap,
                                  H, K, Cin, Cout, extent, infl, 0, 1, D(scale), D(shift), None, 0.2,
                                  P(out), P(ws), ws.numel(), _lib.stream(), P(cnt), P(cnt)), "d3f_kpconv_forward")
    torch.cuda.synchronize()
    ref, mag, alt = kpconv_ref(s[:m], s[:m], idx[:m], f[:m], Kp, W, extent, spec["infl"], "sum",
                               None if off is None else off[:m], None if mod is None else mod[:m],
                               deform=spec["deform"], epi=(scale, shift, 0.2))
    assert_close(out[:m].cpu().numpy(), ref, mag, TOL, "kpconv row count %s n=%d" % (fam, n), alt=alt)
    check_tail(out, m, "kpconv " + fam)


# ---- pools, normalisation, scores, stand-alone epilogue -------------------------------------------------------------

def _pool_case(n, rng, C=40, H=9):
    m = max(n, 0)
    n2 = max(m // 2, 0) if n != 1 else 1
    x = rng.normal(size=(CAP, C)).astype(np.float32)
    inds = np.full((CAP, H), m, np.int32)
    if m:
        inds[:n2] = rng.integers(0, m + 1, (n2, H))                 # real rows: supports [0, m], shadow = m
        inds[:n2:3] = m                                             # some all-shadow rows
    inds = wrong_indices(inds, n2, rng)
    return m, n2, x, inds


@pytest.mark.parametrize("n", COUNTS)
def test_pools_row_count(cuda, n):
    from d3feat_b200 import _lib
    D = Keep(cuda)
    L = _lib.lib()
    rng = np.random.default_rng(n + 10)
    m, n2, x, inds = _pool_case(n, rng)
    C = x.shape[1]
    xd, idd = t(poisoned(x, m), cuda), t(inds, cuda)
    n1d, n2d = dev_count(n if n < 0 else m, cuda), dev_count(n2, cuda)
    ws = _lib.workspace(L.d3f_ind_max_pool_workspace_bytes(C), cuda)
    out = sentinel_out(CAP, C, cuda)
    call(L.d3f_ind_max_pool(P(xd), P(idd), CAP, CAP, inds.shape[1], C, P(out), P(ws), ws.numel(), _lib.stream(),
                            P(n1d), P(n2d)), "d3f_ind_max_pool")
    torch.cuda.synchronize()
    if m:
        assert np.array_equal(out[:n2].cpu().numpy(), ok.ind_max_pool(x[:m], inds[:n2]))
    check_tail(out, n2, "ind_max_pool")
    out = sentinel_out(CAP, C, cuda)
    call(L.d3f_closest_pool(P(xd), P(idd), CAP, CAP, inds.shape[1], C, P(out), _lib.stream(), P(n1d), P(n2d)),
         "d3f_closest_pool")
    torch.cuda.synchronize()
    assert np.array_equal(out[:n2].cpu().numpy(), ok.closest_pool(x[:m], inds[:n2]))
    check_tail(out, n2, "closest_pool")


@pytest.mark.parametrize("n", COUNTS)
def test_row_wise_epilogues_row_count(cuda, n):
    from d3feat_b200 import _lib
    D = Keep(cuda)
    L, m = _lib.lib(), max(n, 0)
    rng = np.random.default_rng(n + 5)
    C = 36
    x = rng.normal(size=(CAP, C)).astype(np.float32)
    res = rng.normal(size=(CAP, C)).astype(np.float32)
    scale = rng.uniform(0.5, 1.5, C).astype(np.float32)
    shift = rng.normal(size=C).astype(np.float32)
    cnt = dev_count(n, cuda)
    xd = t(poisoned(x, m), cuda)
    # l2 normalisation: each element is x / |x|, off by a few ulp of itself
    out = sentinel_out(CAP, C, cuda)
    call(L.d3f_l2_normalize(P(xd), CAP, C, 1e-10, P(out), _lib.stream(), P(cnt)), "d3f_l2_normalize")
    torch.cuda.synchronize()
    x64 = x[:m].astype(np.float64)
    ref = x64 / np.sqrt(np.maximum((x64 * x64).sum(1, keepdims=True), 1e-10))
    assert_close(out[:m].cpu().numpy(), ref, np.abs(ref), TOL, "l2_normalize n=%d" % n)
    check_tail(out, m, "l2_normalize")
    # batch norm + residual + LeakyReLU
    out = sentinel_out(CAP, C, cuda)
    call(L.d3f_affine_leaky(P(xd), CAP, C, D(scale), D(shift), D(poisoned(res, m)), 0.2,
                            P(out), _lib.stream(), P(cnt)), "d3f_affine_leaky")
    torch.cuda.synchronize()
    ref, mag = epilogue(x64, np.abs(x64), scale, shift, residual=res[:m], alpha=0.2)
    assert_close(out[:m].cpu().numpy(), ref, mag, TOL, "affine_leaky n=%d" % n)
    check_tail(out, m, "affine_leaky")


SCORE_ROW_CASES = [(n, None) for n in COUNTS] + [(CAP // 2 + 3, e) for e in (0, 37, -37)]


def _score_lengths(m, excess):
    """Seven clouds (empty and one-point ones among them) whose lengths sum to m + excess."""
    lens = np.array([0, 1, 40, 0, 35, 1, 0], np.int64)
    lens[-1] = m + excess - lens.sum()
    assert lens[-1] > 0
    return lens.astype(np.int32)


@pytest.mark.parametrize("n,excess", SCORE_ROW_CASES,
                         ids=[str(n) if e is None else "B7_excess%+d" % e for n, e in SCORE_ROW_CASES])
def test_detection_scores_row_count(cuda, n, excess):
    """One cloud of exactly n rows, or (excess given) seven clouds whose lengths sum to n + excess: more than n cuts
    the last cloud at n, less than n leaves rows past the last cloud that belong to no cloud. Those rows hold a huge
    maximum: they must not change any real row's score (compared with the oracle, and bit for bit with the same clouds
    at n = sum of the lengths); their own score is unspecified. Element by element against float64."""
    from d3feat_b200 import _lib
    D = Keep(cuda)
    L, m = _lib.lib(), max(n, 0)
    rng = np.random.default_rng(n + 9 + (0 if excess is None else 1000 + excess))
    dim, H = 32, 12
    x = np.abs(rng.normal(size=(CAP, dim))).astype(np.float32)
    x[rng.uniform(size=CAP) < 0.1] = 0.0
    lengths = np.array([m], np.int32) if excess is None else _score_lengths(m, excess)
    start = np.minimum(np.concatenate([[0], np.cumsum(lengths)]), m)
    real = int(start[-1])                                          # rows that belong to a cloud
    nbr = np.full((CAP, H), m, np.int32)
    for b in range(len(lengths)):                                  # neighbours within the cloud, or the shadow m
        a, e = start[b], start[b + 1]
        if e > a:
            blk = rng.integers(a, e + 1, (e - a, H)).astype(np.int32)
            blk[blk == e] = m
            nbr[a:e] = blk
    x[real:m] = 1e6                                                # rows of no cloud: a huge maximum
    nbr = wrong_indices(nbr, m, rng)
    ws = _lib.workspace(L.d3f_detection_scores_workspace_bytes(CAP, len(lengths)), cuda)
    out = sentinel_out(CAP, 1, cuda)
    call(L.d3f_detection_scores(D(poisoned(x, m)), D(nbr), D(lengths), len(lengths), CAP, H, dim,
                                P(out), P(ws), ws.numel(), _lib.stream(), D(dev_count(n, cuda))),
         "d3f_detection_scores")
    torch.cuda.synchronize()
    ref, mag, alt = ok.detection_scores(x[:m].astype(np.float64), nbr[:m], lengths, magnitude=True)
    assert_close(out[:real].cpu().numpy(), ref[:real], mag[:real], TOL, "detection_scores n=%d lengths %s" % (
        n, "[%d]" % m if excess is None else "sum n%+d" % excess), alt=alt[:real])
    check_tail(out, m, "detection_scores")
    if excess is not None and excess < 0:                          # the same clouds without the rows of no cloud
        nb_real = np.where(nbr[:real] == m, real, nbr[:real])
        ws = _lib.workspace(L.d3f_detection_scores_workspace_bytes(real, len(lengths)), cuda)
        alone = torch.empty((real, 1), dtype=torch.float32, device=cuda)
        call(L.d3f_detection_scores(D(x[:real]), D(nb_real), D(lengths), len(lengths), real, H, dim, P(alone), P(ws),
                                    ws.numel(), _lib.stream(), None), "d3f_detection_scores")
        torch.cuda.synchronize()
        assert torch.equal(out[:real], alone), "rows past the last cloud changed a real row's score"
