"""The element-wise check (tests/_oracle.py) is tight enough to matter: it rejects numpy emulations of the ways a KPConv,
GEMM or detection-score kernel typically goes wrong, at the shapes of the GPU tests, and accepts the float32 evaluation
of the same restatement (what an honest fp32 kernel with another summation order computes). The many-cloud batches of
the subsampling and neighbour tests change the oracle's result under every emulated batch-assignment bug. No GPU
needed."""
import numpy as np
import pytest

from oracle import kpconv_np as ok

from _oracle import TOL, assert_close, gemm_mag, epilogue, ratio, tf32, f64
from test_gpu_kpconv import make_case
from test_gpu_widen import SCORE_CASES, score_case


def rejects(out, ref, mag, alt=None):
    with pytest.raises(AssertionError):
        assert_close(out, ref, mag, TOL, "emulated bug", alt=alt)


# ---- GEMM (unary convolution, and the KPConv contraction [Nq, K*Cin] @ [K*Cin, Cout]) --------------------------------

GEMM_SHAPES = [(3000, 64, 32), (3000, 32, 128), (645, 1024, 256), (700, 960, 64)]


def _gemm_case(N, Cin, Cout):
    rng = np.random.default_rng(N + Cin + Cout)
    x = rng.normal(size=(N, Cin)).astype(np.float32)
    w = (rng.normal(size=(Cin, Cout)) * np.sqrt(2.0 / Cout)).astype(np.float32)
    return x, w, f64(x) @ f64(w), gemm_mag(x, w)


@pytest.mark.parametrize("N,Cin,Cout", GEMM_SHAPES)
def test_float32_gemm_is_accepted(N, Cin, Cout):
    x, w, ref, mag = _gemm_case(N, Cin, Cout)
    assert_close(x @ w, ref, mag, TOL, "fp32 gemm %dx%dx%d" % (N, Cin, Cout))
    rng = np.random.default_rng(1)
    scale = rng.uniform(0.5, 1.5, Cout).astype(np.float32)
    shift = rng.normal(size=Cout).astype(np.float32)
    res = rng.normal(size=(N, Cout)).astype(np.float32)
    y, m = epilogue(ref, mag, scale, shift, residual=res, alpha=0.2)
    y32 = (x @ w) * scale + shift + res
    y32 = np.where(y32 > 0, y32, np.float32(0.2) * y32)
    assert_close(y32, y, m, TOL, "fp32 gemm + epilogue")


@pytest.mark.parametrize("N,Cin,Cout", GEMM_SHAPES)
def test_one_pass_tf32_gemm_is_rejected(N, Cin, Cout):
    x, w, ref, mag = _gemm_case(N, Cin, Cout)
    rejects(tf32(x) @ tf32(w), ref, mag)


@pytest.mark.parametrize("N,Cin,Cout", GEMM_SHAPES)
def test_3xtf32_without_the_al_bh_term_is_rejected(N, Cin, Cout):
    x, w, ref, mag = _gemm_case(N, Cin, Cout)
    xh, wh = f64(tf32(x)), f64(tf32(w))
    wl = f64(w) - wh
    rejects(xh @ wh + xh @ wl, ref, mag)           # Ah.Bh + Ah.Bl; the Al.Bh correction is missing
    xl = f64(x) - xh
    assert_close(xh @ wh + xl @ wh + xh @ wl, ref, mag, TOL, "complete 3xTF32")


@pytest.mark.parametrize("N,Cin,Cout", GEMM_SHAPES)
def test_ragged_last_tile_left_at_zero_is_rejected(N, Cin, Cout):
    x, w, ref, mag = _gemm_case(N, Cin, Cout)
    assert N % 128 != 0
    out = (x @ w).copy()
    out[N // 128 * 128:] = 0
    rejects(out, ref, mag)


# ---- KPConv ---------------------------------------------------------------------------------------------------------

KP_SHAPES = [(32, 32, 800, 800, 32, 0.1), (64, 64, 900, 3000, 37, 0.06), (48, 40, 500, 500, 40, 0.12)]


def _kp_case(Cin, Cout, Nq, Ns, H, extent):
    rng = np.random.default_rng(Cin * 7 + H)
    q, s, idx, f, Kp, W = make_case(rng, Nq, Ns, H, Cin, Cout, extent=extent)
    f[::5] = -np.abs(f[::5])          # some supports do not count towards nn
    return q, s, idx, f, Kp, W


def _nn(f, idx):
    fs = np.concatenate([f.astype(np.float64), np.zeros((1, f.shape[1]))], 0)
    return np.maximum((fs[idx].sum(-1) > 0).sum(-1), 1)


@pytest.mark.parametrize("Cin,Cout,Nq,Ns,H,extent", KP_SHAPES)
def test_kpconv_bugs_are_rejected_and_float32_accepted(Cin, Cout, Nq, Ns, H, extent):
    q, s, idx, f, Kp, W = _kp_case(Cin, Cout, Nq, Ns, H, extent)
    args = (Kp, W, extent, "linear", "sum")
    ref, mag, alt = ok.kpconv_ops(q, s, idx, f, *args, dtype=np.float64, magnitude=True)
    assert np.array_equal(ref, ok.kpconv_ops(q, s, idx, f, *args, dtype=np.float64))
    out32 = ok.kpconv_ops(q, s, idx, f, *args, dtype=np.float32)
    assert_close(out32, ref, mag, TOL, "fp32 kpconv Cin %d" % Cin, alt=alt)
    # tensor-core operands rounded to TF32 once (1xTF32)
    rejects(ok.kpconv_ops(q, s, idx, tf32(f), Kp, tf32(W), extent, "linear", "sum"), ref, mag, alt)
    # one neighbour column skipped in one row: the real neighbour with the largest weight of row 7
    r = 7
    real = np.where(idx[r] < Ns)[0]
    j = real[np.argmin(np.linalg.norm(s[idx[r, real]] - q[r], axis=1))]
    idx_bug = idx.copy()
    idx_bug[r, j] = Ns
    rejects(ok.kpconv_ops(q, s, idx_bug, f, *args), ref, mag, alt)
    # nn off by one in one row
    nn = _nn(f, idx)
    out = ref.copy()
    out[r] *= nn[r] / (nn[r] + 1.0)
    rejects(out, ref, mag, alt)
    # two output rows swapped (a row map shifted by one slot)
    out = ref.copy()
    out[[10, 11]] = out[[11, 10]]
    rejects(out, ref, mag, alt)
    # ragged last tile of the contraction left at zero
    out = ref.copy()
    out[Nq // 128 * 128:] = 0
    rejects(out, ref, mag, alt)


@pytest.mark.parametrize("influence", ["constant", "linear", "gaussian"])
@pytest.mark.parametrize("mode", ["sum", "closest"])
def test_float32_accepted_every_influence_and_mode(influence, mode):
    q, s, idx, f, Kp, W = _kp_case(32, 48, 800, 800, 32, 0.1)
    ref, mag, alt = ok.kpconv_ops(q, s, idx, f, Kp, W, 0.1, influence, mode, magnitude=True)
    out32 = ok.kpconv_ops(q, s, idx, f, Kp, W, 0.1, influence, mode, dtype=np.float32)
    assert_close(out32, ref, mag, TOL, "fp32 kpconv %s %s" % (influence, mode), alt=alt)
    rng = np.random.default_rng(3)
    off = (rng.normal(size=(800, 15, 3)) * 0.03).astype(np.float32)
    mods = rng.uniform(0.5, 1.5, (800, 15)).astype(np.float32)
    ref, mag, alt = ok.kpconv_deform_ops(q, s, idx, f, Kp, off, mods, W, 0.1, influence, mode, magnitude=True)
    out32 = ok.kpconv_deform_ops(q, s, idx, f, Kp, off, mods, W, 0.1, influence, mode, dtype=np.float32)
    assert_close(out32, ref, mag, TOL, "fp32 deformable %s %s" % (influence, mode), alt=alt)
    out = ref.copy()
    out[5] *= 1.0 + 1e-3                                     # a 1e-3 slip in one row
    rejects(out, ref, mag, alt)


def test_nn_predicate_ambiguity_is_marked_but_exact_zero_rows_are_not():
    """Rows summing to exactly zero ([a, -a, b, -b, ...], or all zero) are deterministic 'not > 0' in every summation
    order and must not be marked; a row sum that is nonzero but within rounding of zero is marked (alt flips its nn
    vote)."""
    q, s, idx, f, Kp, W = _kp_case(32, 32, 400, 400, 24, 0.12)
    used = np.unique(idx[idx < 400])
    a, b, c = used[:3]
    f[a] = 0
    f[b, 0::2] = np.abs(f[b, 0::2])
    f[b, 1::2] = -f[b, 0::2]                                  # exactly cancelling
    ref, mag, alt = ok.kpconv_ops(q, s, idx, f, Kp, W, 0.12, "linear", "sum", magnitude=True)
    assert np.array_equal(ref, alt)
    f[c] = f[b]
    f[c, 0] += np.float32(1e-6) * abs(f[c, 0])               # sum = tiny positive, far inside the rounding band
    assert 0 < f64(f[c]).sum() < ok.NN_SUM_ULPS * np.abs(f64(f[c])).sum()
    ref, mag, alt = ok.kpconv_ops(q, s, idx, f, Kp, W, 0.12, "linear", "sum", magnitude=True)
    rows = np.any(idx == c, axis=1)
    assert rows.any()
    assert not np.array_equal(ref[rows], alt[rows])
    assert np.array_equal(ref[~rows], alt[~rows])


def test_closest_mode_ties_are_marked():
    q, s, idx, f, Kp, W = _kp_case(32, 32, 400, 400, 24, 0.12)
    Kp = Kp.copy()
    # put a support exactly halfway between two kernel points of query 0 (in float32 input coordinates)
    sup = int(idx[0, 0])
    s = s.copy()
    Kp[2] = Kp[1] + np.float32(0.02) * np.array([1, 0, 0], np.float32)
    s[sup] = q[0] + (Kp[1] + Kp[2]) / 2
    ref, mag, alt = ok.kpconv_ops(q, s, idx, f, Kp, W, 0.12, "linear", "closest", magnitude=True)
    assert not np.array_equal(ref[0], alt[0])
    assert np.array_equal(ref[1:], alt[1:]) or np.any(idx[1:] == sup)


# ---- detection scores -------------------------------------------------------------------------------------------------

SCORE_LENGTHS = [0, 1, 700, 600, 650, 500, 550, 450, 1, 0, 600, 520]    # every kind of score_case, twice over
SCORE_BUGS = ("mean_over_h", "skip_last_column", "prev_cloud_max_first_row", "row_max", "softplus_cut_2")


def _emulated_scores(x, nbr, lengths, bug=None):
    """float32 emulation of the detection-score kernel (csrc/pool.cu): one scale 1/(M + 1e-6) per row applied to the
    row and its neighbourhood, the count_nonzero vote on the raw row sum, one optional injected bug."""
    f32 = np.float32
    x = np.asarray(x, f32)
    N, D = x.shape
    start = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    cloud = np.searchsorted(start[1:], np.arange(N), side="right")
    M = np.zeros(len(lengths), f32)
    for b in range(len(lengths)):
        if start[b + 1] > start[b]:
            M[b] = x[start[b]:start[b + 1]].max()
    if bug == "prev_cloud_max_first_row":
        cloud = cloud[np.maximum(np.arange(N) - 1, 0)]            # the lookup shifted by one row
    inv = f32(1) / (M[cloud] + f32(1e-6))
    if bug == "row_max":
        inv = f32(1) / (x.max(axis=1) + f32(1e-6))
    inv = inv[:, None]
    if bug == "skip_last_column":
        nbr = nbr[:, :-1]
    xs = np.concatenate([x, np.zeros((1, D), f32)], 0)
    votes = np.concatenate([x.sum(axis=1) != 0, [False]])
    cnt = np.maximum(votes[nbr].sum(axis=1), 1).astype(f32)[:, None]
    if bug == "mean_over_h":
        cnt = np.full_like(cnt, max(nbr.shape[1], 1))
    f = x * inv
    mean = (xs[nbr] * inv[:, :, None]).sum(axis=1) / cnt
    d = f - mean
    cut = f32(2) if bug == "softplus_cut_2" else f32(20)
    sp = np.where(d > cut, d, np.log1p(np.exp(np.minimum(d, f32(20)))))
    return (sp * (f / (f32(1e-6) + f.max(axis=1, keepdims=True)))).max(axis=1, keepdims=True)


def test_detection_score_oracle_accepts_float32_and_rejects_bugs():
    x, nbr, lengths = score_case(5, SCORE_LENGTHS, 32, 24)
    ref, mag, alt = ok.detection_scores(f64(x), nbr, lengths, magnitude=True)
    assert np.array_equal(ref, ok.detection_scores(f64(x), nbr, lengths))
    rows = np.sort(np.random.default_rng(0).choice(x.shape[0], 500, replace=False))
    r2, m2, a2 = ok.detection_scores(f64(x), nbr, lengths, magnitude=True, rows=rows, chunk=128)
    assert np.array_equal(r2, ref[rows]) and np.array_equal(m2, mag[rows]) and np.array_equal(a2, alt[rows])
    # the case reaches what it is built for: both softplus branches, and marked cancelling rows
    assert (ref > 20).any() and ((ref > 2) & (ref < 20)).any()
    assert not np.array_equal(ref, alt)
    # honest float32 evaluations: the restatement in float32 and the kernel's own arithmetic, 10x inside the bar
    worst = 0.0
    for what, out in (("fp32 restatement", ok.detection_scores(x, nbr, lengths)),
                      ("fp32 kernel emulation", _emulated_scores(x, nbr, lengths))):
        worst = max(worst, assert_close(out, ref, mag, TOL / 10, "detection scores " + what, alt=alt))
    print("detection scores: float32 headroom %.0fx (largest |err|/mag %.3e)" % (TOL / max(worst, 1e-300), worst))
    weakest = None
    for bug in SCORE_BUGS:
        out = _emulated_scores(x, nbr, lengths, bug)
        rejects(out, ref, mag, alt)
        r = float(ratio(out, ref, mag, alt).max()) / TOL
        print("detection scores, emulated bug %-26s largest |err|/mag = %.3g x TOL" % (bug, r))
        weakest = r if weakest is None else min(weakest, r)
    print("detection scores: weakest rejection %.3g x TOL" % weakest)


def test_detection_score_oracle_cloud_bounds():
    """Lengths summing to more than N cut the last cloud at N; rows past the last cloud belong to no cloud, so they do
    not change any real row's score."""
    x, nbr, lengths = score_case(6, [300, 0, 200, 250], 32, 12)
    ref = ok.detection_scores(f64(x), nbr, lengths)
    short = np.array([300, 0, 200, 200], np.int32)             # the last 50 rows belong to no cloud
    big = x.copy()
    big[700:] = 1e6
    nb2 = nbr.copy()
    nb2[(nb2 >= 700) & (nb2 < 750)] = 750                       # real rows do not reach them
    got = ok.detection_scores(f64(big), nb2, short)
    want = ok.detection_scores(f64(x[:700]), np.where(nb2[:700] == 750, 700, nb2[:700]), short)
    assert np.array_equal(got[:700], want)
    cut = ok.detection_scores(f64(x), nbr, np.array([300, 0, 200, 400], np.int32))
    assert np.array_equal(cut, ref)


@pytest.mark.parametrize("case", sorted(SCORE_CASES))
def test_detection_score_emulation_accepted_on_every_gpu_case(case):
    """The honest float32 kernel emulation passes the bar on every case test_detection_scores_match_restatement runs."""
    lengths, D, H = SCORE_CASES[case]
    x, nbr, lengths = score_case(sum(map(ord, case)), lengths, D, H)
    ref, mag, alt = ok.detection_scores(f64(x), nbr, lengths, magnitude=True)
    assert_close(_emulated_scores(x, nbr, lengths), ref, mag, TOL / 10, "fp32 kernel emulation " + case, alt=alt)


# ---- batch assignment: grid subsampling and radius neighbours of many clouds ----------------------------------------

def _differs(a, b):
    return a.shape != b.shape or not np.array_equal(a, b)


def _first_row_to_previous_cloud(L):
    """Lengths as a search that assigns the first row of every cloud to the previous non-empty cloud sees them."""
    L = L.copy()
    prev = None
    for b in range(len(L)):
        if L[b] > 0:
            if prev is not None:
                L[prev] += 1
                L[b] -= 1
            prev = b
    return L


def _empty_cloud_takes_next_row(L):
    """Lengths as a search that gives an empty cloud the first row of the next cloud sees them."""
    L = L.copy()
    for b in range(len(L) - 1):
        if L[b] == 0 and L[b + 1] > 0:
            L[b], L[b + 1] = 1, L[b + 1] - 1
    return L


def _supports_of_the_neighbouring_cloud(q, qb, s, sb, r):
    """Each query searched among the supports of the next cloud (the previous one for the last cloud)."""
    from oracle import native as on
    qs, ss = np.concatenate([[0], np.cumsum(qb)]), np.concatenate([[0], np.cumsum(sb)])
    rows = []
    for b in range(len(qb)):
        o = b + 1 if b + 1 < len(qb) else b - 1
        nb = on.port_batch_neighbors(q[qs[b]:qs[b + 1]], s[ss[o]:ss[o + 1]], [qb[b]], [sb[o]], r, pad_value=-1)
        rows.append(np.where(nb >= 0, nb + ss[o], len(s)))
    width = max(x.shape[1] for x in rows)
    return np.concatenate([np.pad(x, ((0, 0), (0, width - x.shape[1])), constant_values=len(s)) for x in rows], 0)


@pytest.mark.parametrize("case", ["B17", "B33", "B300", "B1024", "B1024_lone"])
def test_many_cloud_batches_catch_batch_assignment_bugs(case):
    """On the batches of tests/test_gpu_many_clouds.py, the oracle's result changes under each emulated way of putting a
    row into the wrong cloud: the first row of every cloud in the previous non-empty cloud, an empty cloud taking the
    next cloud's first row, the supports taken from the query's neighbouring cloud, and rows past the last cloud
    joined to cloud B - 1."""
    from test_gpu_many_clouds import DL, R, batch, oracle_neighbors, oracle_subsampling, search_args, tail_batch
    P, L = batch(case)
    ref_sub = oracle_subsampling(P, L, DL)
    ref_nb = oracle_neighbors(P, L, P, L, R)[0]
    bugs = {"first row in the previous cloud": _first_row_to_previous_cloud(L),
            "empty cloud takes the next row": _empty_cloud_takes_next_row(L)}
    for what, Lb in bugs.items():
        if np.array_equal(Lb, L):
            assert case.endswith("lone"), what          # no cloud to take a row from
            continue
        assert _differs(oracle_subsampling(P, Lb, DL)[0], ref_sub[0]), what
        assert _differs(oracle_neighbors(P, Lb, P, Lb, R)[0], ref_nb), what
    q, qb, s, sb, r = search_args(P, L, "pool")
    assert _differs(_supports_of_the_neighbouring_cloud(q, qb, s, sb, r), oracle_neighbors(q, qb, s, sb, r)[0])
    B = len(L)
    P, L = tail_batch(B, -37)
    Lb = L.copy()
    Lb[-1] += 37                                            # the 37 rows of no cloud joined to cloud B - 1
    assert _differs(oracle_subsampling(P, Lb, DL)[0], oracle_subsampling(P, L, DL)[0])
    assert _differs(oracle_neighbors(P, Lb, P, Lb, R)[0], oracle_neighbors(P, L, P, L, R)[0])
