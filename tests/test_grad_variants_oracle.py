"""CPU: the element-wise check of tests/test_gpu_grad_variants.py has teeth. At the table's shapes and index edges,
numpy float32 emulations of the feature and weight gradients, computed the way the kernels compute them (the feature
gradient as a forward KPConv over the transposed neighbourhood, the weight gradient in 2048-row blocks summed in
float64), pass assert_close at TOL against the float64 restatement (tests/_kpconv_grad_oracle.py), and each of these
plausible mistakes is rejected:
  * +Kp instead of -Kp in the transposed problem;
  * W instead of W^T on a square layer;
  * df divided by the support's own neighbour count instead of by nn of each query that reaches it;
  * a support named twice in one row counted once in the reverse table;
  * the reverse table one column short, which drops the hub's last query;
  * dW without its last 2048-row block (KPConv and unary), or without its last query chunk.
No GPU needed.
"""
import numpy as np
import pytest

import _kpconv_grad_oracle as og
from _oracle import TOL, assert_close, ratio
from test_gpu_grad_variants import CASES, FAMILIES, case_inputs, edge_case
from test_gpu_kpconv_grad import make_case

f32 = np.float32


def weights(rel, Kp, ext, infl, mode):
    """Correlation weights [..., K] of neighbours at rel [..., 3] (float32), closest mode applied."""
    d2 = np.sum(np.square(rel[..., None, :] - Kp), axis=-1)
    if infl == "constant":
        w = np.ones_like(d2)
    elif infl == "linear":
        w = np.maximum(f32(1) - np.sqrt(d2 + f32(1e-10)) / (f32(2) * ext), f32(0))
    else:
        sigma = ext * f32(0.3)
        w = np.exp(-d2 / (f32(2) * np.square(sigma) + f32(1e-9)))
    if mode == "closest":
        w = w * (np.arange(Kp.shape[0]) == np.argmin(d2, axis=-1)[..., None])
    return w.astype(f32)


def neighbour_counts(f, ii):
    """nn of every query: its neighbours whose feature row sums to > 0 (the shadow row is 0), at least 1."""
    fx = np.concatenate([f, np.zeros((1, f.shape[1]), f32)])
    return np.maximum(np.sum(fx[ii].sum(-1) > 0, axis=-1), 1).astype(f32)


def reverse_table(ii, Nq, Ns, once=False, cut=0):
    """rev[s, j] = the j-th query reaching s, ascending (q, h), padded with Nq (the transposed problem's shadow)."""
    keys = ii.ravel()
    vals = np.repeat(np.arange(Nq), ii.shape[1])
    keys, vals = keys[keys < Ns], vals[keys < Ns]
    if once:                                          # bug: a support named twice in one row counted once
        u = np.unique(keys.astype(np.int64) * Nq + vals)
        keys, vals = u // Nq, u % Nq
    order = np.argsort(keys, kind="stable")
    keys, vals = keys[order], vals[order]
    counts = np.bincount(keys, minlength=Ns)
    pos = np.arange(len(keys)) - (np.cumsum(counts) - counts)[keys]
    Hr = max(int(counts.max(initial=0)) - cut, 0)    # bug: cut > 0 drops the last column(s)
    rev = np.full((Ns, max(Hr, 1)), Nq, np.int64)
    keep = pos < Hr
    rev[keys[keep], pos[keep]] = vals[keep]
    return rev


def emulate_df(q, s, idx, f, Kp, W, ext, infl, mode, dout, kp_sign=-1, transpose=True, nn="query", once=False,
               cut=0):
    """dL/df in float32 as the kernels compute it: G = dout / nn, then a forward KPConv over the transposed
    neighbourhood (queries at 1e6 as its shadow, kernel points kp_sign * Kp, weights W^T, no normalisation)."""
    q, s, f, Kp, W, dout = (np.asarray(a, f32) for a in (q, s, f, Kp, W, dout))
    Nq, Ns = len(q), len(s)
    ii = np.where((idx < 0) | (idx > Ns), Ns, idx)
    nnq = neighbour_counts(f, ii)
    G = dout / nnq[:, None] if nn == "query" else dout
    rev = reverse_table(ii, Nq, Ns, once, cut)
    qx = np.concatenate([q, np.full((1, 3), 1e6, f32)])
    Gx = np.concatenate([G, np.zeros((1, G.shape[1]), f32)])
    WT = np.transpose(W, (0, 2, 1)) if transpose else W
    df = np.zeros((Ns, W.shape[1]), f32)
    for a in range(0, Ns, 128):
        r = rev[a:a + 128]
        w = weights(qx[r] - s[a:a + 128, None, :], f32(kp_sign) * Kp, f32(ext), infl, mode)   # [n, Hr, K]
        wf = np.einsum("nhk,nho->nko", w, Gx[r])
        df[a:a + 128] = np.einsum("nko,koc->nc", wf, WT)
    if nn == "support":                               # bug: the support's own row count instead of nn of its queries
        df /= np.concatenate([nnq, np.ones(max(Ns - Nq, 0), f32)])[:Ns, None]
    return df


def block_sum(A, B, rows, block=2048):
    """sum over the first `rows` rows of A^T B: float32 partials per 2048-row block, summed in float64."""
    out = np.zeros((A.shape[1], B.shape[1]))
    for a in range(0, rows, block):
        b = min(rows, a + block)
        out += A[a:b].T @ B[a:b]
    return out.astype(f32)


def emulate_dW(q, s, idx, f, Kp, W, ext, infl, mode, dout, rows=None):
    """dL/dW in float32: wf recomputed per query, then wf^T G in 2048-row blocks over the first `rows` queries."""
    q, s, f, Kp, W, dout = (np.asarray(a, f32) for a in (q, s, f, Kp, W, dout))
    Nq, Ns = len(q), len(s)
    ii = np.where((idx < 0) | (idx > Ns), Ns, idx)
    G = dout / neighbour_counts(f, ii)[:, None]
    sx = np.concatenate([s, np.full((1, 3), 1e6, f32)])
    fx = np.concatenate([f, np.zeros((1, f.shape[1]), f32)])
    w = weights(sx[ii] - q[:, None, :], Kp, f32(ext), infl, mode)       # [Nq, H, K]
    wf = np.einsum("nhk,nhc->nkc", w, fx[ii]).reshape(Nq, -1)
    return block_sum(wf, G, Nq if rows is None else rows).reshape(W.shape)


def table(id):
    c = next(c for c in CASES if c["id"] == id)
    return case_inputs(c) + (c["extent"], c["infl"], c["mode"])


def edge(fam, name):
    q, s, idx, f, Kp, W, dout, ext, _ = edge_case(fam, name)
    return q, s, idx, f, Kp, W, dout, ext, FAMILIES[fam].get("infl", "linear"), "sum"


def chunked():
    """The 128-query chunk shape of the multi-chunk test: 3 chunks and a ragged fourth."""
    n = 3 * 128 + 64 - 3
    ext = round(0.9 * n ** (-1 / 3), 4)
    return make_case(np.random.default_rng(133), n, n, 36, 32, 32, extent=ext, unreached=3) + (ext, "linear", "sum")


SOURCES = {
    "fast4_32x32": lambda: table("fast4_32x32"),
    "mma4_32x32_closest": lambda: table("mma4_32x32_closest"),
    "mma8_64x64_constant": lambda: table("mma8_64x64_constant"),
    "generic_48x40": lambda: table("generic_48x40"),
    "anyk_k7_1x20": lambda: table("anyk_k7_1x20"),
    "cin1_64x1_gaussian_closest": lambda: table("cin1_64x1_gaussian_closest"),
    "fused32_4000": lambda: table("fused32_4000"),
    "edge_fast_duplicates": lambda: edge("fast", "duplicates"),
    "edge_mma_padding": lambda: edge("mma", "padding"),
    "edge_fast_hub": lambda: edge("fast", "hub"),
    "edge_cin1_hub": lambda: edge("cin1", "hub"),
    "chunk128": chunked,
}
_memo = {}


def source(name):
    if name not in _memo:
        _memo[name] = SOURCES[name]()
    return _memo[name]


def refs(name):
    """float64 (ref, mag, alt) of dL/df and of dL/dW."""
    if ("ref", name) not in _memo:
        q, s, idx, f, Kp, W, dout, ext, infl, mode = source(name)
        a = (q, s, idx, f, Kp, W, ext, infl, mode, dout)
        _memo["ref", name] = og.kpconv_features_grad(*a), og.kpconv_weights_grad(*a)
    return _memo["ref", name]


@pytest.mark.parametrize("name", sorted(SOURCES))
def test_float32_emulation_is_accepted(name):
    q, s, idx, f, Kp, W, dout, ext, infl, mode = source(name)
    (dref, dmag, dalt), (wref, wmag, walt) = refs(name)
    assert_close(emulate_df(q, s, idx, f, Kp, W, ext, infl, mode, dout), dref, dmag, TOL, "fp32 df " + name,
                 alt=dalt)
    assert_close(emulate_dW(q, s, idx, f, Kp, W, ext, infl, mode, dout), wref, wmag, TOL, "fp32 dW " + name,
                 alt=walt)


DF_BUGS = {
    "plus_kp": dict(kp_sign=1),
    "w_not_transposed": dict(transpose=False),
    "nn_of_support": dict(nn="support"),
    "duplicate_counted_once": dict(once=True),
    "reverse_table_one_column_short": dict(cut=1),
}
DF_BUG_CASES = [("plus_kp", "fast4_32x32"), ("plus_kp", "mma4_32x32_closest"), ("plus_kp", "anyk_k7_1x20"),
                ("plus_kp", "cin1_64x1_gaussian_closest"),
                ("w_not_transposed", "fast4_32x32"), ("w_not_transposed", "mma8_64x64_constant"),
                ("w_not_transposed", "edge_mma_padding"),
                ("nn_of_support", "fast4_32x32"), ("nn_of_support", "generic_48x40"),
                ("duplicate_counted_once", "fast4_32x32"), ("duplicate_counted_once", "edge_fast_duplicates"),
                ("reverse_table_one_column_short", "edge_fast_hub"),
                ("reverse_table_one_column_short", "edge_cin1_hub")]


def rejected(out, ref, mag, alt, what):
    worst = float(ratio(out, ref, mag, alt).max())
    print("REJECTED %-60s worst ratio %.3e" % (what, worst))
    with pytest.raises(AssertionError):
        assert_close(out, ref, mag, TOL, what, alt=alt)


@pytest.mark.parametrize("bug,name", DF_BUG_CASES)
def test_feature_gradient_bug_is_rejected(bug, name):
    q, s, idx, f, Kp, W, dout, ext, infl, mode = source(name)
    if bug == "w_not_transposed":
        assert W.shape[1] == W.shape[2]
    if bug == "reverse_table_one_column_short":   # the hub is named by every query: its last query is the one cut
        ii = np.where((idx < 0) | (idx > len(s)), len(s), idx)
        assert np.bincount(ii[ii < len(s)]).argmax() == 0 and (ii == 0).any(1).all()
    (ref, mag, alt), _ = refs(name)
    rejected(emulate_df(q, s, idx, f, Kp, W, ext, infl, mode, dout, **DF_BUGS[bug]), ref, mag, alt,
             "df %s %s" % (bug, name))


@pytest.mark.parametrize("bug,name", [("last_2048_row_block", "fused32_4000"), ("last_chunk", "chunk128")])
def test_weight_gradient_bug_is_rejected(bug, name):
    q, s, idx, f, Kp, W, dout, ext, infl, mode = source(name)
    n = len(q)
    rows = (n - 1) // 2048 * 2048 if bug == "last_2048_row_block" else (n - 1) // 128 * 128
    assert 0 < rows < n
    _, (ref, mag, alt) = refs(name)
    rejected(emulate_dW(q, s, idx, f, Kp, W, ext, infl, mode, dout, rows=rows), ref, mag, alt,
             "dW %s %s" % (bug, name))


@pytest.mark.parametrize("N", [2049, 4097])
@pytest.mark.parametrize("Cout", [32, 64])
def test_unary_weight_gradient_without_its_last_block_is_rejected(N, Cout):
    rng = np.random.default_rng(N + Cout)
    x, g = rng.normal(size=(N, 48)).astype(f32), rng.normal(size=(N, Cout)).astype(f32)
    ref, mag, alt = og.unary_weights_grad(x, None, g)
    assert_close(block_sum(x, g, N), ref, mag, TOL, "fp32 unary dW N=%d" % N, alt=alt)
    rejected(block_sum(x, g, (N - 1) // 2048 * 2048), ref, mag, alt, "unary dW last block N=%d Cout=%d" % (N, Cout))
