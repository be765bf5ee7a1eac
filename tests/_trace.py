"""Test infrastructure: record every fused op the GPU encoder and decoder launch (KPConv, unary GEMMs, both pools, the
detection scores; inputs and output, device tensors) so that the numpy restatement can be evaluated on a SAMPLE OF
ROWS of each op at sizes where the full float64 restatement is too slow (BASELINE configs[1]/[2]/[3] at their real sizes). Each op is independent per output row, so checking
sampled rows against the oracle on the op's real inputs is an oracle comparison, not a path-vs-path one.
"""
import contextlib

import numpy as np

from oracle import kpconv_np as _ok

import _oracle as _o


class Trace:
    def __init__(self):
        self.records = []


@contextlib.contextmanager
def record_ops():
    from d3feat_b200 import convolution_ops as co
    from d3feat_b200 import network_blocks as nb
    tr = Trace()
    orig = dict(kp=co.KPConv_ops, kd=co.KPConv_deform_ops, un=co.unary_convolution, up=co.unary_pair_convolution,
                mp=nb.ind_max_pool, cp=nb.closest_pool, ds=nb.detection_scores)

    def kp(q, s, idx, f, Kp, W, extent, infl, mode, *, epilogue=None, bias=None, query_order=None, **rows):
        out = orig["kp"](q, s, idx, f, Kp, W, extent, infl, mode, epilogue=epilogue, bias=bias, query_order=query_order,
                         **rows)
        tr.records.append(dict(op="kpconv", q=q, s=s, idx=idx, f=f, Kp=Kp, W=W, extent=extent, infl=infl, mode=mode,
                               epilogue=epilogue, bias=bias, out=out, rows_q=rows.get("rows_q"),
                               rows_s=rows.get("rows_s")))
        return out

    def kd(q, s, idx, f, Kp, off, mod, W, extent, infl, mode, *, epilogue=None, query_order=None, **rows):
        out = orig["kd"](q, s, idx, f, Kp, off, mod, W, extent, infl, mode, epilogue=epilogue, query_order=query_order,
                         **rows)
        tr.records.append(dict(op="kpconv_deform", q=q, s=s, idx=idx, f=f, Kp=Kp, off=off, mod=mod, W=W, extent=extent,
                               infl=infl, mode=mode, epilogue=epilogue, out=out, rows_q=rows.get("rows_q"),
                               rows_s=rows.get("rows_s")))
        return out

    def un(x, w, *, epilogue=None, residual=None, rows=None):
        out = orig["un"](x, w, epilogue=epilogue, residual=residual, rows=rows)
        tr.records.append(dict(op="unary", x=x, w=w, epilogue=epilogue, residual=residual, out=out, rows_q=rows))
        return out

    def up(x1, w1, a1, x2, w2, a2, alpha, *, rows=None):
        out = orig["up"](x1, w1, a1, x2, w2, a2, alpha, rows=rows)
        tr.records.append(dict(op="unary_pair", x1=x1, w1=w1, a1=a1, x2=x2, w2=w2, a2=a2, alpha=alpha, out=out,
                               rows_q=rows))
        return out

    def mp(x, inds, **rows):
        out = orig["mp"](x, inds, **rows)
        tr.records.append(dict(op="max_pool", x=x, inds=inds, out=out, rows_q=rows.get("rows_out"),
                               rows_s=rows.get("rows_x")))
        return out

    def cp(x, inds, **rows):
        out = orig["cp"](x, inds, **rows)
        tr.records.append(dict(op="closest_pool", x=x, inds=inds, out=out, rows_q=rows.get("rows_out"),
                               rows_s=rows.get("rows_x")))
        return out

    def ds(features, neighbors, lengths, *, rows=None):
        out = orig["ds"](features, neighbors, lengths, rows=rows)
        tr.records.append(dict(op="detection_scores", features=features, neighbors=neighbors, lengths=lengths, out=out,
                               rows_q=rows))
        return out

    co.KPConv_ops, co.KPConv_deform_ops, co.unary_convolution, co.unary_pair_convolution = kp, kd, un, up
    nb.ind_max_pool, nb.closest_pool, nb.detection_scores = mp, cp, ds
    try:
        yield tr
    finally:
        co.KPConv_ops, co.KPConv_deform_ops, co.unary_convolution, co.unary_pair_convolution = (
            orig["kp"], orig["kd"], orig["un"], orig["up"])
        nb.ind_max_pool, nb.closest_pool, nb.detection_scores = orig["mp"], orig["cp"], orig["ds"]


def _np(t):
    return None if t is None else t.detach().cpu().numpy()


def _count(rows, default):
    """Actual row count of a capacity-sized tensor (device scalar), or its full length."""
    return default if rows is None else max(int(rows.reshape(-1)[0].item()), 0)


def _epi(y, mag, epilogue, residual=None):
    scale = shift = alpha = None
    if epilogue is not None:
        scale, shift, alpha = epilogue
    return _o.epilogue(y, mag, _np(scale), _np(shift), residual=residual, alpha=alpha)


def check_sampled_rows(trace, n_rows, rng, rtol, min_kpconv=None, tol=_o.TOL, what=""):
    """For every recorded op: float64 restatement on `n_rows` sampled output rows (all rows when the op has fewer) vs
    the GPU output rows, on the op's real inputs. Two checks per op:
      * max-norm relative PER TENSOR (< rtol): the denominator is the max |value| of the op's GPU output rows, the
        numerator the max error over the sample (what test_gpu_kpconv.py normalises by);
      * element by element, |out - ref| <= tol * mag (tests/_oracle.py).
    Capacity-sized launches (the static pyramid) pass their device row counts (rows / rows_q / rows_s): only rows
    below the count are sampled, and supports and features are cut to their count, so that the shadow index is the
    count as it is on the device. Returns a list of (op, shape, err, element ratio) for the report."""
    report = []
    n_kp = 0
    for k, r in enumerate(trace.records):
        out = _np(r["out"])
        N = _count(r.get("rows_q"), out.shape[0])
        out = out[:N]
        if N == 0:
            report.append((r["op"], out.shape, 0.0, 0.0))
            continue
        rows = np.arange(N) if N <= n_rows else np.sort(rng.choice(N, n_rows, replace=False))
        denom = max(float(np.abs(out).max()), 1e-30)
        alt = None
        if r["op"] in ("kpconv", "kpconv_deform"):
            Ns = _count(r.get("rows_s"), r["s"].shape[0])
            q, s, idx, f = _np(r["q"])[rows], _np(r["s"])[:Ns], _np(r["idx"])[rows], _np(r["f"])[:Ns]
            assert idx.min(initial=0) >= 0 and idx.max(initial=0) <= Ns, "%s: index past the support count" % r["op"]
            if r["op"] == "kpconv":
                ref, mag, alt = _ok.kpconv_ops(q, s, idx, f, _np(r["Kp"]), _np(r["W"]), r["extent"], r["infl"],
                                               r["mode"], dtype=np.float64, magnitude=True)
                if r["bias"] is not None:      # the offset head of the deformable block: bias, no batch norm (:327-339)
                    assert r["epilogue"] is None
                    b = _np(r["bias"]).astype(np.float64)
                    ref, alt, mag = ref + b, alt + b, mag + np.abs(b)
            else:
                ref, mag, alt = _ok.kpconv_deform_ops(q, s, idx, f, _np(r["Kp"]), _np(r["off"])[rows],
                                                      None if r["mod"] is None else _np(r["mod"])[rows], _np(r["W"]),
                                                      r["extent"], r["infl"], r["mode"], dtype=np.float64,
                                                      magnitude=True)
            alt, _ = _epi(alt, mag, r["epilogue"])
            ref, mag = _epi(ref, mag, r["epilogue"])
            n_kp += 1
        elif r["op"] == "unary":
            x, w = _np(r["x"])[rows], _np(r["w"])
            res = None if r["residual"] is None else _np(r["residual"])[rows].astype(np.float64)
            ref, mag = _epi(x.astype(np.float64) @ w.astype(np.float64), _o.gemm_mag(x, w), r["epilogue"], res)
        elif r["op"] == "unary_pair":
            (s1, t1), (s2, t2) = r["a1"], r["a2"]
            x1, w1, x2, w2 = _np(r["x1"])[rows], _np(r["w1"]), _np(r["x2"])[rows], _np(r["w2"])
            y1, m1 = _o.epilogue(x1.astype(np.float64) @ w1, _o.gemm_mag(x1, w1), _np(s1), _np(t1))
            y2, m2 = _o.epilogue(x2.astype(np.float64) @ w2, _o.gemm_mag(x2, w2), _np(s2), _np(t2))
            ref, mag = _o.epilogue(y1 + y2, m1 + m2, alpha=r["alpha"])
        elif r["op"] == "max_pool":
            x = _np(r["x"])[:_count(r.get("rows_s"), r["x"].shape[0])]
            ref = _ok.ind_max_pool(x, _np(r["inds"])[rows])
            assert np.array_equal(out[rows], ref), "ind_max_pool rows differ (exact op)"
            report.append((r["op"], out.shape, 0.0, 0.0))
            continue
        elif r["op"] == "closest_pool":
            x = _np(r["x"])[:_count(r.get("rows_s"), r["x"].shape[0])]
            ref = _ok.closest_pool(x, _np(r["inds"])[rows])
            assert np.array_equal(out[rows], ref), "closest_pool rows differ (exact op)"
            report.append((r["op"], out.shape, 0.0, 0.0))
            continue
        elif r["op"] == "detection_scores":
            # features and neighbours cut to the device count: the shadow index is the count, as on the device
            x, nbr = _np(r["features"])[:N].astype(np.float64), _np(r["neighbors"])[:N]
            assert nbr.min(initial=0) >= 0 and nbr.max(initial=0) <= N, "detection_scores: index past the row count"
            ref, mag, alt = _ok.detection_scores(x, nbr, _np(r["lengths"]), magnitude=True, rows=rows)
        else:
            raise AssertionError(r["op"])
        err = float(np.abs(out[rows].astype(np.float64) - ref).max()) / denom
        assert err < rtol, "%s %s: sampled-row error %.3g" % (r["op"], out.shape, err)
        ratio = _o.assert_close(out[rows], ref, mag, tol, "%s#%d %s %s" % (what, k, r["op"], out.shape), alt=alt)
        report.append((r["op"], out.shape, err, ratio))
    if min_kpconv is not None:
        assert n_kp >= min_kpconv, "only %d KPConv launches recorded" % n_kp
    return report
