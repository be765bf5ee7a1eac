"""Element-wise tolerance against the float64 restatement.

The max-norm check of the older tests, max|out - ref| / max|ref|, lets a wrong row, tile or chunk hide under the
largest element of the tensor. assert_close checks every element against the rounding-error scale OF THAT ELEMENT:

    |out - ref| <= tol * mag

where `mag` is the same float64 computation evaluated on absolute values (|A| @ |W| for a GEMM; for KPConv the
oracle's magnitude=True mode). Any fp32 summation order of a sum of n products is off by at most ~n * 2^-24 * mag, and
in practice by ~sqrt(n) * 2^-24 * mag, so tol does not depend on the data's scale or sign pattern.

TOL: the kernels are 3xTF32 / fp32 FFMA, whose float32 restatement stays far below 1e-5 * mag
(tests/test_oracle_sensitivity.py) while every emulated kernel bug there is caught. The largest ratio each test sees is
recorded in RATIOS and printed, so the headroom on an H100 can be read off any run.
"""
import numpy as np

TOL = 1e-5

RATIOS = {}          # what -> largest |out - ref| / mag seen


def f64(a):
    return np.asarray(a, np.float64)


def gemm_mag(x, w):
    """|x| @ |w| in float64: the rounding-error scale of x @ w."""
    return np.abs(f64(x)) @ np.abs(f64(w))


def epilogue(y, mag, scale=None, shift=None, bias=None, residual=None, alpha=None):
    """The block epilogue (y*scale + shift, + bias, + residual, LeakyReLU) on a float64 result and its magnitude.
    LeakyReLU is 1-Lipschitz, so it adds nothing to the magnitude."""
    y, mag = f64(y), f64(mag)
    if scale is not None:
        y = y * f64(scale) + f64(shift)
        mag = mag * np.abs(f64(scale)) + np.abs(f64(shift))
    if bias is not None:
        y = y + f64(bias)
        mag = mag + np.abs(f64(bias))
    if residual is not None:
        y = y + f64(residual)
        mag = mag + np.abs(f64(residual))
    if alpha is not None:
        y = np.where(y > 0, y, alpha * y)
    return y, mag


def ratio(out, ref, mag, alt=None):
    """Per-element |out - ref| / mag (the smaller of the two branches where `alt` is given)."""
    out, ref, mag = f64(out), f64(ref), f64(mag)
    err = np.abs(out - ref)
    if alt is not None:
        err = np.minimum(err, np.abs(out - f64(alt)))
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(err == 0, 0.0, err / np.maximum(mag, 1e-300))
    return np.where(np.isnan(r), np.inf, r)


def assert_close(out, ref, mag, tol=TOL, what="", alt=None):
    """Every element: |out - ref| <= tol * mag (or |out - alt| <= tol * mag where the oracle marked an ambiguous
    decision). On failure: the worst element's (row, column), its ratio, and the old max-norm figure."""
    out = f64(out)
    ref = f64(ref)
    assert out.shape == ref.shape, "%s: shape %s vs %s" % (what, out.shape, ref.shape)
    if out.size == 0:
        return 0.0
    r = ratio(out, ref, mag, alt)
    worst = float(r.max())
    RATIOS[what] = max(RATIOS.get(what, 0.0), worst)
    print("RATIO %-60s %.3e" % (what, worst))
    if not worst <= tol:
        i = np.unravel_index(int(np.argmax(r)), r.shape)
        maxnorm = np.abs(out - ref).max() / max(np.abs(ref).max(), 1e-30)
        raise AssertionError("%s: element %s: out %.9g ref %.9g mag %.3g -> |err|/mag %.3g > %.1g "
                             "(max-norm relative error of the tensor: %.3g; %d elements over)" % (
                                 what, tuple(int(x) for x in i), out[i], ref[i], f64(mag)[i], worst, tol, maxnorm,
                                 int((r > tol).sum())))
    return worst


def kpconv_ref(q, s, idx, f, Kp, W, extent, influence="linear", mode="sum", offsets=None, modulations=None,
               deform=False, epi=None, bias=None):
    """float64 (ref, mag, alt) of a rigid (or, deform=True, deformable) KPConv with an optional BN + LeakyReLU
    epilogue `epi` = (scale, shift, alpha) as numpy arrays / float, and an optional bias."""
    from oracle import kpconv_np as ok
    if deform:
        ref, mag, alt = ok.kpconv_deform_ops(q, s, idx, f, Kp, offsets, modulations, W, extent, influence, mode,
                                             magnitude=True)
    else:
        ref, mag, alt = ok.kpconv_ops(q, s, idx, f, Kp, W, extent, influence, mode, magnitude=True)
    scale, shift, alpha = epi if epi is not None else (None, None, None)
    y, m = epilogue(ref, mag, scale, shift, bias=bias, alpha=alpha)
    ya, _ = epilogue(alt, mag, scale, shift, bias=bias, alpha=alpha)
    return y, m, ya


def tf32(a):
    """Round float32 values to TF32 (10 explicit mantissa bits, round to nearest) -- what a tensor core reads."""
    b = np.ascontiguousarray(a, np.float32).view(np.uint32)
    return ((b + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)
