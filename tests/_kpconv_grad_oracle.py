"""Float64 restatement of the gradients of rigid KPConv and of the unary convolution, for the tests.

What tf.gradients gives the reference's training scripts (training_3DMatch.py, utils/trainer.py) for
kernels/convolution_ops.py:161-255 (KPConv_ops) and :90-99 (unary_convolution), with the neighbour count nn held
constant as in the TF graph (it comes from tf.greater and a cast, which have no gradient). It reuses the forward
restatement's decisions (oracle/kpconv_np.py: influences, modes, the closest-tie and nn-vote margins), so every
ambiguous decision is marked exactly where the forward's oracle marks it. Each function returns (ref, mag, alt) as
kpconv_ops(magnitude=True) does.
"""
import numpy as np

from oracle.kpconv_np import CLOSEST_TIE_RTOL, INFLUENCES, MODES, NN_SUM_ULPS, _chunks


def _kpconv_grad_terms(q, s, f, Kp, ii, qa, ext, KP_influence, aggregation_mode, dt):
    """Per query chunk: the correlation weights w [n,K,H] (closest mode applied), the gathered rows nf [n,H,Cin], nn,
    and the same with every ambiguous decision taken the other way (w2, nn2), exactly as kpconv_ops decides them."""
    n_kp = Kp.shape[0]
    nb = s[ii] - qa[:, None, :]
    diff = nb[:, :, None, :] - Kp[None, None, :, :]
    d2 = np.sum(np.square(diff), axis=3)
    if KP_influence == "constant":
        w = np.ones_like(d2)
    elif KP_influence == "linear":
        w = np.maximum(1 - np.sqrt(d2 + dt(1e-10)) / (2 * ext), dt(0.0))
    else:
        sigma = ext * dt(0.3)
        w = np.exp(-d2 / (2 * np.square(sigma) + dt(1e-9)))
    w_all = np.transpose(w, (0, 2, 1))
    w = w_all
    w2 = w_all
    if aggregation_mode == "closest":
        nn1 = np.argmin(d2, axis=2)
        w = w_all * (np.arange(n_kp)[None, :, None] == nn1[:, None, :]).astype(dt)
        w2 = w
        if n_kp > 1:
            srt = np.sort(d2, axis=2)
            tie = srt[:, :, 1] - srt[:, :, 0] <= CLOSEST_TIE_RTOL * srt[:, :, 1]
            nn2 = np.where(tie, np.argsort(d2, axis=2, kind="stable")[:, :, 1], nn1)
            w2 = w_all * (np.arange(n_kp)[None, :, None] == nn2[:, None, :]).astype(dt)
    nf = f[ii]
    nsum = np.sum(nf, axis=-1)
    nnum = np.maximum(np.sum((nsum > 0).astype(dt), axis=-1), 1)
    amb = (nsum != 0) & (np.abs(nsum) < NN_SUM_ULPS * np.sum(np.abs(nf), axis=-1))
    nnum2 = np.maximum(np.sum(((nsum > 0) ^ amb).astype(dt), axis=-1), 1)
    return w, w2, nf, nnum, nnum2


def _kpconv_grad_setup(query_points, support_points, neighbors_indices, features, K_points, K_values,
                       KP_influence, aggregation_mode, grad_out, dt):
    if KP_influence not in INFLUENCES:
        raise ValueError("Unknown influence function type (config.KP_influence)")
    if aggregation_mode not in MODES:
        raise ValueError("Unknown convolution mode. Should be 'closest' or 'sum'")
    q = np.asarray(query_points, dt)
    Ns = np.asarray(support_points).shape[0]
    s = np.concatenate([np.asarray(support_points, dt), np.full((1, 3), 1e6, dt)], 0)
    f = np.concatenate([np.asarray(features, dt), np.zeros((1, features.shape[1]), dt)], 0)
    idx = np.asarray(neighbors_indices).astype(np.int64)
    idx = np.where((idx < 0) | (idx > Ns), Ns, idx)                    # -1 padding and the shadow: row Ns
    return q, s, f, np.asarray(K_points, dt), np.asarray(K_values, dt), idx, np.asarray(grad_out, dt), Ns


def kpconv_weights_grad(query_points, support_points, neighbors_indices, features, K_points, K_values, KP_extent,
                        KP_influence, aggregation_mode, grad_out, dtype=np.float64, chunk=2048):
    """dL/dK_values [K,Cin,Cout] of kpconv_ops for dL/dout = grad_out, nn held constant:
        dW[k,c,o] = sum_q wf[q,k,c] grad_out[q,o] / nn_q,      wf[q,k,c] = sum_h w(q,h,k) f[idx[q,h],c]
    Returns (ref, mag, alt) as kpconv_ops(magnitude=True): mag = the same sum over |f| and |grad_out|, alt = every
    ambiguous decision (closest tie, nn vote) taken the other way."""
    dt = dtype
    q, s, f, Kp, W, idx, G0, _ = _kpconv_grad_setup(query_points, support_points, neighbors_indices, features,
                                                    K_points, K_values, KP_influence, aggregation_mode, grad_out, dt)
    ref, alt, mag1, mag2 = (np.zeros(W.shape, dt) for _ in range(4))
    for a, b in _chunks(q.shape[0], chunk):
        w, w2, nf, nnum, nnum2 = _kpconv_grad_terms(q, s, f, Kp, idx[a:b], q[a:b], dt(KP_extent), KP_influence,
                                                    aggregation_mode, dt)
        G, G2 = G0[a:b] / nnum[:, None], G0[a:b] / nnum2[:, None]
        ref += np.einsum("nkc,no->kco", np.matmul(w, nf), G)
        alt += np.einsum("nkc,no->kco", np.matmul(w2, nf), G2)
        mag1 += np.einsum("nkc,no->kco", np.matmul(w, np.abs(nf)), np.abs(G))
        mag2 += np.einsum("nkc,no->kco", np.matmul(w2, np.abs(nf)), np.abs(G2))
    return ref, np.maximum(mag1, mag2), alt


def kpconv_features_grad(query_points, support_points, neighbors_indices, features, K_points, K_values, KP_extent,
                         KP_influence, aggregation_mode, grad_out, dtype=np.float64, chunk=2048):
    """dL/dfeatures [Ns,Cin] of kpconv_ops for dL/dout = grad_out, nn held constant:
        df[s,c] = sum_{(q,h): idx[q,h] = s} sum_k w(q,h,k) sum_o grad_out[q,o] W[k,c,o] / nn_q
    Shadow entries contribute nothing. Returns (ref, mag, alt) as kpconv_weights_grad."""
    dt = dtype
    q, s, f, Kp, W, idx, G0, Ns = _kpconv_grad_setup(query_points, support_points, neighbors_indices, features,
                                                     K_points, K_values, KP_influence, aggregation_mode, grad_out, dt)
    Cin = W.shape[1]
    ref, alt, mag1, mag2 = (np.zeros((Ns + 1, Cin), dt) for _ in range(4))
    aW = np.abs(W)
    for a, b in _chunks(q.shape[0], chunk):
        ii = idx[a:b]
        w, w2, _, nnum, nnum2 = _kpconv_grad_terms(q, s, f, Kp, ii, q[a:b], dt(KP_extent), KP_influence,
                                                   aggregation_mode, dt)
        G, G2 = G0[a:b] / nnum[:, None], G0[a:b] / nnum2[:, None]
        np.add.at(ref, ii, np.einsum("nkh,nkc->nhc", w, np.einsum("no,kco->nkc", G, W)))
        np.add.at(alt, ii, np.einsum("nkh,nkc->nhc", w2, np.einsum("no,kco->nkc", G2, W)))
        np.add.at(mag1, ii, np.einsum("nkh,nkc->nhc", w, np.einsum("no,kco->nkc", np.abs(G), aW)))
        np.add.at(mag2, ii, np.einsum("nkh,nkc->nhc", w2, np.einsum("no,kco->nkc", np.abs(G2), aW)))
    return ref[:Ns], np.maximum(mag1, mag2)[:Ns], alt[:Ns]


def unary_features_grad(features, K_values, grad_out, dtype=np.float64):
    """dL/dfeatures = grad_out @ K_values^T of unary_convolution, as (ref, mag, alt) (no ambiguous decision)."""
    g, w = np.asarray(grad_out, dtype), np.asarray(K_values, dtype)
    ref = g @ w.T
    return ref, np.abs(g) @ np.abs(w).T, ref


def unary_weights_grad(features, K_values, grad_out, dtype=np.float64):
    """dL/dK_values = features^T @ grad_out of unary_convolution, as (ref, mag, alt)."""
    x, g = np.asarray(features, dtype), np.asarray(grad_out, dtype)
    ref = x.T @ g
    return ref, np.abs(x).T @ np.abs(g), ref
