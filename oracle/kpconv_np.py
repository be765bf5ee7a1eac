"""TEST INFRASTRUCTURE ONLY -- numpy restatement of the TF1 graph half of the D3Feat hot path.

Each function follows the reference line ranges quoted in its docstring (paths relative to
/root/reference). TensorFlow 1.12 is not installable here, so this is a *restatement*, not the
reference itself: "parity unpinned" for these functions (no reference test or golden vector pins the
TF kernels' summation order). The contract is therefore mathematical: the CUDA path must agree with
the fp64 evaluation of this restatement to 1e-4 (see tests/), and the fp32 evaluation is used to show
how much of that budget fp32 summation-order noise consumes on its own.

Only tests/, __graft_entry__.smoke() and bench.py's CPU-baseline legs may import this module.
"""
import numpy as np

INFLUENCES = ("constant", "linear", "gaussian")
MODES = ("sum", "closest")


def _chunks(n, rows_per_chunk):
    for a in range(0, n, rows_per_chunk):
        yield a, min(n, a + rows_per_chunk)


def unary_convolution(features, K_values):
    """kernels/convolution_ops.py:90-99 -- tf.matmul(features, K_values)."""
    return features @ K_values


# Discontinuities of the graph that fp32 and fp64 may legitimately resolve differently (magnitude=True marks them):
CLOSEST_TIE_RTOL = 1e-5            # closest mode: the two nearest kernel points' d2 differ by less than this, relative
NN_SUM_ULPS = 64 * 2.0 ** -24      # nn predicate: |row sum| < this * sum |row| (a float64 sum of exactly 0 is exact)
IN_RANGE_RTOL = 1e-5               # deformable in-range / constant weight: |d2 - extent^2| < this * extent^2



def kpconv_ops(query_points, support_points, neighbors_indices, features, K_points, K_values, KP_extent,
               KP_influence="linear", aggregation_mode="sum", dtype=np.float64, chunk=2048, magnitude=False):
    """kernels/convolution_ops.py:161-255 (KPConv_ops), steps 1-11 of SURVEY.md section 3.2.

    dtype=np.float64 evaluates the same graph in double (the tolerance oracle); np.float32 mimics the
    reference's arithmetic type (summation order of tf.matmul / reduce_sum is not reproducible).

    magnitude=True returns (out, mag, alt):
      mag  the same contraction on absolute values, sum_k w^T |f| @ |W_k| / nn (the influence weights are
           non-negative; nn is counted on the SIGNED features), the scale of the rounding error of any
           summation order of out, per element;
      alt  out with every ambiguous decision taken the other way: a closest-mode neighbour whose two nearest
           kernel points are tied within CLOSEST_TIE_RTOL goes to the second one, a support whose feature-row sum
           is within NN_SUM_ULPS of zero (but not exactly zero) flips its nn vote. alt == out on rows without
           such a decision; mag covers both branches.
    """
    if KP_influence not in INFLUENCES:
        raise ValueError("Unknown influence function type (config.KP_influence)")
    if aggregation_mode not in MODES:
        raise ValueError("Unknown convolution mode. Should be 'closest' or 'sum'")
    dt = dtype
    q = np.asarray(query_points, dt)
    # :190-191 shadow support point at 1e6
    s = np.concatenate([np.asarray(support_points, dt), np.full((1, 3), 1e6, dt)], 0)
    # :234 shadow feature row of zeros
    f = np.concatenate([np.asarray(features, dt), np.zeros((1, features.shape[1]), dt)], 0)
    Kp = np.asarray(K_points, dt)
    W = np.asarray(K_values, dt)
    idx = np.asarray(neighbors_indices)
    n_kp = Kp.shape[0]
    Nq = q.shape[0]
    out = np.zeros((Nq, W.shape[2]), dt)
    if magnitude:
        mag, alt, mag_alt = np.zeros_like(out), np.zeros_like(out), np.zeros_like(out)
    ext = dt(KP_extent)
    for a, b in _chunks(Nq, chunk):
        ii = idx[a:b]
        nb = s[ii] - q[a:b, None, :]                                   # :194-197  [n,H,3]
        diff = nb[:, :, None, :] - Kp[None, None, :, :]                # :200-202  [n,H,K,3]
        d2 = np.sum(np.square(diff), axis=3)                           # :205      [n,H,K]
        if KP_influence == "constant":
            w = np.ones_like(d2)                                       # :208-211
        elif KP_influence == "linear":
            w = np.maximum(1 - np.sqrt(d2 + dt(1e-10)) / (2 * ext), dt(0.0))   # :213-216 (note the factor 2)
        else:
            sigma = ext * dt(0.3)                                      # :218-222, radius_gaussian :48-55
            w = np.exp(-d2 / (2 * np.square(sigma) + dt(1e-9)))
        w = np.transpose(w, (0, 2, 1))                                 # [n,K,H]
        w_all = w
        if aggregation_mode == "closest":                              # :227-229
            nn1 = np.argmin(d2, axis=2)                                # [n,H]
            onehot = (np.arange(n_kp)[None, :, None] == nn1[:, None, :]).astype(dt)
            w = w * onehot
        nf = f[ii]                                                     # :237      [n,H,Cin]
        wf = np.matmul(w, nf)                                          # :240      [n,K,Cin]
        ko = np.einsum("nkc,kco->no", wf, W)                           # :243-247  sum_k wf_k @ W_k
        nsum = np.sum(nf, axis=-1)                                     # :250
        nnum = np.sum((nsum > 0).astype(dt), axis=-1)                  # :251
        nnum = np.maximum(nnum, 1)                                     # :252
        out[a:b] = ko / nnum[:, None]                                  # :253
        if not magnitude:
            continue
        aW = np.abs(W)
        mag[a:b] = np.einsum("nkc,kco->no", np.matmul(w, np.abs(nf)), aW) / nnum[:, None]
        w2 = w
        if aggregation_mode == "closest" and n_kp > 1:
            srt = np.sort(d2, axis=2)
            tie = srt[:, :, 1] - srt[:, :, 0] <= CLOSEST_TIE_RTOL * srt[:, :, 1]
            second = np.argsort(d2, axis=2, kind="stable")[:, :, 1]
            nn2 = np.where(tie, second, nn1)
            w2 = w_all * (np.arange(n_kp)[None, :, None] == nn2[:, None, :]).astype(dt)
        asum = np.sum(np.abs(nf), axis=-1)
        amb = (nsum != 0) & (np.abs(nsum) < NN_SUM_ULPS * asum)
        nnum2 = np.maximum(np.sum(((nsum > 0) ^ amb).astype(dt), axis=-1), 1)
        alt[a:b] = np.einsum("nkc,kco->no", np.matmul(w2, nf), W) / nnum2[:, None]
        mag_alt[a:b] = np.einsum("nkc,kco->no", np.matmul(w2, np.abs(nf)), aW) / nnum2[:, None]
    if magnitude:
        return out, np.maximum(mag, mag_alt), alt
    return out


def kpconv_deform_ops(query_points, support_points, neighbors_indices, features, K_points, offsets,
                      modulations, K_values, KP_extent, KP_influence="linear", mode="sum",
                      dtype=np.float64, chunk=1024, magnitude=False):
    """kernels/convolution_ops.py:379-499 (KPConv_deform_ops).

    The top_k compaction (:435-451) is restated as its net effect: a neighbour that is in range of no
    deformed kernel point is re-pointed to the shadow row (zero features); the kept ones keep their
    sq_distances. No neighbour-count normalisation in this op.

    magnitude=True returns (out, mag, alt) as kpconv_ops does (modulations are positive, so they enter mag as
    they are); the ambiguous decisions here are the closest-mode ties and every d2 < extent^2 comparison with
    |d2 - extent^2| < IN_RANGE_RTOL * extent^2 (the in-range test and the constant influence).
    """
    if KP_influence not in INFLUENCES:
        raise ValueError("Unknown influence function type (config.KP_influence)")
    if mode not in MODES:
        raise ValueError("Unknown convolution mode. Should be 'closest' or 'sum'")
    dt = dtype
    q = np.asarray(query_points, dt)
    s = np.concatenate([np.asarray(support_points, dt), np.full((1, 3), 1000.0, dt)], 0)   # :414
    f = np.concatenate([np.asarray(features, dt), np.zeros((1, features.shape[1]), dt)], 0)  # :480
    Kp = np.asarray(K_points, dt)
    W = np.asarray(K_values, dt)
    off = np.asarray(offsets, dt)
    idx = np.asarray(neighbors_indices)
    n_kp = Kp.shape[0]
    Nq = q.shape[0]
    ext = dt(KP_extent)
    out = np.zeros((Nq, W.shape[2]), dt)
    if magnitude:
        mag, alt = np.zeros_like(out), np.zeros_like(out)
    for a, b in _chunks(Nq, chunk):
        ii = idx[a:b]
        nb = s[ii] - q[a:b, None, :]                                   # :417-420
        dKp = off[a:b] + Kp[None]                                      # :424      [n,K,3]
        diff = nb[:, :, None, :] - dKp[:, None, :, :]                  # :427-429  [n,H,K,3]
        d2 = np.sum(np.square(diff), axis=3)                           # :432
        mod = None if modulations is None else np.asarray(modulations, dt)[a:b, :, None]

        def contract(inside, nn1, feats):
            in_range = np.any(inside, axis=2)                          # :435      [n,H]
            if KP_influence == "constant":
                w = inside.astype(dt)                                  # :456
            elif KP_influence == "linear":
                w = np.maximum(1 - np.sqrt(d2 + dt(1e-10)) / ext, dt(0.0))  # :461 (no factor 2)
            else:
                sigma = ext * dt(0.3)
                w = np.exp(-d2 / (2 * np.square(sigma) + dt(1e-9)))
            w = np.transpose(w, (0, 2, 1))
            if mode == "closest":
                w = w * (np.arange(n_kp)[None, :, None] == nn1[:, None, :]).astype(dt)
            nf = feats * in_range[:, :, None].astype(dt)               # :441-451, 483
            wf = np.matmul(w, nf)                                      # :486
            if mod is not None:
                wf = wf * mod                                          # :489-490
            return wf

        inside = d2 < ext ** 2
        nn1 = np.argmin(d2, axis=2)
        out[a:b] = np.einsum("nkc,kco->no", contract(inside, nn1, f[ii]), W)   # :493-497
        if not magnitude:
            continue
        near = np.abs(d2 - ext ** 2) < IN_RANGE_RTOL * ext ** 2
        nn2 = nn1
        if mode == "closest" and n_kp > 1:
            srt = np.sort(d2, axis=2)
            tie = srt[:, :, 1] - srt[:, :, 0] <= CLOSEST_TIE_RTOL * srt[:, :, 1]
            nn2 = np.where(tie, np.argsort(d2, axis=2, kind="stable")[:, :, 1], nn1)
        aW = np.abs(W)
        alt[a:b] = np.einsum("nkc,kco->no", contract(inside ^ near, nn2, f[ii]), W)
        mag[a:b] = np.maximum(np.einsum("nkc,kco->no", contract(inside, nn1, np.abs(f[ii])), aW),
                              np.einsum("nkc,kco->no", contract(inside ^ near, nn2, np.abs(f[ii])), aW))
    if magnitude:
        return out, mag, alt
    return out


def kpconv_deformable(query_points, support_points, neighbors_indices, features, K_points, K_values,
                      K_values0, b0, KP_extent, KP_influence="linear", aggregation_mode="sum",
                      modulated=False, dtype=np.float64):
    """kernels/convolution_ops.py:258-376 with explicit kernel points / offset-head weights."""
    dt = dtype
    n_kp = K_points.shape[0]
    f0 = kpconv_ops(query_points, support_points, neighbors_indices, features, K_points, K_values0,
                    KP_extent, KP_influence, aggregation_mode, dtype=dt) + np.asarray(b0, dt)   # :327-339
    if modulated:
        offsets = f0[:, :3 * n_kp].reshape(-1, n_kp, 3)                # :341-345
        modulations = 2 / (1 + np.exp(-f0[:, 3 * n_kp:]))              # :348
    else:
        offsets = f0.reshape(-1, n_kp, 3)                              # :352-353
        modulations = None
    offsets = offsets * dt(KP_extent)                                  # :359
    return kpconv_deform_ops(query_points, support_points, neighbors_indices, features, K_points, offsets,
                             modulations, K_values, KP_extent, KP_influence, aggregation_mode, dtype=dt)


# ----------------------------------------------------------------------------------------------------
#  block epilogues  (models/network_blocks.py)
# ----------------------------------------------------------------------------------------------------

def ind_max_pool(x, inds):
    """models/network_blocks.py:51-66 -- shadow row = column-wise minimum."""
    x = np.concatenate([x, np.min(x, axis=0, keepdims=True)], 0)
    return np.max(x[inds], axis=1)


def closest_pool(x, inds):
    """models/network_blocks.py:69-83 -- shadow row = zeros, first column only."""
    x = np.concatenate([x, np.zeros((1, x.shape[1]), x.dtype)], 0)
    return x[inds[:, 0]]


def batch_norm_inference(x, bn, eps=1e-6):
    """models/network_blocks.py:149-160 in inference form (training = dropout_prob < 0.99 is False at
    test, :1071 + utils/tester.py:199): gamma * (x - mean) / sqrt(var + 1e-6) + beta."""
    dt = x.dtype
    g, b, m, v = (np.asarray(bn[k], dt) for k in ("gamma", "beta", "moving_mean", "moving_variance"))
    return g * (x - m) / np.sqrt(v + dt.type(eps)) + b


def leaky_relu(x, alpha=0.2):
    """models/network_blocks.py:185-186."""
    return np.where(x > 0, x, x * x.dtype.type(alpha))


class EncoderOracle:
    """Block-for-block restatement of assemble_CNN_blocks (models/network_blocks.py:1052-1118) and the
    block functions it dispatches to (:222-244 simple, :321-368 resnetb, :561-612 resnetb_strided,
    :424-471 resnetb_deformable, :672-723 resnetb_deformable_strided, :207-219 unary, :194-205 last_unary,
    :971-979 nearest_upsample)."""

    def __init__(self, config, params, dtype=np.float64):
        self.cfg = config
        self.p = params
        self.dt = dtype

    # -- helpers ---------------------------------------------------------------------------------
    def _w(self, scope):
        return np.asarray(self.p[scope + "/weights"], self.dt)

    def _bn(self, scope, x):
        if not self.cfg.use_batch_norm:
            return x + np.asarray(self.p[scope + "/offset"], self.dt)
        bn = {k: self.p[scope + "/batch_normalization/" + k] for k in
              ("gamma", "beta", "moving_mean", "moving_variance")}
        return batch_norm_inference(x, bn)

    def _kpconv(self, scope, q, s, idx, x, radius, deformable=False):
        cfg = self.cfg
        extent = cfg.KP_extent * radius / cfg.density_parameter          # network_blocks.py:92, 112
        Kp = self.p[scope + "/kernel_points"]
        if deformable:
            return kpconv_deformable(q, s, idx, x, Kp, self.p[scope + "/weights"],
                                     self.p[scope + "/offset_conv_weights"], self.p[scope + "/offset_conv_bias"],
                                     extent, cfg.KP_influence, cfg.convolution_mode, bool(cfg.modulated),
                                     dtype=self.dt)
        return kpconv_ops(q, s, idx, x, Kp, self.p[scope + "/weights"], extent, cfg.KP_influence,
                          cfg.convolution_mode, dtype=self.dt)

    # -- blocks ----------------------------------------------------------------------------------
    def unary_block(self, scope, x):
        return leaky_relu(self._bn(scope, unary_convolution(x, self._w(scope))))

    def last_unary_block(self, scope, x):
        return unary_convolution(x, self._w(scope))

    def simple_block(self, scope, layer, inputs, x, r):
        pts = inputs["points"][layer]
        x = self._kpconv(scope, pts, pts, inputs["neighbors"][layer], x, r)
        return leaky_relu(self._bn(scope, x))

    def resnetb_block(self, scope, layer, inputs, feats, r, strided=False, deformable=False):
        x = leaky_relu(self._bn(scope + "/conv1", unary_convolution(feats, self._w(scope + "/conv1"))))
        if strided:
            q, s, idx = inputs["points"][layer + 1], inputs["points"][layer], inputs["pools"][layer]
        else:
            q = s = inputs["points"][layer]
            idx = inputs["neighbors"][layer]
        x = self._kpconv(scope + "/conv2", q, s, idx, x, r, deformable)
        x = leaky_relu(self._bn(scope + "/conv2", x))
        x = self._bn(scope + "/conv3", unary_convolution(x, self._w(scope + "/conv3")))
        if strided:
            shortcut = ind_max_pool(feats, inputs["pools"][layer])        # :600
        else:
            shortcut = feats
        if (scope + "/shortcut/weights") in self.p:                       # dims differ (:355-362, :604-610)
            shortcut = self._bn(scope + "/shortcut",
                                unary_convolution(shortcut, self._w(scope + "/shortcut")))
        return leaky_relu(x + shortcut)

    # -- encoder ---------------------------------------------------------------------------------
    def encoder(self, inputs, return_all=False):
        """assemble_CNN_blocks (:1052-1118). inputs: dict(points, neighbors, pools, features)."""
        cfg = self.cfg
        r = cfg.first_subsampling_dl * cfg.density_parameter
        layer = 0
        feats = np.asarray(inputs["features"], self.dt)
        inputs = dict(inputs)
        inputs["points"] = [np.asarray(p, self.dt) for p in inputs["points"]]
        F = []
        trace = []
        block_in_layer = 0
        for block in cfg.architecture:
            if any(t in block for t in ("pool", "strided", "upsample", "global")):
                F.append(feats)
            if "upsample" in block:
                break
            scope = "layer_{:d}/{:s}_{:d}".format(layer, block.replace("_deformable", ""), block_in_layer)
            deform = "deformable" in block
            if block == "simple":
                feats = self.simple_block(scope, layer, inputs, feats, r)
            elif block in ("resnetb", "resnetb_deformable"):
                feats = self.resnetb_block(scope, layer, inputs, feats, r, False, deform)
            elif block in ("resnetb_strided", "resnetb_deformable_strided"):
                feats = self.resnetb_block(scope, layer, inputs, feats, r, True, deform)
            elif block == "unary":
                feats = self.unary_block(scope, feats)
            else:
                raise ValueError("Unknown block name in the architecture definition : " + block)
            trace.append((scope, feats))
            block_in_layer += 1
            if "pool" in block or "strided" in block:
                layer += 1
                r *= 2
                block_in_layer = 0
        if not any("upsample" in b for b in cfg.architecture):
            F.append(feats)
        return (F, trace) if return_all else F

    def decoder(self, inputs, F, return_scores=False):
        """models/D3Feat.py:15-65: (nearest_upsample, concat, unary)* + last_unary + l2_normalize.
        Variable scopes are 'uplayer_{layer}/{block}_{i}' (D3Feat.py:37). return_scores=True also evaluates the
        detection branch (:67-115) on the un-normalised features -> (descriptors, scores)."""
        cfg = self.cfg
        arch = list(cfg.architecture)
        start = next(i for i, b in enumerate(arch) if "upsample" in b)
        layer = cfg.num_layers - 1
        feats = F[-1]
        block_in_layer = 0
        for block in arch[start:]:
            scope = "uplayer_{:d}/{:s}_{:d}".format(layer, block, block_in_layer)
            if "upsample" in block:
                feats = closest_pool(feats, inputs["upsamples"][layer - 1])   # network_blocks.py:971-979
            elif block == "unary":
                feats = self.unary_block(scope, feats)
            elif block == "last_unary":
                feats = self.last_unary_block(scope, feats)
            else:
                raise ValueError("Unknown block name in the architecture definition : " + block)
            block_in_layer += 1
            if "upsample" in block:
                layer -= 1
                block_in_layer = 0
                feats = np.concatenate([feats, F[layer]], axis=1)          # D3Feat.py:63
        # tf.nn.l2_normalize(features, axis=1, epsilon=1e-10): x * rsqrt(max(sum(x^2), eps))
        norm = np.sqrt(np.maximum(np.sum(feats * feats, axis=1, keepdims=True), self.dt(1e-10)))
        if return_scores:
            return feats / norm, detection_scores(feats, inputs["neighbors"][0], inputs["lengths"][0])
        return feats / norm


def detection_scores(features, neighbors, lengths, magnitude=False, rows=None, chunk=4096):
    """Detection branch, models/D3Feat.py:67-115, for any number of stacked clouds (the reference writes it out for
    exactly two: first_pcd / second_pcd of in_batches).

      :71      features ++ zero shadow row
      :75-84   per cloud: features / (max over all points and channels of that cloud + 1e-6)
      :87-93   neighbour rows gathered through neighbors[0]; neighbour_num = count_nonzero(sum over channels), >= 1;
               mean = sum over neighbours / neighbour_num; local_max_score = softplus(features - mean)
      :96-97   depth_wise_max_score = features / (1e-6 + max over channels)
      :99-104  score = max over channels of the product; the shadow row is dropped.

    A cloud reaching past the N rows is cut at N; rows past the last cloud belong to no cloud (scaled to zero, in no
    cloud's maximum). rows= evaluates the score of those rows only (the cloud maxima still come from whole clouds).

    magnitude=True returns (score, mag, alt), all [len(rows), 1]:
      mag  the first-order rounding-error scale of the score on absolute values: the cloud scale 1/(M + 1e-6) carries
           the cancellation factor k = (|M| + 1e-6) / |M + 1e-6| into every scaled feature (mag_f = k |f|); the
           neighbour mean sum_h k |f_h| / cnt; softplus adds slope sigma(d) times the error of d plus its own rounding;
           the channel ratio f / (1e-6 + dmax) the relative errors of both operands, its denominator with the
           cancellation factor of 1e-6 + dmax; the max over channels is 1-Lipschitz (mag = max over channels). One
           float32 underflow step (FLT_MIN) is added to the softplus and the score.
      alt  the score with the count_nonzero vote flipped for every neighbour whose channel sum is within NN_SUM_ULPS
           of zero, exact zero included (a kernel sums the raw row in its own order, the restatement the scaled row;
           either may come out at exactly zero). Rows whose channels are all zero are not marked. mag covers both.
    """
    x = np.asarray(features)
    dt = x.dtype.type
    N, D = x.shape
    lengths = np.asarray(lengths, np.int64)
    start = np.minimum(np.concatenate([[0], np.cumsum(lengths)]), N)
    scaled = np.zeros((N + 1, D), x.dtype)
    kappa = np.ones((N + 1, 1))                              # cancellation factor of the row's cloud scale
    with np.errstate(divide="ignore", invalid="ignore"):
        for b in range(len(lengths)):
            a, e = start[b], start[b + 1]
            if e > a:
                m = x[a:e].max()
                scaled[a:e] = x[a:e] / (m + dt(1e-6))
                kappa[a:e] = (abs(float(m)) + 1e-6) / abs(float(m) + 1e-6)
    rows = np.arange(N) if rows is None else np.asarray(rows, np.int64)
    nb_all = np.asarray(neighbors, np.int64)
    out = np.zeros((rows.shape[0], 1), x.dtype)
    if magnitude:
        mag, alt = np.zeros((rows.shape[0], 1)), np.zeros((rows.shape[0], 1), x.dtype)
    tiny = float(np.finfo(np.float32).tiny)
    for a, b in _chunks(rows.shape[0], chunk):
        r = rows[a:b]
        nb = nb_all[r]
        nf = scaled[nb]                                       # [n, H, D]; shadow index N -> zero row
        f = scaled[r]
        nsum = nf.sum(axis=-1)
        vote = nsum != 0
        dmax = f.max(axis=1, keepdims=True)
        ratio = f / (dt(1e-6) + dmax)

        def branch(vote):
            num = np.maximum(np.count_nonzero(vote, axis=-1), 1).astype(x.dtype)[:, None]
            mean = nf.sum(axis=1) / num
            d = f - mean
            softplus = np.where(d > 20, d, np.log1p(np.exp(np.minimum(d, dt(20)))))
            return (softplus * ratio).max(axis=1, keepdims=True), num, d, softplus

        score, num, d, softplus = branch(vote)
        out[a:b] = score
        if not magnitude:
            continue
        asum = np.abs(nf).sum(axis=-1)
        amb = np.abs(nsum) < NN_SUM_ULPS * asum
        score2, num2, d2, softplus2 = branch(vote ^ amb)
        alt[a:b] = score2
        k = kappa[r]
        af = k * np.abs(f)
        dmax64 = dmax.astype(np.float64)
        e = 1e-6 + dmax64
        ae = k * np.abs(dmax64) + 1e-6
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            aratio = (af + np.abs(ratio) * ae) / np.abs(e)
            an = (kappa[nb] * np.abs(nf)).sum(axis=1)          # sum_h k |f_h|
            m = None
            for nm, dd, sp in ((num, d, softplus), (num2, d2, softplus2)):
                sig = 0.5 * (1.0 + np.tanh(0.5 * np.float64(dd)))
                asp = sig * (af + an / nm) + np.abs(sp) + tiny
                mp = (asp * np.abs(ratio) + np.abs(sp) * aratio).max(axis=1, keepdims=True)
                m = mp if m is None else np.maximum(m, mp)
        mag[a:b] = m + tiny
    if magnitude:
        return out, mag, alt
    return out


# ----------------------------------------------------------------------------------------------------
#  input pyramid  (datasets/common.py:1301-1413)
# ----------------------------------------------------------------------------------------------------

def descriptor_input_pyramid(config, stacked_points, stacked_lengths, neighborhood_limits, neighbors_fn,
                             subsampling_fn):
    """Pyramid loop of Dataset.tf_descriptor_input with big_neighborhood_filter (:399-406).

    neighbors_fn(q, s, qb, sb, r) / subsampling_fn(p, b, dl) are the native ops (oracle 'ref' or 'port').
    """
    r_normal = config.first_subsampling_dl * config.KP_extent * 2.5
    layer_blocks = []
    pts_l, nb_l, pool_l, up_l, len_l = [], [], [], [], []
    arch = list(config.architecture)
    pts = np.asarray(stacked_points, np.float32)
    lens = np.asarray(stacked_lengths, np.int32)
    for block_i, block in enumerate(arch):
        if "global" in block or "upsample" in block:
            break
        if not ("pool" in block or "strided" in block):
            layer_blocks.append(block)
            if block_i < len(arch) - 1 and "upsample" not in arch[block_i + 1]:
                continue
        if layer_blocks:
            if any("deformable" in b for b in layer_blocks[:-1]):
                r = r_normal * config.density_parameter / (config.KP_extent * 2.5)
            else:
                r = r_normal
            conv_i = neighbors_fn(pts, pts, lens, lens, r)
        else:
            conv_i = np.zeros((0, 1), np.int32)
        if "pool" in block or "strided" in block:
            dl = 2 * r_normal / (config.KP_extent * 2.5)
            pool_p, pool_b = subsampling_fn(pts, lens, dl)
            if "deformable" in block:
                r = r_normal * config.density_parameter / (config.KP_extent * 2.5)
            else:
                r = r_normal
            pool_i = neighbors_fn(pool_p, pts, pool_b, lens, r)
            up_i = neighbors_fn(pts, pool_p, lens, pool_b, 2 * r)
        else:
            pool_i = np.zeros((0, 1), np.int32)
            pool_p = np.zeros((0, 3), np.float32)
            pool_b = np.zeros((0,), np.int32)
            up_i = np.zeros((0, 1), np.int32)
        lim = neighborhood_limits[len(pts_l)]
        conv_i, pool_i, up_i = conv_i[:, :lim], pool_i[:, :lim], up_i[:, :lim]
        pts_l.append(pts)
        nb_l.append(conv_i)
        pool_l.append(pool_i)
        up_l.append(up_i)
        len_l.append(lens)
        pts, lens = pool_p, pool_b
        r_normal *= 2
        layer_blocks = []
    return dict(points=pts_l, neighbors=nb_l, pools=pool_l, upsamples=up_l, lengths=len_l)
