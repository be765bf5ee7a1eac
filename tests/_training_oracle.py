"""Float64 torch-on-CPU restatement of the D3Feat training graph (d3feat_b200/training.py) and of its new ops.

Every function evaluates the TF graph in float64 with torch autograd supplying the adjoint; the choices that make
the autograd gradient TF's own are explicit:
  * reduce_max / reduce_min are amax / amin, whose gradients split ties evenly (TF's _MinOrMaxGrad);
  * tf.maximum(s, eps) in l2_normalize is where(s >= eps, s, eps): the tie goes to the first input;
  * LeakyReLU is where(y > 0, y, alpha*y): LeakyReluGrad tests y > 0;
  * KPConv's neighbour count nn and detection's count_nonzero are computed from detached tensors (no gradient);
  * softplus' = sigmoid (SoftplusGrad), written out below.
The tolerances scale with mag(ref), the largest |ref| of the tensor compared.
`decisions` collects the decision margins of a whole-network run: the gaps that fp32 must not close for the fp32
graph to take the same branches as this restatement.

Only tests/ import this module.
"""
import numpy as np
import torch

D = torch.float64


def t64(a):
    return torch.as_tensor(np.asarray(a, np.float64))


def mag(t):
    return float(t.detach().abs().max()) if t.numel() else 0.0


def leaky(y, alpha):
    return y if alpha is None else torch.where(y > 0, y, alpha * y)


def batch_norm_train(x, gamma, beta, residual=None, alpha=None, eps=1e-6):
    """tf.layers.batch_normalization(training=True) (+ residual, LeakyReLU) -> (out, batch mean, batch variance).
    gamma None: x + beta (use_batch_norm = False). N = 0: the statistics are None."""
    if gamma is None:
        y, mean, var = x + beta, None, None
    else:
        if x.shape[0] == 0:
            return x + 0 * beta, None, None
        mean = x.mean(0)
        var = ((x - mean.detach()) ** 2).mean(0)          # tf.nn.moments: stop_gradient(mean) in the variance
        inv = torch.rsqrt(var + eps) * gamma
        y = x * inv + (beta - mean * inv)
    if residual is not None:
        y = y + residual
    return leaky(y, alpha), mean, var


def ind_max_pool(x, inds):
    """reduce_max(gather(x || reduce_min(x), inds)); an index outside [0, N1) is the shadow (the forward's rule)."""
    N1 = x.shape[0]
    xs = torch.cat([x, x.amin(0, keepdim=True)], 0)
    inds = torch.as_tensor(np.asarray(inds, np.int64))
    ii = torch.where((inds < 0) | (inds >= N1), N1, inds)
    return xs[ii].amax(1)


def gather_rows(x, inds):
    """(x || zeros)[inds]: closest_pool on the first index column, tf.gather."""
    N1 = x.shape[0]
    xs = torch.cat([x, torch.zeros((1, x.shape[1]), dtype=x.dtype)], 0)
    inds = torch.as_tensor(np.asarray(inds, np.int64))
    return xs[torch.where((inds < 0) | (inds >= N1), N1, inds)]


def l2_normalize(x, eps=1e-10):
    s = (x * x).sum(1, keepdim=True)
    return x * torch.rsqrt(torch.where(s >= eps, s, torch.full_like(s, eps)))


def softplus(d):
    """softplus with SoftplusGrad's derivative sigmoid(d) everywhere (the forward switches to d above 20)."""
    class _Sp(torch.autograd.Function):
        @staticmethod
        def forward(ctx, d):
            ctx.save_for_backward(d)
            return torch.where(d > 20, d, torch.log1p(torch.exp(torch.clamp_max(d, 20.0))))

        @staticmethod
        def backward(ctx, g):
            d, = ctx.saved_tensors
            return g * torch.sigmoid(d)
    return _Sp.apply(d)


def detection_scores(x, neighbors, lengths, decisions=None):
    """The detection branch as pool.cu computes it (models/D3Feat.py:67-115 for B stacked clouds): per-cloud maximum
    M (all elements of the cloud), inv = 1/(M + 1e-6) (0 for rows of no cloud), mean over the neighbour rows scaled by
    the row's own inv, divided by the detached count of neighbours with a non-zero raw row sum."""
    N, Dm = x.shape
    lengths = np.asarray(lengths, np.int64)
    start = np.minimum(np.concatenate([[0], np.cumsum(lengths)]), N)
    inv = torch.zeros((N, 1), dtype=x.dtype)
    for b in range(len(lengths)):
        a, e = int(start[b]), int(start[b + 1])
        if e > a:
            M = x[a:e].amax()
            inv[a:e] = 1.0 / (M + 1e-6)
            if decisions is not None:
                v = x[a:e].detach().flatten()
                below = v[v < M.detach()]
                if below.numel():
                    decisions.setdefault("cloud_max_gap", []).append(float((M.detach() - below.max()) / abs(M.detach())))
    nb = torch.as_tensor(np.asarray(neighbors, np.int64))
    valid = (nb >= 0) & (nb < N)
    ii = torch.where(valid, nb, N)
    xs = torch.cat([x, torch.zeros((1, Dm), dtype=x.dtype)], 0)
    nonzero = torch.cat([x.detach().sum(1) != 0, torch.zeros(1, dtype=torch.bool)])
    cnt = torch.clamp_min((nonzero[ii] & valid).sum(1, keepdim=True), 1).to(x.dtype)
    f = x * inv
    mean = xs[ii].sum(1) * inv / cnt
    d = f - mean
    dmax = f.amax(1, keepdim=True)
    ratio = f / (1e-6 + dmax)
    p = softplus(d) * ratio
    score = p.amax(1, keepdim=True)
    if decisions is not None:
        pd = p.detach()
        top = pd.amax(1, keepdim=True)
        second = torch.where(pd < top, pd, torch.full_like(pd, -np.inf)).amax(1)
        decisions["score_rows_gap"] = ((top[:, 0] - second) / top[:, 0].abs().clamp_min(1e-30)).numpy()
    return score


def kpconv(q, s, idx, f, Kp, W, extent, influence="linear", mode="sum"):
    """Rigid KPConv_ops (kernels/convolution_ops.py:161-255) with the neighbour count nn detached."""
    Ns = s.shape[0]
    idx = torch.as_tensor(np.asarray(idx, np.int64))
    ii = torch.where((idx < 0) | (idx > Ns), Ns, idx)
    s_ = torch.cat([t64(s), torch.full((1, 3), 1e6, dtype=D)], 0)
    f_ = torch.cat([f, torch.zeros((1, f.shape[1]), dtype=f.dtype)], 0)
    nbp = s_[ii] - t64(q)[:, None, :]
    d2 = ((nbp[:, :, None, :] - t64(Kp)[None, None]) ** 2).sum(-1)                  # [n, H, K]
    if influence == "constant":
        w = torch.ones_like(d2)
    elif influence == "linear":
        w = torch.clamp_min(1 - torch.sqrt(d2 + 1e-10) / (2 * extent), 0.0)
    else:
        sigma = extent * 0.3
        w = torch.exp(-d2 / (2 * sigma ** 2 + 1e-9))
    if mode == "closest":
        w = w * torch.nn.functional.one_hot(d2.argmin(2), d2.shape[2]).to(D)
    nf = f_[ii]                                                                     # [n, H, C]
    out = torch.einsum("nhk,nhc,kco->no", w, nf, W)
    nn = torch.clamp_min((nf.detach().sum(-1) > 0).sum(-1), 1).to(D)
    return out / nn[:, None]


class Network:
    """The rigid training graph (training.forward) in float64 on the CPU. params: {name: leaf float64 tensor}; the
    moving statistics are updated in the dict as the GPU updates them in the store. decisions: margins (see top)."""

    def __init__(self, config, params, inference=False):
        self.cfg = config
        self.p = params
        self.inference = inference          # batch norm from the moving statistics (the inference graph)
        self.decisions = {"leaky": [], "pool_gap": []}

    def bn(self, scope, x, residual=None, alpha=None):
        cfg = self.cfg
        if cfg.use_batch_norm and self.inference:
            pre = scope + "/batch_normalization/"
            g, b, m, v = (self.p[pre + k] for k in ("gamma", "beta", "moving_mean", "moving_variance"))
            y = g * (x - m) / torch.sqrt(v + 1e-6) + b
            y = y if residual is None else y + residual
        elif cfg.use_batch_norm:
            pre = scope + "/batch_normalization/"
            y, mean, var = batch_norm_train(x, self.p[pre + "gamma"], self.p[pre + "beta"], residual, None)
            if mean is not None:
                dec = 1.0 - cfg.batch_norm_momentum
                for k, v in (("moving_mean", mean), ("moving_variance", var)):
                    m = self.p[pre + k]
                    self.p[pre + k] = m - (m - v.detach()) * dec
        else:
            y, _, _ = batch_norm_train(x, None, self.p[scope + "/offset"], residual, None)
        if alpha is not None:
            a = y.detach().abs()
            self.decisions["leaky"].append(a / max(float(a.max()), 1e-30))
        return leaky(y, alpha)

    def conv(self, scope, q, s, idx, x, radius):
        cfg = self.cfg
        ext = cfg.KP_extent * radius / cfg.density_parameter
        return kpconv(q, s, idx, x, self.p[scope + "/kernel_points"].detach().numpy(), self.p[scope + "/weights"], ext,
                      cfg.KP_influence, cfg.convolution_mode)

    def pool(self, x, inds):
        out = ind_max_pool(x, inds)
        xs = torch.cat([x, x.amin(0, keepdim=True)], 0).detach()
        inds = torch.as_tensor(np.asarray(inds, np.int64))
        v = xs[torch.where((inds < 0) | (inds >= x.shape[0]), x.shape[0], inds)]
        top = v.amax(1, keepdim=True)
        below = torch.where(v < top, v, torch.full_like(v, -np.inf)).amax(1)
        gap = (top[:, 0] - below) / max(float(top.abs().max()), 1e-30)
        self.decisions["pool_gap"].append(gap[torch.isfinite(gap)])
        return out

    def block(self, block, scope, layer, inputs, x, r, fdim):
        P, w = inputs["points"], lambda s: self.p[s + "/weights"]
        if block == "unary":
            return self.bn(scope, x @ w(scope), alpha=0.2)
        if block == "last_unary":
            return x @ w(scope)
        if block == "simple":
            return self.bn(scope, self.conv(scope, P[layer], P[layer], inputs["neighbors"][layer], x, r), alpha=0.2)
        if block in ("resnetb", "resnetb_strided"):
            strided = block == "resnetb_strided"
            y = self.bn(scope + "/conv1", x @ w(scope + "/conv1"), alpha=0.2)
            if strided:
                y = self.conv(scope + "/conv2", P[layer + 1], P[layer], inputs["pools"][layer], y, r)
            else:
                y = self.conv(scope + "/conv2", P[layer], P[layer], inputs["neighbors"][layer], y, r)
            y = self.bn(scope + "/conv2", y, alpha=0.2)
            sc = self.pool(x, inputs["pools"][layer]) if strided else x
            if sc.shape[1] != 2 * fdim:
                sc = self.bn(scope + "/shortcut", sc @ w(scope + "/shortcut"))
            return self.bn(scope + "/conv3", y @ w(scope + "/conv3"), residual=sc, alpha=0.2)
        if block == "nearest_upsample":
            return gather_rows(x, np.asarray(inputs["upsamples"][layer - 1])[:, 0])
        raise ValueError(block)

    def forward(self, inputs):
        cfg = self.cfg
        r = cfg.first_subsampling_dl * cfg.density_parameter
        layer, fdim, bil = 0, cfg.first_features_dim, 0
        x = t64(inputs["features"])
        F = []
        arch = list(cfg.architecture)
        for block in arch:
            if any(t in block for t in ("pool", "strided", "upsample", "global")):
                F.append(x)
            if "upsample" in block:
                break
            x = self.block(block, "layer_{:d}/{:s}_{:d}".format(layer, block, bil), layer, inputs, x, r, fdim)
            bil += 1
            if "strided" in block:
                layer, r, fdim, bil = layer + 1, r * 2, fdim * 2, 0
        layer = cfg.num_layers - 1
        r = cfg.first_subsampling_dl * cfg.density_parameter * 2 ** layer
        fdim = cfg.first_features_dim * 2 ** layer
        x = F[-1]
        bil = 0
        for block in arch[next(i for i, b in enumerate(arch) if "upsample" in b):]:
            x = self.block(block, "uplayer_{:d}/{:s}_{:d}".format(layer, block, bil), layer, inputs, x, r, fdim)
            bil += 1
            if "upsample" in block:
                layer, r, fdim, bil = layer - 1, r * 0.5, fdim // 2, 0
                x = torch.cat([x, F[layer]], 1)
        s = (x * x).sum(1)
        self.decisions["l2_sum_vs_eps"] = float(s.detach().min())
        return l2_normalize(x), detection_scores(x, inputs["neighbors"][0], inputs["lengths"][0], self.decisions)


def cdist(a, b):
    return torch.sqrt(((a[:, None, :] - b[None, :, :]) ** 2).sum(-1) + 1e-12)


def d3feat_loss(desc, scores, anc, pos, points, config, weights, decisions=None):
    """models/KPFCNN_model.py:142-188 with utils/loss.py circle_loss / det_loss, plus the L2 regulariser over
    `weights` -> (loss, desc_loss, det_loss, accuracy, d_pos, d_neg)."""
    anc, pos = torch.as_tensor(np.asarray(anc, np.int64)), torch.as_tensor(np.asarray(pos, np.int64))
    k = anc.shape[0]
    reg = config.weights_decay * sum(0.5 * (w * w).sum() for w in weights)
    if k < 0.5 * config.keypts_num:
        z = torch.zeros((), dtype=D)
        return reg, z, z, z - 1, z, z
    kp = t64(points)[anc]
    kd = cdist(kp, kp)
    dists = cdist(desc[anc], desc[pos])
    same = torch.eye(k, dtype=torch.bool)
    fneg = (kd < config.safe_radius) & ~same
    negm = ~same & ~fneg
    fp = (dists * same.to(D)).amax(1)
    cn = (dists + 1e5 * same.to(D)).amin(1)
    avg_neg = (dists * negm.to(D)).mean() * k / (k - 1.0)
    acc = ((fp - cn) <= 0).to(D).sum() / k
    neg = dists + 1e8 * fneg.to(D) + 1e8 * same.to(D)
    lse_n = torch.logsumexp(25 * (1.4 - neg) * torch.clamp_min(1.4 - neg, 0.0).detach(), dim=-1)
    desc_loss = (torch.nn.functional.softplus(25 * (fp - 0.1) + lse_n) / 25).mean()
    det = config.det_loss_weight * ((fp - cn)[:, None] * (scores[anc] + scores[pos] + 1e-6)).mean()
    if decisions is not None:
        # a repeated keypoint repeats a column exactly (the same rows, the same arithmetic): not a decision
        dd = dists.detach() + 1e5 * same.to(D)
        lo = dd.amin(1, keepdim=True)
        second = torch.where(dd > lo, dd, torch.full_like(dd, np.inf)).amin(1)
        decisions["closest_negative_gap"] = float(((second - lo[:, 0]) / second).min())
        decisions["keypoint_score_gap"] = float(np.min(decisions["score_rows_gap"][np.concatenate([anc, pos])]))
    return desc_loss + det + reg, desc_loss, det, acc, fp.mean(), avg_neg
