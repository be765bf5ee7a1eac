"""Training graph of D3Feat on the GPU: the rigid blocks of models/network_blocks.py and the decoder of
models/D3Feat.py with training = True, and the loss of models/KPFCNN_model.py:142-188 / utils/loss.py.

    store = ParamStore(training.initial_params(config, seed), "cuda")   # or a restored snapshot
    params = training.trainable(store)               # weights, gamma, beta, offset require grad
    opt = training.MomentumClip(params, config.learning_rate, config.momentum, config.grad_clip_norm)
    with use_params(store):
        desc, scores = training.forward(inputs, config)       # inputs: exact-shape pyramid (pyramid.descriptor_input)
        loss, *stats = training.d3feat_loss(desc, scores, anc_inds, pos_inds, points, config)
    opt.zero_grad(); loss.backward()
    opt.step()                                       # tf.clip_by_norm per gradient + tf.train.MomentumOptimizer

The differentiable ops are torch.autograd.Functions over sm_90a kernels (train_ops.cu): batch norm in training mode
(batch statistics, moving-average update in place), ind_max_pool, closest_pool / gather_rows, l2_normalize and
detection_scores. The update is MomentumClip over optim.cu. The convolutions are the differentiable conv_ops.KPConv /
unary_convolution. forward walks the same schedule of scopes, radii and widths as the inference path
(network_blocks.architecture), with its own blocks; the inference blocks still refuse training = True. Because the
moving statistics are updated in place, ParamStore.bn_affine picks the trained statistics up. The loss is small tensor
algebra on the keypoints and stays in torch.

The step is not graph-capturable (the KPConv feature gradient reads its reverse width back to the host), so inputs
must have exact shapes: a static (capacity-sized) pyramid is refused with ValueError. Deformable blocks have no
gradient here and raise NotImplementedError.
"""
import types

import numpy as np
import torch
import torch.nn.functional as Fn

from . import _lib
from . import network_blocks as nb
from . import variables as V
from .variables import variable_scope

_F32, _I32 = torch.float32, torch.int32
BN_EPSILON = 1e-6        # models/network_blocks.py:155
L2_EPSILON = 1e-10       # tf.nn.l2_normalize default (models/D3Feat.py:65)

# training_3DMatch.py:79-113 (weights_decay: utils/config.py:137)
# lr_decays (:107) is read-only: every Config built from these dicts shares it (assign a new dict to change it)
TRAINING_3DMATCH = dict(batch_norm_momentum=0.98, learning_rate=1e-1, momentum=0.98, grad_clip_norm=100.0,
                        weights_decay=1e-6, det_loss_weight=1.0, safe_radius=0.1, keypts_num=256,
                        lr_decays=types.MappingProxyType({i: 0.1 ** (1 / 80) for i in range(1, 200)}))
# training_KITTI.py:63-113
TRAINING_KITTI = dict(TRAINING_3DMATCH, first_subsampling_dl=0.30, safe_radius=1.0, keypts_num=1024)

TRAINABLE = ("weights", "gamma", "beta", "offset")


# ----------------------------------------------------------------------------------------------------
#  direct entry points
# ----------------------------------------------------------------------------------------------------

def batch_norm_forward(x, gamma, beta, moving_mean, moving_var, momentum, residual=None, alpha=None):
    """tf.layers.batch_normalization(training=True, epsilon=1e-6) on x[N, C], then + residual and LeakyReLU(alpha)
    when given. Updates moving_mean / moving_var in place (moving -= (moving - batch) * (1 - momentum)) and returns
    (out, batch mean, invstd). gamma = None: use_batch_norm = False, out = x + beta (beta is the 'offset'), no
    statistics (mean and invstd are None). N = 0 leaves the moving statistics as they are."""
    op = "batch_norm_forward"
    x = _lib.tensor_arg(x, op + ": x", _F32, (None, None))
    dev = x.device
    N, C = x.shape
    beta = _lib.tensor_arg(beta, op + ": beta", _F32, (C,), dev)
    res = _lib.tensor_arg(residual, op + ": residual", _F32, (N, C), dev, optional=True)
    mean = invstd = None
    if gamma is not None:
        gamma = _lib.tensor_arg(gamma, op + ": gamma", _F32, (C,), dev)
        for t, n in ((moving_mean, "moving_mean"), (moving_var, "moving_variance")):
            if not (torch.is_tensor(t) and t.is_contiguous()):
                raise ValueError("%s: %s must be a contiguous tensor (it is updated in place)" % (op, n))
            _lib.tensor_arg(t, "%s: %s" % (op, n), _F32, (C,), dev)
        mean = torch.zeros((C,), dtype=_F32, device=dev)
        invstd = torch.zeros((C,), dtype=_F32, device=dev)
    out = torch.empty((N, C), dtype=_F32, device=dev)
    L = _lib.lib()
    ws = _lib.workspace(L.d3f_batch_norm_train_workspace_bytes(N, C), dev)
    _lib.check(L.d3f_batch_norm_train_forward(_lib.ptr(x), N, C, _lib.ptr(gamma), _lib.ptr(beta),
                                              _lib.ptr(moving_mean if gamma is not None else None),
                                              _lib.ptr(moving_var if gamma is not None else None),
                                              float(np.float32(1.0 - momentum)), BN_EPSILON, _lib.ptr(res),
                                              -1.0 if alpha is None else float(alpha), _lib.ptr(out), _lib.ptr(mean),
                                              _lib.ptr(invstd), _lib.ptr(ws), ws.numel(), _lib.stream()),
               "d3f_batch_norm_train_forward")
    if gamma is not None and N > 0:
        # written by the kernel: tell autograd and the cached inference folds (ParamStore.bn_affine) they changed
        torch.autograd.graph.increment_version(moving_mean)
        torch.autograd.graph.increment_version(moving_var)
    return out, mean, invstd


def batch_norm_backward(x, out, grad_out, gamma, mean, invstd, alpha=None, *, x_grad=True, residual_grad=False,
                        gamma_grad=True, beta_grad=True):
    """Gradients of batch_norm_forward for grad_out[N, C]: (dx, dresidual, dgamma, dbeta), None where not asked for.
    dz = grad_out * LeakyReluGrad (out > 0), dbeta = sum dz, dgamma = sum dz*xhat,
    dx = gamma*invstd*(dz - dbeta/N - xhat*dgamma/N) (dx = dz without gamma), dresidual = dz."""
    op = "batch_norm_backward"
    x = _lib.tensor_arg(x, op + ": x", _F32, (None, None))
    dev = x.device
    N, C = x.shape
    out = _lib.tensor_arg(out, op + ": out", _F32, (N, C), dev)
    g = _lib.tensor_arg(grad_out, op + ": grad_out", _F32, (N, C), dev)
    if gamma is not None:
        gamma = _lib.tensor_arg(gamma, op + ": gamma", _F32, (C,), dev)
        mean = _lib.tensor_arg(mean, op + ": mean", _F32, (C,), dev)
        invstd = _lib.tensor_arg(invstd, op + ": invstd", _F32, (C,), dev)
    else:
        gamma_grad, mean, invstd = False, None, None
    new = lambda want, shape: torch.empty(shape, dtype=_F32, device=dev) if want else None
    dx, dres = new(x_grad, (N, C)), new(residual_grad, (N, C))
    dgamma, dbeta = new(gamma_grad, (C,)), new(beta_grad, (C,))
    L = _lib.lib()
    ws = _lib.workspace(L.d3f_batch_norm_train_workspace_bytes(N, C), dev)
    _lib.check(L.d3f_batch_norm_train_backward(_lib.ptr(x), _lib.ptr(out), _lib.ptr(g), N, C, _lib.ptr(gamma),
                                               _lib.ptr(mean), _lib.ptr(invstd),
                                               -1.0 if alpha is None else float(alpha), _lib.ptr(dx), _lib.ptr(dres),
                                               _lib.ptr(dgamma), _lib.ptr(dbeta), _lib.ptr(ws), ws.numel(),
                                               _lib.stream()), "d3f_batch_norm_train_backward")
    return dx, dres, dgamma, dbeta


def ind_max_pool_backward(x, inds, out, grad_out):
    """Gradient of network_blocks.ind_max_pool(x, inds) -> out for grad_out[N2, C]: dx[N1, C] (TF's reduce_max and
    reduce_min gradients: ties split evenly, the shadow's shares go to the rows equal to the column minimum)."""
    op = "ind_max_pool_backward"
    x = _lib.tensor_arg(x, op + ": x", _F32, (None, None))
    dev = x.device
    N1, C = x.shape
    inds = _lib.tensor_arg(inds, op + ": inds", _I32, (None, None), dev)
    N2, H = inds.shape
    out = _lib.tensor_arg(out, op + ": out", _F32, (N2, C), dev)
    g = _lib.tensor_arg(grad_out, op + ": grad_out", _F32, (N2, C), dev)
    if N1 == 0:
        raise ValueError("%s: x has no rows" % op)
    dx = torch.empty((N1, C), dtype=_F32, device=dev)
    L = _lib.lib()
    ws = _lib.workspace(L.d3f_ind_max_pool_backward_workspace_bytes(N1, N2, H, C), dev)
    _lib.check(L.d3f_ind_max_pool_backward(_lib.ptr(x), _lib.ptr(inds), _lib.ptr(out), _lib.ptr(g), N1, N2, H, C,
                                           _lib.ptr(dx), _lib.ptr(ws), ws.numel(), _lib.stream()),
               "d3f_ind_max_pool_backward")
    return dx


def gather_rows_backward(inds, grad_out, n_rows):
    """Gradient of the row gather out[q] = (x || zeros)[inds[q]] for grad_out[N2, C]: dx[n_rows, C], the sum of the
    rows of grad_out gathered from each row, in ascending q; indices outside [0, n_rows) lose their gradient."""
    op = "gather_rows_backward"
    inds = _lib.tensor_arg(inds, op + ": inds", _I32, (None,))
    dev = inds.device
    N2 = inds.shape[0]
    g = _lib.tensor_arg(grad_out, op + ": grad_out", _F32, (N2, None), dev)
    C = g.shape[1]
    dx = torch.empty((int(n_rows), C), dtype=_F32, device=dev)
    L = _lib.lib()
    ws = _lib.workspace(L.d3f_gather_rows_backward_workspace_bytes(int(n_rows), N2), dev)
    _lib.check(L.d3f_gather_rows_backward(_lib.ptr(inds), _lib.ptr(g), int(n_rows), N2, C, _lib.ptr(dx), _lib.ptr(ws),
                                          ws.numel(), _lib.stream()), "d3f_gather_rows_backward")
    return dx


def l2_normalize_backward(x, grad_out):
    """Gradient of network_blocks.l2_normalize(x) for grad_out[N, C]."""
    op = "l2_normalize_backward"
    x = _lib.tensor_arg(x, op + ": x", _F32, (None, None))
    g = _lib.tensor_arg(grad_out, op + ": grad_out", _F32, tuple(x.shape), x.device)
    dx = torch.empty_like(x)
    _lib.check(_lib.lib().d3f_l2_normalize_backward(_lib.ptr(x), _lib.ptr(g), x.shape[0], x.shape[1], L2_EPSILON,
                                                    _lib.ptr(dx), _lib.stream()), "d3f_l2_normalize_backward")
    return dx


def detection_scores_backward(features, neighbors, lengths, grad_scores):
    """Gradient of network_blocks.detection_scores(features, neighbors, lengths) for grad_scores[N, 1]: dfeatures."""
    op = "detection_scores_backward"
    x = _lib.tensor_arg(features, op + ": features", _F32, (None, None))
    dev = x.device
    N, D = x.shape
    nbr = _lib.tensor_arg(neighbors, op + ": neighbors", _I32, (N, None), dev)
    lens = _lib.tensor_arg(lengths, op + ": lengths", _I32, (None,), dev)
    g = _lib.tensor_arg(grad_scores, op + ": grad_scores", _F32, (N, 1), dev)
    B, H = int(lens.shape[0]), int(nbr.shape[1])
    dx = torch.empty_like(x)
    L = _lib.lib()
    ws = _lib.workspace(L.d3f_detection_scores_backward_workspace_bytes(N, H, B, D), dev)
    _lib.check(L.d3f_detection_scores_backward(_lib.ptr(x), _lib.ptr(nbr), _lib.ptr(lens), _lib.ptr(g), B, N, H, D,
                                               _lib.ptr(dx), _lib.ptr(ws), ws.numel(), _lib.stream()),
               "d3f_detection_scores_backward")
    return dx


# ----------------------------------------------------------------------------------------------------
#  autograd Functions
# ----------------------------------------------------------------------------------------------------

class _BatchNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, gamma, beta, residual, moving_mean, moving_var, momentum, alpha):
        out, mean, invstd = batch_norm_forward(x, gamma, beta, moving_mean, moving_var, momentum, residual, alpha)
        ctx.save_for_backward(x, out, gamma, mean, invstd)
        ctx.alpha = alpha
        return out

    @staticmethod
    def backward(ctx, grad_out):
        x, out, gamma, mean, invstd = ctx.saved_tensors
        need = ctx.needs_input_grad
        dx, dres, dgamma, dbeta = batch_norm_backward(x, out, grad_out, gamma, mean, invstd, ctx.alpha,
                                                      x_grad=need[0], residual_grad=need[3],
                                                      gamma_grad=need[1] and gamma is not None, beta_grad=need[2])
        return dx, dgamma, dbeta, dres, None, None, None, None


class _MaxPoolFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, inds):
        out = nb.ind_max_pool(x, inds)
        ctx.save_for_backward(x, inds, out)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        x, inds, out = ctx.saved_tensors
        return ind_max_pool_backward(x, inds, out, grad_out), None


class _GatherFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, inds):
        ctx.save_for_backward(inds)
        ctx.n_rows = x.shape[0]
        return nb.closest_pool(x, inds[:, None])

    @staticmethod
    def backward(ctx, grad_out):
        inds, = ctx.saved_tensors
        return gather_rows_backward(inds, grad_out, ctx.n_rows), None


class _L2Fn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        ctx.save_for_backward(x)
        return nb.l2_normalize(x)

    @staticmethod
    def backward(ctx, grad_out):
        x, = ctx.saved_tensors
        return l2_normalize_backward(x, grad_out)


class _DetectionFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, neighbors, lengths):
        ctx.save_for_backward(x, neighbors, lengths)
        return nb.detection_scores(x, neighbors, lengths)

    @staticmethod
    def backward(ctx, grad_out):
        x, neighbors, lengths = ctx.saved_tensors
        return detection_scores_backward(x, neighbors, lengths, grad_out), None, None


def batch_norm(x, scope, config, residual=None, alpha=None):
    """models/network_blocks.py:149-165 with training = True, + residual and LeakyReLU(alpha) when given. Reads
    gamma / beta and the moving statistics of `scope` (or its 'offset' without batch norm) from the active ParamStore
    and updates the moving statistics in place."""
    store = V.current_store()
    if store is None:
        raise RuntimeError("batch_norm: no ParamStore active (wrap the call in variables.use_params)")
    gamma, beta, mm, mv = store.bn_variables(scope, config.use_batch_norm)
    return _BatchNormFn.apply(x, gamma, beta, residual, mm, mv, float(config.batch_norm_momentum), alpha)


def ind_max_pool(x, inds):
    """network_blocks.ind_max_pool with a gradient."""
    return _MaxPoolFn.apply(x, _lib.tensor_arg(inds, "ind_max_pool: inds", _I32, (None, None), x.device))


def closest_pool(x, inds):
    """network_blocks.closest_pool with a gradient: the row gather through the first index column."""
    inds = _lib.tensor_arg(inds, "closest_pool: inds", _I32, (None, None), x.device)
    return _GatherFn.apply(x, inds[:, 0].contiguous())


def gather_rows(x, inds):
    """tf.gather(x, inds) of rows with a gradient (repeated indices sum their gradients; no atomics)."""
    return _GatherFn.apply(x, _lib.tensor_arg(inds, "gather_rows: inds", _I32, (None,), x.device))


def l2_normalize(x):
    """network_blocks.l2_normalize with a gradient."""
    return _L2Fn.apply(x)


def detection_scores(x, neighbors, lengths):
    """network_blocks.detection_scores with a gradient with respect to the features."""
    return _DetectionFn.apply(x, neighbors, lengths)


# ----------------------------------------------------------------------------------------------------
#  blocks (training = True), signature of network_blocks: layer_ind, inputs, features, radius, fdim, config
# ----------------------------------------------------------------------------------------------------

def unary_block(layer_ind, inputs, features, radius, fdim, config):
    """:207-219."""
    w = nb.weight_variable([int(features.shape[1]), fdim])
    x = nb.conv_ops.unary_convolution(features, w)
    return batch_norm(x, V.current_scope(), config, alpha=0.2)


def last_unary_block(layer_ind, inputs, features, radius, fdim, config):
    """:194-205."""
    w = nb.weight_variable([int(features.shape[1]), 32])
    return nb.conv_ops.unary_convolution(features, w)


def simple_block(layer_ind, inputs, features, radius, fdim, config):
    """:222-244."""
    w = nb.weight_variable([config.num_kernel_points, int(features.shape[1]), fdim])
    pts = inputs["points"][layer_ind]
    x = nb.KPConv(pts, pts, inputs["neighbors"][layer_ind], features, w, radius, config)
    return batch_norm(x, V.current_scope(), config, alpha=0.2)


def _resnetb(layer_ind, inputs, features, radius, fdim, config, strided):
    with variable_scope("conv1"):
        w = nb.weight_variable([int(features.shape[1]), fdim // 2])
        x = batch_norm(nb.conv_ops.unary_convolution(features, w), V.current_scope(), config, alpha=0.2)
    with variable_scope("conv2"):
        w = nb.weight_variable([config.num_kernel_points, int(x.shape[1]), fdim // 2])
        if strided:
            x = nb.KPConv(inputs["points"][layer_ind + 1], inputs["points"][layer_ind], inputs["pools"][layer_ind], x,
                          w, radius, config)
        else:
            x = nb.KPConv(inputs["points"][layer_ind], inputs["points"][layer_ind], inputs["neighbors"][layer_ind], x,
                          w, radius, config)
        x = batch_norm(x, V.current_scope(), config, alpha=0.2)
    with variable_scope("shortcut"):
        shortcut = ind_max_pool(features, inputs["pools"][layer_ind]) if strided else features
        if int(shortcut.shape[1]) != 2 * fdim:
            w = nb.weight_variable([int(shortcut.shape[1]), 2 * fdim])
            shortcut = batch_norm(nb.conv_ops.unary_convolution(shortcut, w), V.current_scope(), config)
    with variable_scope("conv3"):
        w = nb.weight_variable([int(x.shape[1]), 2 * fdim])
        # leaky_relu(batch_norm(conv3) + shortcut) (:343-368)
        return batch_norm(nb.conv_ops.unary_convolution(x, w), V.current_scope(), config, residual=shortcut,
                          alpha=0.2)


def resnetb_block(layer_ind, inputs, features, radius, fdim, config):
    """:321-368."""
    return _resnetb(layer_ind, inputs, features, radius, fdim, config, False)


def resnetb_strided_block(layer_ind, inputs, features, radius, fdim, config):
    """:561-612."""
    return _resnetb(layer_ind, inputs, features, radius, fdim, config, True)


def nearest_upsample_block(layer_ind, inputs, features, radius, fdim, config):
    """:971-979."""
    with variable_scope("nearest_upsample"):
        return closest_pool(features, inputs["upsamples"][layer_ind - 1])


BLOCKS = {
    "unary": unary_block,
    "last_unary": last_unary_block,
    "simple": simple_block,
    "resnetb": resnetb_block,
    "resnetb_strided": resnetb_strided_block,
    "nearest_upsample": nearest_upsample_block,
}


def get_block_ops(block_name):
    if "deformable" in block_name:
        raise NotImplementedError("%s: the deformable blocks have no gradient in d3feat_b200" % block_name)
    if block_name not in BLOCKS:
        raise ValueError("Unknown block name in the architecture definition : " + block_name)
    return BLOCKS[block_name]


def forward(inputs, config):
    """assemble_FCNN_blocks (models/D3Feat.py:5-115) with training = True, under the active ParamStore: the schedule
    of network_blocks.architecture run with the blocks above -> (l2-normalised descriptors [N, 32], scores [N, 1]).
    Updates the moving statistics of every batch norm in place. Before anything runs: ValueError for a static
    (capacity-sized) pyramid or an architecture without a decoder, NotImplementedError for a deformable one."""
    if inputs.get("rows"):
        raise ValueError("training: the inputs are a static (capacity-sized) pyramid; training needs exact shapes "
                         "(pyramid.descriptor_input without static=True)")
    for block in config.architecture:
        get_block_ops(block)
    encoder, decoder = nb.architecture(config)
    if not decoder:
        raise ValueError("training: the architecture has no upsample block, so no decoder")
    F = []
    features = nb.run_blocks(encoder, get_block_ops, inputs, inputs["features"], F, config)
    features = nb.run_blocks(decoder, get_block_ops, inputs, features, F, config)
    return l2_normalize(features), detection_scores(features, inputs["neighbors"][0], inputs["lengths"][0])


def initial_params(config, seed=0):
    """The variables a new run of the reference starts from, {name: float32 array} under the schedule of
    network_blocks.variables (ready for ParamStore):
      weights              weight_variable (models/network_blocks.py:37-41): normal with std sqrt(2 / shape[-1]),
                           redrawn beyond 2 std (tf.truncated_normal), then round(x * 1000) / 1000, in float32
      batch norm           gamma 1, beta 0, moving mean 0, moving variance 1 (tf.layers.batch_normalization); with
                           config.use_batch_norm off the '<scope>/offset' bias, 0 (:162-165)
      offset_conv_*        0 (kernels/convolution_ops.py:327-328)
      kernel_points        kernel_points.load_kernels(1.5 * KP_extent, K, 1, 3, config.fixed_kernel_points): one
                           disposition optimised once for the run, each KPConv with its own rotation and noise
                           (kernels/convolution_ops.py:127-148)
    Draws are counter-based splitmix64 of `seed` (kernel_points.draw), so a seed gives the same bits everywhere; numpy's
    and TF's random streams are not reproduced."""
    from . import kernel_points as kp
    K, fixed = config.num_kernel_points, config.fixed_kernel_points
    D = None
    p = {}
    for i, v in enumerate(nb.variables(config)):
        if v.kind == "weights":
            n = int(np.prod(v.shape))
            e = np.arange(n, dtype=np.uint64) * np.uint64(64)
            z = kp.normal(kp.sub_seed(seed, i), kp.WEIGHTS, e).astype(np.float32)
            for a in range(1, 64):                        # tf.truncated_normal redraws beyond 2 std
                bad = np.nonzero(np.abs(z) > 2)[0]
                if bad.size == 0:
                    break
                z[bad] = kp.normal(kp.sub_seed(seed, i), kp.WEIGHTS, e[bad] + np.uint64(a)).astype(np.float32)
            w = z * np.float32(np.sqrt(2 / v.shape[-1]))
            p[v.name] = (np.round(w * np.float32(1000)) / np.float32(1000)).astype(np.float32).reshape(v.shape)
        elif v.kind == "kernel_points":
            if D is None:
                D = kp.shared_disposition(K, fixed, seed)
            p[v.name] = kp.load_kernels(v.radius, K, 1, 3, fixed, seed=kp.sub_seed(seed, i), disposition=D)[0].astype(
                np.float32)
        elif v.kind == "batch_norm":
            if config.use_batch_norm:
                for name, x in zip(V.ParamStore.bn_names(v.name), (1, 0, 0, 1)):
                    p[name] = np.full(v.shape, x, np.float32)
            else:
                p[v.name + "/offset"] = np.zeros(v.shape, np.float32)
        else:                                             # offset_conv_weights, offset_conv_bias
            p[v.name] = np.zeros(v.shape, np.float32)
    return p


def trainable(store):
    """Mark every 'weights', 'gamma', 'beta' and 'offset' of the ParamStore as requiring grad and return them (in
    name order). Kernel points and moving statistics stay non-trainable."""
    out = []
    for name in sorted(store.t):
        if name.rsplit("/", 1)[-1] in TRAINABLE:
            out.append(store.t[name].requires_grad_(True))
    return out


# ----------------------------------------------------------------------------------------------------
#  loss (models/KPFCNN_model.py:128-188, utils/loss.py)
# ----------------------------------------------------------------------------------------------------

def cdist(a, b):
    """utils/loss.py cdist(metric='euclidean'): sqrt(sum (a_i - b_j)^2 + 1e-12)."""
    return torch.sqrt(((a[:, None, :] - b[None, :, :]) ** 2).sum(-1) + 1e-12)


def d3feat_loss(descriptors, scores, anc_inds, pos_inds, backup_points, config):
    """The training loss of D3Feat for one pair: (loss, desc_loss, det_loss, accuracy, d_pos, d_neg).

    anc_inds / pos_inds: int32 [k] keypoint rows of the stacked batch (drawn with replacement, so they repeat),
    backup_points [N, 3] the stacked points the keypoint distances are measured on. Circle loss (log_scale 25, margins
    0.1 / 1.4, false negatives within config.safe_radius masked), detection loss times config.det_loss_weight, both
    zero (accuracy -1) with fewer than 0.5 * config.keypts_num correspondences, plus the L2 regulariser
    config.weights_decay * sum 1/2 |w|^2 over every 'weights' of the active ParamStore."""
    store = V.current_store()
    if store is None:
        raise RuntimeError("d3feat_loss: no ParamStore active (wrap the call in variables.use_params)")
    k = int(anc_inds.shape[0])
    reg = sum(0.5 * (w * w).sum() for n, w in sorted(store.t.items()) if "weights" in n)
    reg = config.weights_decay * reg
    if k < 0.5 * config.keypts_num:
        zero = torch.zeros((), dtype=_F32, device=descriptors.device)
        return reg + zero, zero, zero, zero - 1.0, zero, zero
    with torch.no_grad():
        anc_pts = backup_points.index_select(0, anc_inds.long())
        keypts_distance = cdist(anc_pts, anc_pts)
    dists = cdist(gather_rows(descriptors, anc_inds), gather_rows(descriptors, pos_inds))
    same = torch.eye(k, dtype=torch.bool, device=dists.device)
    false_negative = (keypts_distance < config.safe_radius) & ~same
    negative = ~same & ~false_negative
    same_f, fn_f = same.to(dists.dtype), false_negative.to(dists.dtype)
    # circle_loss (pos_margin 0.1, neg_margin 1.4)
    furthest_positive = (dists * same_f).amax(1)
    closest_negative = (dists + 1e5 * same_f).amin(1)
    average_negative = (dists * negative.to(dists.dtype)).mean() * k / (k - 1.0)
    diff = furthest_positive - closest_negative
    accuracy = (diff <= 0).to(dists.dtype).sum() / k
    log_scale, pos_margin, neg_margin = 25.0, 0.1, 1.4
    lse_positive = log_scale * (furthest_positive - pos_margin)
    neg = dists + 1e8 * fn_f + 1e8 * same_f
    lse_negative = torch.logsumexp(log_scale * (neg_margin - neg) * torch.clamp_min(neg_margin - neg, 0.0).detach(),
                                   dim=-1)
    desc_loss = (Fn.softplus(lse_positive + lse_negative) / log_scale).mean()
    d_pos, d_neg = furthest_positive.mean(), average_negative
    if config.det_loss_weight != 0:
        # det_loss: its own furthest positive / closest negative (the same values, a second path to dists)
        fp = (dists * same_f).amax(1)
        cn = (dists + 1e5 * same_f).amin(1)
        s = gather_rows(scores, anc_inds) + gather_rows(scores, pos_inds) + 1e-6
        det_loss = config.det_loss_weight * ((fp - cn)[:, None] * s).mean()
    else:
        det_loss = torch.zeros((), dtype=dists.dtype, device=dists.device)
    return desc_loss + det_loss + reg, desc_loss, det_loss, accuracy, d_pos, d_neg


# ----------------------------------------------------------------------------------------------------
#  the update (utils/trainer.py:116-156, 376-381)
# ----------------------------------------------------------------------------------------------------

def learning_rate(config, epoch):
    """The learning rate during epoch `epoch` (0-based) of the reference's trainer: a float32 variable that starts at
    config.learning_rate and, at the end of every epoch e in config.lr_decays, is assigned fl32(lr * fl32(decay))
    (utils/trainer.py:376-381). No lr_decays: no decay."""
    lr = np.float32(config.learning_rate)
    decays = getattr(config, "lr_decays", None) or {}
    for e in range(int(epoch)):
        if e in decays:
            lr = lr * np.float32(decays[e])
    return float(lr)


def _momentum_table(op, vars_, accums, grads):
    """The device table of d3f_momentum_clip_update: int64 [T, 4] = (var, accum, grad, numel), copied from pinned
    memory without a synchronisation. vars_ and accums are updated in place (contiguous, or ValueError); a strided
    grad is read through a contiguous copy. The returned list keeps every tensor the table names alive, so none of its
    addresses can be freed and handed to another tensor while the table is in use. Refused (RuntimeError) while the
    current stream is being captured into a CUDA graph: the graph would copy from a pinned buffer that does not outlive
    the capture."""
    dev, rows, keep = None, [], []
    for i, (v, a, g) in enumerate(zip(vars_, accums, grads)):
        for t, n in ((v, "var"), (a, "accum")):
            if not (torch.is_tensor(t) and t.is_contiguous()):
                raise ValueError("%s: %s[%d] must be a contiguous tensor (it is updated in place)" % (op, n, i))
        v = _lib.tensor_arg(v, "%s: var[%d]" % (op, i), _F32, None, dev)
        dev = v.device
        a = _lib.tensor_arg(a, "%s: accum[%d]" % (op, i), _F32, tuple(v.shape), dev)
        g = _lib.tensor_arg(g, "%s: grad[%d]" % (op, i), _F32, tuple(v.shape), dev)
        keep += [v, a, g]
        rows.append((v.data_ptr(), a.data_ptr(), g.data_ptr(), v.numel()))
    if torch.cuda.is_current_stream_capturing():
        raise RuntimeError("%s: the table of tensor addresses cannot be built during CUDA graph capture; run one eager "
                           "step with the same tensors before capturing" % op)
    host = torch.tensor(rows, dtype=torch.int64).reshape(-1, 4).pin_memory()
    return host.to(dev, non_blocking=True), keep, sum(r[3] for r in rows)


def _momentum_launch(op, table, T, numel, lr, momentum, clip_norm, dev):
    L = _lib.lib()
    ws = _lib.workspace(L.d3f_momentum_clip_workspace_bytes(T, numel), dev)
    _lib.check(L.d3f_momentum_clip_update(_lib.ptr(table), T, numel, float(np.float32(lr)),
                                          float(np.float32(momentum)), float(np.float32(clip_norm)), _lib.ptr(ws),
                                          ws.numel(), _lib.stream()), op)


def momentum_clip_update(vars_, accums, grads, lr, momentum, clip_norm):
    """One update of the reference's trainer for every tensor of the lists, in place (utils/trainer.py:116-156):
    gc = tf.clip_by_norm(g, clip_norm) (none for clip_norm <= 0), accum = accum * momentum + gc, var -= accum * lr.
    The exact contract, with the fp64 block-ordered norm, is oracle/optim_np.py. Two kernels for all tensors, no
    synchronisation. It copies a fresh table of addresses every call, so it cannot be captured in a CUDA graph; a
    MomentumClip step can."""
    op = "momentum_clip_update"
    vars_, accums, grads = list(vars_), list(accums), list(grads)
    if not len(vars_) == len(accums) == len(grads):
        raise ValueError("%s: %d vars, %d accums and %d grads" % (op, len(vars_), len(accums), len(grads)))
    if not vars_:
        return
    table, keep, numel = _momentum_table(op, vars_, accums, grads)
    _momentum_launch("d3f_momentum_clip_update", table, len(vars_), numel, lr, momentum, clip_norm, table.device)
    for v in vars_:
        torch.autograd.graph.increment_version(v)


class MomentumClip:
    """The reference's update: tf.clip_by_norm on each gradient on its own, then tf.train.MomentumOptimizer
    (utils/trainer.py:116-156), as two sm_90a kernels for all parameters together (d3f_momentum_clip_update). It
    differs from torch.optim.SGD + clip_grad_norm_: torch adds 1e-6 to the norm and leaves g alone below the threshold,
    where TF always computes g * c / max(norm, c), which can move g by an ulp; and SGD's momentum applies lr to the
    gradient before the accumulator, not after. The norm is summed in fp64 in fixed blocks (oracle/optim_np.py), so
    every step is bitwise reproducible.

    params: float32 contiguous CUDA tensors on one device (updated in place). state: the accumulators (TF's Momentum
    slots), zero-initialised, one per parameter. lr, momentum, clip_norm are read at every step() (clip_norm <= 0: no
    clipping), rounded to float32. A parameter whose .grad is None is skipped, as TF skips a None gradient. An entry of
    state (or the whole list) may be replaced, e.g. by restored slots, and a parameter's storage may be replaced
    (p.data = ...): the next step() uses the new tensors.

    step() never synchronises. It keeps a device table of the parameters', accumulators' and gradients' addresses and
    rebuilds it (one pinned copy) only when one of them moves or changes size; zero_grad() zeroes the gradients in
    place, so the addresses stay. To capture step() in a CUDA graph, run one eager step() with the same tensors first:
    a step that would rebuild the table during the capture raises RuntimeError. The graph then replays on those
    tensors, with the lr, momentum and clip_norm of the capture."""

    def __init__(self, params, lr, momentum, clip_norm):
        self.params = list(params)
        dev = None
        for i, p in enumerate(self.params):
            if not (torch.is_tensor(p) and p.is_contiguous()):
                raise ValueError("MomentumClip: params[%d] must be a contiguous tensor (it is updated in place)" % i)
            dev = _lib.tensor_arg(p, "MomentumClip: params[%d]" % i, _F32, None, dev).device
        self.lr, self.momentum, self.clip_norm = float(lr), float(momentum), float(clip_norm)
        self.state = [torch.zeros_like(p, memory_format=torch.contiguous_format) for p in self.params]
        self._key, self._table = None, None

    def zero_grad(self):
        """Zero every existing gradient in place (addresses kept)."""
        with torch.no_grad():
            for p in self.params:
                if p.grad is not None:
                    p.grad.zero_()

    def step(self):
        live = [i for i, p in enumerate(self.params) if p.grad is not None]
        if not live:
            return
        if len(self.state) != len(self.params):
            raise ValueError("MomentumClip.step: %d accumulators in state for %d parameters" % (
                len(self.state), len(self.params)))
        triples = [(self.params[i].detach(), self.state[i], self.params[i].grad) for i in live]
        # every address and size the kernel reads or writes through: a moved parameter, accumulator or gradient
        # rebuilds the table
        key = tuple((i,) + tuple((t.data_ptr(), t.numel(), t.is_contiguous()) if torch.is_tensor(t) else (id(t),)
                                 for t in ts) for i, ts in zip(live, triples))
        if key != self._key or not all(g.is_contiguous() for _, _, g in triples):
            self._table = _momentum_table("MomentumClip.step", *zip(*triples))
            self._key = key
        table, _, numel = self._table
        _momentum_launch("d3f_momentum_clip_update", table, len(live), numel, self.lr, self.momentum, self.clip_norm,
                         table.device)
        for i in live:
            torch.autograd.graph.increment_version(self.params[i])
