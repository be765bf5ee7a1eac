"""Mirror of models/network_blocks.py (the blocks the D3Feat encoder/decoder uses) on top of the fused ops.

Same function names and signatures as the reference so that architecture lists and call sites carry over:
  weight_variable(shape)                          network_blocks.py:37-41  (restored from the ParamStore)
  ind_max_pool(x, inds) / closest_pool(x, inds)   :51-66 / :69-83
  KPConv / KPConv_deformable(q, s, idx, features, K_values, radius, config)   :86-124
  batch_norm(x, use_batch_norm, momentum, training) / leaky_relu(features, alpha)   :149-165 / :185-186
  unary_block, last_unary_block, simple_block, resnetb_block, resnetb_strided_block,
  resnetb_deformable_block, resnetb_deformable_strided_block, nearest_upsample_block   :194-244, 321-368,
                                                                       424-471, 561-612, 672-723, 971-979
  get_block_ops(block_name)                       :982-1042
  assemble_CNN_blocks(inputs, config, dropout_prob)   :1052-1118  (the ENCODER)
  assemble_FCNN_blocks / assemble_FCNN_decoder    models/D3Feat.py:5-115

The blocks are inference only (training = dropout_prob < 0.99 must be False, like utils/tester.py:199 feeds 1.0):
batch norm uses the moving statistics and is folded, together with the LeakyReLU and the residual add, into the
epilogue of the producing kernel. Parameters are looked up in the active ParamStore under the reference's
variable-scope names. The schedule of scopes, radii and widths (architecture, run_blocks) is shared with the training
blocks (training.forward); the variables it creates (variables) are shared by the seeded parameters
(synth.make_params) and the initial parameters of a new run (training.initial_params).
"""
from collections import namedtuple

import torch

from . import _lib
from . import convolution_ops as conv_ops
from . import variables as V
from .variables import variable_scope


# ----------------------------------------------------------------------------------------------------
#  utilities
# ----------------------------------------------------------------------------------------------------

def weight_variable(shape):
    """The reference draws N(0, sqrt(2/shape[-1])) rounded to 1e-3 (:37-41) and the Saver overwrites it at
    test time; here the value comes from the ParamStore ('<scope>/weights')."""
    store = V.current_store()
    if store is None:
        raise RuntimeError("weight_variable: no ParamStore active (wrap the call in variables.use_params)")
    w = store.get(V.scoped("weights"))
    if tuple(w.shape) != tuple(int(s) for s in shape):
        raise ValueError("weights '%s' have shape %s, block expects %s" % (V.scoped("weights"), tuple(w.shape), tuple(shape)))
    return w


def _rows(inputs, level):
    """Device scalar with the actual row count of pyramid level `level` when the pyramid was built in its static
    (capacity-sized, sync-free) form, else None: the tensors then have exact shapes."""
    rows = inputs.get("rows") if isinstance(inputs, dict) else None
    if not rows or level >= len(rows):
        return None
    return rows[level]


_F32, _I32 = torch.float32, torch.int32


def _pool_args(op, x, inds, rows_x, rows_out):
    conv_ops._refuse_op_grad(op, x)
    x = _lib.tensor_arg(x, op + ": x", _F32, (None, None))
    inds = _lib.tensor_arg(inds, op + ": inds", _I32, (None, None), x.device)
    return (x, inds, _lib.row_count_arg(rows_x, op + ": rows_x", x.device),
            _lib.row_count_arg(rows_out, op + ": rows_out", x.device))


def ind_max_pool(x, inds, *, rows_x=None, rows_out=None):
    """:51-66 -- max over the pooled rows; shadow index -> column-wise minimum of x."""
    x, inds, rows_x, rows_out = _pool_args("ind_max_pool", x, inds, rows_x, rows_out)
    N1, C = x.shape
    N2, H = inds.shape
    L = _lib.lib()
    ws = _lib.workspace(L.d3f_ind_max_pool_workspace_bytes(C), x.device)
    out = torch.empty((N2, C), dtype=torch.float32, device=x.device)
    _lib.check(L.d3f_ind_max_pool(_lib.ptr(x), _lib.ptr(inds), N1, N2, H, C, _lib.ptr(out), _lib.ptr(ws), ws.numel(),
                                  _lib.stream(), _lib.ptr(rows_x), _lib.ptr(rows_out)), "d3f_ind_max_pool")
    return out


def closest_pool(x, inds, *, rows_x=None, rows_out=None):
    """:69-83 -- features of the closest pooled point (first index column); shadow -> zeros."""
    x, inds, rows_x, rows_out = _pool_args("closest_pool", x, inds, rows_x, rows_out)
    N1, C = x.shape
    N2, H = inds.shape
    out = torch.empty((N2, C), dtype=torch.float32, device=x.device)
    _lib.check(_lib.lib().d3f_closest_pool(_lib.ptr(x), _lib.ptr(inds), N1, N2, H, C, _lib.ptr(out), _lib.stream(),
                                           _lib.ptr(rows_x), _lib.ptr(rows_out)), "d3f_closest_pool")
    return out


def _affine_leaky(x, scale, shift, residual, alpha, rows=None):
    op = "affine_leaky"
    x = _lib.tensor_arg(x, op + ": x", _F32, (None, None))
    N, C = x.shape
    scale = _lib.tensor_arg(scale, op + ": scale", _F32, (C,), x.device, optional=True)
    shift = _lib.tensor_arg(shift, op + ": shift", _F32, (C,), x.device, optional=True)
    residual = _lib.tensor_arg(residual, op + ": residual", _F32, (N, C), x.device, optional=True)
    rows = _lib.row_count_arg(rows, op + ": rows", x.device)
    out = torch.empty_like(x)
    _lib.check(_lib.lib().d3f_affine_leaky(_lib.ptr(x), N, C, _lib.ptr(scale), _lib.ptr(shift), _lib.ptr(residual),
                                           -1.0 if alpha is None else float(alpha), _lib.ptr(out), _lib.stream(),
                                           _lib.ptr(rows)), "d3f_affine_leaky")
    return out


def _bn_affine(use_batch_norm):
    """(scale, shift) of the current scope's inference batch norm (:149-160), or scale 1 and the 'offset' bias without
    batch norm (:162-165)."""
    store, scope = V.current_store(), V.current_scope()
    if use_batch_norm:
        return store.bn_affine(scope)
    shift = store.bn_variables(scope, False)[1]
    return torch.ones_like(shift), shift


def _bn_epilogue(config, alpha):
    """(scale, shift, alpha): the current scope's batch norm and LeakyReLU as a kernel epilogue."""
    return _bn_affine(config.use_batch_norm) + (alpha,)


def batch_norm(x, use_batch_norm=True, momentum=0.99, training=True):
    """:149-165, inference form only (moving statistics, epsilon 1e-6)."""
    if training:
        raise NotImplementedError("d3feat_b200 implements the inference path (training = dropout_prob < 0.99 is False)")
    return _affine_leaky(x, *_bn_affine(use_batch_norm), None, None)


def leaky_relu(features, alpha=0.2):
    """:185-186."""
    return _affine_leaky(features, None, None, None, alpha)


def _order(inputs, layer_ind):
    orders = inputs.get("orders") if isinstance(inputs, dict) else None
    if not orders or layer_ind >= len(orders):
        return None
    o = orders[layer_ind]
    return o if (o is not None and o.numel() > 0) else None


def KPConv(query_points, support_points, neighbors_indices, features, K_values, radius, config, *, epilogue=None,
           query_order=None, rows_q=None, rows_s=None):
    """:86-103."""
    extent = config.KP_extent * radius / config.density_parameter
    return conv_ops.KPConv(query_points, support_points, neighbors_indices, features, K_values,
                           fixed=config.fixed_kernel_points, KP_extent=extent, KP_influence=config.KP_influence,
                           aggregation_mode=config.convolution_mode, epilogue=epilogue, query_order=query_order,
                           rows_q=rows_q, rows_s=rows_s)


def KPConv_deformable(query_points, support_points, neighbors_indices, features, K_values, radius, config, *,
                      epilogue=None, query_order=None, rows_q=None, rows_s=None):
    """:106-124."""
    extent = config.KP_extent * radius / config.density_parameter
    return conv_ops.KPConv_deformable(query_points, support_points, neighbors_indices, features, K_values,
                                      fixed=config.fixed_kernel_points, KP_extent=extent,
                                      KP_influence=config.KP_influence, aggregation_mode=config.convolution_mode,
                                      modulated=config.modulated, epilogue=epilogue, query_order=query_order,
                                      rows_q=rows_q, rows_s=rows_s)


# ----------------------------------------------------------------------------------------------------
#  blocks  (signature: layer_ind, inputs, features, radius, fdim, config, training)
# ----------------------------------------------------------------------------------------------------

def _no_training(training):
    if training:
        raise NotImplementedError("d3feat_b200 implements the inference path only")


def last_unary_block(layer_ind, inputs, features, radius, fdim, config, training):
    """:194-205."""
    w = weight_variable([int(features.shape[1]), 32])
    return conv_ops.unary_convolution(features, w, rows=_rows(inputs, layer_ind))


def unary_block(layer_ind, inputs, features, radius, fdim, config, training):
    """:207-219 -- 1x1 conv + BN + LeakyReLU (one kernel)."""
    _no_training(training)
    w = weight_variable([int(features.shape[1]), fdim])
    return conv_ops.unary_convolution(features, w, epilogue=_bn_epilogue(config, 0.2), rows=_rows(inputs, layer_ind))


def simple_block(layer_ind, inputs, features, radius, fdim, config, training):
    """:222-244."""
    _no_training(training)
    w = weight_variable([config.num_kernel_points, int(features.shape[1]), fdim])
    r0 = _rows(inputs, layer_ind)
    return KPConv(inputs["points"][layer_ind], inputs["points"][layer_ind], inputs["neighbors"][layer_ind], features,
                  w, radius, config, epilogue=_bn_epilogue(config, 0.2), query_order=_order(inputs, layer_ind),
                  rows_q=r0, rows_s=r0)


def _resnetb(layer_ind, inputs, features, radius, fdim, config, training, strided, deformable):
    _no_training(training)
    conv = KPConv_deformable if deformable else KPConv
    r_in = _rows(inputs, layer_ind)                                   # rows of this level
    r_out = _rows(inputs, layer_ind + 1) if strided else r_in         # rows the block produces
    with variable_scope("conv1"):
        w = weight_variable([int(features.shape[1]), fdim // 2])
        x = conv_ops.unary_convolution(features, w, epilogue=_bn_epilogue(config, 0.2), rows=r_in)
    with variable_scope("conv2"):
        w = weight_variable([config.num_kernel_points, int(x.shape[1]), fdim // 2])
        if strided:
            x = conv(inputs["points"][layer_ind + 1], inputs["points"][layer_ind], inputs["pools"][layer_ind], x, w,
                     radius, config, epilogue=_bn_epilogue(config, 0.2), rows_q=r_out, rows_s=r_in)
        else:
            x = conv(inputs["points"][layer_ind], inputs["points"][layer_ind], inputs["neighbors"][layer_ind], x, w,
                     radius, config, epilogue=_bn_epilogue(config, 0.2), query_order=_order(inputs, layer_ind),
                     rows_q=r_in, rows_s=r_in)
    pair = None
    with variable_scope("shortcut"):
        shortcut = (ind_max_pool(features, inputs["pools"][layer_ind], rows_x=r_in, rows_out=r_out) if strided
                    else features)
        if int(shortcut.shape[1]) != 2 * fdim:
            w_s = weight_variable([int(shortcut.shape[1]), 2 * fdim])
            pair = (w_s, _bn_epilogue(config, None)[:2])
    with variable_scope("conv3"):
        w = weight_variable([int(x.shape[1]), 2 * fdim])
        if pair is not None:
            # conv3 + BN, shortcut unary + BN, add, LeakyReLU (:343-368) as one GEMM over the concatenated K
            return conv_ops.unary_pair_convolution(x, w, _bn_epilogue(config, None)[:2], shortcut, pair[0], pair[1],
                                                   0.2, rows=r_out)
        # conv3 + BN + shortcut add + LeakyReLU in one kernel
        return conv_ops.unary_convolution(x, w, epilogue=_bn_epilogue(config, 0.2), residual=shortcut, rows=r_out)


def resnetb_block(layer_ind, inputs, features, radius, fdim, config, training):
    """:321-368."""
    return _resnetb(layer_ind, inputs, features, radius, fdim, config, training, False, False)


def resnetb_strided_block(layer_ind, inputs, features, radius, fdim, config, training):
    """:561-612."""
    return _resnetb(layer_ind, inputs, features, radius, fdim, config, training, True, False)


def resnetb_deformable_block(layer_ind, inputs, features, radius, fdim, config, training):
    """:424-471."""
    return _resnetb(layer_ind, inputs, features, radius, fdim, config, training, False, True)


def resnetb_deformable_strided_block(layer_ind, inputs, features, radius, fdim, config, training):
    """:672-723."""
    return _resnetb(layer_ind, inputs, features, radius, fdim, config, training, True, True)


def nearest_upsample_block(layer_ind, inputs, features, radius, fdim, config, training):
    """:971-979."""
    with variable_scope("nearest_upsample"):
        return closest_pool(features, inputs["upsamples"][layer_ind - 1], rows_x=_rows(inputs, layer_ind),
                            rows_out=_rows(inputs, layer_ind - 1))


def get_block_ops(block_name):
    """:982-1042 (the blocks reachable from the D3Feat / KPConv-deformable architectures)."""
    table = {
        "unary": unary_block,
        "last_unary": last_unary_block,
        "simple": simple_block,
        "resnetb": resnetb_block,
        "resnetb_deformable": resnetb_deformable_block,
        "resnetb_strided": resnetb_strided_block,
        "resnetb_deformable_strided": resnetb_deformable_strided_block,
        "nearest_upsample": nearest_upsample_block,
    }
    if block_name not in table:
        raise ValueError("Unknown block name in the architecture definition : " + block_name)
    return table[block_name]


# ----------------------------------------------------------------------------------------------------
#  architectures
# ----------------------------------------------------------------------------------------------------

# One block of the schedule: its name, pyramid layer, variable scope, radius and width (fdim). skip: the running
# features join the skip list F before the block; concat: F[layer - 1] is concatenated to the block's output.
Step = namedtuple("Step", "block layer scope radius fdim skip concat")


def architecture(config):
    """The schedule of config.architecture as (encoder, decoder), two lists of Steps: the walk of assemble_CNN_blocks
    (models/network_blocks.py:1052-1118) and of the decoder loop of models/D3Feat.py:15-63, which starts at the first
    upsample block (no decoder without one). Scopes are 'layer_{l}/{block}_{i}' without '_deformable' and
    'uplayer_{l}/{block}_{i}'. Radius (from first_subsampling_dl * density_parameter) and fdim (from first_features_dim)
    double after every pool / strided block; the decoder starts them at the deepest layer and halves them after every
    upsample block. The inference blocks, training.forward and synth.make_params all walk this one schedule."""
    arch = list(config.architecture)
    start = next((i for i, b in enumerate(arch) if "upsample" in b), len(arch))
    r0, f0 = config.first_subsampling_dl * config.density_parameter, config.first_features_dim
    encoder, decoder = [], []
    layer, r, fdim, i = 0, r0, f0, 0
    for block in arch[:start]:
        down = "pool" in block or "strided" in block
        scope = "layer_{:d}/{:s}_{:d}".format(layer, block.replace("_deformable", ""), i)
        encoder.append(Step(block, layer, scope, r, fdim, down or "global" in block, False))
        layer, r, fdim, i = (layer + 1, r * 2, fdim * 2, 0) if down else (layer, r, fdim, i + 1)
    layer = config.num_layers - 1
    r, fdim, i = r0 * 2 ** layer, f0 * 2 ** layer, 0
    for block in arch[start:]:
        up = "upsample" in block
        decoder.append(Step(block, layer, "uplayer_{:d}/{:s}_{:d}".format(layer, block, i), r, fdim, False, up))
        layer, r, fdim, i = (layer - 1, r * 0.5, fdim // 2, 0) if up else (layer, r, fdim, i + 1)
    return encoder, decoder


# One variable of the schedule: its name (for kind "batch_norm" the scope of the batch norm's variables), shape and
# kind: "weights", "kernel_points" (radius: the KPConv's 1.5 * KP_extent), "batch_norm" (shape (width,)),
# "offset_conv_weights" or "offset_conv_bias".
Variable = namedtuple("Variable", "name shape kind radius")


def variables(config):
    """The model variables of architecture(config), in creation order: what the blocks of :194-723 and
    models/D3Feat.py:15-63 create under their scopes. synth.make_params and training.initial_params both fill this one
    schedule."""
    K, cin, skip_dims, out = config.num_kernel_points, config.in_features_dim, [], []
    encoder, decoder = architecture(config)

    def add(name, shape, kind, radius=None):
        out.append(Variable(name, tuple(int(x) for x in shape), kind, radius))

    for step in encoder:
        block, scope, fdim = step.block, step.scope, step.fdim
        if step.skip:
            skip_dims.append(cin)
        radius = 1.5 * config.KP_extent * step.radius / config.density_parameter
        if block == "simple":
            add(scope + "/weights", (K, cin, fdim), "weights")
            add(scope + "/kernel_points", (K, 3), "kernel_points", radius)
            add(scope, (fdim,), "batch_norm")
            cin = fdim
        elif block.startswith("resnetb"):
            mid = fdim // 2
            add(scope + "/conv1/weights", (cin, mid), "weights")
            add(scope + "/conv1", (mid,), "batch_norm")
            add(scope + "/conv2/weights", (K, mid, mid), "weights")
            add(scope + "/conv2/kernel_points", (K, 3), "kernel_points", radius)
            add(scope + "/conv2", (mid,), "batch_norm")
            if "deformable" in block:
                od = (4 if config.modulated else 3) * K
                add(scope + "/conv2/offset_conv_weights", (K, mid, od), "offset_conv_weights")
                add(scope + "/conv2/offset_conv_bias", (od,), "offset_conv_bias")
            add(scope + "/conv3/weights", (mid, 2 * fdim), "weights")
            add(scope + "/conv3", (2 * fdim,), "batch_norm")
            if cin != 2 * fdim:
                add(scope + "/shortcut/weights", (cin, 2 * fdim), "weights")
                add(scope + "/shortcut", (2 * fdim,), "batch_norm")
            cin = 2 * fdim
        else:
            raise ValueError("Unknown block name in the architecture definition : " + block)
    for step in decoder:
        if step.block == "unary":
            add(step.scope + "/weights", (cin, step.fdim), "weights")
            add(step.scope, (step.fdim,), "batch_norm")
            cin = step.fdim
        elif step.block == "last_unary":
            add(step.scope + "/weights", (cin, 32), "weights")
            cin = 32
        if step.concat:
            cin += skip_dims[step.layer - 1]
    return out


def run_blocks(steps, block_ops, inputs, features, F, config, *args):
    """Run `steps` of architecture(config) on `features`, each under its variable scope, as
    block_ops(step.block)(layer, inputs, features, radius, fdim, config, *args). The running features are appended to
    F before a step with .skip; F[layer - 1] is concatenated to the output of one with .concat. Returns the last
    features."""
    for s in steps:
        if s.skip:
            F.append(features)
        with variable_scope(s.scope):
            features = block_ops(s.block)(s.layer, inputs, features, s.radius, s.fdim, config, *args)
        if s.concat:
            features = torch.cat((features, F[s.layer - 1]), dim=1)
    return features


def assemble_CNN_blocks(inputs, config, dropout_prob):
    """:1052-1118 -- the KPFCNN encoder. Returns F, the list of per-level skip features with the final features as
    the last entry."""
    F = []
    features = run_blocks(architecture(config)[0], get_block_ops, inputs, inputs["features"], F, config,
                          dropout_prob < 0.99)
    return F + [features]


def detection_scores(features, neighbors, lengths, *, rows=None):
    """Detection branch of models/D3Feat.py:67-115 on the decoder output BEFORE l2 normalisation: per-cloud max
    normalisation, softplus(x - mean over the non-zero neighbours), channel-max ratio, max over channels -> [N, 1].
    The reference hard-codes two clouds per batch (anchor || positive); here any number of stacked clouds."""
    op = "detection_scores"
    x = _lib.tensor_arg(features, op + ": features", _F32, (None, None))
    nbr = _lib.tensor_arg(neighbors, op + ": neighbors", _I32, (x.shape[0], None), x.device)
    lens = _lib.tensor_arg(lengths, op + ": lengths", _I32, (None,), x.device)
    rows = _lib.row_count_arg(rows, op + ": rows", x.device)
    N, D = int(x.shape[0]), int(x.shape[1])
    B, H = int(lens.shape[0]), int(nbr.shape[1])
    out = torch.empty((N, 1), dtype=torch.float32, device=x.device)
    lib = _lib.lib()
    ws = _lib.workspace(lib.d3f_detection_scores_workspace_bytes(N, B), x.device)
    _lib.check(lib.d3f_detection_scores(_lib.ptr(x), _lib.ptr(nbr), _lib.ptr(lens), B, N, H, D, _lib.ptr(out),
                                        _lib.ptr(ws), ws.numel(), _lib.stream(), _lib.ptr(rows)),
               "d3f_detection_scores")
    return out


def l2_normalize(features, *, rows=None):
    """models/D3Feat.py:65 -- x * rsqrt(max(sum x^2, 1e-10)) per row."""
    x = _lib.tensor_arg(features, "l2_normalize: features", _F32, (None, None))
    rows = _lib.row_count_arg(rows, "l2_normalize: rows", x.device)
    out = torch.empty_like(x)
    _lib.check(_lib.lib().d3f_l2_normalize(_lib.ptr(x), x.shape[0], x.shape[1], 1e-10, _lib.ptr(out), _lib.stream(),
                                           _lib.ptr(rows)), "d3f_l2_normalize")
    return out


def assemble_FCNN_blocks(inputs, config, dropout_prob=1.0):
    """models/D3Feat.py:5-115 in one call: encoder + decoder -> (l2-normalised descriptors [N,32], scores [N,1])."""
    F = assemble_CNN_blocks(inputs, config, dropout_prob)
    return assemble_FCNN_decoder(inputs, config, F, dropout_prob, with_scores=True)


def assemble_FCNN_decoder(inputs, config, F, dropout_prob=1.0, with_scores=False):
    """models/D3Feat.py:15-65 -- decoder loop + l2-normalised 32-d descriptors; with_scores=True also runs the
    detection branch (:67-115) and returns (descriptors, scores). ValueError for an architecture without a decoder."""
    decoder = architecture(config)[1]
    if not decoder:
        raise ValueError("assemble_FCNN_decoder: the architecture has no upsample block, so no decoder")
    features = run_blocks(decoder, get_block_ops, inputs, F[-1], F, config, dropout_prob < 0.99)
    out = l2_normalize(features, rows=_rows(inputs, 0))
    if with_scores:
        return out, detection_scores(features, inputs["neighbors"][0], inputs["lengths"][0], rows=_rows(inputs, 0))
    return out
