"""Record one real training step op by op, and replay each op against the direct entry points and float64.

    rec = Recorder()
    with rec.patched(), use_params(store):
        desc, scores = training.forward(inputs, config)
        loss = training.d3feat_loss(desc, scores, anc, pos, backup, config)[0]
    loss.backward()

For the duration of the `with`, the module attributes the training blocks call are wrapped: training.batch_norm,
ind_max_pool, closest_pool, gather_rows, l2_normalize and detection_scores, and convolution_ops.KPConv_ops and
unary_convolution. A call is recorded only when its output is a graph node (the no-grad forward that _UnaryFn and
_KPConvFn run inside their own forward is not). Each record keeps the op's inputs (detached), its GPU output, and the
gradient that reaches that output (out.register_hook: the summed upstream gradient the Function's backward receives).

direct(r) recomputes the op's gradients with the direct entry points fed the recorded gradient; reference(h) gives
their float64 (ref, mag, alt) from the record moved to the host. With weights_decay = 0 every parameter is used by
exactly one op, so its .grad must equal that op's recomputed weight / gamma / beta gradient bit for bit
(param_grads(r)).

Only tests/ import this module.
"""
import contextlib

import numpy as np
import torch

import _kpconv_grad_oracle as og
import _training_oracle as ot

KINDS = ("kpconv", "kpconv_strided", "unary", "bn", "pool", "gather", "l2", "det")


def expected_calls(config):
    """Calls per op kind of one training.forward + d3feat_loss, walked from config.architecture and the channel
    counts (kpconv_strided counts the strided KPConvs among kpconv)."""
    n = dict.fromkeys(KINDS, 0)
    fdim, c = config.first_features_dim, config.in_features_dim
    F = []
    arch = list(config.architecture)
    up = next(i for i, b in enumerate(arch) if "upsample" in b)

    def block(b, c, fdim):
        if b in ("unary", "simple"):
            n["unary" if b == "unary" else "kpconv"] += 1
            n["bn"] += 1
            return fdim
        if b == "last_unary":
            n["unary"] += 1
            return 32
        if b in ("resnetb", "resnetb_strided"):
            n["unary"] += 2
            n["kpconv"] += 1
            n["bn"] += 3
            if b == "resnetb_strided":
                n["kpconv_strided"] += 1
                n["pool"] += 1
            if c != 2 * fdim:
                n["unary"] += 1
                n["bn"] += 1
            return 2 * fdim
        if b == "nearest_upsample":
            n["gather"] += 1
            return c
        raise ValueError(b)
    for b in arch[:up]:
        if "strided" in b:
            F.append(c)
        c = block(b, c, fdim)
        if "strided" in b:
            fdim *= 2
    fdim = config.first_features_dim * 2 ** (config.num_layers - 1)
    for b in arch[up:]:
        c = block(b, c, fdim)
        if "upsample" in b:
            fdim //= 2
            c += F.pop()
    n["l2"] += 1
    n["det"] += 1
    n["gather"] += 4 if config.det_loss_weight != 0 else 2       # descriptors and scores at the anchors / positives
    return n


def counts(calls):
    n = dict.fromkeys(KINDS, 0)
    for r in calls:
        n[r["kind"]] += 1
        n["kpconv_strided"] += int(r.get("strided", False))
    return n


class Recorder:
    def __init__(self):
        self.calls = []

    def _keep(self, kind, out, **rec):
        if not (torch.is_tensor(out) and out.requires_grad):
            return out
        rec.update(kind=kind, index=len(self.calls), out=out.detach(), grad_out=None)

        def hook(g, rec=rec):
            rec["grad_out"] = g.detach().clone()
        out.register_hook(hook)
        self.calls.append(rec)
        return out

    @contextlib.contextmanager
    def patched(self):
        from d3feat_b200 import convolution_ops as co, training as T, variables as V
        orig = {(m, n): getattr(m, n) for m, n in (
            (T, "batch_norm"), (T, "ind_max_pool"), (T, "closest_pool"), (T, "gather_rows"), (T, "l2_normalize"),
            (T, "detection_scores"), (co, "KPConv_ops"), (co, "unary_convolution"))}
        keep = self._keep

        def batch_norm(x, scope, config, residual=None, alpha=None):
            store = V.current_store()
            if config.use_batch_norm:
                pre = scope + "/batch_normalization/"
                gamma, beta = store.get(pre + "gamma"), store.get(pre + "beta")
                mm, mv = store.get(pre + "moving_mean"), store.get(pre + "moving_variance")
                before = (mm.detach().clone(), mv.detach().clone())
            else:
                gamma, beta, mm, mv, before = None, store.get(scope + "/offset"), None, None, (None, None)
            out = orig[T, "batch_norm"](x, scope, config, residual, alpha)
            return keep("bn", out, scope=scope, x=x.detach(), x_grad=x.requires_grad,
                        residual=None if residual is None else residual.detach(), gamma=gamma, beta=beta,
                        moving_before=before,
                        moving_after=(None, None) if mm is None else (mm.detach().clone(), mv.detach().clone()),
                        momentum=float(config.batch_norm_momentum), alpha=alpha)

        def ind_max_pool(x, inds):
            return keep("pool", orig[T, "ind_max_pool"](x, inds), x=x.detach(), inds=inds)

        def closest_pool(x, inds):
            return keep("gather", orig[T, "closest_pool"](x, inds), inds=inds[:, 0].contiguous(), n_rows=x.shape[0])

        def gather_rows(x, inds):
            return keep("gather", orig[T, "gather_rows"](x, inds), inds=inds, n_rows=x.shape[0])

        def l2_normalize(x):
            return keep("l2", orig[T, "l2_normalize"](x), x=x.detach())

        def detection_scores(x, neighbors, lengths):
            return keep("det", orig[T, "detection_scores"](x, neighbors, lengths), x=x.detach(), neighbors=neighbors,
                        lengths=lengths)

        def KPConv_ops(q, s, idx, f, Kp, W, extent, influence, mode, **kw):
            out = orig[co, "KPConv_ops"](q, s, idx, f, Kp, W, extent, influence, mode, **kw)
            if any(v is not None for v in kw.values()):
                raise AssertionError("KPConv_ops: the training blocks pass no epilogue, bias, order or row counts")
            return keep("kpconv", out, q=q, s=s, idx=idx, f=f.detach(), f_grad=f.requires_grad, Kp=Kp, W=W,
                        extent=float(extent), influence=influence, mode=mode, strided=q.data_ptr() != s.data_ptr())

        def unary_convolution(features, K_values, **kw):
            out = orig[co, "unary_convolution"](features, K_values, **kw)
            if any(v is not None for v in kw.values()):
                raise AssertionError("unary_convolution: the training blocks pass no epilogue, residual or rows")
            return keep("unary", out, x=features.detach(), x_grad=features.requires_grad, W=K_values)

        new = dict(batch_norm=batch_norm, ind_max_pool=ind_max_pool, closest_pool=closest_pool,
                   gather_rows=gather_rows, l2_normalize=l2_normalize, detection_scores=detection_scores,
                   KPConv_ops=KPConv_ops, unary_convolution=unary_convolution)
        for (m, n) in orig:
            setattr(m, n, new[n])
        try:
            yield self
        finally:
            for (m, n), fn in orig.items():
                setattr(m, n, fn)


# ----------------------------------------------------------------------------------------------------
#  replay
# ----------------------------------------------------------------------------------------------------

def direct(r):
    """The op's gradients (and the training-only forward values) from the direct entry points, fed r's grad_out:
    {name: tensor}. Also checks that the recomputed forward of batch norm gives the recorded bits."""
    from d3feat_b200 import convolution_ops as co, training as T
    k, g = r["kind"], r["grad_out"]
    if k == "kpconv":
        df, dW = co.kpconv_backward(r["q"], r["s"], r["idx"], r["f"], r["Kp"], r["W"].detach(), r["extent"],
                                    r["influence"], r["mode"], g, features_grad=r["f_grad"])
        return dict(dW=dW) if df is None else dict(df=df, dW=dW)
    if k == "unary":
        dx, dW = co.unary_backward(r["x"], r["W"].detach(), g, features_grad=r["x_grad"])
        return dict(dW=dW) if dx is None else dict(dx=dx, dW=dW)
    if k == "bn":
        gamma = None if r["gamma"] is None else r["gamma"].detach()
        mm, mv = (None if t is None else t.clone() for t in r["moving_before"])
        out, mean, invstd = T.batch_norm_forward(r["x"], gamma, r["beta"].detach(), mm, mv, r["momentum"],
                                                 r["residual"], r["alpha"])
        assert torch.equal(out, r["out"]), "%s: the recomputed batch norm differs from the step's" % r["scope"]
        res = dict(out=out)
        if gamma is not None:
            assert torch.equal(mm, r["moving_after"][0]) and torch.equal(mv, r["moving_after"][1]), r["scope"]
            res.update(mean=mean, invstd=invstd, moving_mean=mm, moving_var=mv)
        dx, dres, dgamma, dbeta = T.batch_norm_backward(r["x"], out, g, gamma, mean, invstd, r["alpha"],
                                                        residual_grad=r["residual"] is not None)
        res.update(dx=dx, dbeta=dbeta)
        if dres is not None:
            res["dres"] = dres
        if dgamma is not None:
            res["dgamma"] = dgamma
        return res
    if k == "pool":
        return dict(dx=T.ind_max_pool_backward(r["x"], r["inds"], r["out"], g))
    if k == "gather":
        return dict(dx=T.gather_rows_backward(r["inds"], g, r["n_rows"]))
    if k == "l2":
        return dict(dx=T.l2_normalize_backward(r["x"], g))
    if k == "det":
        return dict(dx=T.detection_scores_backward(r["x"], r["neighbors"], r["lengths"], g))
    raise ValueError(k)


def param_grads(r, d):
    """[(parameter, its gradient from this op)] for the trainable tensors op r reads."""
    if r["kind"] in ("kpconv", "unary"):
        return [(r["W"], d["dW"])]
    if r["kind"] == "bn":
        return ([] if r["gamma"] is None else [(r["gamma"], d["dgamma"])]) + [(r["beta"], d["dbeta"])]
    return []


def host(r, d):
    """The record and its direct gradients as numpy arrays (parameters as values)."""
    cv = lambda v: v.detach().cpu().numpy() if torch.is_tensor(v) else v
    h = {k: (tuple(cv(t) for t in v) if isinstance(v, tuple) else cv(v)) for k, v in r.items()}
    h["gpu"] = {k: cv(v) for k, v in d.items()}
    return h


def reference(h):
    """{name: (ref, mag, alt)} in float64 for every name of h["gpu"]; for "det", h["ambiguous"] is set to the rows
    the oracle marked."""
    k, g = h["kind"], h["grad_out"]
    if k == "kpconv":
        args = (h["q"], h["s"], h["idx"], h["f"], h["Kp"], h["W"], h["extent"], h["influence"], h["mode"], g)
        res = dict(dW=og.kpconv_weights_grad(*args))
        if "df" in h["gpu"]:
            res["df"] = og.kpconv_features_grad(*args)
        return res
    if k == "unary":
        res = dict(dW=og.unary_weights_grad(h["x"], h["W"], g))
        if "dx" in h["gpu"]:
            res["dx"] = og.unary_features_grad(h["x"], h["W"], g)
        return res
    if k == "bn":
        decay = float(np.float32(1.0 - h["momentum"]))
        fw = ot.batch_norm_train_forward_ref(h["x"], h["gamma"], h["beta"], h["residual"], h["alpha"],
                                             h["moving_before"][0], h["moving_before"][1], decay)
        bw = ot.batch_norm_train_grads(h["x"], h["gpu"]["out"], g, h["gamma"], h["alpha"],
                                       mean=h["gpu"].get("mean"), invstd=h["gpu"].get("invstd"))
        both = dict(fw, **bw)
        return {n: both[n] + (None,) for n in h["gpu"]}
    if k == "pool":
        return dict(dx=ot.ind_max_pool_grad(h["x"], h["inds"], g) + (None,))
    if k == "gather":
        return dict(dx=ot.gather_rows_grad(h["inds"], g, h["n_rows"]) + (None,))
    if k == "l2":
        return dict(dx=ot.l2_normalize_grad(h["x"], g) + (None,))
    if k == "det":
        ref, mag, alt, amb = ot.detection_scores_grad(h["x"], h["neighbors"], h["lengths"], g)
        h["ambiguous"] = amb
        return dict(dx=(ref, mag, alt))
    raise ValueError(k)
