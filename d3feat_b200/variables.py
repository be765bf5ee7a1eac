"""Minimal stand-in for TF1 variable scopes: the reference blocks create their weights with
`weight_variable(shape)` / `tf.Variable(..., name='kernel_points')` under nested `tf.variable_scope`s and, at
test time, a Saver restores them by name (utils/tester.py:143-162). Here the restored checkpoint is a dict
{scoped name: array}; the mirrored blocks look their parameters up under the same names."""
import contextlib
import threading

import numpy as np
import torch

from . import _lib

# The active store and scope are per host thread: two threads running two models must not see each other's scopes
# (every library call releases the GIL, so their `use_params` / `variable_scope` blocks interleave).
class _ThreadState(threading.local):
    def __init__(self):
        self.scope = []
        self.store = None


_state = _ThreadState()


class ParamStore:
    """Device-resident parameters keyed by the reference's variable names (e.g.
    'layer_1/resnetb_0/conv2/weights', '.../kernel_points', '.../batch_normalization/gamma')."""

    def __init__(self, params, device):
        self.device = torch.device(device)
        self.t = {}
        for k, v in params.items():
            a = np.ascontiguousarray(np.asarray(v, dtype=np.float32))
            self.t[k] = torch.from_numpy(a).to(self.device)
        self._bn = {}

    def __contains__(self, name):
        return name in self.t

    def __len__(self):
        return len(self.t)

    def get(self, name):
        try:
            return self.t[name]
        except KeyError:
            raise KeyError("variable '%s' is not in the parameter store" % name)

    @staticmethod
    def bn_names(scope):
        """The variables tf.layers.batch_normalization creates under `scope` (models/network_blocks.py:149-160):
        '<scope>/batch_normalization/' + gamma, beta, moving_mean, moving_variance."""
        return tuple(scope + "/batch_normalization/" + k for k in ("gamma", "beta", "moving_mean", "moving_variance"))

    def bn_variables(self, scope, use_batch_norm=True):
        """(gamma, beta, moving_mean, moving_variance) of `scope`'s batch norm; with use_batch_norm off,
        (None, offset, None, None): the '<scope>/offset' bias that replaces it (models/network_blocks.py:162-165)."""
        if use_batch_norm:
            return tuple(self.get(n) for n in self.bn_names(scope))
        return None, self.get(scope + "/offset"), None, None

    def bn_affine(self, scope, eps=1e-6):
        """Inference batch norm folded to y = x*scale + shift (models/network_blocks.py:149-160 with moving
        statistics): scale = gamma / sqrt(var + eps), shift = beta - mean * scale. Folded in float64, once per
        scope, and again when one of the four tensors is replaced or updated in place."""
        src = self.bn_variables(scope)
        key = (scope, eps)
        hit = self._bn.get(key)
        if hit is not None and all(a is b and a._version == v for a, b, v in zip(src, hit[0], hit[1])):
            return hit[2]
        g, b, m, v = (a.double() for a in src)
        scale = g / torch.sqrt(v + eps)
        shift = b - m * scale
        res = (scale.float().contiguous(), shift.float().contiguous())
        if _lib.publish_ready(self.device):
            self._bn[key] = (src, tuple(a._version for a in src), res)
        return res


@contextlib.contextmanager
def use_params(store):
    prev, _state.store = _state.store, store
    try:
        yield store
    finally:
        _state.store = prev


@contextlib.contextmanager
def variable_scope(name):
    scope = _state.scope
    scope.append(name)
    try:
        yield
    finally:
        scope.pop()


def current_scope():
    return "/".join(_state.scope)


def current_store():
    return _state.store


def scoped(name):
    s = current_scope()
    return s + "/" + name if s else name
