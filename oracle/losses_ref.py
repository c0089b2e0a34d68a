"""ORACLE (test infrastructure) -- the reference's own python/depthmotionnet/v2/losses.py (and the helpers it star-imports),
imported unmodified from the reference tree next to DEMON_REF_SRC and run eagerly in numpy.

Minimal stand-ins are injected for the two modules it imports: `tensorflow` (sqrt, reduce_sum, reduce_mean, concat, split,
exp, abs, add_n, stop_gradient, name_scope, and tensors with get_shape()) and `lmbspecialops` (replace_nonfinite and the
C oracle of oracle/ops.py for scale_invariant_gradient, median3x3_downsample, depth_to_flow and depth_to_normals).  The
stand-ins are removed from sys.modules again after the import.  tests/golden/make_losses_golden.py stores what this
module computes.
"""
import contextlib
import importlib
import os
import sys
import types

import numpy as np

from . import ops
from .ref import REF_SRC


class Tensor(np.ndarray):
    """An ndarray with TF's static-shape accessor."""

    def get_shape(self):
        shape = list(self.shape)
        return types.SimpleNamespace(as_list=lambda: shape)


def tensor(x):
    return np.asarray(x).view(Tensor)


def _tf():
    tf = types.ModuleType("tensorflow")
    tf.sqrt = lambda x: tensor(np.sqrt(x))
    tf.reduce_sum = lambda x, axis=None: tensor(np.sum(x, axis=axis))
    tf.reduce_mean = lambda x, axis=None: tensor(np.mean(x, axis=axis))
    tf.concat = lambda values, axis: tensor(np.concatenate(values, axis=axis))
    tf.split = lambda value, num_or_size_splits, axis=0: [tensor(v) for v in np.split(value, num_or_size_splits, axis=axis)]
    tf.exp = lambda x: tensor(np.exp(x))
    tf.abs = lambda x: tensor(np.abs(x))

    def add_n(inputs):
        total = inputs[0]
        for x in inputs[1:]:
            total = total + x
        return tensor(total)
    tf.add_n = add_n
    tf.stop_gradient = lambda x: x
    tf.name_scope = lambda name: contextlib.nullcontext()
    return tf


def _sops():
    s = types.ModuleType("lmbspecialops")
    s.replace_nonfinite = lambda x, value=0.0: tensor(np.where(np.isfinite(x), x, np.asarray(x).dtype.type(value)))
    s.scale_invariant_gradient = lambda input, deltas, weights, epsilon=0.001: tensor(
        ops.scale_invariant_gradient(np.asarray(input), deltas, weights, epsilon))
    s.median3x3_downsample = lambda input: tensor(ops.median3x3_downsample(np.asarray(input)))
    s.depth_to_flow = lambda depth, intrinsics, rotation, translation, rotation_format="angleaxis3", inverse_depth=False, \
        normalize_flow=False, name=None: tensor(ops.depth_to_flow(np.asarray(depth), intrinsics, rotation, translation, rotation_format,
                                                                  inverse_depth, normalize_flow))
    s.depth_to_normals = lambda depth, intrinsics, inverse_depth=False: tensor(
        ops.depth_to_normals(np.asarray(depth), intrinsics, inverse_depth))
    s.leaky_relu = lambda x, leak=0.1: tensor(ops.leaky_relu(np.asarray(x), leak))
    return s


def reference_python_dir():
    """<reference>/python next to DEMON_REF_SRC (<reference>/lmbspecialops/src), or None."""
    if not REF_SRC:
        return None
    path = os.path.normpath(os.path.join(REF_SRC, "..", "..", "python"))
    return path if os.path.isfile(os.path.join(path, "depthmotionnet", "v2", "losses.py")) else None


def load():
    """The reference's v2/losses.py module over the stand-ins, or None where the reference tree is absent."""
    root = reference_python_dir()
    if root is None:
        return None
    names = ("tensorflow", "lmbspecialops", "depthmotionnet", "depthmotionnet.helpers", "depthmotionnet.v2", "depthmotionnet.v2.helpers",
             "depthmotionnet.v2.losses")
    saved = {k: sys.modules.get(k) for k in names}
    try:
        sys.modules["tensorflow"] = _tf()
        sys.modules["lmbspecialops"] = _sops()
        pkg = types.ModuleType("depthmotionnet")
        pkg.__path__ = [os.path.join(root, "depthmotionnet")]
        v2 = types.ModuleType("depthmotionnet.v2")
        v2.__path__ = [os.path.join(root, "depthmotionnet", "v2")]
        sys.modules["depthmotionnet"], sys.modules["depthmotionnet.v2"] = pkg, v2
        return importlib.import_module("depthmotionnet.v2.losses")
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
