"""Variable table of the DeMoN v2 graphs (python/depthmotionnet/v2/blocks.py) and a seeded synthetic weight generator.

Names and layouts are the ones TensorFlow creates for the v2 graph, so a checkpoint written by training/v2/training.py
feeds this package unchanged (same conventions as demon_b200.weights: conv [kh,kw,cin,cout], conv2d_transpose
[kh,kw,cout,cin], dense [in,out]).  No trained v2 weights are published, so tests and benchmarks use
`synthetic_weights`.
"""
from collections import OrderedDict

import numpy as np

from .. import weights as _v1


def _sep(name, k, cin, cmid, cout):
    """convrelu2 (v2/helpers.py:46-91): (k x 1) then (1 x k)."""
    return [(name + "y", "conv", (k, 1, cin, cmid)), (name + "x", "conv", (1, k, cmid, cout))]


def _trunk(flow, iterative):
    """v2/blocks.py:140-215 (flow) and :349-414 (depth and motion)."""
    wide2 = flow and not iterative
    specs = _sep("conv1", 9, 6, 24, 32)
    specs += _sep("conv2", 7, 32, 48 if wide2 else 32, 64 if wide2 else 32)
    if not wide2:
        specs += _sep("conv2_extra_inputs", 3, 9 if flow else (8 if iterative else 7), 32, 32)
    specs += _sep("conv2_1", 3, 64, 64, 64)
    specs += _sep("conv3", 5, 64, 96, 128)
    specs += _sep("conv3_1", 3, 128, 128, 128)
    specs += _sep("conv4", 5, 128, 192, 256)
    specs += _sep("conv4_1", 3, 256, 256, 256)
    specs += _sep("conv5", 5 if flow else 3, 256, 384, 384)
    specs += _sep("conv5_1", 3, 384, 384, 384)
    specs += [("dense5", "dense", (4608, 4608))]
    return specs


def flow_block_specs(iterative):
    """flow_block, v2/blocks.py:120-253."""
    return _trunk(True, iterative) + [
        ("predict_flow5/conv1", "conv", (3, 3, 480, 24)),
        ("predict_flow5/conv2", "conv", (3, 3, 24, 4)),
        ("upsample_flow5to4/upconv", "deconv", (4, 4, 2, 4)),
        ("refine4/upconv", "deconv", (4, 4, 256, 480)),
        ("refine3/upconv", "deconv", (4, 4, 128, 514)),
        ("refine2/upconv", "deconv", (4, 4, 64, 256)),
        ("predict_flow2/conv1", "conv", (3, 3, 128, 24)),
        ("predict_flow2/conv2", "conv", (3, 3, 24, 4)),
    ]


def depthmotion_block_specs(iterative):
    """depthmotion_block, v2/blocks.py:317-494."""
    return _trunk(False, iterative) + _sep("motion_conv3", 5, 64, 64, 64) + _sep("motion_conv4", 5, 64, 64, 64) + \
        _sep("motion_conv5a", 3, 64, 64, 64) + [
        ("motion_conv5b", "conv", (3, 3, 480, 64)),
        ("motion_fc1", "dense", (6144, 1024)),
        ("motion_fc2", "dense", (1024, 128)),
        ("motion_fc3", "dense", (128, 7)),
        ("refine4/upconv", "deconv", (4, 4, 256, 384)),
        ("refine3/upconv", "deconv", (4, 4, 128, 512)),
        ("refine2/upconv", "deconv", (4, 4, 64, 256)),
        ("predict_depthnormal2/conv1", "conv", (3, 3, 128, 24)),
        ("predict_depthnormal2/conv2", "conv", (3, 3, 24, 4)),
    ]


def refine_block_specs():
    """depth_refine_block, v2/blocks.py:499-560: as v1's, with depth0 and normal0 out of predict_depth0/conv2."""
    return [s if s[0] != "predict_depth0/conv2" else ("predict_depth0/conv2", "conv", (3, 3, 16, 4))
            for s in _v1.refine_block_specs()]


# scope -> block specs (v2/networks.py:33,39,100,116,195)
SCOPES = OrderedDict([
    ("netFlow1", lambda: flow_block_specs(False)),
    ("netDM1", lambda: depthmotion_block_specs(False)),
    ("netFlow2", lambda: flow_block_specs(True)),
    ("netDM2", lambda: depthmotion_block_specs(True)),
    ("netRefine", refine_block_specs),
])


def variable_specs():
    """OrderedDict: full variable name -> (kind, shape) for kernels and biases, in the order the device plan lists them."""
    out = OrderedDict()
    for scope, fn in SCOPES.items():
        for name, kind, shape in fn():
            out["%s/%s/kernel" % (scope, name)] = (kind, tuple(shape))
            out["%s/%s/bias" % (scope, name)] = ("bias", (shape[2] if kind == "deconv" else shape[-1],))
    return out


# output resolution of every conv, input resolution of every transposed conv (as demon_b200.weights._TRUNK_RES)
_TRUNK_RES = dict(_v1._TRUNK_RES, **{
    "motion_conv3y": (24, 64), "motion_conv3x": (24, 32), "motion_conv4y": (12, 32), "motion_conv4x": (12, 16),
    "motion_conv5ay": (6, 16), "motion_conv5ax": (6, 8), "motion_conv5b": (6, 8)})


def layer_macs(refine_hw=(192, 256)):
    """OrderedDict: layer name -> multiply-accumulates per image pair and call, counted as demon_b200.weights.layer_macs
    counts v1's (conv: output pixels x kh x kw x cin x cout; transposed conv: input pixels x 16 x cin x cout; dense:
    in x out)."""
    h, w = refine_hw
    refine_res = {"conv0": (h, w), "conv1": (h // 2, w // 2), "conv1_1": (h // 2, w // 2), "conv2": (h // 4, w // 4),
                  "conv2_1": (h // 4, w // 4), "refine1/upconv": (h // 4, w // 4), "refine0/upconv": (h // 2, w // 2),
                  "predict_depth0/conv1": (h, w), "predict_depth0/conv2": (h, w)}
    out = OrderedDict()
    for scope, fn in SCOPES.items():
        res = refine_res if scope == "netRefine" else _TRUNK_RES
        for name, kind, shape in fn():
            if kind == "dense":
                out[scope + "/" + name] = shape[0] * shape[1]
            else:
                rh, rw = res[name]
                out[scope + "/" + name] = rh * rw * shape[0] * shape[1] * shape[2] * shape[3]
    return out


def macs_per_pair(iterations=3):
    """Multiply-accumulates of one pair through bootstrap + `iterations` x iterative + refinement at 256x192, per block
    and in all ("pipeline")."""
    lm = layer_macs()
    tot = {scope: sum(v for k, v in lm.items() if k.startswith(scope + "/")) for scope in SCOPES}
    tot["pipeline"] = tot["netFlow1"] + tot["netDM1"] + iterations * (tot["netFlow2"] + tot["netDM2"]) + tot["netRefine"]
    return tot


def synthetic_weights(seed=0, dtype=np.float32):
    """Seeded stand-in for a trained v2 checkpoint, made like demon_b200.weights.synthetic_weights: fan-in scaled normal
    kernels, small non-zero biases, and prediction heads rescaled into the geometrically self-consistent regime the
    geometry ops between the blocks need (inverse depth ~0.5, small rotation, translation ~(0.9, 0.1, -0.05), scale ~1,
    flow ~ the flow that depth and motion imply).  normal0 gets the bias of normal2."""
    rng = np.random.RandomState(seed)
    out = OrderedDict()
    for name, (kind, shape) in variable_specs().items():
        if kind == "bias":
            out[name] = rng.uniform(-0.05, 0.05, size=shape).astype(dtype)
            continue
        fan_in = shape[0] if kind == "dense" else (shape[3] * 4 if kind == "deconv" else shape[0] * shape[1] * shape[2])
        out[name] = (rng.standard_normal(size=shape) * np.sqrt(2.0 / fan_in)).astype(dtype)

    def rescale(prefix, wscale, bias):
        out[prefix + "/kernel"] = (out[prefix + "/kernel"] * wscale).astype(dtype)
        out[prefix + "/bias"] = np.asarray(bias, dtype=dtype)

    for scope in ("netFlow1", "netFlow2"):
        rescale(scope + "/predict_flow5/conv2", 0.02, [0.381, 0.035, 0.3, 0.3])
        rescale(scope + "/predict_flow2/conv2", 0.02, [0.381, 0.035, 0.3, 0.3])
    for scope in ("netDM1", "netDM2"):
        rescale(scope + "/predict_depthnormal2/conv2", 0.1, [0.5, 0.0, 0.0, -0.8])
        rescale(scope + "/motion_fc3", 0.05, [0.02, -0.03, 0.01, 0.9, 0.1, -0.05, 1.0])
    rescale("netRefine/predict_depth0/conv2", 0.2, [0.5, 0.0, 0.0, -0.8])
    return out
