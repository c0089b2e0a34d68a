"""ORACLE (test infrastructure) -- training/v2/training.py's objective on the CPU in float64: the blocks of
oracle/network_v2.py on each sample's own camera, the losses of oracle/losses.py, the ground truth of its
prepare_ground_truth_tensors, composed per evolution as training.py:170-495 composes them.  Table of selected losses,
built blocks and default weights: demon_b200.v2.objective, which tests/test_objective.py checks against training.py.

oracle/network_v2.py runs depth_to_flow and flow_to_depth on the networks' constant camera; `CameraOps` hands it the
batch's INTRINSICS instead, through the `ops` argument its blocks take.  image2_2 is the float32 area resize the device
makes bit for bit (oracle/resize_area.py), then widened, so both sides start from the same input.
"""
import numpy as np
import torch

from demon_b200.v2 import objective as dobj
from demon_b200.v2 import weights as W2
from oracle import losses as ol
from oracle import ops as oops
from oracle.network import Weights
from oracle.network_v2 import depthmotion_block, flow_block, refine_block
from oracle.resize_area import resize_area


class CameraOps:
    """oracle.ops with the intrinsics of depth_to_flow / flow_to_depth replaced by `intrinsics` [B,4]."""

    def __init__(self, intrinsics):
        self.intrinsics = np.asarray(intrinsics)

    def depth_to_flow(self, depth, intrinsics, *args, **kwargs):
        return oops.depth_to_flow(depth, self.intrinsics.astype(np.asarray(intrinsics).dtype), *args, **kwargs)

    def flow_to_depth(self, flow, intrinsics, *args, **kwargs):
        return oops.flow_to_depth(flow, self.intrinsics.astype(np.asarray(intrinsics).dtype), *args, **kwargs)

    def __getattr__(self, name):
        return getattr(oops, name)


def regularization(tf_weights, evolution):
    """0.0004 * sum over the built blocks' kernels of sum(k^2) / 2, one numpy float64 sum per kernel."""
    total = 0.0
    for name, (kind, _) in W2.variable_specs().items():
        if kind != "bias" and name.split("/", 1)[0] in dobj.built_scopes(evolution):
            k = np.asarray(tf_weights[name], np.float64)
            total += 0.5 * float(np.sum(k * k))
    return dobj.REGULARIZATION_SCALE * total


def _np(t):
    return t.detach().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)


def run_blocks(W, ip, image2_2, K, evolution, prev_predictions=None):
    """{scope: the block's result dict (numpy)} for the blocks `evolution` builds, as training.py wires them."""
    t = lambda a: torch.as_tensor(np.asarray(a, np.float64))
    ops = CameraOps(K)
    B = ip.shape[0]
    new = B if prev_predictions is None else B - prev_predictions["predict_rotation"].shape[0]
    res = {}
    f1 = flow_block(W, "netFlow1", t(ip[:new]))
    res["netFlow1"] = f1
    if evolution >= "1_dm1":
        fc2 = f1["predict_flowconf2"]
        res["netDM1"] = depthmotion_block(W, "netDM1", t(ip[:new]), t(image2_2[:new]), fc2[:, 0:2].contiguous(), fc2)
    if evolution >= "2_flow2":
        dm1 = res["netDM1"]
        prev = {k: dm1[k] if prev_predictions is None else torch.cat((dm1[k], t(prev_predictions[k])))
                for k in ("predict_depth2", "predict_normal2", "predict_rotation", "predict_translation")}
        res["netFlow2"] = flow_block(W, "netFlow2", t(ip), t(image2_2), prev, ops=ops)
    if evolution >= "3_dm2":
        fc2 = res["netFlow2"]["predict_flowconf2"]
        res["netDM2"] = depthmotion_block(W, "netDM2", t(ip), t(image2_2), fc2[:, 0:2].contiguous(), fc2, prev["predict_rotation"],
                                          prev["predict_translation"], ops=ops)
    if evolution == "5_refine":
        res["netRefine"] = refine_block(W, "netRefine", t(ip[:, 0:3]), res["netDM2"]["predict_depth2"])
    return {s: {k: _np(v) for k, v in r.items()} for s, r in res.items()}


def objective(tf_weights, batch, evolution, prev_predictions=None, **weights):
    """demon_b200.v2.objective.objective on the CPU in float64: a dict of Python floats."""
    w = dobj._weights(evolution, weights)
    ip, motion, depth, K = (np.asarray(batch[k], np.float64) for k in ("IMAGE_PAIR", "MOTION", "DEPTH", "INTRINSICS"))
    image2_2 = resize_area(np.asarray(batch["IMAGE_PAIR"], np.float32)[:, 3:6], (48, 64)).astype(np.float64)
    rot, tr = np.ascontiguousarray(motion[:, 0:3]), np.ascontiguousarray(motion[:, 3:6])
    gt = ol.prepare_ground_truth_tensors(depth, rot, tr, K)
    res = run_blocks(Weights(tf_weights, torch.float64), ip, image2_2, K, evolution, prev_predictions)
    scored = {prefix[:-1] for prefix, _ in dobj.SELECTED_LOSSES[evolution]}
    got = {}
    for scope in ("netFlow1", "netFlow2"):
        if scope in scored:
            fc5, fc2 = res[scope]["predict_flowconf5"], res[scope]["predict_flowconf2"]
            c = lambda a, s: np.ascontiguousarray(a[:, s])
            got.update(ol.flow_loss_block(gt["flow2"], gt["flow5"], gt["flow2_sig"], c(fc2, slice(0, 2)), c(fc5, slice(0, 2)),
                                          c(fc2, slice(2, 4)), c(fc5, slice(2, 4)), w["flow_weight"], w["conf_weight"],
                                          w["flow_sig_weight"], w["conf_sig_weight"], conf_diff_scale=10,
                                          level5_factor=w["level5_factor"], loss_prefix=scope + "_"))
    for scope in ("netDM1", "netDM2"):
        if scope in scored:
            r = res[scope]
            got.update(ol.depthnormal_loss_block(gt["depth2"], gt["depth2_sig"], gt["normal2"], rot, tr, r["predict_depth2"],
                                                 r["predict_normal2"], r["predict_rotation"], r["predict_translation"],
                                                 w["depth_weight"], w["depth_sig_weight"], w["normal_weight"], w["rotation_weight"],
                                                 w["translation_weight"], 1, loss_prefix=scope + "_"))
    if "netRefine" in scored:
        r = res["netRefine"]
        got.update(ol.depth_refine_loss_block(gt["depth0"], gt["depth0_sig"], gt["normal0"], r["predict_depth0"], r["predict_normal0"],
                                              w["depth_weight"], w["depth_sig_weight"], w["normal_weight"], loss_prefix="netRefine_"))
    out = {}
    for prefix, names in dobj.SELECTED_LOSSES[evolution]:
        for name in names:
            out[prefix + name] = float(got[prefix + name])
    out["regularization"] = regularization(tf_weights, evolution)
    out["total"] = sum(out.values())
    return out
