"""Generates tests/golden/losses_golden.npz by running the REFERENCE's own python/depthmotionnet/v2/losses.py (imported
unmodified by oracle/losses_ref.py over numpy stand-ins for tensorflow and lmbspecialops) in float64 on seeded inputs:
prepare_ground_truth_tensors, every combination of flow_loss_block's optional arguments, depthnormal_loss_block,
depth_refine_loss_block and the module's small functions, for N = 1 and 3 at odd sizes with NaN / +-inf / 0 / negative
values in ground truth and prediction.  Needs the reference tree (DEMON_REF_SRC):
    DEMON_REF_SRC=<reference>/lmbspecialops/src python tests/golden/make_losses_golden.py
"""
import hashlib
import itertools
import os
import sys

import numpy as np

_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if _ROOT not in sys.path:
    sys.path.insert(0, _ROOT)

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "losses_golden.npz")

SIZES = [(1, 23, 34), (3, 40, 70)]
FLOW_ARGS = dict(flow_weight=1.7, conf_weight=0.3, flow_sig_weight=2.5, conf_sig_weight=0.8)
DN_ARGS = dict(depth_weight=300.0, depth_sig_weight=1500.0, normal_weight=50.0, rotation_weight=160.0, translation_weight=15.0,
               translation_factor=1.3)
REFINE_ARGS = dict(depth_weight=300.0, depth_sig_weight=1500.0, normal_weight=100.0)


def flow_combos():
    """(use pr_conf2, use pr_conf5, flow_sig_weight set, conf_sig_weight set, conf_diff_scale, level5_factor, prefix)"""
    out = [c + (1, 0.5, '') for c in itertools.product((True, False), repeat=4)]
    out += [(True, True, True, True, 10, 0.0, 'netFlow1_'), (True, False, True, True, 2.5, 0.25, 'netFlow2_')]
    return out


def make_inputs(ci):
    n, h, w = SIZES[ci]
    rng = np.random.RandomState(4242 + ci)
    depth = rng.uniform(0.2, 2.0, (n, 1, h, w))
    bad = rng.rand(n, 1, h, w)
    depth[bad < 0.02] = np.nan
    depth[(bad >= 0.02) & (bad < 0.03)] = 0.0
    depth[(bad >= 0.03) & (bad < 0.035)] = np.inf
    depth[(bad >= 0.035) & (bad < 0.04)] = -0.5
    k = np.tile([0.89115971, 1.18821287, 0.5, 0.5], (n, 1)) + rng.uniform(-0.02, 0.02, (n, 4))
    rot = rng.uniform(-0.1, 0.1, (n, 3))
    tr = rng.uniform(-0.5, 0.5, (n, 3)) + np.array([0.5, 0.0, 0.1])
    return {"depth": depth, "intrinsics": k, "rotation": rot, "translation": tr}


def make_predictions(ci, gt):
    rng = np.random.RandomState(777 + ci)

    def noisy(a, s, invalid=True):
        b = np.where(np.isfinite(a), a, 0.5) + rng.normal(0, s, a.shape)
        if invalid:
            m = rng.rand(*a.shape)
            b[m < 0.01] = np.nan
            b[(m >= 0.01) & (m < 0.015)] = np.inf
            b[(m >= 0.015) & (m < 0.02)] = -np.inf
            b[(m >= 0.02) & (m < 0.03)] = 0.0
        return b
    n = gt["depth2"].shape[0]
    return {"pr_flow2": noisy(gt["flow2"], 0.01), "pr_flow5": noisy(gt["flow5"], 0.01),
            "pr_conf2": rng.uniform(0.05, 1.0, gt["flow2"].shape), "pr_conf5": rng.uniform(0.05, 1.0, gt["flow5"].shape),
            "pr_depth2": np.abs(noisy(gt["depth2"], 0.05)) + 0.01, "pr_normal2": noisy(gt["normal2"], 0.1),
            "pr_depth0": np.abs(noisy(gt["depth0"], 0.05)) + 0.01, "pr_normal0": noisy(gt["normal0"], 0.1),
            "pr_rotation": rng.uniform(-0.1, 0.1, (n, 3)), "pr_translation": rng.uniform(-0.5, 0.5, (n, 3))}


def run(mod, ci, inputs, gt_stored=None):
    """What `mod` (the reference module or oracle/losses) computes for case ci -> {name: array}.  The blocks run on
    gt_stored (the stored ground truth) when given, so that both sides see the same inputs."""
    from oracle.losses_ref import tensor
    out = {}
    inp = {k: tensor(v) for k, v in inputs.items()}
    gt = mod.prepare_ground_truth_tensors(inp["depth"], inp["rotation"], inp["translation"], inp["intrinsics"])
    for k, v in gt.items():
        out["gt/" + k] = np.asarray(v)
    g = gt_stored if gt_stored is not None else {k: np.asarray(v) for k, v in gt.items()}
    pr = make_predictions(ci, g)
    for k, v in pr.items():
        out["pr/" + k] = v
    g = {k: tensor(v) for k, v in g.items()}
    pr = {k: tensor(v) for k, v in pr.items()}
    for j, (c2, c5, fs, cs, scale, l5, prefix) in enumerate(flow_combos()):
        r = mod.flow_loss_block(g["flow2"], g["flow5"], g["flow2_sig"], pr["pr_flow2"], pr["pr_flow5"], pr["pr_conf2"] if c2 else None,
                                pr["pr_conf5"] if c5 else None, FLOW_ARGS["flow_weight"], FLOW_ARGS["conf_weight"],
                                FLOW_ARGS["flow_sig_weight"] if fs else None, FLOW_ARGS["conf_sig_weight"] if cs else None,
                                conf_diff_scale=scale, level5_factor=l5, loss_prefix=prefix)
        out["flow%d/keys" % j] = np.array(list(r.keys()))
        out["flow%d/values" % j] = np.array([float(np.asarray(v)) for v in r.values()])
    r = mod.depthnormal_loss_block(g["depth2"], g["depth2_sig"], g["normal2"], inp["rotation"], inp["translation"], pr["pr_depth2"],
                                   pr["pr_normal2"], pr["pr_rotation"], pr["pr_translation"], loss_prefix="netDM1_", **DN_ARGS)
    out["dn/keys"], out["dn/values"] = np.array(list(r.keys())), np.array([float(np.asarray(v)) for v in r.values()])
    r = mod.depth_refine_loss_block(g["depth0"], g["depth0_sig"], g["normal0"], pr["pr_depth0"], pr["pr_normal0"], loss_prefix="netRefine_",
                                    **REFINE_ARGS)
    out["refine/keys"], out["refine/values"] = np.array(list(r.keys())), np.array([float(np.asarray(v)) for v in r.values()])
    out["conf2"] = np.asarray(mod.compute_confidence_map(pr["pr_flow2"], g["flow2"], 3))
    out["l1"] = np.array([float(np.asarray(mod.l1_loss(pr["pr_rotation"] - inp["rotation"], 0.00001))),
                          float(np.asarray(mod.l1_loss(pr["pr_translation"] - inp["translation"], 0)))])
    out["l2"] = np.array([float(np.asarray(mod.pointwise_l2_loss(pr["pr_normal2"], g["normal2"], 0.00001))),
                          float(np.asarray(mod.pointwise_l2_loss(pr["pr_flow2"], g["flow2"], 0)))])
    return out


def digest(a):
    a = np.ascontiguousarray(a)
    return "%s %s %s" % (a.dtype.str, "x".join(map(str, a.shape)), hashlib.sha256(a.tobytes()).hexdigest())


def sig_loss_value(mod, ci, g):
    from oracle.losses_ref import tensor
    pr = make_predictions(ci, g)
    s = mod.scale_invariant_gradient(tensor(pr["pr_depth2"]), deltas=[1, 2, 4, 8, 16], weights=[1, 1, 1, 1, 1], epsilon=0.01)
    return float(np.asarray(mod.scale_invariant_gradient_loss(tensor(s), tensor(g["depth2_sig"]), 0.00001)))


def main():
    from oracle import losses_ref
    ref = losses_ref.load()
    if ref is None:
        sys.exit("needs the reference tree: set DEMON_REF_SRC to <reference>/lmbspecialops/src")
    out = {}
    for ci in range(len(SIZES)):
        inputs = make_inputs(ci)
        for k, v in inputs.items():
            out["c%d/in/%s" % (ci, k)] = v
        res = run(ref, ci, inputs)
        for k, v in res.items():
            if k.startswith("gt/"):
                out["c%d/%s" % (ci, k)] = np.array(digest(v))   # the ground truth is stored as its digest only
            elif not k.startswith("pr/"):
                out["c%d/%s" % (ci, k)] = v
        g = {k[3:]: v for k, v in res.items() if k.startswith("gt/")}
        out["c%d/sig_loss" % ci] = np.float64(sig_loss_value(ref, ci, g))
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
