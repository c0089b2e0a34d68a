"""CPU: the float64 objective oracle (tests/objective_oracle.py) against direct calls of oracle/losses.py, the
regularisation against a numpy sum over the kernels, and the per-evolution tables of demon_b200.v2.objective against the
reference's training/v2/training.py where that tree is present."""
import ast
import os
import re

import numpy as np
import pytest
import torch

from demon_b200.v2 import objective as dobj
from demon_b200.v2 import weights as W2
from oracle import losses as ol
from oracle.network import Weights

import objective_oracle as oobj


@pytest.fixture(scope="module")
def weights():
    return W2.synthetic_weights(0)


def synthetic_batch(b, seed):
    """A batch shaped like datareader.build_batch's: inverse depth around 0.5, unit translations, small rotations, and
    each sample's own principal point (as rot180 / mirror_x make it)."""
    rng = np.random.RandomState(seed)
    t = rng.normal(size=(b, 3)) * 0.2 + np.array([0.9, 0.1, -0.05])
    t /= np.linalg.norm(t, axis=1, keepdims=True)
    k = np.tile(np.array([0.89115971, 1.18821287, 0.5, 0.5]), (b, 1))
    k[:, 2:] += rng.uniform(-0.02, 0.02, (b, 2))
    return {"IMAGE_PAIR": rng.uniform(-0.5, 0.5, (b, 6, 192, 256)).astype(np.float32),
            "MOTION": np.concatenate((rng.uniform(-0.03, 0.03, (b, 3)), t), axis=1).astype(np.float32),
            "DEPTH": rng.uniform(0.3, 0.7, (b, 1, 192, 256)).astype(np.float32),
            "INTRINSICS": k.astype(np.float32)}


def test_oracle_objective_equals_direct_loss_calls(weights):
    """4_iterative with one new sample and one earlier iteration: the oracle's dict equals oracle/losses.py's blocks
    called by hand on the oracle's block outputs, plus the regularisation, summed in order."""
    batch = synthetic_batch(2, 3)
    prev = {"predict_depth2": np.full((1, 1, 48, 64), 0.5), "predict_normal2": np.tile(np.array([0, 0, -1.0])[None, :, None, None], (1, 1, 48, 64)),
            "predict_rotation": np.array([[0.01, -0.02, 0.01]]), "predict_translation": np.array([[0.9, 0.1, -0.05]])}
    got = oobj.objective(weights, batch, "4_iterative", prev)

    ip = batch["IMAGE_PAIR"].astype(np.float64)
    i22 = oobj.resize_area(batch["IMAGE_PAIR"][:, 3:6], (48, 64)).astype(np.float64)
    res = oobj.run_blocks(Weights(weights, torch.float64), ip, i22, batch["INTRINSICS"].astype(np.float64), "4_iterative", prev)
    m = batch["MOTION"].astype(np.float64)
    rot, tr = m[:, 0:3].copy(), m[:, 3:6].copy()
    gt = ol.prepare_ground_truth_tensors(batch["DEPTH"].astype(np.float64), rot, tr, batch["INTRINSICS"].astype(np.float64))
    f, d = res["netFlow2"], res["netDM2"]
    c = np.ascontiguousarray
    fl = ol.flow_loss_block(gt["flow2"], gt["flow5"], gt["flow2_sig"], c(f["predict_flowconf2"][:, 0:2]), c(f["predict_flowconf5"][:, 0:2]),
                            c(f["predict_flowconf2"][:, 2:4]), c(f["predict_flowconf5"][:, 2:4]), 500.0, 25.0, 250.0, 25.0,
                            conf_diff_scale=10, level5_factor=0, loss_prefix="netFlow2_")
    dl = ol.depthnormal_loss_block(gt["depth2"], gt["depth2_sig"], gt["normal2"], rot, tr, d["predict_depth2"], d["predict_normal2"],
                                   d["predict_rotation"], d["predict_translation"], 150.0, 375.0, 25.0, 160, 45, 1, loss_prefix="netDM2_")
    want = [fl["netFlow2_" + k] for k in ("loss_flow5", "loss_flow2", "loss_flow2_sig", "loss_conf5", "loss_conf2", "loss_conf2_sig")]
    want += [dl["netDM2_" + k] for k in ("loss_depth2", "loss_depth2_sig", "loss_normal2", "loss_rotation", "loss_translation")]
    assert list(got)[:-2] == [k for p, names in dobj.SELECTED_LOSSES["4_iterative"] for k in (p + n for n in names)]
    assert [got[k] for k in list(got)[:-2]] == [float(v) for v in want]
    assert got["netFlow2_loss_flow5"] == 0.0 and got["netFlow2_loss_conf5"] == 0.0   # level5_factor 0
    assert all(np.isfinite(v) and v > 0 for k, v in got.items() if "5" not in k)
    assert got["total"] == sum(float(v) for v in want) + got["regularization"]
    # the netFlow2 block saw each sample's camera: the constant one gives another flow from depth and motion
    same = oobj.run_blocks(Weights(weights, torch.float64), ip, i22, np.tile(np.array([0.89115971, 1.18821287, 0.5, 0.5]), (2, 1)),
                           "2_flow2", prev)
    assert not np.array_equal(same["netFlow2"]["predict_flowconf2"], f["predict_flowconf2"])


def test_regularization_is_a_numpy_sum_over_the_kernels(weights):
    """0.0004 * sum of sum(k^2)/2 over every kernel of the built scopes, biases excluded; Session.kernel_l2 caches it per
    load_weights."""
    from demon_b200.v2.networks import Session
    kernels = {}
    for name, a in weights.items():
        if name.endswith("/kernel"):
            kernels.setdefault(name.split("/")[0], []).append(np.asarray(a, np.float64))
    s = Session()
    s.load_weights(weights)
    for evo in dobj.EVOLUTIONS:
        ref = 0.0004 * sum(0.5 * np.sum(k ** 2) for scope in dobj.built_scopes(evo) for k in kernels[scope])
        assert dobj.regularization(s, evo) == pytest.approx(ref, rel=1e-12)
        assert oobj.regularization(weights, evo) == pytest.approx(ref, rel=1e-12)
    assert dobj.built_scopes("0_flow1") == ("netFlow1",)
    assert dobj.built_scopes("4_iterative") == ("netFlow1", "netDM1", "netFlow2", "netDM2")
    assert dobj.built_scopes("5_refine") == dobj.SCOPES
    first = s.kernel_l2()
    assert s.kernel_l2() is first
    w2 = dict(weights)
    w2["netRefine/conv0/kernel"] = weights["netRefine/conv0/kernel"] * 2
    s.load_weights(w2)
    assert s.kernel_l2()["netRefine"] > first["netRefine"] and s.kernel_l2()["netFlow1"] == first["netFlow1"]


def test_weights_and_arguments():
    assert dobj._weights("5_refine", {})["depth_sig_weight"] == 0.5 * 0.25 * 1500
    assert dobj._weights("3_dm2", {})["depth_sig_weight"] == 0.25 * 1500
    assert dobj._weights("2_flow2", {"level5_factor": 0.5})["level5_factor"] == 0.5
    with pytest.raises(TypeError, match="flow_weigth"):
        dobj._weights("0_flow1", {"flow_weigth": 1.0})
    with pytest.raises(ValueError, match="evolution"):
        dobj.objective(None, {}, "6_more")


def _training_py():
    from oracle.ref import REF_SRC
    path = os.path.normpath(os.path.join(REF_SRC, "..", "..", "training", "v2", "training.py")) if REF_SRC else ""
    if not os.path.isfile(path):
        pytest.skip("the reference tree (DEMON_REF_SRC) is absent")
    with open(path) as f:
        return f.read()


def test_selected_losses_equal_training_py():
    """Each `selected_losses = (...)` of training.py with its loss prefix, under the `if trainer.current_evo ...` that
    guards its block, gives the table of demon_b200.v2.objective; so do the constants behind DEFAULT_WEIGHTS."""
    src = _training_py()
    lines = src.splitlines()
    table = {e: [] for e in dobj.EVOLUTIONS}
    for i, line in enumerate(lines):
        m = re.match(r"(\s*)selected_losses = (\(.*\))\s*$", line)
        if not m:
            continue
        names = ast.literal_eval(m.group(2))
        prefix = re.search(r"losses\['(\w+)'\+l\]", lines[i + 2]).group(1)
        indent = len(m.group(1))
        for j in range(i - 1, -1, -1):   # the guarding condition: the nearest one indented less
            c = re.match(r"(\s*)if trainer\.current_evo (==|in) (.*):\s*$", lines[j])
            if c and len(c.group(1)) < indent:
                evos = ast.literal_eval(c.group(3))
                evos = (evos,) if isinstance(evos, str) else evos
                break
        for e in evos:
            table[e].append((prefix, tuple(names)))
    assert {e: tuple(v) for e, v in table.items()} == dobj.SELECTED_LOSSES
    consts = dict(re.findall(r"^(_\w+_weight) = (.+)$", src, re.M))
    w = dobj.DEFAULT_WEIGHTS
    for key, const in (("flow_weight", "_flow_loss_weight"), ("flow_sig_weight", "_flow_grad_loss_weight"),
                       ("conf_weight", "_flow_conf_loss_weight"), ("conf_sig_weight", "_flow_conf_grad_loss_weight"),
                       ("depth_weight", "_depth_loss_weight"), ("depth_sig_weight", "_depth_grad_loss_weight"),
                       ("normal_weight", "_normal_loss_weight"), ("rotation_weight", "_rotation_loss_weight"),
                       ("translation_weight", "_translation_loss_weight")):
        assert w[key] == eval(consts[const], {}), key
    assert "l2_regularizer(%s)" % dobj.REGULARIZATION_SCALE in src
