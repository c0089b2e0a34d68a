"""CPU, no device: the v2 network's variable table, the oracle's 'same' convolution, and the plan the library lays out for
v2 (demon_debug_describe_plan builds it without a device): tap offsets, channel padding and the planner's choice per layer."""
import ctypes
import re

import numpy as np
import pytest
import torch

from demon_b200 import _lib
from demon_b200.v2 import weights as W2


def describe_plan(variant, batch=64, refine_hw=(192, 256), precision=1):
    buf = ctypes.create_string_buffer(1 << 20)
    n = _lib.load().demon_debug_describe_plan(variant, batch, refine_hw[0], refine_hw[1], precision, buf, len(buf))
    assert n > 0
    out = {}
    for line in buf.value.decode().splitlines():
        name, rest = line.split(None, 1)
        parts = [p.strip() for p in rest.split(" : ")]
        geo = dict(zip(parts[0].split()[1::2], map(int, parts[0].split()[2::2])))
        geo["kind"] = parts[0].split()[0]
        tap0 = tuple(map(int, parts[1].split()[1:])) if parts[1].startswith("tap0") else None
        out[name] = (geo, tap0, parts[-1])
    return out


def family(plan_text):
    """'simt', 'dense', or the tensor-core mode: 'halo', 'per-tap', 'cin8'."""
    if plan_text.startswith("dense"):
        return "dense"
    if plan_text.startswith("simt"):
        return "simt"
    return plan_text.split()[1]


def tf_pad_before(n, k, s):
    out = -(-n // s)
    return max((out - 1) * s + k - n, 0) // 2


@pytest.fixture(scope="module")
def weights():
    return W2.synthetic_weights(0)


def test_variable_table_is_what_the_oracle_reads_and_the_plan_holds(weights):
    """Every v2 variable the CPU oracle reads, with the shapes it reads, is in the table, and nothing else; the device plan
    has exactly one layer per kernel of the table, in the table's order."""
    from oracle.network_v2 import OracleNetsV2

    class Recording(dict):
        def __init__(self, d):
            super().__init__(d)
            self.read = set()

        def __getitem__(self, k):
            self.read.add(k)
            return dict.__getitem__(self, k)

    rec = Recording(weights)
    orc = OracleNetsV2(rec)
    g = torch.Generator().manual_seed(3)
    ip = (torch.rand(1, 6, 192, 256, generator=g) - 0.5).numpy()
    i22 = np.ascontiguousarray(ip[:, 3:6, ::4, ::4])
    r = orc.bootstrap(ip, i22)
    r = orc.iterative(ip, i22, r["predict_depth2"], r["predict_normal2"], r["predict_rotation"], r["predict_translation"])
    d = orc.refine(ip[:, 0:3], r["predict_depth2"], r["predict_normal2"])
    assert d["predict_depth0"].shape == (1, 1, 192, 256) and d["predict_normal0"].shape == (1, 3, 192, 256)
    specs = W2.variable_specs()
    assert rec.read == set(specs)
    for name, (_, shape) in specs.items():
        assert weights[name].shape == shape, name
    plan = describe_plan(2)
    assert [n + "/kernel" for n in plan] == [k for k in specs if k.endswith("/kernel")]
    for name, (geo, _, _) in plan.items():
        kind, shape = specs[name + "/kernel"]
        assert geo["kind"] == kind, name
        if kind == "conv":
            assert (geo["kh"], geo["kw"], geo["cin"], geo["cout"]) == shape, name
        elif kind == "deconv":
            assert (geo["cout"], geo["cin"]) == shape[2:], name
        else:
            assert (geo["cin"], geo["cout"]) == shape, name


def _same_conv_loop(x, k, b, sy, sx):
    """tf.nn.conv2d padding='SAME' as TensorFlow documents it: out = ceil(in / s); pad_along = max((out - 1) s + k - in,
    0); pad_top = pad_along // 2; out[i, j] = sum_{di, dj} in[i s + di - pad_top, j s + dj - pad_left] k[di, dj]."""
    C, H, Wd = x.shape
    kh, kw, _, co = k.shape
    Ho, Wo = -(-H // sy), -(-Wd // sx)
    pt = max((Ho - 1) * sy + kh - H, 0) // 2
    pl = max((Wo - 1) * sx + kw - Wd, 0) // 2
    out = np.tile(b.astype(np.float64)[:, None, None], (1, Ho, Wo))
    for i in range(Ho):
        for j in range(Wo):
            for di in range(kh):
                for dj in range(kw):
                    y, xx = i * sy + di - pt, j * sx + dj - pl
                    if 0 <= y < H and 0 <= xx < Wd:
                        out[:, i, j] += x[:, y, xx] @ k[di, dj]
    return out


@pytest.mark.parametrize("stride", (1, 2))
@pytest.mark.parametrize("size", ((6, 8), (7, 9), (12, 5)))
def test_oracle_same_conv_matches_tf_definition(stride, size):
    from oracle.network import Weights
    from oracle.network_v2 import conv2d_same
    rng = np.random.RandomState(stride * 100 + size[0])
    for k in range(1, 10):
        for kh, kw, sy, sx in ((k, 1, stride, 1), (1, k, 1, stride), (k, k, stride, stride)):
            x = rng.standard_normal((3,) + size)
            ker = rng.standard_normal((kh, kw, 3, 2))
            bias = rng.standard_normal(2)
            w = Weights({"c/kernel": ker, "c/bias": bias}, torch.float64)
            got = conv2d_same(w, "c", torch.from_numpy(x)[None], (sy, sx))[0].numpy()
            np.testing.assert_allclose(got, _same_conv_loop(x, ker, bias, sy, sx), rtol=1e-12, atol=1e-12,
                                       err_msg=str((k, kh, kw, sy, sx, size)))


@pytest.mark.parametrize("refine_hw", ((192, 256), (200, 300), (768, 1024)))
def test_v2_tap_offsets_follow_tf_same_padding(refine_hw):
    """Every v2 conv's first tap is minus TF's pad_before at its own input size: one row (y conv) or column (x conv) later
    than caffe padding for a stride-2 layer on an even input, equal to it otherwise.  The transposed convs are v1's."""
    plan = describe_plan(2, 1, refine_hw)
    v1 = describe_plan(1, 1, refine_hw)
    later = 0
    for name, (geo, tap0, _) in plan.items():
        if geo["kind"] != "conv":
            assert tap0 is None, name
            continue
        dy, dx = tap0
        assert dy == -tf_pad_before(geo["H"], geo["kh"], geo["sy"]), name
        assert dx == -tf_pad_before(geo["W"], geo["kw"], geo["sx"]), name
        if geo["sy"] == 2 and geo["H"] % 2 == 0:
            assert dy == -(geo["kh"] // 2) + 1, name
            later += 1
        elif geo["sx"] == 2 and geo["W"] % 2 == 0:
            assert dx == -(geo["kw"] // 2) + 1, name
            later += 1
        else:
            assert (dy, dx) == (-(geo["kh"] // 2), -(geo["kw"] // 2)), name
    # conv1..conv5 (y and x) of four trunks, motion_conv3/4/5a (y and x) of two, and the refinement block's conv1 / conv2
    assert later == 4 * 10 + 2 * 6 + 2
    assert all(tap0 is None for _, tap0, _ in v1.values())


# The planner's decision for every v2 layer at 3xTF32 (batch 64 and batch 1): the tensor-core mode, 'simt' or 'dense'.
# Per layer name within a block (the same in the four trunk blocks unless listed per block).
EXPECTED_FAMILY = {
    "conv1y": "cin8", "conv1x": "halo", "conv2y": "halo", "conv2x": "halo",
    "conv2_extra_inputsy": "halo", "conv2_extra_inputsx": "halo", "conv2_1y": "halo", "conv2_1x": "halo",
    "conv3y": "per-tap", "conv3x": "per-tap", "conv3_1y": "per-tap", "conv3_1x": "per-tap",
    "conv4y": "per-tap", "conv4x": "per-tap", "conv4_1y": "per-tap", "conv4_1x": "per-tap",
    "conv5y": "per-tap", "conv5x": "per-tap", "conv5_1y": "per-tap", "conv5_1x": "per-tap", "dense5": "dense",
    "predict_flow5/conv1": "per-tap", "predict_flow5/conv2": "simt", "upsample_flow5to4/upconv": "simt",
    "refine4/upconv": "per-tap", "refine3/upconv": "per-tap", "refine2/upconv": "per-tap",
    "predict_flow2/conv1": "halo", "predict_flow2/conv2": "simt",
    "motion_conv3y": "per-tap", "motion_conv3x": "per-tap", "motion_conv4y": "per-tap", "motion_conv4x": "per-tap",
    "motion_conv5ay": "per-tap", "motion_conv5ax": "per-tap", "motion_conv5b": "per-tap",
    "motion_fc1": "dense", "motion_fc2": "dense", "motion_fc3": "dense",
    "predict_depthnormal2/conv1": "halo", "predict_depthnormal2/conv2": "simt",
}
EXPECTED_REFINE = {"conv0": "cin8", "conv1": "halo", "conv1_1": "halo", "conv2": "halo", "conv2_1": "halo",
                   "refine1/upconv": "halo", "refine0/upconv": "halo", "predict_depth0/conv1": "halo", "predict_depth0/conv2": "simt"}


@pytest.mark.parametrize("batch", (64, 1))
def test_planner_decision_for_every_v2_layer(batch):
    plan = describe_plan(2, batch)
    for name, (geo, _, text) in plan.items():
        scope, layer = name.split("/", 1)
        want = EXPECTED_REFINE[layer] if scope == "netRefine" else EXPECTED_FAMILY[layer]
        assert family(text) == want, (name, text)
    # the 24 / 48-channel y halves sit in 32 / 64-channel pixels: the x convs read whole chunks of 32 on the tensor cores
    for scope in ("netFlow1", "netDM1", "netFlow2", "netDM2"):
        g1 = plan[scope + "/conv1x"][0]
        assert (g1["cin"], g1["cin_buf"], g1["in_pitch"]) == (24, 32, 32)
        g2 = plan[scope + "/conv2x"][0]
        assert (g2["cin"], g2["cin_buf"]) == ((48, 64) if scope == "netFlow1" else (32, 32))
    # conv5_1_dense5: conv5_1 in channels 0..383 of one 480-channel buffer, read whole by predict_flow5/conv1, refine4 of
    # the flow block and motion_conv5b, and as its first 384 channels by refine4 of the DM block
    for scope in ("netFlow1", "netFlow2"):
        assert (plan[scope + "/conv5_1x"][0]["out_pitch"], plan[scope + "/predict_flow5/conv1"][0]["cin"]) == (480, 480)
        assert plan[scope + "/refine4/upconv"][0]["cin"] == 480
    for scope in ("netDM1", "netDM2"):
        assert (plan[scope + "/motion_conv5b"][0]["cin"], plan[scope + "/motion_conv5b"][0]["out_off"]) == (480, 64)
        assert (plan[scope + "/refine4/upconv"][0]["cin"], plan[scope + "/refine4/upconv"][0]["in_pitch"]) == (384, 480)
    assert plan["netRefine/predict_depth0/conv2"][0]["cout"] == 4


def test_v1_plan_has_no_v2_layer():
    v1 = describe_plan(1)
    assert not any("dense5" in n or "motion_conv5b" in n for n in v1)
    assert "netDM1/motion_conv1" in v1


def test_v2_macs_per_pair():
    t = W2.macs_per_pair()
    lm = W2.layer_macs()
    assert lm["netFlow1/dense5"] == 4608 * 4608
    assert lm["netDM1/motion_conv5b"] == 6 * 8 * 9 * 480 * 64
    assert t["pipeline"] == t["netFlow1"] + t["netDM1"] + 3 * (t["netFlow2"] + t["netDM2"]) + t["netRefine"]
    print("\nv2 GFLOP per pair (bootstrap + 3 iterations + refinement): %.3f" % (2 * t["pipeline"] / 1e9))


def test_session_restore_reads_a_v2_checkpoint(weights, tmp_path):
    """Session.restore of demon_b200.v2.networks: a TF bundle with the v2 variables (float64 here, converted to float32)
    comes back under the same names; a variable of the wrong shape is refused by name."""
    from demon_b200 import checkpoint as ck
    from demon_b200.v2.networks import Session
    tensors = {k: v.astype(np.float64) for k, v in weights.items()}
    tensors["global_step"] = np.array(7, np.int64)   # a training checkpoint holds more than the graph's variables
    prefix = ck.save_checkpoint(str(tmp_path / "v2"), tensors)
    s = Session()
    s.restore(prefix)
    assert list(s.weights) == list(W2.variable_specs()) or set(s.weights) == set(W2.variable_specs())
    for k, v in weights.items():
        assert s.weights[k].dtype == np.float32 and np.array_equal(s.weights[k], v), k
    bad = dict(tensors)
    bad["netDM1/motion_conv5b/kernel"] = np.zeros((3, 3, 384, 64), np.float32)
    prefix = ck.save_checkpoint(str(tmp_path / "bad"), bad)
    with pytest.raises(ValueError, match="netDM1/motion_conv5b/kernel"):
        Session().restore(prefix)


def test_oracle_clip_by_value_follows_tf_1_4():
    """maximum(minimum(x, 50), 0) with std::min / std::max compare order: +inf -> 50, -inf -> 0, NaN stays NaN; the kernel
    (clip_0_50 in csrc/net.cu) is written the same way and the v2 layer trace compares the two bit for bit."""
    from oracle.network_v2 import clip_by_value
    x = torch.tensor([float("inf"), float("-inf"), float("nan"), -0.0, 0.0, 1e-45, 50.0, 50.000004, 3.0e38, -1.0])
    y = clip_by_value(x, 0.0, 50.0)
    assert y[0] == 50 and y[1] == 0 and torch.isnan(y[2])
    assert y[3:].tolist() == [-0.0, 0.0, x[5].item(), 50.0, 50.0, 50.0, 0.0]
