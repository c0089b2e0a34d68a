"""CPU: pins the torch calls of oracle/network.py against naive numpy loops written from TensorFlow's
documented definitions of the layers the reference graph uses, checks the variable table against the
numbers in SURVEY.md / BASELINE.md, replays the committed golden outputs (BASELINE.json configs[0]), and checks that
forcing the oracle's layer outputs (the hook tests/test_gpu_layer_trace.py uses) changes nothing else."""
import os
import re

import numpy as np
import pytest
import torch

from demon_b200 import weights as W
from oracle import network as onet


def tf_conv2d_valid(x, k, b, strides):
    """tf.nn.conv2d, NHWC, VALID: out[b,i,j,o] = sum_{di,dj,q} x[b, s0*i+di, s1*j+dj, q] * k[di,dj,q,o]."""
    B, H, Wd, C = x.shape
    kh, kw, _, O = k.shape
    Ho, Wo = (H - kh) // strides[0] + 1, (Wd - kw) // strides[1] + 1
    out = np.zeros((B, Ho, Wo, O))
    for i in range(Ho):
        for j in range(Wo):
            patch = x[:, strides[0] * i:strides[0] * i + kh, strides[1] * j:strides[1] * j + kw, :]
            out[:, i, j, :] = np.tensordot(patch, k, axes=([1, 2, 3], [0, 1, 2]))
    return out + b


def tf_conv2d_transpose_valid(x, k, b, stride):
    """tf.nn.conv2d_transpose (the gradient of conv2d), NHWC, VALID, kernel [kh,kw,out,in]:
    out[b, s*i+di, s*j+dj, o] += x[b,i,j,q] * k[di,dj,o,q]."""
    B, H, Wd, C = x.shape
    kh, kw, O, _ = k.shape
    out = np.zeros((B, (H - 1) * stride + kh, (Wd - 1) * stride + kw, O))
    for i in range(H):
        for j in range(Wd):
            out[:, stride * i:stride * i + kh, stride * j:stride * j + kw, :] += np.einsum("bq,yxoq->byxo", x[:, i, j, :], k)
    return out + b


def leaky(x):
    return np.maximum(np.float32(0.1).astype(x.dtype) * x, x)


def nchw(x):
    return np.ascontiguousarray(x.transpose(0, 3, 1, 2))


def test_convrelu2_caffe_padding_matches_tf_definition():
    """helpers.py:105-153 with stride 2 and k 5 on an odd-sized input."""
    rng = np.random.RandomState(0)
    x = rng.randn(2, 9, 12, 3)
    w = {"s/cy/kernel": rng.randn(5, 1, 3, 4), "s/cy/bias": rng.randn(4), "s/cx/kernel": rng.randn(1, 5, 4, 6), "s/cx/bias": rng.randn(6)}
    pad = 2
    t = leaky(tf_conv2d_valid(np.pad(x, ((0, 0), (pad, pad), (0, 0), (0, 0))), w["s/cy/kernel"], w["s/cy/bias"], (2, 1)))
    ref = leaky(tf_conv2d_valid(np.pad(t, ((0, 0), (0, 0), (pad, pad), (0, 0))), w["s/cx/kernel"], w["s/cx/bias"], (1, 2)))
    got = onet.convrelu2_caffe_padding(onet.Weights(w, torch.float64), "s/c", torch.from_numpy(nchw(x)), 2).numpy()
    assert got.shape == (2, 6, 5, 6)   # ceil(9/2), ceil(12/2)
    np.testing.assert_allclose(got, nchw(ref), rtol=1e-12, atol=1e-12)


def test_conv2d_caffe_padding_matches_tf_definition():
    rng = np.random.RandomState(1)
    x = rng.randn(1, 7, 6, 5)
    w = {"c/kernel": rng.randn(3, 3, 5, 2), "c/bias": rng.randn(2)}
    ref = tf_conv2d_valid(np.pad(x, ((0, 0), (1, 1), (1, 1), (0, 0))), w["c/kernel"], w["c/bias"], (2, 2))
    got = onet.conv2d_caffe_padding(onet.Weights(w, torch.float64), "c", torch.from_numpy(nchw(x)), 2).numpy()
    np.testing.assert_allclose(got, nchw(ref), rtol=1e-12, atol=1e-12)


def test_refine_upconv_matches_tf_definition():
    """blocks_original.py:97-110: conv2d_transpose(k4, s2, VALID) -> leaky -> slice begin (1,1), size 2n."""
    rng = np.random.RandomState(2)
    x = rng.randn(2, 3, 4, 5)
    w = {"r/upconv/kernel": rng.randn(4, 4, 6, 5), "r/upconv/bias": rng.randn(6)}
    full = leaky(tf_conv2d_transpose_valid(x, w["r/upconv/kernel"], w["r/upconv/bias"], 2))
    assert full.shape == (2, 8, 10, 6)    # 2n+2
    ref = full[:, 1:7, 1:9, :]
    direct = rng.randn(2, 7, 6, 8)
    got = onet.refine_caffe_padding(onet.Weights(w, torch.float64), "r", torch.from_numpy(nchw(x)), torch.from_numpy(direct)).numpy()
    np.testing.assert_allclose(got[:, :6], nchw(ref), rtol=1e-12, atol=1e-12)
    assert np.array_equal(got[:, 6:], direct)          # concat order: upsampled features first (blocks_original.py:111)


def test_nearest_neighbour_upsample_and_flatten_order():
    W_ = W.synthetic_weights(0)
    rng = np.random.RandomState(3)
    img = rng.rand(1, 3, 16, 24).astype(np.float32)
    d = rng.rand(1, 1, 4, 6).astype(np.float32)
    # conv0 sees concat(image1, depth[y//4, x//4]) (blocks_original.py:475,482)
    out = onet.refine_block(onet.Weights(W_), "netRefine", torch.from_numpy(img), torch.from_numpy(d))["predict_depth0"]
    assert tuple(out.shape) == (1, 1, 16, 24)
    up = np.repeat(np.repeat(d, 4, axis=2), 4, axis=3)
    x = torch.from_numpy(np.concatenate((img, up), axis=1))
    c0 = onet.convrelu_caffe_padding(onet.Weights(W_), "netRefine/conv0", x, 1)
    iy = torch.div(torch.arange(16) * 4, 16, rounding_mode="floor")
    assert iy.tolist() == [y // 4 for y in range(16)]
    assert c0.shape == (1, 32, 16, 24)


def test_variable_table_matches_survey_numbers():
    specs = W.variable_specs()
    assert len(specs) == 2 * (26 + 29 + 28 + 29 + 9)          # 121 layers, kernel + bias
    assert sum(int(np.prod(s)) for _, s in specs.values()) == 45753883   # 45.75 M parameters
    m = W.macs_per_pair()
    assert abs(m["pipeline"] / 1e6 - 15176.3) < 0.1            # 30.353 GFLOP / pair
    assert abs(m["refine_fn"](768, 1024) / 1e6 - 49337.6) < 0.1
    assert specs["netFlow2/refine3/upconv/kernel"] == ("deconv", (4, 4, 128, 514))
    assert specs["netDM1/motion_fc1/kernel"] == ("dense", (6144, 1024))


def test_golden_config1_netflow1_on_sculpture_pair(sculpture, synthetic_weights, golden_dir):
    """BASELINE.json configs[0]: single sculpture pair, netFlow1 only, CPU."""
    g = np.load(os.path.join(golden_dir, "oracle_config1.npz"))
    with torch.no_grad():
        f = onet.flow_block(onet.Weights(synthetic_weights), "netFlow1", torch.from_numpy(sculpture["image_pair"]))
    assert tuple(f["predict_flowconf2"].shape) == (1, 4, 48, 64)
    np.testing.assert_allclose(f["predict_flowconf2"].numpy(), g["predict_flowconf2"], rtol=0, atol=2e-5)
    np.testing.assert_allclose(f["predict_flowconf5"].numpy(), g["predict_flowconf5"], rtol=0, atol=2e-5)


def test_golden_pipeline_fp32_vs_fp64(golden_dir):
    """The committed fp32 and fp64 oracle outputs agree far inside the 1e-4 budget: the budget is the
    CUDA path's, not the oracle's."""
    g = np.load(os.path.join(golden_dir, "oracle_pipeline.npz"))
    d32, d64 = g["predict_depth0_f32"], g["predict_depth0_f64"]
    assert np.abs(d32 - d64).sum() / np.abs(d64).sum() < 1e-6
    f32, f64 = g["predict_flow2_f32"], g["predict_flow2_f64"]
    assert np.sqrt(((f32 - f64) ** 2).sum(1)).mean() < 1e-6


# stride of the strided layers (helpers.py:105-153 / blocks_original.py:459-465): conv1..conv5 of the trunks split into a y
# and an x conv, netRefine's conv1 and conv2; every other layer has stride 1
_STRIDED = re.compile(r"net\w+/conv[1-5]([yx]?)")
_LINEAR = ("predict_flow5/conv2", "predict_flow2/conv2", "predict_depthnormal2/conv2", "predict_depth0/conv2",
           "upsample_flow5to4/upconv", "motion_fc3")   # the layers without a leaky ReLU


def own_layer_outputs(W_, record):
    """A `force` for the oracle that computes every layer itself, with the oracle's own arithmetic, and records its name.
    The scaled depth channel of predict_depthnormal2/conv2 is scale * conv, with the scale of the same block's motion_fc3."""
    scales = {}

    def force(name, x):
        assert name not in record, "layer %s forced twice" % name
        record.append(name)
        act = not name.endswith(_LINEAR)
        if name.endswith("upconv"):
            y = onet._upconv(W_, name, x)
            return onet.my_leaky_relu(y) if act else y
        if name.split("/")[-1].startswith("motion_fc"):
            y = onet.dense(W_, name, x, act)
            if name.endswith("motion_fc3"):
                scales[name.split("/")[0]] = y[:, 6:7]
            return y
        m = _STRIDED.fullmatch(name)
        stride = 1 if not m else {"y": (2, 1), "x": (1, 2), "": 2}[m.group(1)]
        y = onet.conv2d_caffe_padding(W_, name, x, stride, activation=act)
        if name.endswith("predict_depthnormal2/conv2"):
            y = torch.cat((scales[name.split("/")[0]].reshape(-1, 1, 1, 1) * y[:, 0:1], y[:, 1:4]), dim=1)
        return y
    return force


def test_forced_oracle_with_its_own_layer_outputs_is_the_oracle(sculpture, synthetic_weights):
    """The oracle's `force` hook changes nothing but where each layer's output comes from: forced with its own fp32 layer
    outputs, all three stages reproduce the unforced oracle bit for bit, and every one of the 121 layers is forced once."""
    nets = onet.OracleNets(synthetic_weights)
    ip, i22 = sculpture["image_pair"], sculpture["image2_2"]
    record = []
    force = own_layer_outputs(nets.W, record)
    stages = []
    r0 = nets.bootstrap(ip, i22, full=True)
    stages.append((r0, nets.bootstrap(ip, i22, full=True, force=force)))
    args = tuple(r0[k].numpy() for k in ("predict_depth2", "predict_normal2", "predict_rotation", "predict_translation"))
    stages.append((nets.iterative(ip, i22, *args, full=True), nets.iterative(ip, i22, *args, full=True, force=force)))
    image1 = np.ascontiguousarray(ip[:, 0:3])
    stages.append((nets.refine(image1, r0["predict_depth2"]), nets.refine(image1, r0["predict_depth2"], force=force)))
    for want, got in stages:
        assert set(want) == set(got)
        for k in want:
            assert torch.equal(want[k], got[k]), k
    layers = sorted({n.rsplit("/", 1)[0] for n in W.variable_specs()})
    assert sorted(record) == layers
