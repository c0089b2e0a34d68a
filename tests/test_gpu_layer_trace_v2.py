"""GPU: every layer of the v2 network traced on the device and checked on its own, as tests/test_gpu_layer_trace.py does
for v1 (its steps 1-3), with the v2 oracle (oracle/network_v2.py) forced by the GPU's output taps:

1. input wiring, bit for bit: each layer's input tap equals the input the oracle builds from the GPU's outputs with its
   own concats, NCHW flattens and geometry ops (demon_b200.lmbspecialops), including dense5's input permutation, the
   480-channel conv5_1_dense5 and the motion concat, and the clip of depth_from_flow to [0, 50]; padding channels are
   exactly zero.
2. output against float64 of the GPU's own input tap under the per-element bounds of the v1 trace: tc_error_bound for
   the tensor-core layers, gamma_n for the SIMT and dense layers.  The float64 convolutions use TF's 'same' padding, so
   every v2 tap set is checked; dense5's reference applies TF's NCHW flatten and reshape to the taps.
3. each stage output equals, bit for bit, the tap it is exported from (depth0 and normal0 included).
"""
import re

import numpy as np
import pytest
import torch

from demon_b200 import _lib
from demon_b200 import lmbspecialops as sops
from demon_b200.v2 import weights as W2
from demon_b200.v2.networks import BootstrapNet, IterativeNet, RefinementNet, Session
from oracle import ops as oops
from oracle.network_v2 import OracleNetsV2
from test_conv_variants import _PLAN_RE, tc_error_bound
from test_gpu_conv_variants import ref64
from test_gpu_conv_variants_v2 import plan_of, ref64_same
from test_gpu_layer_trace import PRECISIONS, STAGE_SCOPES, U, check_bitwise, dev, first_mismatch, gamma, traced, where

pytestmark = pytest.mark.gpu
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    yield
    for prec, (ratio, share, name) in sorted(WORST.items()):
        print("\nv2 layer trace, %s: largest |err| / S = %.3g (%.3g of the bound) at %s" % (prec, ratio, share, name))


@pytest.fixture(scope="module")
def weights():
    return W2.synthetic_weights(0)


@pytest.fixture(scope="module")
def sessions(weights):
    out = {}
    for prec in PRECISIONS:
        out[prec] = Session(precision=prec)
        out[prec].load_weights(weights)
    return out


@pytest.fixture(scope="module")
def random_pairs():
    g = torch.Generator().manual_seed(4321)
    ip = (torch.rand(2, 6, 192, 256, generator=g) - 0.5).numpy()
    i22 = oops.median3x3_downsample(oops.median3x3_downsample(np.ascontiguousarray(ip[:, 3:6])))
    return ip, i22


def pixel_major(x, c, hw):
    """[B, c*hw] in TF's NCHW flatten order -> the buffer's [B, hw*c] pixel-major order (and back with c, hw swapped)."""
    return x.reshape(x.shape[0], c, hw).transpose(1, 2).reshape(x.shape[0], -1)


def forced(trace, run):
    """oracle stage `run(force)` forced with the trace's output taps; dense5's tap is turned into TF's column order."""
    seen = {}

    def force(name, x):
        assert name not in seen, "layer %s forced twice" % name
        seen[name] = x
        y = trace.out(name)
        if name.endswith("/dense5"):
            y = pixel_major(y, 48, 96)
        return (y.permute(0, 3, 1, 2) if y.dim() == 4 else y).cpu()

    res = run(force)
    assert sorted(seen) == sorted(trace.taps), set(seen) ^ set(trace.taps)
    return seen, res


def nhwc_order(name, x, g):
    x = x.cuda()
    if x.dim() == 4:
        return x.permute(0, 2, 3, 1)
    if name.endswith("motion_fc1"):
        return pixel_major(x, g["in_pitch"], g["H"] * g["W"])
    if name.endswith("/dense5"):
        return pixel_major(x, 96, 48)
    return x


def check_layer(name, kind, g, plan, x_oracle, tap_in, tap_out, weights, precision, scale=None):
    cin, cin_buf, B = g["cin"], g["cin_buf"], tap_in.shape[0]
    plan = plan_of(plan)
    # 1. wiring
    x_tap = tap_in[..., :cin]
    want = nhwc_order(name, x_oracle, g)
    assert tuple(want.shape) == tuple(x_tap.shape), (name, tuple(want.shape), tuple(x_tap.shape))
    i, count = first_mismatch(x_tap, want)
    if i is not None:
        pytest.fail("input of %s: %d of %d elements differ from the oracle's, first %s: got %r, oracle %r"
                    % (name, count, x_tap.numel(), where(name, i), x_tap[i].item(), want[i].item()))
    if cin_buf > cin:
        nz = (tap_in[..., cin:] != 0).nonzero()
        assert nz.shape[0] == 0, "padding channels of %s's input are not 0 (%d elements)" % (name, nz.shape[0])
    # 2. output against float64 of the GPU's own input
    k, b = weights[name + "/kernel"], weights[name + "/bias"]
    if kind == "dense":
        x64 = x_tap.double()
        if name.endswith("motion_fc1"):
            x64 = pixel_major(x64, g["H"] * g["W"], g["in_pitch"])
        elif name.endswith("/dense5"):
            x64 = pixel_major(x64, 48, 96)
        kt, bt = (torch.from_numpy(np.asarray(a, np.float64)).cuda() for a in (k, b))
        y, S = x64 @ kt + bt, x64.abs() @ kt.abs() + bt.abs()
        if name.endswith("/dense5"):   # TF's reshape to [96,6,8], in the buffer's pixel order
            y, S = pixel_major(y, 96, 48), pixel_major(S, 96, 48)
    else:
        geom = (g["kh"], g["kw"], g["sy"], g["sx"])
        if kind == "deconv":
            y, S = ref64(x_tap, k, b, geom, True), ref64(x_tap.abs(), np.abs(k), np.abs(b), geom, True)
        else:
            y, S = ref64_same(x_tap, k, b, geom), ref64_same(x_tap.abs(), np.abs(k), np.abs(b), geom)
    if g["leaky"]:
        y = torch.maximum(float(np.float32(0.1)) * y, y)
    m = _PLAN_RE.match(plan)
    if m:
        c = tc_error_bound(precision, cin_buf, g["kh"], g["kw"], kind == "deconv", int(m.group(9)))
    else:
        taps = 1 if kind == "dense" else (4 if kind == "deconv" else g["kh"] * g["kw"])
        ksplit = int(re.search(r"ksplit (\d+)", plan).group(1)) if kind == "dense" else 1
        c = gamma(taps * cin_buf / ksplit + ksplit + 3)
    bound = c * S
    if g["scale"]:
        s = scale.double().reshape(B, 1, 1)
        y[..., 0] = s * y[..., 0]
        S[..., 0] = s.abs() * S[..., 0]
        bound[..., 0] = c * S[..., 0] + U * y[..., 0].abs()
    got = tap_out.double()
    err = (got - y).abs()
    bad = (~(err <= bound) & ~(torch.isnan(got) & torch.isnan(y))).nonzero()
    if bad.shape[0]:
        j = tuple(bad[0].tolist())
        pytest.fail("output of %s: %d elements over the bound %.3g S, first %s: got %r, float64 %r, S %r; plan %s"
                    % (name, bad.shape[0], c, where(name, j), got[j].item(), y[j].item(), S[j].item(), plan))
    pos = S > 0
    ratio = (err[pos] / S[pos]).nan_to_num(0.0).max().item() if pos.any() else 0.0
    return ratio, ratio / c


def check_stage(trace, seen, weights, prec_name):
    scales = {}
    for name, kind, g, plan in trace.layers:
        a, b = trace.taps[name]
        sc = scales.get(name.split("/")[0]) if g["scale"] else None
        assert not g["scale"] or sc is not None, name
        ratio, share = check_layer(name, kind, g, plan, seen[name], a, b, weights, PRECISIONS[prec_name], sc)
        if name.endswith("motion_fc3"):
            scales[name.split("/")[0]] = b[:, 6]
        if ratio > WORST.get(prec_name, (-1.0,))[0]:
            WORST[prec_name] = (ratio, share, name)


def check_exports(stage, trace, out):
    nchw = lambda t: t.permute(0, 3, 1, 2)
    if stage == "refine":
        t = trace.out("netRefine/predict_depth0/conv2")
        check_bitwise(out["predict_depth0"], nchw(t[..., 0:1]), "predict_depth0 against its tap")
        check_bitwise(out["predict_normal0"], nchw(t[..., 1:4]), "predict_normal0 against its tap")
        return
    f, d = STAGE_SCOPES[stage]
    pairs = {"predict_flow5": nchw(trace.out(f + "predict_flow5/conv2")[..., 0:2]),
             "predict_flow2": nchw(trace.out(f + "predict_flow2/conv2")[..., 0:2]),
             "predict_depth2": nchw(trace.out(d + "predict_depthnormal2/conv2")[..., 0:1]),
             "predict_normal2": nchw(trace.out(d + "predict_depthnormal2/conv2")[..., 1:4]),
             "predict_rotation": trace.out(d + "motion_fc3")[:, 0:3],
             "predict_translation": trace.out(d + "motion_fc3")[:, 3:6]}
    for k, want in pairs.items():
        check_bitwise(out[k], want, "%s against its tap" % k)


def run_stage(sess, prec, weights, stage, B, inputs, refine_hw=(192, 256)):
    """One traced v2 stage-wise call and all its checks; returns (the call's outputs, the forced oracle's full outputs)."""
    net = sess.net(B, refine_hw)
    oracle = OracleNetsV2(weights)
    if stage == "bootstrap":
        ip, i22 = inputs
        out, t = traced(net, STAGE_SCOPES[stage], lambda: BootstrapNet(sess, "channels_first", B).eval(dev(ip), dev(i22)))
        seen, res = forced(t, lambda force: oracle.bootstrap(ip, i22, full=True, force=force, ops=sops))
    elif stage == "iterative":
        out, t = traced(net, STAGE_SCOPES[stage], lambda: IterativeNet(sess, "channels_first", B).eval(*(dev(a) for a in inputs)))
        seen, res = forced(t, lambda force: oracle.iterative(*inputs, full=True, force=force, ops=sops))
    else:
        image1, depth2 = inputs
        out, t = traced(net, STAGE_SCOPES[stage],
                        lambda: RefinementNet(sess, "channels_first", B, image_size=refine_hw).eval(dev(image1), dev(depth2), None))
        seen, res = forced(t, lambda force: oracle.refine(image1, depth2, force=force))
    check_exports(stage, t, out)
    check_stage(t, seen, weights, prec)
    del t, seen
    return out, res


def iterative_inputs(ip, i22, r, translation_scale=1.0):
    return (ip, i22, r["predict_depth2"].cpu().numpy(), r["predict_normal2"].cpu().numpy(), r["predict_rotation"].cpu().numpy(),
            r["predict_translation"].cpu().numpy() * np.float32(translation_scale))


@pytest.mark.parametrize("prec", sorted(PRECISIONS))
def test_trace_v2_random_pairs(sessions, weights, random_pairs, prec):
    """Batch 2: bootstrap, iterative fed the GPU bootstrap's outputs, refine fed the GPU iterative's depth2."""
    ip, i22 = random_pairs
    r0, _ = run_stage(sessions[prec], prec, weights, "bootstrap", 2, (ip, i22))
    r1, _ = run_stage(sessions[prec], prec, weights, "iterative", 2, iterative_inputs(ip, i22, r0))
    run_stage(sessions[prec], prec, weights, "refine", 2, (np.ascontiguousarray(ip[:, 0:3]), r1["predict_depth2"].cpu().numpy()))


def adversarial(weights):
    """test_gpu_network.py's adversarial weights on the v2 variables."""
    w = dict(weights)
    for scope in ("netDM1", "netDM2"):
        w[scope + "/predict_depthnormal2/conv2/bias"] = np.array([0.0, 0, 0, -0.8], np.float32)
        w[scope + "/predict_depthnormal2/conv2/kernel"] = weights[scope + "/predict_depthnormal2/conv2/kernel"] * 5
        w[scope + "/motion_fc3/bias"] = np.array([0.3, -0.2, 0.1, 2.5, 0.5, -0.7, 1.0], np.float32)
    for scope in ("netFlow1", "netFlow2"):
        w[scope + "/predict_flow2/conv2/bias"] = np.array([0.01, -0.01, 0.3, 0.3], np.float32)
    return w


@pytest.mark.parametrize("translation_scale", (1.0, 1e-3), ids=["adversarial", "adversarial_short_translation"])
def test_trace_v2_adversarial(weights, translation_scale):
    """Adversarial weights, iterative stage: depth_to_flow gives NaN and flows the gate zeroes, warp2d leaves the image and
    flow_to_depth triangulates from flows that contradict the motion; with the previous translation shortened 1000-fold the
    triangulated inverse depths go far above 50, so the clip of v2/blocks.py:379 acts.  netDM2's extra inputs must still
    be the oracle's bit for bit, the clip included."""
    w = adversarial(weights)
    s = Session("3xtf32")
    s.load_weights(w)
    g = torch.Generator().manual_seed(99)
    ip = (torch.rand(1, 6, 192, 256, generator=g) - 0.5).numpy()
    i22 = oops.median3x3_downsample(oops.median3x3_downsample(np.ascontiguousarray(ip[:, 3:6])))
    r0 = BootstrapNet(s, "channels_first", 1).eval(dev(ip), dev(i22))
    torch.cuda.synchronize()
    _, res = run_stage(s, "3xtf32", w, "iterative", 1, iterative_inputs(ip, i22, r0, translation_scale))
    raw = res["depth_from_flow_unclipped"].numpy()
    assert (res["flow_from_depth_motion"].numpy() == 0).mean() > 0.05
    if translation_scale != 1.0:
        assert (raw > 50).sum() > 100, (raw > 50).sum()
        assert (res["depth_from_flow"].numpy() == 50).sum() == (raw > 50).sum()


@pytest.mark.parametrize("hw,B", [((200, 300), 2), ((768, 1024), 1)], ids=["200x300", "768x1024"])
def test_trace_v2_refinement_sizes(sessions, weights, hw, B):
    rng = np.random.RandomState(hw[0] + hw[1])
    image1 = rng.uniform(-0.5, 0.5, (B, 3) + hw).astype(np.float32)
    depth2 = rng.uniform(0.2, 0.8, (B, 1, hw[0] // 4, hw[1] // 4)).astype(np.float32)
    run_stage(sessions["3xtf32"], "3xtf32", weights, "refine", B, (image1, depth2), refine_hw=hw)
