"""GPU: every layer of the network traced on the device (demon_debug_trace_layers), each one checked on its own.

A stage-wise call (bootstrap, iterative, refine) runs with a trace that copies every layer's input slice just before the
layer runs and its output slice just after.  The CPU oracle then runs forced (oracle/network.py): every layer returns the
GPU's output tap instead of computing, while the oracle builds each layer's input from those taps in the reference's own
order (its concats, nearest-neighbour upsampling, NCHW flatten, |flow| < 1 gate) with the device's standalone geometry ops
(demon_b200.lmbspecialops, pinned against the oracle and the reference's sources by the op tests).  For every layer:

1. input wiring, bit for bit: channels [0, cin) of the GPU's input tap equal the oracle's input (NaN equals NaN, -0 equals
   +0), and the padding channels [cin, cin_buf), which carry zero weights, are exactly zero.  This covers every skip-concat
   and channel slice, the import of the caller's tensors and the three fused glue kernels (flow_extra_kernel,
   dm_extra_kernel, refine_input_kernel) against the standalone ops composed by the oracle's own graph.
2. output against float64 of the GPU's own input tap, computed on the device, under a per-element bound |err| <= c * S with
   S = sum |x||w| + |b|: tensor-core layers with tc_error_bound (tests/test_conv_variants.py) and their plan's split-K, the
   fp32 SIMT and dense layers with gamma_n, n = K / ksplit + ksplit + 3 (K = taps x cin_buf).  motion_fc1's reference is the
   NCHW flatten of its NHWC input tap times the TF-layout kernel, so the row permutation of its upload is checked;
   predict_depthnormal2/conv2's depth channel is scale * conv, the scale taken from the same stage's motion_fc3 tap.  Every
   layer is isolated, so errors do not compound and a failure names the layer.
3. each stage output equals, bit for bit, the tap it is exported from.
"""
import ctypes
import re
import time

import numpy as np
import pytest
import torch

from demon_b200 import _lib
from demon_b200 import lmbspecialops as sops
from demon_b200.networks_original import BootstrapNet, DemonPipeline, IterativeNet, RefinementNet, Session
from oracle import ops as oops
from oracle.network import OracleNets
from test_conv_variants import _PLAN_RE, FP32, TF32, X3TF32, tc_error_bound
from test_gpu_conv_variants import describe_layers, ref64

pytestmark = pytest.mark.gpu

PRECISIONS = {"fp32": FP32, "3xtf32": X3TF32, "tf32": TF32}
STAGE_SCOPES = {"bootstrap": ("netFlow1/", "netDM1/"), "iterative": ("netFlow2/", "netDM2/"), "refine": ("netRefine/",)}
U = 2.0 ** -24
WORST = {}   # precision name -> (largest |err| / S, its share of the bound, layer)


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    yield
    for prec, (ratio, bound_ratio, name) in sorted(WORST.items()):
        print("\nlayer trace, %s: largest |err| / S = %.3g (%.3g of the bound) at %s" % (prec, ratio, bound_ratio, name))


@pytest.fixture(scope="module")
def sessions(synthetic_weights):
    out = {}
    for prec in PRECISIONS:
        s = Session(precision=prec)
        s.load_weights(synthetic_weights)
        out[prec] = s
    return out


@pytest.fixture(scope="module")
def random_pairs():
    """tests/test_gpu_network.py's random_pairs."""
    g = torch.Generator().manual_seed(1234)
    ip = (torch.rand(2, 6, 192, 256, generator=g) - 0.5).numpy()
    i22 = oops.median3x3_downsample(oops.median3x3_downsample(np.ascontiguousarray(ip[:, 3:6])))
    return ip, i22


def gamma(n):
    return n * U / (1 - n * U)


def out_hw(kind, g):
    if kind == "deconv":
        return 2 * g["H"], 2 * g["W"]
    return -(-g["H"] // g["sy"]), -(-g["W"] // g["sx"])


class Trace:
    """The input and output taps of the layers of `scopes` on the net `net` (a _NetHandle), set until close().  Taps are
    NaN before the call, so a copy that never happened shows."""

    def __init__(self, net, scopes):
        self.net = net
        self.layers = [L for L in describe_layers(net.ptr) if L[0].startswith(scopes)]
        B = net.batch
        n = _lib.load().demon_net_num_layers(net.ptr)
        names = [_lib.load().demon_net_layer_name(net.ptr, i).decode() for i in range(n)]
        ins, outs = (ctypes.c_void_p * n)(), (ctypes.c_void_p * n)()
        self.taps = {}
        for name, kind, g, plan in self.layers:
            if kind == "dense":
                shapes = (B, g["cin_buf"]), (B, g["cout"])
            else:
                shapes = (B, g["H"], g["W"], g["cin_buf"]), (B,) + out_hw(kind, g) + (g["cout"],)
            a, b = (torch.full(s, float("nan"), device="cuda") for s in shapes)
            i = names.index(name)
            ins[i], outs[i] = a.data_ptr(), b.data_ptr()
            self.taps[name] = (a, b)
        _lib.check(_lib.load().demon_debug_trace_layers(net.ptr, ctypes.cast(ins, ctypes.c_void_p), ctypes.cast(outs, ctypes.c_void_p)))

    def close(self):
        _lib.check(_lib.load().demon_debug_trace_layers(self.net.ptr, None, None))

    def out(self, name):
        return self.taps[name][1]


def traced(net, scopes, call):
    """Runs `call()` (a stage-wise entry on `net`) with a trace of `scopes`; returns (its outputs, the trace)."""
    t = Trace(net, scopes)
    try:
        out = call()
        torch.cuda.synchronize()
    finally:
        t.close()
    assert _lib.load().demon_check_errors() == 0, "a pipeline wait timed out or a CUDA error is pending"
    return out, t


def forced(trace, run):
    """Runs the oracle stage `run(force)` forced with the trace's output taps; returns ({layer: oracle input}, its outputs)."""
    seen = {}

    def force(name, x):
        assert name not in seen, "layer %s forced twice" % name
        seen[name] = x
        y = trace.out(name)
        return (y.permute(0, 3, 1, 2) if y.dim() == 4 else y).cpu()

    res = run(force)
    assert sorted(seen) == sorted(trace.taps), set(seen) ^ set(trace.taps)
    return seen, res


def nhwc_order(name, x, g):
    """The oracle's input of a layer in the GPU tap's layout: NCHW -> NHWC; motion_fc1's NCHW flatten -> NHWC flatten."""
    x = x.cuda()
    if x.dim() == 4:
        return x.permute(0, 2, 3, 1)
    if name.endswith("motion_fc1"):
        return x.reshape(x.shape[0], g["in_pitch"], g["H"], g["W"]).permute(0, 2, 3, 1).reshape(x.shape[0], -1)
    return x


def first_mismatch(got, want):
    """Index of the first element where got and want differ in bits (NaN equals NaN, -0 equals +0), and the count."""
    bad = ((got + 0.0).view(torch.int32) != (want + 0.0).view(torch.int32)) & ~(torch.isnan(got) & torch.isnan(want))
    idx = bad.nonzero()
    return (tuple(idx[0].tolist()) if idx.shape[0] else None), idx.shape[0]


def where(name, i):
    return "%s at %s %s" % (name, "[n, channel]" if len(i) == 2 else "[n, y, x, channel]", list(i))


def check_bitwise(got, want, what):
    i, count = first_mismatch(got, want)
    if i is not None:
        pytest.fail("%s: %d of %d elements differ, first %s: got %r, want %r"
                    % (what, count, got.numel(), where("", i), got[i].item(), want[i].item()))


def check_layer(name, kind, g, plan, x_oracle, tap_in, tap_out, weights, precision, scale=None):
    """The three per-layer checks of the module docstring (1 and 2) for one layer; returns (|err| / S, its share of the bound)."""
    cin, cin_buf, B = g["cin"], g["cin_buf"], tap_in.shape[0]
    # 1. wiring
    x_tap = tap_in[..., :cin]
    want = nhwc_order(name, x_oracle, g)
    assert tuple(want.shape) == tuple(x_tap.shape), (name, tuple(want.shape), tuple(x_tap.shape))
    i, count = first_mismatch(x_tap, want)
    if i is not None:
        pytest.fail("input of %s: %d of %d elements differ from the oracle's, first at input channel %d, %s: got %r, oracle %r"
                    % (name, count, x_tap.numel(), i[-1], where(name, i), x_tap[i].item(), want[i].item()))
    if cin_buf > cin:
        pad = tap_in[..., cin:]
        nz = (pad != 0).nonzero()   # NaN != 0 as well
        if nz.shape[0]:
            j = tuple(nz[0].tolist())
            pytest.fail("padding channel %d of %s's input is %r, not 0 (%d such elements), first %s"
                        % (cin + j[-1], name, pad[j].item(), nz.shape[0], where(name, j[:-1] + (cin + j[-1],))))
    # 2. output against float64 of the GPU's own input
    k = weights[name + "/kernel"]
    b = weights[name + "/bias"]
    if kind == "dense":
        x64 = x_tap.double()
        if name.endswith("motion_fc1"):   # the reference's NCHW flatten of the NHWC tap
            x64 = x64.reshape(B, g["H"], g["W"], g["in_pitch"]).permute(0, 3, 1, 2).reshape(B, -1)
        kt, bt = (torch.from_numpy(np.asarray(a, np.float64)).cuda() for a in (k, b))
        y, S = x64 @ kt + bt, x64.abs() @ kt.abs() + bt.abs()
    else:
        geom = (g["kh"], g["kw"], g["sy"], g["sx"])
        y = ref64(x_tap, k, b, geom, kind == "deconv")
        S = ref64(x_tap.abs(), np.abs(k), np.abs(b), geom, kind == "deconv")
    if g["leaky"]:
        y = torch.maximum(float(np.float32(0.1)) * y, y)
    m = _PLAN_RE.match(plan)
    if m:   # tensor cores
        c = tc_error_bound(precision, cin_buf, g["kh"], g["kw"], kind == "deconv", int(m.group(9)))
    else:
        taps = 1 if kind == "dense" else (4 if kind == "deconv" else g["kh"] * g["kw"])
        ksplit = int(re.search(r"ksplit (\d+)", plan).group(1)) if kind == "dense" else 1
        c = gamma(taps * cin_buf / ksplit + ksplit + 3)
    bound = c * S
    if g["scale"]:   # channel 0 = scale * conv: one more rounding, of |scale * y|
        s = scale.double().reshape(B, 1, 1)
        y[..., 0] = s * y[..., 0]
        S[..., 0] = s.abs() * S[..., 0]
        bound[..., 0] = c * S[..., 0] + U * y[..., 0].abs()
    got = tap_out.double()
    err = (got - y).abs()
    bad = ~(err <= bound) & ~(torch.isnan(got) & torch.isnan(y))
    idx = bad.nonzero()
    if idx.shape[0]:
        j = tuple(idx[0].tolist())
        pytest.fail("output of %s: %d elements over the bound %.3g S, first at output channel %d, %s: got %r, float64 %r, S %r; plan %s"
                    % (name, idx.shape[0], c, j[-1], where(name, j), got[j].item(), y[j].item(), S[j].item(), plan))
    pos = S > 0
    ratio = (err[pos] / S[pos]).nan_to_num(0.0).max().item() if pos.any() else 0.0
    return ratio, ratio / c


def check_stage(stage, trace, seen, weights, prec_name, scale=None):
    """Checks 1 and 2 for every layer of a traced stage, one layer at a time."""
    precision = PRECISIONS[prec_name]
    scales = {}
    for name, kind, g, plan in trace.layers:
        a, b = trace.taps[name]
        sc = scales.get(name.split("/")[0]) if g["scale"] else None
        assert not g["scale"] or sc is not None, name
        ratio, share = check_layer(name, kind, g, plan, seen[name], a, b, weights, precision, sc)
        if name.endswith("motion_fc3"):
            scales[name.split("/")[0]] = b[:, 6]
        if ratio > WORST.get(prec_name, (-1.0,))[0]:
            WORST[prec_name] = (ratio, share, name)


def check_exports(stage, trace, out):
    """3. every stage output equals the tap it is exported from (channels_first outputs)."""
    nchw = lambda t: t.permute(0, 3, 1, 2)
    if stage == "refine":
        check_bitwise(out["predict_depth0"], nchw(trace.out("netRefine/predict_depth0/conv2")), "predict_depth0 against its tap")
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


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


def run_stage(sess, prec, weights, stage, B, inputs, refine_hw=(192, 256)):
    """One traced stage-wise call on the session's net and all its checks; returns the call's outputs (torch, device)."""
    net = sess.net(B, refine_hw)
    oracle = OracleNets(weights)
    if stage == "bootstrap":
        ip, i22 = inputs
        out, t = traced(net, STAGE_SCOPES[stage], lambda: BootstrapNet(sess, "channels_first", B).eval(dev(ip), dev(i22)))
        seen, _ = forced(t, lambda force: oracle.bootstrap(ip, i22, force=force, ops=sops))
    elif stage == "iterative":
        out, t = traced(net, STAGE_SCOPES[stage], lambda: IterativeNet(sess, "channels_first", B).eval(*(dev(a) for a in inputs)))
        seen, _ = forced(t, lambda force: oracle.iterative(*inputs, force=force, ops=sops))
    else:
        image1, depth2 = inputs
        out, t = traced(net, STAGE_SCOPES[stage],
                        lambda: RefinementNet(sess, "channels_first", B, image_size=refine_hw).eval(dev(image1), dev(depth2)))
        seen, _ = forced(t, lambda force: oracle.refine(image1, depth2, force=force))
    check_exports(stage, t, out)
    check_stage(stage, t, seen, weights, prec)
    del t, seen
    return out


def iterative_inputs(ip, i22, r):
    return (ip, i22) + tuple(r[k].cpu().numpy() for k in ("predict_depth2", "predict_normal2", "predict_rotation", "predict_translation"))


def run_all_stages(sess, prec, weights, ip, i22):
    """bootstrap, iterative fed with the GPU bootstrap's outputs, refine fed with the GPU iterative's depth."""
    B = ip.shape[0]
    r0 = run_stage(sess, prec, weights, "bootstrap", B, (ip, i22))
    r1 = run_stage(sess, prec, weights, "iterative", B, iterative_inputs(ip, i22, r0))
    run_stage(sess, prec, weights, "refine", B, (np.ascontiguousarray(ip[:, 0:3]), r1["predict_depth2"].cpu().numpy()))
    return r0, r1


@pytest.mark.parametrize("prec", sorted(PRECISIONS))
def test_trace_random_pairs(sessions, synthetic_weights, random_pairs, prec):
    """Batch 2, every stage at every precision."""
    run_all_stages(sessions[prec], prec, synthetic_weights, *random_pairs)


def test_trace_sculpture_pair(sessions, synthetic_weights, sculpture):
    run_all_stages(sessions["3xtf32"], "3xtf32", synthetic_weights, sculpture["image_pair"], sculpture["image2_2"])


def test_trace_adversarial_weights(synthetic_weights):
    """The adversarial weights of test_gpu_network.py's test_adversarial_weights_exercise_invalid_geometry_branches, iterative
    stage: the previous depth straddles 0, depth_to_flow gives NaN and flows the gate zeroes, warp2d leaves the image and
    flow_to_depth triangulates from flows that contradict the motion.  Those are the branches of the fused glue; the inputs
    it makes must still be the oracle's bit for bit."""
    w = dict(synthetic_weights)
    for scope in ("netDM1", "netDM2"):
        w[scope + "/predict_depthnormal2/conv2/bias"] = np.array([0.0, 0, 0, -0.8], np.float32)
        w[scope + "/predict_depthnormal2/conv2/kernel"] = synthetic_weights[scope + "/predict_depthnormal2/conv2/kernel"] * 5
        w[scope + "/motion_fc3/bias"] = np.array([0.3, -0.2, 0.1, 2.5, 0.5, -0.7, 1.0], np.float32)
    for scope in ("netFlow1", "netFlow2"):
        w[scope + "/predict_flow2/conv2/bias"] = np.array([0.01, -0.01, 0.3, 0.3], np.float32)
    s = Session("3xtf32")
    s.load_weights(w)
    g = torch.Generator().manual_seed(99)
    ip = (torch.rand(1, 6, 192, 256, generator=g) - 0.5).numpy()
    i22 = oops.median3x3_downsample(oops.median3x3_downsample(np.ascontiguousarray(ip[:, 3:6])))
    r0 = BootstrapNet(s, "channels_first", 1).eval(dev(ip), dev(i22))
    torch.cuda.synchronize()
    args = iterative_inputs(ip, i22, r0)
    assert (args[2] <= 0).mean() > 0.05
    ref = OracleNets(w).iterative(*args, full=True)
    assert (ref["flow_from_depth_motion"].numpy() == 0).mean() > 0.05       # NaN / gated pixels
    run_stage(s, "3xtf32", w, "iterative", 1, args)


def l1_rel(a, r):
    return float(np.abs(a - r).sum() / np.abs(r).sum())


@pytest.mark.parametrize("hw,B", [((192, 256), 2), ((200, 300), 2), ((8, 12), 2), ((768, 1024), 1)],
                         ids=["192x256", "200x300", "8x12", "768x1024"])
def test_trace_refinement_sizes(sessions, synthetic_weights, hw, B):
    """The refinement block at sizes other than the pipeline's: per-tap plans with ragged tiles at every level.  At 200x300
    and 8x12 predict_depth0 is also compared with the CPU oracle at test_gpu_network.py's bar (L1-rel 1e-4)."""
    rng = np.random.RandomState(hw[0] + hw[1])
    image1 = rng.uniform(-0.5, 0.5, (B, 3) + hw).astype(np.float32)
    depth2 = rng.uniform(0.2, 0.8, (B, 1, hw[0] // 4, hw[1] // 4)).astype(np.float32)
    out = run_stage(sessions["3xtf32"], "3xtf32", synthetic_weights, "refine", B, (image1, depth2), refine_hw=hw)
    if hw in ((200, 300), (8, 12)):
        ref = OracleNets(synthetic_weights).refine(image1, depth2)["predict_depth0"].numpy()
        assert l1_rel(out["predict_depth0"].cpu().numpy(), ref) < 1e-4


def test_trace_batch64_iterative(synthetic_weights):
    """Batch 64, iterative stage, 3xTF32: the b64 plans and the glue kernels' grid over images.  The bootstrap runs untraced
    to make the iterative stage's inputs; every layer's float64 reference runs on all 64 images, one layer at a time."""
    s = Session("3xtf32")
    s.load_weights(synthetic_weights)
    g = torch.Generator().manual_seed(1234)
    ip = (torch.rand(64, 6, 192, 256, generator=g) - 0.5).numpy()
    i22 = sops.median3x3_downsample(sops.median3x3_downsample(np.ascontiguousarray(ip[:, 3:6])))
    r0 = BootstrapNet(s, "channels_first", 64).eval(dev(ip), dev(i22))
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    run_stage(s, "3xtf32", synthetic_weights, "iterative", 64, iterative_inputs(ip, i22, r0))
    print("\nbatch 64 iterative trace: %.1f s, peak torch allocation %.2f GB"
          % (time.perf_counter() - t0, torch.cuda.max_memory_allocated() / 2 ** 30))


def test_trace_after_staging_and_pipeline_refusal(synthetic_weights, random_pairs):
    """A uint8 host call and a resize call of the fused pipeline leave their staging bytes in concat0, pd0a and c1y (see
    build_plan); the stage-wise layers traced afterwards on the same net must still read zero padding and the oracle's
    inputs.  While a trace is set every pipeline entry refuses (DEMON_E_STATE); clearing the trace restores them."""
    s = Session("3xtf32")
    s.load_weights(synthetic_weights)
    ip, i22 = random_pairs
    pipe = DemonPipeline(s, batch_size=2, iterations=1)
    rng = np.random.RandomState(11)
    u8 = rng.randint(0, 256, (2, 2, 192, 256, 3)).astype(np.uint8)
    d0 = np.empty((2, 1, 192, 256), np.float32)
    rot, tr = np.empty((2, 3), np.float32), np.empty((2, 3), np.float32)
    pipe.forward_host_u8(u8, None, d0, rot, tr)
    big = torch.from_numpy(rng.randint(0, 256, (2, 2, 150, 210, 3)).astype(np.uint8)).cuda()
    pipe.forward_images(big, resample="bilinear", image2_2="resize")
    torch.cuda.synchronize()
    _lib.check_errors()
    run_all_stages(s, "3xtf32", synthetic_weights, ip, i22)
    lib = _lib.load()
    t = Trace(s.net(2), STAGE_SCOPES["refine"])
    try:
        with pytest.raises(RuntimeError, match="error -3"):
            pipe.forward(dev(ip), dev(i22))
        with pytest.raises(RuntimeError, match="error -3"):
            pipe.forward_host_u8(u8, None, d0, rot, tr)
    finally:
        t.close()
    out = pipe.forward(dev(ip), dev(i22))
    torch.cuda.synchronize()
    assert lib.demon_check_errors() == 0
    assert torch.isfinite(out["predict_depth0"]).all()
