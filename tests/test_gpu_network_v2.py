"""GPU: the v2 network (demon_b200.v2.networks over the v2 plan) against the CPU oracle (oracle/network_v2.py), the fused
v2 pipeline against the stage-wise entries, graph replay, batch independence, refinement sizes, the handle-kind checks of
the C ABI, and the layer trace's evidence for what v2 adds: padded channels, dense5's two permutations and the two
concats it feeds."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from demon_b200 import _lib
from demon_b200.v2 import weights as W2
from oracle import ops as oops
from oracle.network_v2 import OracleNetsV2

TOL = 1e-4
BARS = {"fp32": TOL, "3xtf32": TOL, "tf32": 3e-2}   # tf32: single-pass TF32 products (~1e-3 relative per layer)


def l1_rel(a, r):
    return float(np.abs(a - r).sum() / np.abs(r).sum())


def epe(a, r):
    return float(np.sqrt(((a - r) ** 2).sum(axis=1)).mean())


@pytest.fixture(scope="module")
def weights():
    return W2.synthetic_weights(0)


@pytest.fixture(scope="module")
def sessions(weights):
    from demon_b200.v2.networks import Session
    out = {}
    for prec in ("fp32", "3xtf32", "tf32"):
        out[prec] = Session(precision=prec)
        out[prec].load_weights(weights)
    return out


@pytest.fixture(scope="module")
def oracle64(weights):
    return OracleNetsV2(weights, torch.float64)


@pytest.fixture(scope="module")
def pairs():
    g = torch.Generator().manual_seed(4321)
    ip = (torch.rand(2, 6, 192, 256, generator=g) - 0.5).numpy()
    i22 = oops.median3x3_downsample(oops.median3x3_downsample(np.ascontiguousarray(ip[:, 3:6])))
    return ip, i22


def check(out, ref, bar, keys_flow=("predict_flow2", "predict_flow5"), keys_depth=("predict_depth2",),
          keys_other=("predict_normal2", "predict_rotation", "predict_translation")):
    n = lambda t: t.numpy() if hasattr(t, "numpy") else t
    for k in keys_flow:
        assert epe(out[k], n(ref[k])) < bar, (k, epe(out[k], n(ref[k])))
    for k in keys_depth:
        assert l1_rel(out[k], n(ref[k])) < bar, (k, l1_rel(out[k], n(ref[k])))
    for k in keys_other:   # normals: mean absolute error per component; motion: largest absolute error
        err = np.abs(out[k] - n(ref[k]))
        assert (err.mean() if "normal" in k else err.max()) < bar, (k, float(err.mean()), float(err.max()))


@pytest.mark.parametrize("prec", ("fp32", "3xtf32", "tf32"))
def test_stages_against_fp64_oracle(sessions, oracle64, pairs, prec):
    """BootstrapNet, IterativeNet (fed the oracle's bootstrap output) and RefinementNet (fed the oracle's depth2), each
    against the float64 oracle, inside v1's bars."""
    from demon_b200.v2.networks import BootstrapNet, IterativeNet, RefinementNet
    ip, i22 = pairs
    s, bar = sessions[prec], BARS[prec]
    out = BootstrapNet(s, "channels_first", 2).eval(ip, i22)
    ref = oracle64.bootstrap(ip, i22)
    assert set(out) == {"predict_flow5", "predict_flow2", "predict_depth2", "predict_normal2", "predict_rotation", "predict_translation"}
    check(out, ref, bar)
    args = (ip, i22, ref["predict_depth2"].numpy().astype(np.float32), ref["predict_normal2"].numpy().astype(np.float32),
            ref["predict_rotation"].numpy().astype(np.float32), ref["predict_translation"].numpy().astype(np.float32))
    out = IterativeNet(s, "channels_first", 2).eval(*args)
    check(out, oracle64.iterative(*args), bar)
    image1 = np.ascontiguousarray(ip[:, 0:3])
    d2 = args[2]
    o = RefinementNet(s, "channels_first", 2).eval(image1, d2, args[3])
    r = oracle64.refine(image1, d2)
    assert set(o) == {"predict_depth0", "predict_normal0"} and o["predict_normal0"].shape == (2, 3, 192, 256)
    assert l1_rel(o["predict_depth0"], r["predict_depth0"].numpy()) < bar
    assert np.abs(o["predict_normal0"] - r["predict_normal0"].numpy()).mean() < bar


def test_clip_of_depth_from_flow_with_adversarial_weights(weights):
    """Weights that make the bootstrap depth straddle zero, the motion large and the flow contradict it: flow_to_depth
    triangulates near the singularity, and a previous translation shortened 1000-fold puts inverse depths far above 50,
    which v2 clips (v2/blocks.py:379).  The flow
    block only passes through exact ops and must match tightly; the DM block passes through the singular triangulation."""
    from demon_b200.v2.networks import IterativeNet, Session
    w = dict(weights)
    for scope in ("netDM1", "netDM2"):
        w[scope + "/predict_depthnormal2/conv2/bias"] = np.array([0.0, 0, 0, -0.8], np.float32)
        w[scope + "/predict_depthnormal2/conv2/kernel"] = weights[scope + "/predict_depthnormal2/conv2/kernel"] * 5
        w[scope + "/motion_fc3/bias"] = np.array([0.3, -0.2, 0.1, 2.5, 0.5, -0.7, 1.0], np.float32)
    for scope in ("netFlow1", "netFlow2"):
        w[scope + "/predict_flow2/conv2/bias"] = np.array([0.01, -0.01, 0.3, 0.3], np.float32)
    s = Session("3xtf32")
    s.load_weights(w)
    g = torch.Generator().manual_seed(99)
    ip = (torch.rand(1, 6, 192, 256, generator=g) - 0.5).numpy()
    i22 = oops.median3x3_downsample(oops.median3x3_downsample(np.ascontiguousarray(ip[:, 3:6])))
    orc = OracleNetsV2(w)
    r0 = orc.bootstrap(ip, i22)
    # a translation 1000 x shorter than the bootstrap's: the flow now triangulates to tiny depths, inverse depth >> 50
    args = (ip, i22, r0["predict_depth2"].numpy(), r0["predict_normal2"].numpy(), r0["predict_rotation"].numpy(),
            r0["predict_translation"].numpy() * np.float32(1e-3))
    ref = orc.iterative(*args, full=True)
    raw = ref["depth_from_flow_unclipped"].numpy()
    assert (raw > 50).sum() > 0 and (ref["depth_from_flow"].numpy() == 50).sum() == (raw > 50).sum()
    out = IterativeNet(s, "channels_first", 1).eval(*args)
    assert all(np.isfinite(v).all() for v in out.values())
    assert epe(out["predict_flow2"], ref["predict_flow2"].numpy()) < TOL
    assert l1_rel(out["predict_depth2"], ref["predict_depth2"].numpy()) < 0.2


def test_pipeline_equals_stagewise_chain_and_graph_replay(sessions, pairs):
    """demon_pipeline_run on a v2 handle == bootstrap, three iterations and refinement through the stage-wise entries, bit for
    bit; image2_2=None is the median pair; the replayed CUDA graph equals the eager first call, also on new content."""
    from demon_b200.v2.networks import BootstrapNet, DemonPipelineV2, IterativeNet, RefinementNet
    ip, i22 = pairs
    s = sessions["3xtf32"]
    r = BootstrapNet(s, "channels_first", 2).eval(ip, i22)
    it = IterativeNet(s, "channels_first", 2)
    for _ in range(3):
        r = it.eval(ip, i22, r["predict_depth2"], r["predict_normal2"], r["predict_rotation"], r["predict_translation"])
    d0 = RefinementNet(s, "channels_first", 2).eval(np.ascontiguousarray(ip[:, 0:3]), r["predict_depth2"], r["predict_normal2"])
    pipe = DemonPipelineV2(s, batch_size=2, iterations=3)
    x = torch.from_numpy(ip).cuda()
    eager = {k: v.clone() for k, v in pipe.forward(x, None).items()}
    torch.cuda.synchronize()
    got = {k: v.cpu().numpy() for k, v in eager.items()}
    for k in ("predict_flow2", "predict_depth2", "predict_normal2", "predict_rotation", "predict_translation"):
        assert np.array_equal(got[k], r[k]), k
    for k in ("predict_depth0", "predict_normal0"):
        assert np.array_equal(got[k], d0[k]), k
    for _ in range(3):   # capture, replay, replay
        out = pipe.forward(x, None)
    torch.cuda.synchronize()
    for k in eager:
        assert torch.equal(eager[k], out[k]), k
    flipped = torch.flip(x, dims=[0]).contiguous()
    ref = {k: v.clone() for k, v in DemonPipelineV2(s, batch_size=2, iterations=3).forward(flipped, None).items()}   # eager
    out = pipe.forward(flipped, None)                                                                                # replay
    torch.cuda.synchronize()
    for k in eager:
        assert torch.equal(ref[k], out[k]), k
    assert pipe.launches() > 0


def test_batch_64_pairs_equal_their_batch_1_results(sessions, weights):
    """Every pair of a batch of 64 comes out as it does alone (up to the tensor-core path's tile-dependent summation order,
    as for v1) and one of them is inside the bar against the float64 oracle's pipeline."""
    from demon_b200.v2.networks import DemonPipelineV2
    g = torch.Generator().manual_seed(1234)
    ip = torch.rand(64, 6, 192, 256, generator=g) - 0.5
    s = sessions["3xtf32"]
    a = {k: v.clone() for k, v in DemonPipelineV2(s, batch_size=64).forward(ip.cuda()).items()}
    torch.cuda.synchronize()
    for k in a:
        assert torch.isfinite(a[k]).all(), k
    one = DemonPipelineV2(s, batch_size=1)
    for i in (0, 37, 63):
        o = one.forward(ip[i:i + 1].cuda())
        torch.cuda.synchronize()
        assert l1_rel(o["predict_depth0"][0].cpu().numpy(), a["predict_depth0"][i].cpu().numpy()) < 2e-6, i
        np.testing.assert_allclose(o["predict_translation"][0].cpu().numpy(), a["predict_translation"][i].cpu().numpy(), atol=2e-6)
    ipn = ip[37:38].numpy()
    i22 = oops.median3x3_downsample(oops.median3x3_downsample(np.ascontiguousarray(ipn[:, 3:6])))
    ref = OracleNetsV2(weights, torch.float64).pipeline(ipn, i22)
    got = {k: v[37:38].cpu().numpy() for k, v in a.items()}
    assert l1_rel(got["predict_depth0"], ref["predict_depth0"].numpy()) < TOL
    assert l1_rel(got["predict_depth2"], ref["predict_depth2"].numpy()) < TOL
    assert epe(got["predict_flow2"], ref["predict_flow2"].numpy()) < TOL
    np.testing.assert_allclose(got["predict_translation"], ref["predict_translation"].numpy(), atol=1e-5)


@pytest.mark.parametrize("hw", ((192, 256), (200, 300), (768, 1024)))
def test_refinement_sizes(sessions, weights, hw):
    """The v2 refinement block at 256x192, at 300x200 (odd 50x75 at its coarsest level) and at 1024x768, against the
    float32 oracle (one image; the oracle takes ~10 s at 1024x768)."""
    from demon_b200.v2.networks import RefinementNet
    H, W_ = hw
    rng = np.random.RandomState(H)
    image1 = rng.uniform(-0.5, 0.5, (1, 3, H, W_)).astype(np.float32)
    depth2 = rng.uniform(0.2, 0.8, (1, 1, H // 4, W_ // 4)).astype(np.float32)
    o = RefinementNet(sessions["3xtf32"], "channels_first", 1, image_size=hw).eval(image1, depth2, None)
    r = OracleNetsV2(weights).refine(image1, depth2)
    assert o["predict_depth0"].shape == (1, 1, H, W_) and o["predict_normal0"].shape == (1, 3, H, W_)
    assert l1_rel(o["predict_depth0"], r["predict_depth0"].numpy()) < TOL
    assert np.abs(o["predict_normal0"] - r["predict_normal0"].numpy()).mean() < TOL


def test_stage_entries_refuse_the_other_kind_and_the_pipeline_takes_both(sessions, weights, pairs):
    """v1 forward entries refuse a v2 handle and v2 entries a v1 handle (DEMON_E_INVALID); the fused pipeline takes both and
    refuses what only v2 has on a v1 handle (normal0, image2_2_mode 2); the variable table, describe, trace and profile
    entries take both."""
    from demon_b200.networks_original import Session as SessionV1
    from demon_b200 import weights as W1
    lib = _lib.load()
    v2 = sessions["3xtf32"].net(1)
    s1 = SessionV1("3xtf32")
    s1.load_weights(W1.synthetic_weights(0))
    v1 = s1.net(1)
    assert lib.demon_net_variant(v2.ptr) == 2 and lib.demon_net_variant(v1.ptr) == 1
    assert v2.variable_names() == list(W2.variable_specs().keys())
    x = torch.zeros(1, 6, 192, 256, device="cuda")
    i2 = torch.zeros(1, 3, 48, 64, device="cuda")
    o = [torch.zeros(1, 8, 192, 256, device="cuda") for _ in range(7)]
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    assert lib.demon_bootstrap_forward(v2.ptr, x.data_ptr(), i2.data_ptr(), *(t.data_ptr() for t in o[:6]), 0, s) == -1
    assert lib.demon_refine_forward(v2.ptr, x.data_ptr(), i2.data_ptr(), o[0].data_ptr(), 0, s) == -1
    assert lib.demon_bootstrap_forward_v2(v1.ptr, x.data_ptr(), i2.data_ptr(), *(t.data_ptr() for t in o[:6]), 0, s) == -1
    outs = dict(zip(("depth0", "normal0", "rotation", "translation", "flow2", "depth2", "normal2"), (t.data_ptr() for t in o)))
    assert lib.demon_pipeline_run(v1.ptr, _lib.PipelineArgs(input=_lib.INPUT_F32, images=x.data_ptr(), iterations=1, **outs), s) == -1
    del outs["normal0"]
    assert lib.demon_pipeline_run(v1.ptr, _lib.PipelineArgs(input=_lib.INPUT_F32, images=x.data_ptr(), image2_2_mode=2, iterations=1,
                                                            **outs), s) == -1
    assert lib.demon_refine_forward_v2(v1.ptr, x.data_ptr(), i2.data_ptr(), None, o[0].data_ptr(), None, 0, s) == -1
    buf = ctypes.create_string_buffer(1 << 20)
    assert lib.demon_debug_describe_layers(v2.ptr, buf, len(buf)) > 0
    ref = ctypes.create_string_buffer(1 << 20)
    lib.demon_debug_describe_plan(2, 1, 192, 256, 1, ref, len(ref))
    assert buf.value.split(b"\n")[0].split(b" : ")[:2] == ref.value.split(b"\n")[0].split(b" : ")[:2]
    _lib.check(lib.demon_net_profile_begin(v2.ptr))
    from demon_b200.v2.networks import BootstrapNet
    BootstrapNet(sessions["3xtf32"], "channels_first", 1).eval(pairs[0][:1], pairs[1][:1])
    torch.cuda.synchronize()
    _lib.check(lib.demon_net_profile_end(v2.ptr))
    ms, calls, launches = ctypes.c_double(), ctypes.c_int64(), ctypes.c_int()
    names = [lib.demon_net_layer_name(v2.ptr, i).decode() for i in range(lib.demon_net_num_layers(v2.ptr))]
    i = names.index("netFlow1/dense5")
    _lib.check(lib.demon_net_layer_profile(v2.ptr, i, ctypes.byref(ms), ctypes.byref(calls), ctypes.byref(launches), None))
    assert calls.value == 1 and ms.value > 0 and launches.value == 4   # gather, dense, split-K reduction, scatter


def test_layer_trace_padding_dense5_and_concats(sessions, weights, pairs):
    """The layer trace on the v2 stage-wise entries: the padded channels of the y halves the x convs read are exactly zero;
    dense5's input is conv5_1's first 96 channels in the buffer's pixel-major order, its output lands in channels 384..479
    of conv5_1_dense5 as TF's reshape [96,6,8] puts it, and motion_fc1 reads motion_conv5a ++ motion_conv5b; all bit for
    bit.  dense5's output is also checked against the float64 dense layer of its own traced input (the oracle's
    permutations), inside the per-element bound of the trace test."""
    from demon_b200.v2.networks import BootstrapNet, IterativeNet
    lib = _lib.load()
    s = sessions["3xtf32"]
    net = s.net(2)
    L = lib.demon_net_num_layers(net.ptr)
    names = [lib.demon_net_layer_name(net.ptr, i).decode() for i in range(L)]
    buf = ctypes.create_string_buffer(1 << 20)
    lib.demon_debug_describe_layers(net.ptr, buf, len(buf))
    geo = {}
    for line in buf.value.decode().splitlines():
        nm, rest = line.split(None, 1)
        toks = rest.split(" : ")[0].split()
        geo[nm] = dict(zip(toks[1::2], map(int, toks[2::2])), kind=toks[0])

    def shape(nm, inp):
        g = geo[nm]
        if g["kind"] == "dense":
            return (2, g["cin_buf"] if inp else g["cout"])
        if inp:
            return (2, g["H"], g["W"], g["cin_buf"])
        if g["kind"] == "deconv":
            return (2, 2 * g["H"], 2 * g["W"], g["cout"])
        return (2, -(-g["H"] // g["sy"]), -(-g["W"] // g["sx"]), g["cout"])

    tin = [torch.full(shape(n, True), float("nan"), device="cuda") for n in names]
    tout = [torch.full(shape(n, False), float("nan"), device="cuda") for n in names]
    pin = (ctypes.c_void_p * L)(*[t.data_ptr() for t in tin])
    pout = (ctypes.c_void_p * L)(*[t.data_ptr() for t in tout])
    ip, i22 = pairs
    _lib.check(lib.demon_debug_trace_layers(net.ptr, pin, pout))
    try:
        r = BootstrapNet(s, "channels_first", 2).eval(ip, i22)
        IterativeNet(s, "channels_first", 2).eval(ip, i22, r["predict_depth2"], r["predict_normal2"], r["predict_rotation"],
                                                   r["predict_translation"])
        torch.cuda.synchronize()
    finally:
        lib.demon_debug_trace_layers(net.ptr, None, None)
    T = lambda n, inp: (tin if inp else tout)[names.index(n)].cpu().numpy()
    for scope in ("netFlow1", "netDM1", "netFlow2", "netDM2"):
        x1 = T(scope + "/conv1x", True)
        assert np.isfinite(x1).all() and (x1[..., 24:] == 0).all()
        assert np.array_equal(x1[..., :24], T(scope + "/conv1y", False))
        x2 = T(scope + "/conv2x", True)
        c2 = 48 if scope == "netFlow1" else 32
        assert x2.shape[-1] == (64 if scope == "netFlow1" else 32) and (x2[..., c2:] == 0).all()
        assert np.array_equal(x2[..., :c2], T(scope + "/conv2y", False))
        c51 = T(scope + "/conv5_1x", False)                                        # [B,6,8,384]
        d_in = T(scope + "/dense5", True)                                          # [B,4608]
        assert np.array_equal(d_in, c51[..., :96].reshape(2, -1))
        d_out = T(scope + "/dense5", False)
        k = weights[scope + "/dense5/kernel"].astype(np.float64)
        b = weights[scope + "/dense5/bias"].astype(np.float64)
        nchw_in = d_in.reshape(2, 48, 96).transpose(0, 2, 1).reshape(2, -1).astype(np.float64)   # TF's flatten of [96,6,8]
        y = nchw_in @ k + b
        y = np.maximum(0.1 * y, y).reshape(2, 96, 48).transpose(0, 2, 1).reshape(2, -1)           # TF's reshape, in pixel order
        assert np.abs(d_out - y).max() <= 1e-4 * max(1.0, np.abs(y).max())
        c5d = T(scope + ("/predict_flow5/conv1" if "Flow" in scope else "/motion_conv5b"), True)   # [B,6,8,480]
        assert np.array_equal(c5d[..., :384], c51)
        assert np.array_equal(c5d[..., 384:], d_out.reshape(2, 6, 8, 96))
        if "DM" in scope:
            fc1 = T(scope + "/motion_fc1", True).reshape(2, 6, 8, 128)
            assert np.array_equal(fc1[..., :64], T(scope + "/motion_conv5ax", False))
            assert np.array_equal(fc1[..., 64:], T(scope + "/motion_conv5b", False))
            assert np.array_equal(T(scope + "/refine4/upconv", True), c51)
    # the clip: channel 7 of netDM2's extra inputs lies in [0, 50]
    ex = T("netDM2/conv2_extra_inputsy", True)
    assert (ex[..., 7] >= 0).all() and (ex[..., 7] <= 50).all() and (ex[..., 8:] == 0).all()


def test_channels_last_equals_channels_first(sessions, pairs):
    """data_format is a boundary transpose for the v2 entries too, normal0's export included."""
    from demon_b200.v2.networks import BootstrapNet, RefinementNet
    ip, i22 = pairs
    s = sessions["3xtf32"]
    a = BootstrapNet(s, "channels_first", 2).eval(ip, i22)
    b = BootstrapNet(s, "channels_last", 2).eval(np.ascontiguousarray(ip.transpose(0, 2, 3, 1)), np.ascontiguousarray(i22.transpose(0, 2, 3, 1)))
    for k in ("predict_flow5", "predict_flow2", "predict_depth2", "predict_normal2"):
        assert np.array_equal(a[k], b[k].transpose(0, 3, 1, 2)), k
    image1 = np.ascontiguousarray(ip[:, 0:3])
    ra = RefinementNet(s, "channels_first", 2).eval(image1, a["predict_depth2"], a["predict_normal2"])
    rb = RefinementNet(s, "channels_last", 2).eval(np.ascontiguousarray(image1.transpose(0, 2, 3, 1)), b["predict_depth2"], b["predict_normal2"])
    assert rb["predict_normal0"].shape == (2, 192, 256, 3)
    for k in ("predict_depth0", "predict_normal0"):
        assert np.array_equal(ra[k], rb[k].transpose(0, 3, 1, 2)), k
