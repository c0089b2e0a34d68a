"""GPU: the network graphs through the C ABI (via the networks_original mirror) against the CPU oracle.

The north-star bar: inverse-depth L1-rel <= 1e-4 on predict_depth0 and flow EPE <= 1e-4 on predict_flow2
(normalized units), measured against the fp32 CPU oracle; the fp64 oracle distance is checked too."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from demon_b200 import weights as W
from oracle import ops as oops
from oracle.network import OracleNets

TOL = 1e-4


def l1_rel(a, r):
    """l1 relative error on inverse depth (python/depthmotionnet/evaluation/metrics.py:62-81,151-170 family)."""
    return float(np.abs(a - r).sum() / np.abs(r).sum())


def epe(a, r):
    """compute_flow_epe, python/depthmotionnet/evaluation/metrics.py:377-387."""
    return float(np.sqrt(((a - r) ** 2).sum(axis=1)).mean())


def demeaned_rel(a, r):
    """stricter: error relative to the spatially varying part of the signal"""
    return float(np.abs(a - r).sum() / np.abs(r - r.mean()).sum())


@pytest.fixture(scope="module")
def sessions(synthetic_weights):
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    from demon_b200.networks_original import Session
    out = {}
    for prec in ("fp32", "3xtf32"):
        s = Session(precision=prec)
        s.load_weights(synthetic_weights)
        out[prec] = s
    return out


@pytest.fixture(scope="module")
def oracle32(synthetic_weights):
    return OracleNets(synthetic_weights)


@pytest.fixture(scope="module")
def oracle64(synthetic_weights):
    return OracleNets(synthetic_weights, torch.float64)


def check_predictions(out, ref32, ref64, keys_flow=("predict_flow2",), keys_depth=("predict_depth2",)):
    """The bar (north star): <= 1e-4 against the fp32 CPU path.  The fp32 path itself sits up to ~1e-4 from the
    exact result on inputs where flow_to_depth is ill conditioned (tests/test_gpu_ops.py:
    test_flow_to_depth_matches_oracle), so the assertion is: within TOL of the fp64 oracle, and within
    TOL + 2 x (fp32 oracle's own distance to the fp64 oracle) of the fp32 oracle."""
    n = lambda t: t.numpy() if hasattr(t, "numpy") else t
    for k in keys_flow:
        own = epe(n(ref32[k]), n(ref64[k]))
        assert epe(out[k], n(ref64[k])) < TOL, k
        assert epe(out[k], n(ref32[k])) < TOL + 2 * own, k
    for k in keys_depth:
        own = l1_rel(n(ref32[k]), n(ref64[k]))
        assert l1_rel(out[k], n(ref64[k])) < TOL, k
        assert l1_rel(out[k], n(ref32[k])) < TOL + 2 * own, k
    for k in ("predict_rotation", "predict_translation"):
        if k in out:
            own = float(np.abs(n(ref32[k]) - n(ref64[k])).max())
            np.testing.assert_allclose(out[k], n(ref64[k]), atol=1e-5)
            np.testing.assert_allclose(out[k], n(ref32[k]), atol=1e-5 + 2 * own)


@pytest.fixture(scope="module")
def random_pairs():
    g = torch.Generator().manual_seed(1234)      # SURVEY.md section 8d config 3 generator
    ip = (torch.rand(2, 6, 192, 256, generator=g) - 0.5).numpy()
    i22 = oops.median3x3_downsample(oops.median3x3_downsample(np.ascontiguousarray(ip[:, 3:6])))
    return ip, i22


def test_variable_table_agrees_with_python_table(sessions):
    net = sessions["fp32"].net(1)
    assert net.variable_names() == list(W.variable_specs().keys())


def test_tensor_core_path_is_selected_for_the_big_layers(sessions):
    net = sessions["3xtf32"].net(1)
    for layer in ("netRefine/conv1_1", "netFlow1/conv3x", "netDM2/refine3/upconv", "netRefine/refine0/upconv", "netFlow1/conv1y",
                  "netRefine/conv0", "netDM1/conv2_extra_inputsy", "netFlow2/conv2_extra_inputsy"):   # (7..9 channels in a 32-channel pixel)
        assert net.uses_tensor_cores(layer), layer
    for layer in ("netDM1/motion_fc1", "netRefine/predict_depth0/conv2", "netFlow2/predict_flow2/conv2"):
        assert not net.uses_tensor_cores(layer), layer
    assert not sessions["fp32"].net(1).uses_tensor_cores("netRefine/conv1_1")


@pytest.mark.parametrize("prec", ("fp32", "3xtf32"))
def test_bootstrap_on_sculpture_pair(sessions, oracle32, sculpture, prec):
    """BASELINE.json configs[1], first stage."""
    from demon_b200.networks_original import BootstrapNet
    out = BootstrapNet(sessions[prec], "channels_first", 1).eval(sculpture["image_pair"], sculpture["image2_2"])
    ref = oracle32.bootstrap(sculpture["image_pair"], sculpture["image2_2"])
    assert set(out) == {"predict_flow5", "predict_flow2", "predict_depth2", "predict_normal2", "predict_rotation", "predict_translation"}
    for k in out:
        assert out[k].shape == tuple(ref[k].shape), k
    assert epe(out["predict_flow2"], ref["predict_flow2"].numpy()) < TOL
    assert epe(out["predict_flow5"], ref["predict_flow5"].numpy()) < TOL
    assert l1_rel(out["predict_depth2"], ref["predict_depth2"].numpy()) < TOL
    np.testing.assert_allclose(out["predict_normal2"], ref["predict_normal2"].numpy(), atol=1e-4)
    np.testing.assert_allclose(out["predict_rotation"], ref["predict_rotation"].numpy(), atol=1e-5)
    np.testing.assert_allclose(out["predict_translation"], ref["predict_translation"].numpy(), atol=1e-5)


@pytest.mark.parametrize("prec", ("fp32", "3xtf32"))
def test_iterative_and_refine_stage_by_stage(sessions, oracle32, oracle64, random_pairs, prec):
    """Each eval() fed with the ORACLE's previous outputs: isolates every stage (networks_original.py:154-255)."""
    from demon_b200.networks_original import IterativeNet, RefinementNet
    ip, i22 = random_pairs
    r0 = oracle32.bootstrap(ip, i22)
    args = (ip, i22, r0["predict_depth2"].numpy(), r0["predict_normal2"].numpy(), r0["predict_rotation"].numpy(),
            r0["predict_translation"].numpy())
    out = IterativeNet(sessions[prec], "channels_first", 2).eval(*args)
    ref, ref64 = oracle32.iterative(*args), oracle64.iterative(*args)
    check_predictions(out, ref, ref64)
    image1 = np.ascontiguousarray(ip[:, 0:3])
    d2 = ref["predict_depth2"].numpy()
    o = RefinementNet(sessions[prec], "channels_first", 2).eval(image1, d2)
    r = oracle32.refine(image1, d2)
    assert o["predict_depth0"].shape == (2, 1, 192, 256)
    assert l1_rel(o["predict_depth0"], r["predict_depth0"].numpy()) < TOL
    assert demeaned_rel(o["predict_depth0"], r["predict_depth0"].numpy()) < 10 * TOL


def test_channels_last_equals_channels_first(sessions, random_pairs):
    """data_format is a pure boundary transpose (networks_original.py:37-42)."""
    from demon_b200.networks_original import BootstrapNet, RefinementNet
    ip, i22 = random_pairs
    s = sessions["3xtf32"]
    a = BootstrapNet(s, "channels_first", 2).eval(ip, i22)
    b = BootstrapNet(s, "channels_last", 2).eval(np.ascontiguousarray(ip.transpose(0, 2, 3, 1)), np.ascontiguousarray(i22.transpose(0, 2, 3, 1)))
    assert b["predict_flow2"].shape == (2, 48, 64, 2) and b["predict_normal2"].shape == (2, 48, 64, 3)
    for k in ("predict_flow5", "predict_flow2", "predict_depth2", "predict_normal2"):
        assert np.array_equal(a[k], b[k].transpose(0, 3, 1, 2)), k
    assert np.array_equal(a["predict_rotation"], b["predict_rotation"])
    image1 = np.ascontiguousarray(ip[:, 0:3])
    ra = RefinementNet(s, "channels_first", 2).eval(image1, a["predict_depth2"])
    rb = RefinementNet(s, "channels_last", 2).eval(np.ascontiguousarray(image1.transpose(0, 2, 3, 1)), b["predict_depth2"])
    assert np.array_equal(ra["predict_depth0"], rb["predict_depth0"].transpose(0, 3, 1, 2))


@pytest.mark.parametrize("prec", ("fp32", "3xtf32"))
def test_full_pipeline_against_oracle_and_golden(sessions, oracle32, sculpture, golden_dir, prec):
    """BASELINE.json configs[1]: full pipeline batch 1 on the sculpture pair vs the CPU path, and vs the
    committed golden outputs (fp32 and fp64 oracle)."""
    from demon_b200.networks_original import DemonPipeline
    pipe = DemonPipeline(sessions[prec], batch_size=1, iterations=3)
    out = pipe.forward(torch.from_numpy(sculpture["image_pair"]).cuda(), torch.from_numpy(sculpture["image2_2"]).cuda())
    torch.cuda.synchronize()
    out = {k: v.cpu().numpy() for k, v in out.items()}
    g = np.load(os.path.join(golden_dir, "oracle_pipeline.npz"))
    for sfx in ("_f32", "_f64"):
        assert l1_rel(out["predict_depth0"], g["predict_depth0" + sfx]) < TOL
        assert epe(out["predict_flow2"], g["predict_flow2" + sfx]) < TOL
        assert l1_rel(out["predict_depth2"], g["predict_depth2" + sfx]) < TOL
        np.testing.assert_allclose(out["predict_rotation"], g["predict_rotation" + sfx], atol=1e-5)
        np.testing.assert_allclose(out["predict_translation"], g["predict_translation" + sfx], atol=1e-5)
    print("\n[%s] depth0 L1-rel vs fp64 oracle %.3e (de-meaned %.3e), flow EPE %.3e" % (
        prec, l1_rel(out["predict_depth0"], g["predict_depth0_f64"]), demeaned_rel(out["predict_depth0"], g["predict_depth0_f64"]),
        epe(out["predict_flow2"], g["predict_flow2_f64"])))
    assert pipe.launches() > 0


def test_pipeline_matches_stagewise_api_and_median_image2_2(sessions, random_pairs):
    """The fused pipeline == the five eval() calls of examples/example.py:87-99, bit for bit; image2_2=None
    reproduces median3x3_downsample twice (examples/evaluation.py:170-173)."""
    from demon_b200.networks_original import BootstrapNet, IterativeNet, RefinementNet, DemonPipeline
    ip, i22 = random_pairs
    s = sessions["3xtf32"]
    r = BootstrapNet(s, "channels_first", 2).eval(ip, i22)
    it = IterativeNet(s, "channels_first", 2)
    for _ in range(3):
        r = it.eval(ip, i22, r["predict_depth2"], r["predict_normal2"], r["predict_rotation"], r["predict_translation"])
    d0 = RefinementNet(s, "channels_first", 2).eval(np.ascontiguousarray(ip[:, 0:3]), r["predict_depth2"])["predict_depth0"]
    pipe = DemonPipeline(s, batch_size=2, iterations=3)
    out = pipe.forward(torch.from_numpy(ip).cuda(), None)
    torch.cuda.synchronize()
    assert np.array_equal(out["predict_depth0"].cpu().numpy(), d0)
    assert np.array_equal(out["predict_flow2"].cpu().numpy(), r["predict_flow2"])
    assert np.array_equal(out["predict_rotation"].cpu().numpy(), r["predict_rotation"])
    # host-buffer entry (the e2e path of bench.py)
    hp = torch.from_numpy(ip).pin_memory()
    d0h = torch.empty(2, 1, 192, 256).pin_memory()
    rot, tr = torch.empty(2, 3).pin_memory(), torch.empty(2, 3).pin_memory()
    pipe.forward_host(hp, None, d0h, rot, tr)
    assert np.array_equal(d0h.numpy(), d0) and np.array_equal(rot.numpy(), r["predict_rotation"])
    # async entry, two pipelines (own workspaces) in flight on two streams: same bits
    pipes = [pipe, DemonPipeline(s, batch_size=2, iterations=3, private_net=True)]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    outs = [(torch.zeros(2, 1, 192, 256).pin_memory(), torch.zeros(2, 3).pin_memory(), torch.zeros(2, 3).pin_memory())
            for _ in range(2)]
    for i in range(6):
        k = i % 2
        streams[k].synchronize()
        pipes[k].forward_host_async(hp, None, *outs[k], stream=streams[k])
    torch.cuda.synchronize()
    for k in range(2):
        assert np.array_equal(outs[k][0].numpy(), d0) and np.array_equal(outs[k][2].numpy(), r["predict_translation"])


def test_uint8_entry_equals_fp32_entry_bit_for_bit(sessions, synthetic_weights):
    """SURVEY.md section 8(f2): uint8 images in, `/255 - 0.5` + pair concat + median on the device.  On the repository's own
    sculpture pair (examples/sculpture{1,2}.png, examples/example.py:15-42) and on random bytes the outputs must equal
    those of the fp32 entry fed with numpy's float32 conversion, with image2_2 given (the resized image) and computed."""
    import os
    from demon_b200.networks_original import DemonPipeline
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sculpture_inputs.npz"))
    rng = np.random.RandomState(5)
    rnd = rng.randint(0, 256, (2, 192, 256, 3)).astype(np.uint8)
    u8 = np.stack([np.stack([z["img1"], z["img2"]]).astype(np.uint8), rnd])                          # [2,2,192,256,3]
    i22_u8 = np.stack([z["img2_2"].astype(np.uint8), rnd[1, 2::4, 2::4]])                             # [2,48,64,3]
    f = lambda a: a.astype(np.float32) / 255 - 0.5                                                    # example.py:25-27
    pair = np.concatenate([f(u8[:, 0]).transpose(0, 3, 1, 2), f(u8[:, 1]).transpose(0, 3, 1, 2)], axis=1)
    i22 = f(i22_u8).transpose(0, 3, 1, 2)
    pipe = DemonPipeline(sessions["3xtf32"], batch_size=2, iterations=3)
    for with_i22 in (True, False):
        ref = {k: v.clone() for k, v in pipe.forward(torch.from_numpy(pair).cuda(), torch.from_numpy(i22).cuda() if with_i22 else None).items()}
        got = pipe.forward_u8(torch.from_numpy(u8).cuda(), torch.from_numpy(i22_u8).cuda() if with_i22 else None)
        torch.cuda.synchronize()
        for k in ref:
            assert torch.equal(ref[k], got[k]), (k, with_i22)
    # host entry: bytes in, depth out
    d0 = np.empty((2, 1, 192, 256), np.float32); rot = np.empty((2, 3), np.float32); tr = np.empty((2, 3), np.float32)
    pipe.forward_host_u8(u8, None, d0, rot, tr)
    assert np.array_equal(d0, ref["predict_depth0"].cpu().numpy()) and np.array_equal(tr, ref["predict_translation"].cpu().numpy())


def test_cuda_graph_replay_equals_eager(sessions, random_pairs):
    """demon_pipeline_run replays a CUDA graph from the third call with the same pointer arguments on; the result
    must equal the eager first call bit for bit, also after the input buffer's CONTENT changes."""
    from demon_b200.networks_original import DemonPipeline
    ip, i22 = random_pairs
    pipe = DemonPipeline(sessions["3xtf32"], batch_size=2, iterations=3)
    x = torch.from_numpy(ip).cuda()
    x2 = torch.from_numpy(i22).cuda()
    eager = {k: v.clone() for k, v in pipe.forward(x, x2).items()}          # fresh outputs -> eager
    outs = {k: torch.empty_like(v) for k, v in eager.items()}
    for _ in range(4):                                                       # eager, capture, replay, replay
        pipe.forward(x, x2, outs)
    torch.cuda.synchronize()
    for k in eager:
        assert torch.equal(eager[k], outs[k]), k
    flipped = torch.flip(x, dims=[0]).contiguous()
    ref = {k: v.clone() for k, v in pipe.forward(flipped, torch.flip(x2, dims=[0]).contiguous()).items()}
    x.copy_(flipped); x2.copy_(torch.flip(x2, dims=[0]))
    pipe.forward(x, x2, outs)                                                # replay on new content
    torch.cuda.synchronize()
    for k in ref:
        assert torch.equal(ref[k], outs[k]), k


def test_batch_consistency_and_determinism_at_benchmark_batch(sessions, synthetic_weights):
    """BASELINE.json configs[2] size (batch 64): two runs are bit identical; every sample equals the batch-1
    result of the same pair (pairs are independent, blocks_original.py has no cross-sample op) up to fp32
    rounding -- the tensor-core path picks its N tile, and with it how the 3xTF32 terms are summed, from the
    number of tiles a layer has, so different batch sizes are not bit identical; and a sample checked against the
    CPU oracle is inside the tolerance."""
    from demon_b200.networks_original import DemonPipeline
    g = torch.Generator().manual_seed(1234)
    ip = (torch.rand(64, 6, 192, 256, generator=g) - 0.5)
    s = sessions["3xtf32"]
    pipe = DemonPipeline(s, batch_size=64, iterations=3)
    x = ip.cuda()
    a = {k: v.clone() for k, v in pipe.forward(x, None).items()}
    b = pipe.forward(x, None)
    torch.cuda.synchronize()
    for k in a:
        assert torch.equal(a[k], b[k]), k
        assert torch.isfinite(a[k]).all(), k
    one = DemonPipeline(s, batch_size=1, iterations=3)
    for i in (0, 37, 63):
        o = one.forward(x[i:i + 1], None)
        torch.cuda.synchronize()
        assert l1_rel(o["predict_depth0"][0].cpu().numpy(), a["predict_depth0"][i].cpu().numpy()) < 2e-6, i
        np.testing.assert_allclose(o["predict_translation"][0].cpu().numpy(), a["predict_translation"][i].cpu().numpy(), atol=2e-6)
    i = 37
    ipn = ip[i:i + 1].numpy()
    i22 = oops.median3x3_downsample(oops.median3x3_downsample(np.ascontiguousarray(ipn[:, 3:6])))
    ref = OracleNets(synthetic_weights).pipeline(ipn, i22)
    ref64 = OracleNets(synthetic_weights, torch.float64).pipeline(ipn, i22)
    got = {k: v[i:i + 1].cpu().numpy() for k, v in a.items()}
    check_predictions(got, ref, ref64, keys_depth=("predict_depth0", "predict_depth2"))


def test_adversarial_weights_exercise_invalid_geometry_branches(synthetic_weights):
    """Weights that make the previous depth straddle zero and the motion large: depth_to_flow yields NaN, the
    |flow| < 1 gate (blocks_original.py:165-168) zeroes it, warp2d leaves the image, flow_to_depth triangulates
    behind the camera (-> 0) or near the singularity.  netFlow2's output only passes through the EXACT ops
    (depth_to_flow, gate, warp2d), so it must still match tightly.  netDM2's passes through the singular
    triangulation, where the reference function itself amplifies float rounding of its own flow to percent level
    (see demon_b200/weights.py: synthetic_weights) -- there only finiteness and a loose bound are asserted."""
    from demon_b200.networks_original import Session, IterativeNet
    w = dict(synthetic_weights)
    for scope in ("netDM1", "netDM2"):
        w[scope + "/predict_depthnormal2/conv2/bias"] = np.array([0.0, 0, 0, -0.8], np.float32)      # depth straddles 0
        w[scope + "/predict_depthnormal2/conv2/kernel"] = synthetic_weights[scope + "/predict_depthnormal2/conv2/kernel"] * 5
        w[scope + "/motion_fc3/bias"] = np.array([0.3, -0.2, 0.1, 2.5, 0.5, -0.7, 1.0], np.float32)  # large motion
    for scope in ("netFlow1", "netFlow2"):
        w[scope + "/predict_flow2/conv2/bias"] = np.array([0.01, -0.01, 0.3, 0.3], np.float32)       # flow contradicts the motion
    s = Session("3xtf32")
    s.load_weights(w)
    g = torch.Generator().manual_seed(99)
    ip = (torch.rand(1, 6, 192, 256, generator=g) - 0.5).numpy()
    i22 = oops.median3x3_downsample(oops.median3x3_downsample(np.ascontiguousarray(ip[:, 3:6])))
    orc = OracleNets(w)
    r0 = orc.bootstrap(ip, i22)
    assert (r0["predict_depth2"].numpy() <= 0).mean() > 0.05
    args = (ip, i22, r0["predict_depth2"].numpy(), r0["predict_normal2"].numpy(), r0["predict_rotation"].numpy(),
            r0["predict_translation"].numpy())
    ref = orc.iterative(*args, full=True)
    assert (ref["flow_from_depth_motion"].numpy() == 0).mean() > 0.05       # NaN / gated pixels
    out = IterativeNet(s, "channels_first", 1).eval(*args)
    assert all(np.isfinite(v).all() for v in out.values())
    assert epe(out["predict_flow2"], ref["predict_flow2"].numpy()) < TOL
    assert epe(out["predict_flow5"], ref["predict_flow5"].numpy()) < TOL
    assert l1_rel(out["predict_depth2"], ref["predict_depth2"].numpy()) < 0.2


def test_refinement_at_1024x768_batch_8_equals_eight_single_images(sessions):
    """BASELINE.json configs[4] at its own batch size: RefinementNet at 1024x768, batch 8.  The oracle takes ~10 s per such
    image, so the CPU comparison stays at one image (next test); here every image of the batch must come out as it does
    alone (images are independent: same kernels, same per-pixel arithmetic, only the tile -> CTA assignment changes)."""
    from demon_b200.networks_original import RefinementNet
    rng = np.random.RandomState(5)
    image1 = rng.uniform(-0.5, 0.5, (8, 3, 768, 1024)).astype(np.float32)
    depth2 = rng.uniform(0.2, 0.8, (8, 1, 192, 256)).astype(np.float32)
    o8 = RefinementNet(sessions["3xtf32"], "channels_first", 8, image_size=(768, 1024)).eval(image1, depth2)["predict_depth0"]
    assert o8.shape == (8, 1, 768, 1024) and np.isfinite(o8).all()
    one = RefinementNet(sessions["3xtf32"], "channels_first", 1, image_size=(768, 1024))
    for i in (0, 3, 7):
        o1 = one.eval(image1[i:i + 1], depth2[i:i + 1])["predict_depth0"]
        assert np.abs(o8[i:i + 1] - o1).max() <= 1e-6 * max(1.0, np.abs(o1).max()), i
    from demon_b200 import _lib
    assert _lib.load().demon_debug_tc_timeouts() == 0


def test_refinement_at_1024x768(sessions, synthetic_weights):
    """BASELINE.json configs[4]: RefinementNet at 1024x768, one image against the CPU oracle (which takes ~10 s per image)."""
    from demon_b200.networks_original import RefinementNet
    rng = np.random.RandomState(4)
    image1 = rng.uniform(-0.5, 0.5, (1, 3, 768, 1024)).astype(np.float32)
    depth2 = rng.uniform(0.2, 0.8, (1, 1, 192, 256)).astype(np.float32)
    o = RefinementNet(sessions["3xtf32"], "channels_first", 1, image_size=(768, 1024)).eval(image1, depth2)
    r = OracleNets(synthetic_weights).refine(image1, depth2)
    assert o["predict_depth0"].shape == (1, 1, 768, 1024)
    assert l1_rel(o["predict_depth0"], r["predict_depth0"].numpy()) < TOL
