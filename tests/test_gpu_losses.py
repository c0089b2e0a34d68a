"""DeMoN v2's training losses on the device (demon_b200.v2.losses, csrc/losses.cu) against the mirror ops and the numpy
oracle (oracle/losses.py, itself pinned to the reference's losses.py by tests/test_losses.py)."""
import gc
import importlib.util
import math
import os

import numpy as np
import pytest
import torch

from demon_b200 import _lib
from demon_b200 import lmbspecialops as sops
from demon_b200.v2 import losses as L
from oracle import losses as OL

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
_spec = importlib.util.spec_from_file_location("make_losses_golden", os.path.join(GOLDEN, "make_losses_golden.py"))
GEN = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(GEN)


@pytest.fixture(scope="module", autouse=True)
def leave_the_device_idle():
    """Later modules (tests/test_gpu_op_paths.py) trace kernels with torch.profiler in this process: leave them an idle
    device with this module's buffers and CUDA-graph pools returned."""
    yield
    if torch.cuda.is_available():
        torch.cuda.synchronize()
        gc.collect()
        torch.cuda.empty_cache()


def bits(t):
    t = t.contiguous()
    return t.view(torch.int32 if t.dtype == torch.float32 else torch.int64)


def ulp32(x):
    x = abs(float(x))
    return float(np.spacing(np.float32(x))) if x > 0 else float(np.spacing(np.float32(0)))


def gt_inputs(n, h, w, seed, dtype=torch.float32):
    rng = np.random.RandomState(seed)
    depth = rng.uniform(0.2, 2.0, (n, 1, h, w))
    bad = rng.rand(n, 1, h, w)
    depth[bad < 0.02] = np.nan
    depth[(bad >= 0.02) & (bad < 0.03)] = 0.0
    depth[(bad >= 0.03) & (bad < 0.035)] = np.inf
    depth[(bad >= 0.035) & (bad < 0.04)] = -0.5
    k = np.tile([0.89115971, 1.18821287, 0.5, 0.5], (n, 1)) + rng.uniform(-0.02, 0.02, (n, 4))
    rot = rng.uniform(-0.1, 0.1, (n, 3))
    tr = rng.uniform(-0.5, 0.5, (n, 3)) + np.array([0.5, 0.0, 0.1])
    return [torch.from_numpy(a).to("cuda", dtype) for a in (depth, rot, tr, k)]


def composed_ground_truth(depth, rot, tr, k):
    """prepare_ground_truth_tensors composed from the mirror ops in the reference's order (losses.py:331-356)."""
    lv = [depth]
    for _ in range(5):
        lv.append(sops.median3x3_downsample(lv[-1]))

    def flow(d):
        return sops.depth_to_flow(d, k, rot, tr, inverse_depth=True, normalize_flow=True)

    def sig(x):
        return torch.cat([sops.scale_invariant_gradient(x, [d], [1], 0.001) for d in L.SIG_DELTAS], dim=1)
    f2 = flow(lv[2])
    return {"depth0": depth, "depth0_sig": sig(depth), "depth2": lv[2], "depth2_sig": sig(lv[2]), "flow0": flow(depth), "flow2": f2,
            "flow2_sig": sig(f2), "flow5": flow(lv[5]), "normal0": sops.depth_to_normals(depth, k, True),
            "normal2": sops.depth_to_normals(lv[2], k, True)}


@pytest.mark.parametrize("n,h,w,dtype", [(1, 192, 256, torch.float32), (8, 192, 256, torch.float32), (32, 192, 256, torch.float32),
                                         (3, 37, 53, torch.float32), (2, 192, 256, torch.float64), (3, 37, 53, torch.float64)])
def test_ground_truth_is_the_mirror_composition_bit_for_bit(n, h, w, dtype):
    args = gt_inputs(n, h, w, 10 + n + h, dtype)
    lib = _lib.load()
    c0 = lib.demon_launch_count()
    got = L.prepare_ground_truth_tensors(*args)
    assert lib.demon_launch_count() - c0 == 6
    ref = composed_ground_truth(*args)
    assert list(got) == list(ref)
    for key in ref:
        assert got[key].shape == ref[key].shape, key
        assert torch.equal(bits(got[key]), bits(ref[key])), key
    assert got["depth0"] is args[0]


def _l2_case(seed, shape, dtype=torch.float32):
    rng = np.random.RandomState(seed)
    pr = rng.normal(0, 1, shape)
    gt = rng.normal(0, 1, shape)
    m = rng.rand(*shape)
    pr[m < 0.01] = np.nan
    gt[(m >= 0.01) & (m < 0.02)] = np.inf
    pr[(m >= 0.02) & (m < 0.03)] = -np.inf
    gt[(m >= 0.03) & (m < 0.04)] = pr[(m >= 0.03) & (m < 0.04)]
    return torch.from_numpy(pr).to("cuda", dtype), torch.from_numpy(gt).to("cuda", dtype)


@pytest.mark.parametrize("shape", [(32, 2, 48, 64), (32, 3, 192, 256), (3, 1, 37, 53), (1, 10, 7, 5)])
def test_pointwise_terms_bit_exact_and_mean_within_one_ulp(shape):
    pr, gt = _l2_case(sum(shape), shape)
    terms = L.pointwise_l2_loss(pr, gt, 0.00001, reduction='none')
    ref = OL.terms(pr.cpu().numpy(), gt.cpu().numpy(), 0.00001)
    assert np.array_equal(terms.cpu().numpy().view(np.int32), ref.view(np.int32))
    t64 = terms.double().cpu().numpy().ravel()
    for w in (1.0, 37.5):
        loss = L.pointwise_l2_loss(pr, gt, 0.00001) if w == 1.0 else L.flow_loss_block(
            gt, gt, None, pr, pr, None, None, w, 1.0, None, None)["loss_flow2"] if shape[1] == 2 else None
        if loss is None:
            continue
        want = float(np.float32(math.fsum(t64) / t64.size) * np.float32(w))
        assert abs(float(loss) - want) <= ulp32(want), (float(loss), want)
    a = L.pointwise_l2_loss(pr, gt, 0.00001)
    b = L.pointwise_l2_loss(pr, gt, 0.00001)
    assert torch.equal(bits(a), bits(b))


def _sig_case(n, h, w, seed):
    rng = np.random.RandomState(seed)
    pr = torch.from_numpy(rng.uniform(0.1, 2.0, (n, 1, h, w))).float().cuda()
    gt = torch.from_numpy(rng.uniform(0.1, 2.0, (n, 1, h, w))).float().cuda()
    pr.view(-1)[::97] = float("nan")
    gt_sig = torch.cat([sops.scale_invariant_gradient(gt, [d], [1], 0.001) for d in L.SIG_DELTAS], 1)
    return pr, gt_sig


@pytest.mark.parametrize("n,h,w", [(32, 48, 64), (32, 192, 256), (3, 37, 53)])
def test_sig_loss_within_one_ulp_of_its_terms_and_graph_replay_is_bit_identical(n, h, w):
    pr, gt_sig = _sig_case(n, h, w, n + h)
    # the per-pixel terms of the same loss through the mirror SIG + the L2 terms
    pr_sig = torch.cat([sops.scale_invariant_gradient(pr, [d], [1], 0.01) for d in L.SIG_DELTAS], 1)
    t64 = L.pointwise_l2_loss(pr_sig, gt_sig, 0.00001, reduction='none').double().cpu().numpy().ravel()
    nrm = torch.zeros(n, 3, h, w, device="cuda")
    eager = L.depth_refine_loss_block(pr, gt_sig, nrm, pr, nrm, 1.0, 3.0, 1.0)
    want = float(np.float32(math.fsum(t64) / t64.size) * np.float32(3.0))
    assert abs(float(eager["loss_depth0_sig"]) - want) <= ulp32(want)
    t0 = OL.terms(pr_sig.cpu().numpy(), gt_sig.cpu().numpy(), 0).astype(np.float64).ravel()
    assert abs(float(eager["loss_depth0_sig_unscaled"]) - float(np.float32(math.fsum(t0) / t0.size))) <= ulp32(math.fsum(t0) / t0.size)
    again = L.depth_refine_loss_block(pr, gt_sig, nrm, pr, nrm, 1.0, 3.0, 1.0)
    for k in eager:
        assert torch.equal(bits(eager[k]), bits(again[k])), k
    # forward + backward of the block captured in one CUDA graph
    x = pr.clone().requires_grad_(True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            x.grad = None
            r = L.depth_refine_loss_block(pr, gt_sig, nrm, x, nrm, 1.0, 3.0, 1.0)
            (r["loss_depth0"] + r["loss_depth0_sig"]).backward()
            del r
    torch.cuda.current_stream().wait_stream(s)
    eager_grad = x.grad.clone()
    g = torch.cuda.CUDAGraph()
    x.grad = None
    with torch.cuda.graph(g):
        r = L.depth_refine_loss_block(pr, gt_sig, nrm, x, nrm, 1.0, 3.0, 1.0)
        (r["loss_depth0"] + r["loss_depth0_sig"]).backward()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(bits(r["loss_depth0_sig"]), bits(eager["loss_depth0_sig"]))
    assert torch.equal(bits(x.grad), bits(eager_grad))


def _case(ci, dtype):
    inp = {k: torch.from_numpy(v).to("cuda", dtype) for k, v in GEN.make_inputs(ci).items()}
    gt = L.prepare_ground_truth_tensors(inp["depth"], inp["rotation"], inp["translation"], inp["intrinsics"])
    pr = {k: torch.from_numpy(v).to("cuda", dtype) for k, v in GEN.make_predictions(ci, {k: v.cpu().numpy() for k, v in gt.items()}).items()}
    return inp, gt, pr


def _check_dict(got, want, dtype, keys=None):
    assert list(got) == list(want if keys is None else keys)
    for k, v in want.items():
        a, b = float(got[k].detach()), float(v)
        if dtype == torch.float64:
            assert a == b or abs(a - b) <= 1e-12 * abs(b), (k, a, b)
        else:   # one rounding of the mean; two for the products and the ratio of two such losses
            n_ulp = 2.01 if k.endswith(("loss_translation", "rot_transl_loss_ratio")) else 1.01
            assert abs(a - b) <= n_ulp * ulp32(b), (k, a, b)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("ci", [0, 1])
def test_blocks_equal_the_oracle(ci, dtype):
    inp, gt, pr = _case(ci, dtype)
    g = {k: v.cpu().numpy() for k, v in gt.items()}
    p = {k: v.cpu().numpy() for k, v in pr.items()}
    golden = dict(np.load(os.path.join(GOLDEN, "losses_golden.npz")))
    for j, (c2, c5, fs, cs, scale, l5, prefix) in enumerate(GEN.flow_combos()):
        a = dict(GEN.FLOW_ARGS)
        args = (pr["pr_conf2"] if c2 else None, pr["pr_conf5"] if c5 else None, a["flow_weight"], a["conf_weight"],
                a["flow_sig_weight"] if fs else None, a["conf_sig_weight"] if cs else None)
        got = L.flow_loss_block(gt["flow2"], gt["flow5"], gt["flow2_sig"], pr["pr_flow2"], pr["pr_flow5"], *args, conf_diff_scale=scale,
                                level5_factor=l5, loss_prefix=prefix)
        want = OL.flow_loss_block(g["flow2"], g["flow5"], g["flow2_sig"], p["pr_flow2"], p["pr_flow5"], p["pr_conf2"] if c2 else None,
                                  p["pr_conf5"] if c5 else None, *args[2:], conf_diff_scale=scale, level5_factor=l5, loss_prefix=prefix)
        _check_dict(got, want, dtype, keys=list(golden["c%d/flow%d/keys" % (ci, j)]))
    got = L.depthnormal_loss_block(gt["depth2"], gt["depth2_sig"], gt["normal2"], inp["rotation"], inp["translation"], pr["pr_depth2"],
                                   pr["pr_normal2"], pr["pr_rotation"], pr["pr_translation"], loss_prefix="netDM1_", **GEN.DN_ARGS)
    want = OL.depthnormal_loss_block(g["depth2"], g["depth2_sig"], g["normal2"], inp["rotation"].cpu().numpy(),
                                     inp["translation"].cpu().numpy(), p["pr_depth2"], p["pr_normal2"], p["pr_rotation"], p["pr_translation"],
                                     loss_prefix="netDM1_", **GEN.DN_ARGS)
    _check_dict(got, want, dtype, keys=list(golden["c%d/dn/keys" % ci]))
    got = L.depth_refine_loss_block(gt["depth0"], gt["depth0_sig"], gt["normal0"], pr["pr_depth0"], pr["pr_normal0"], loss_prefix="netRefine_",
                                    **GEN.REFINE_ARGS)
    want = OL.depth_refine_loss_block(g["depth0"], g["depth0_sig"], g["normal0"], p["pr_depth0"], p["pr_normal0"], loss_prefix="netRefine_",
                                      **GEN.REFINE_ARGS)
    _check_dict(got, want, dtype, keys=list(golden["c%d/refine/keys" % ci]))
    conf = L.compute_confidence_map(pr["pr_flow2"], gt["flow2"], 3)
    want = OL.compute_confidence_map(p["pr_flow2"], g["flow2"], 3)
    if dtype == torch.float32:   # exp in double rounded once to float32: the host's bits
        assert np.array_equal(conf.cpu().numpy(), want, equal_nan=True)
    else:                        # CUDA's and the host's double exp may differ in the last bit
        np.testing.assert_allclose(conf.cpu().numpy(), want, rtol=4.5e-16, atol=0)
    assert all(v.shape == () and v.is_cuda for v in got.values())


def test_numpy_in_gives_numpy_out_and_tensor_weights():
    inp, gt, pr = _case(0, torch.float32)
    g = {k: v.cpu().numpy() for k, v in gt.items()}
    p = {k: v.cpu().numpy() for k, v in pr.items()}
    r = L.depth_refine_loss_block(g["depth0"], g["depth0_sig"], g["normal0"], p["pr_depth0"], p["pr_normal0"], 300.0, 1500.0, 100.0)
    assert all(isinstance(v, np.ndarray) for v in r.values())
    w = torch.tensor(1500.0, device="cuda")
    rt = L.depth_refine_loss_block(gt["depth0"], gt["depth0_sig"], gt["normal0"], pr["pr_depth0"], pr["pr_normal0"], 300.0, w, 100.0)
    assert float(rt["loss_depth0_sig"]) == float(r["loss_depth0_sig"])
    lf = L.flow_loss_block(gt["flow2"], gt["flow5"], gt["flow2_sig"], pr["pr_flow2"], pr["pr_flow5"], None, None, torch.tensor(1.7, device="cuda"),
                           0.3, None, None)
    want = np.float32(0.5) * np.float32(1.7) * np.float32(float(L.pointwise_l2_loss(pr["pr_flow5"], gt["flow5"], 0.00001)))
    assert float(lf["loss_flow5"]) == float(want)


def _small(seed, n=2, h=9, w=21):
    rng = np.random.RandomState(seed)

    def t(*s, lo=0.2, hi=2.0):
        return torch.from_numpy(rng.uniform(lo, hi, s)).cuda()
    return t


def test_gradcheck_float64():
    t = _small(5)
    gt_d, pr_d = t(2, 1, 9, 21), t(2, 1, 9, 21).requires_grad_(True)
    gt_n, pr_n = t(2, 3, 9, 21, lo=-1, hi=1), t(2, 3, 9, 21, lo=-1, hi=1).requires_grad_(True)
    gsig = torch.cat([sops.scale_invariant_gradient(gt_d, [d], [1], 0.001) for d in L.SIG_DELTAS], 1)

    def refine(d, nn):
        r = L.depth_refine_loss_block(gt_d, gsig, gt_n, d, nn, 3.0, 7.0, 2.0)
        return r["loss_depth0"], r["loss_depth0_sig"], r["loss_normal0"]
    assert torch.autograd.gradcheck(refine, (pr_d, pr_n), eps=1e-6, atol=1e-7, rtol=1e-5)
    rot_gt, tr_gt = t(2, 3, lo=-0.1, hi=0.1), t(2, 3, lo=-0.5, hi=0.5)
    rot, tr = t(2, 3, lo=-0.1, hi=0.1).requires_grad_(True), t(2, 3, lo=-0.5, hi=0.5).requires_grad_(True)

    def dn(d, nn, r_, t_):
        r = L.depthnormal_loss_block(gt_d, gsig, gt_n, rot_gt, tr_gt, d, nn, r_, t_, 3.0, 7.0, 2.0, 5.0, 4.0, 1.3)
        return r["loss_depth2"], r["loss_depth2_sig"], r["loss_normal2"], r["loss_rotation"], r["loss_translation"], r["loss_translation_no_factor"]
    assert torch.autograd.gradcheck(dn, (pr_d, pr_n, rot, tr), eps=1e-6, atol=1e-7, rtol=1e-5)
    f2g, f5g = t(2, 2, 9, 21, lo=-0.5, hi=0.5), t(2, 2, 3, 5, lo=-0.5, hi=0.5)
    f2, f5 = t(2, 2, 9, 21, lo=-0.5, hi=0.5).requires_grad_(True), t(2, 2, 3, 5, lo=-0.5, hi=0.5).requires_grad_(True)
    c2, c5 = t(2, 2, 9, 21, lo=0.1, hi=1).requires_grad_(True), t(2, 2, 3, 5, lo=0.1, hi=1).requires_grad_(True)
    fsig = torch.cat([sops.scale_invariant_gradient(f2g, [d], [1], 0.001) for d in L.SIG_DELTAS], 1)

    def flow(a, b):   # the flow losses (the confidence target depends on the flows, without gradient: see below)
        r = L.flow_loss_block(f2g, f5g, fsig, a, b, None, None, 3.0, 1.0, 2.0, None)
        return r["loss_flow5"], r["loss_flow2"], r["loss_flow2_sig"]
    assert torch.autograd.gradcheck(flow, (f2, f5), eps=1e-6, atol=1e-7, rtol=1e-5)

    def conf(a, b):
        r = L.flow_loss_block(f2g, f5g, fsig, f2.detach(), f5.detach(), a, b, 3.0, 1.5, 2.0, 0.7)
        return r["loss_conf5"], r["loss_conf2"], r["loss_conf2_sig"]
    assert torch.autograd.gradcheck(conf, (c2, c5), eps=1e-6, atol=1e-7, rtol=1e-5)
    x = t(4, 3, lo=-1, hi=1).requires_grad_(True)
    assert torch.autograd.gradcheck(lambda v: L.l1_loss(v, 0.00001), (x,), eps=1e-6, atol=1e-7, rtol=1e-5)


def test_float32_gradients_within_the_operation_count_bound():
    """Bound per element: |g32 - g64| <= K * u * max|g64| with u = 2^-24 and K = 64 -- a SIG gradient element sums at
    most 5 deltas x 4 neighbour terms, each a chain of about 8 roundings of the loss term and the SIG derivative, over
    addends bounded by max|g64|.  The largest measured ratio is recorded in DESIGN.md."""
    inp, gt, pr = _case(1, torch.float32)
    d = pr["pr_depth0"].clone().requires_grad_(True)
    n = pr["pr_normal0"].clone().requires_grad_(True)
    r = L.depth_refine_loss_block(gt["depth0"], gt["depth0_sig"], gt["normal0"], d, n, 300.0, 1500.0, 100.0)
    (r["loss_depth0"] + r["loss_depth0_sig"] + r["loss_normal0"]).backward()
    g = {k: v.cpu().numpy() for k, v in gt.items()}
    pd, pn = pr["pr_depth0"].cpu().numpy(), pr["pr_normal0"].cpu().numpy()
    want_d = OL.l2_grad(pd, g["depth0"], 1e-5, 300.0) + OL.sig_loss_grad(pd, g["depth0_sig"], 1e-5, 0.01, 1500.0)
    want_n = OL.l2_grad(pn, g["normal0"], 1e-5, 100.0)
    u = 2.0 ** -24
    worst = 0.0
    for got, want in ((d.grad.cpu().numpy(), want_d), (n.grad.cpu().numpy(), want_n)):
        ratio = np.abs(got.astype(np.float64) - want).max() / (u * np.abs(want).max())
        worst = max(worst, ratio)
        assert ratio <= 64, ratio
    print("largest float32 gradient error: %.2f u max|g|" % worst)
    # exactly 0 where the difference is not finite (the normal loss alone acts on pr_normal0)
    dn = pn - g["normal0"]
    assert (n.grad.cpu().numpy()[~np.isfinite(dn)] == 0).all()


def test_no_gradient_through_gt_confidence_target_or_summaries():
    inp, gt, pr = _case(0, torch.float32)
    g2 = gt["flow2"].clone().requires_grad_(True)
    f2 = pr["pr_flow2"].clone().requires_grad_(True)
    c2 = pr["pr_conf2"].clone().requires_grad_(True)
    r = L.flow_loss_block(g2, gt["flow5"], gt["flow2_sig"], f2, pr["pr_flow5"], c2, None, 1.0, 1.0, 1.0, 1.0)
    for k in ("loss_flow2_unscaled", "loss_flow5_unscaled", "loss_conf2_unscaled", "loss_flow2_sig_unscaled", "loss_conf2_sig_unscaled"):
        assert not r[k].requires_grad, k
    (r["loss_conf2"] + r["loss_conf2_sig"]).backward()
    assert g2.grad is None
    assert f2.grad is not None and (f2.grad == 0).all()    # the confidence target carries no gradient into the flow
    assert c2.grad is not None and c2.grad.abs().sum() > 0
    d = pr["pr_depth2"].clone().requires_grad_(True)
    rdn = L.depthnormal_loss_block(gt["depth2"], gt["depth2_sig"], gt["normal2"], inp["rotation"], inp["translation"], d, pr["pr_normal2"],
                                   pr["pr_rotation"], pr["pr_translation"], **GEN.DN_ARGS)
    assert not rdn["rot_transl_loss_ratio"].requires_grad and not rdn["loss_depth2_sig_unscaled"].requires_grad


def test_losses_on_v2_pipeline_outputs():
    from demon_b200.v2 import weights as W2
    from demon_b200.v2.networks import DemonPipelineV2, Session
    s = Session(precision="3xtf32")
    s.load_weights(W2.synthetic_weights(0))
    ip = (torch.rand(8, 6, 192, 256, generator=torch.Generator().manual_seed(9)) - 0.5).cuda()
    out = {k: v.clone() for k, v in DemonPipelineV2(s, batch_size=8, iterations=1).forward(ip).items()}
    inp = gt_inputs(8, 192, 256, 77)
    gt = L.prepare_ground_truth_tensors(*inp)
    pr = {k: v.clone().requires_grad_(True) for k, v in out.items()}
    dn = L.depthnormal_loss_block(gt["depth2"], gt["depth2_sig"], gt["normal2"], inp[1], inp[2], pr["predict_depth2"], pr["predict_normal2"],
                                  pr["predict_rotation"], pr["predict_translation"], **GEN.DN_ARGS)
    rf = L.depth_refine_loss_block(gt["depth0"], gt["depth0_sig"], gt["normal0"], pr["predict_depth0"], pr["predict_normal0"], **GEN.REFINE_ARGS)
    g = {k: v.cpu().numpy() for k, v in gt.items()}
    o = {k: v.cpu().numpy() for k, v in out.items()}
    want = OL.depthnormal_loss_block(g["depth2"], g["depth2_sig"], g["normal2"], inp[1].cpu().numpy(), inp[2].cpu().numpy(), o["predict_depth2"],
                                     o["predict_normal2"], o["predict_rotation"], o["predict_translation"], **GEN.DN_ARGS)
    _check_dict(dn, want, torch.float32)
    want = OL.depth_refine_loss_block(g["depth0"], g["depth0_sig"], g["normal0"], o["predict_depth0"], o["predict_normal0"], **GEN.REFINE_ARGS)
    _check_dict(rf, want, torch.float32)
    total = sum(v for k, v in dn.items() if k in ("loss_depth2", "loss_depth2_sig", "loss_normal2", "loss_rotation", "loss_translation"))
    total = total + rf["loss_depth0"] + rf["loss_depth0_sig"] + rf["loss_normal0"]
    total.backward()
    for k in ("predict_depth2", "predict_normal2", "predict_rotation", "predict_translation", "predict_depth0", "predict_normal0"):
        assert pr[k].grad is not None and torch.isfinite(pr[k].grad).all() and pr[k].grad.abs().sum() > 0, k
