"""GPU: the evaluation run on the device (DemonPipeline.forward_snapshots, csrc/evaluation.cu, the resampled sums and the
motion kernel in csrc/metrics.cu, demon_b200.evaluation.evaluate_batch / Evaluator) against the stage-wise API, the
reference's mask (oracle/view_tools.py) and a table composed from the existing per-sample functions.  Synthetic weights."""
import math

import numpy as np
import pytest
import scipy.ndimage
import torch

pytestmark = pytest.mark.gpu

from demon_b200 import evaluation as ev
from demon_b200 import lmbspecialops as sops
from oracle import view_tools as vt

B = 2
ITER = 3


@pytest.fixture(scope="module")
def session(synthetic_weights):
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    from demon_b200.networks_original import Session
    s = Session()
    s.load_weights(synthetic_weights)
    return s


def random_inputs(seed, n=B):
    g = torch.Generator().manual_seed(seed)
    ip = (torch.rand(n, 6, 192, 256, generator=g) - 0.5).cuda()
    i22 = sops.median3x3_downsample(sops.median3x3_downsample(ip[:, 3:6].contiguous()))
    return ip, i22


def stagewise(session, ip, i22, iterations=ITER):
    """examples/evaluation.py:225-255 with the per-stage entries: snapshots k = 0..iterations, refined depth of each."""
    from demon_b200.networks_original import BootstrapNet, IterativeNet, RefinementNet
    n = ip.shape[0]
    boot, it, ref = BootstrapNet(session, batch_size=n), IterativeNet(session, batch_size=n), RefinementNet(session, batch_size=n)
    snaps = []
    r = boot.eval(ip, i22)
    for k in range(iterations + 1):
        if k:
            r = it.eval(ip, i22, r["predict_depth2"], r["predict_normal2"], r["predict_rotation"], r["predict_translation"])
        r = {key: v.clone() for key, v in r.items()}
        r["predict_depth0"] = ref.eval(ip[:, 0:3].contiguous(), r["predict_depth2"])["predict_depth0"].clone()
        snaps.append(r)
    torch.cuda.synchronize()
    return snaps


KEYS = ("predict_flow2", "predict_depth2", "predict_normal2", "predict_rotation", "predict_translation", "predict_depth0")


def test_snapshots_equal_stagewise_and_forward(session):
    from demon_b200.networks_original import DemonPipeline
    pipe = DemonPipeline(session, batch_size=B, iterations=ITER)
    ip, i22 = random_inputs(11)
    plain = {k: v.clone() for k, v in pipe.forward(ip, i22).items()}
    pipe.forward(ip, i22)
    torch.cuda.synchronize()
    plain_launches = pipe.launches()
    assert plain_launches > 0
    want = stagewise(session, ip, i22)
    runs = []
    for _ in range(3):   # eager, capture + replay, replay
        out = pipe.forward_snapshots(ip, i22)
        runs.append({k: v.clone() for k, v in out.items()})
    torch.cuda.synchronize()
    for out in runs:
        assert set(out) == set(KEYS)
        assert out["predict_depth0"].shape == (ITER + 1, B, 1, 192, 256)
        for k in range(ITER + 1):
            for key in KEYS:
                assert torch.equal(out[key][k], want[k][key]), (k, key)
    # the last snapshot is the plain pipeline's output
    for key in KEYS:
        assert torch.equal(runs[0][key][ITER], plain[key]), key
    # the graph replays with new input contents (same staging buffers, same key)
    ip2, i222 = random_inputs(12)
    out = pipe.forward_snapshots(ip2, i222)
    torch.cuda.synchronize()
    want2 = stagewise(session, ip2, i222)
    for k in range(ITER + 1):
        for key in KEYS:
            assert torch.equal(out[key][k], want2[k][key]), (k, key)
    # without refinement: the same snapshots, no depth0
    out = pipe.forward_snapshots(ip2, i222, refine=False)
    torch.cuda.synchronize()
    assert "predict_depth0" not in out
    for key in KEYS[:-1]:
        assert torch.equal(out[key], torch.stack([want2[k][key] for k in range(ITER + 1)])), key
    # snapshot calls keep their own launch count; the plain pipeline's stays what it was
    assert pipe.launches() == plain_launches
    assert pipe.snapshot_launches() > 0


def test_snapshots_with_median_image2_2(session):
    from demon_b200.networks_original import DemonPipeline
    pipe = DemonPipeline(session, batch_size=B, iterations=1)
    ip, i22 = random_inputs(13)
    a = {k: v.clone() for k, v in pipe.forward_snapshots(ip, None).items()}
    b = pipe.forward_snapshots(ip, i22)
    torch.cuda.synchronize()
    for key in KEYS:
        assert torch.equal(a[key], b[key]), key


def mask_operands(case):
    depth, K1, R1, t1, K2, R2, t2, bx, by = case
    return depth, vt.operands(K1, R1, t1, K2, R2, t2), bx, by


@pytest.mark.parametrize("case", range(len(vt.edge_cases())))
def test_mask_kernel_matches_reference(case):
    c = vt.edge_cases()[case]
    depth, ops, bx, by = mask_operands(c)
    h, w = depth.shape
    got = ev.visible_points_mask(depth[None], *[o[None] for o in ops], w, h, bx, by).cpu().numpy()[0]
    assert np.array_equal(got, vt.visible_points_mask_numpy(depth, *ops, w, h, bx, by))
    if vt.available():
        ref = vt.reference_mask(depth, *c[1:])
        assert ref.matches(got) if isinstance(ref, vt.Recorded) else np.array_equal(got, ref)
    # the inverse-depth entry takes 1/depth in float32 first
    with np.errstate(divide='ignore'):
        inv = (np.float32(1) / depth).astype(np.float32)
        back = (np.float32(1) / inv).astype(np.float32)
    got_inv = ev.visible_points_mask(inv[None], *[o[None] for o in ops], w, h, bx, by, inverse_depth=True).cpu().numpy()[0]
    assert np.array_equal(got_inv, vt.visible_points_mask_numpy(back, *ops, w, h, bx, by))


def test_mask_kernel_batch_and_invalidate():
    """Several samples in one launch, each with its own cameras; invalidate_... sets NaN in place like the reference."""
    rng = np.random.RandomState(5)
    n, h, w = 5, 48, 64
    inv = rng.uniform(0.1, 1.5, (n, h, w)).astype(np.float32)
    inv[rng.rand(n, h, w) < 0.05] = np.nan
    motion = np.concatenate([rng.normal(0, 0.1, (n, 3)), rng.normal(0, 0.5, (n, 3))], axis=1).astype(np.float32)
    intr = np.tile(np.array([[0.89, 1.19, 0.49, 0.51]], dtype=np.float32), (n, 1))
    ops = ev.visible_points_operands(motion, intr, h, w)
    with np.errstate(divide='ignore'):
        absd = (np.float32(1) / inv).astype(np.float32)
    want = np.stack([vt.visible_points_mask_numpy(absd[i], *[o[i] for o in ops], w, h) for i in range(n)])
    assert np.array_equal(ev.visible_points_mask(absd, *ops).cpu().numpy(), want)
    d_np = inv.copy()
    d_t = torch.from_numpy(inv.copy()).cuda()
    ev.invalidate_points_not_visible_in_second_image(d_np, motion, intr)
    ev.invalidate_points_not_visible_in_second_image(d_t, motion, intr)
    ref = inv.copy()
    ref[want == 0] = np.nan
    assert np.array_equal(d_np, ref, equal_nan=True) and np.array_equal(d_t.cpu().numpy(), ref, equal_nan=True)


def materialise(pred, gh, gw, window):
    """skimage.transform.resize(order=0) of the prediction planes [n, c, ph, pw] to [gh, gw] by scipy.ndimage.zoom, cropped."""
    n, c, ph, pw = pred.shape
    out = np.stack([np.stack([scipy.ndimage.zoom(pred[i, j], (gh / ph, gw / pw), order=0, grid_mode=True, mode='grid-constant')
                              for j in range(c)]) for i in range(n)])
    y0, x0, oh, ow = window
    return np.ascontiguousarray(out[:, :, y0:y0 + oh, x0:x0 + ow])


@pytest.mark.parametrize("ph,pw", ((48, 64), (192, 256)))
@pytest.mark.parametrize("crop", (False, True))
@pytest.mark.parametrize("masked", (False, True))
def test_resampled_depth_sums_equal_materialised(ph, pw, crop, masked):
    rng = np.random.RandomState(ph + 2 * crop + masked)
    n, gh, gw = 3, 480, 640
    pred = rng.uniform(0.05, 2.0, (n, 1, ph, pw)).astype(np.float32)
    pred[rng.rand(n, 1, ph, pw) < 0.02] = np.nan
    gt = rng.uniform(0.05, 2.0, (n, gh, gw)).astype(np.float32)
    gt[rng.rand(n, gh, gw) < 0.03] = np.nan
    gt[rng.rand(n, gh, gw) < 0.01] = 0
    valid = (rng.rand(n, gh, gw) > 0.2).astype(np.uint8) if masked else None
    window = ev.EIGEN_CROP if crop else (0, 0, gh, gw)
    y0, x0, oh, ow = window
    gt_m = gt.copy()
    if masked:
        gt_m[valid == 0] = np.nan
    gt_m = np.ascontiguousarray(gt_m[:, y0:y0 + oh, x0:x0 + ow])
    pred_m = materialise(pred, gh, gw, window)[:, 0]
    gt_div = torch.tensor([1.0, 2.5, 0.7], dtype=torch.float32, device="cuda")
    rs = ev._Resampler(ph, pw, gh, gw, window, torch.device("cuda"))
    g = torch.from_numpy(gt).cuda()
    v = None if valid is None else torch.from_numpy(valid).cuda()
    p = torch.from_numpy(pred).cuda()
    got = rs.depth_sums(p, g, v, gt_div)
    want = ev.depth_error_sums(pred_m, gt_m, True, True, gt_div)
    assert torch.equal(got, want)
    scale = ev.depth_scale_factor(want, 'abs')
    assert torch.equal(rs.depth_sums(p, g, v, gt_div, scale), ev.depth_error_sums(pred_m, gt_m, True, True, gt_div, scale))


def test_resampled_flow_sums_equal_materialised():
    rng = np.random.RandomState(9)
    n, gh, gw = 3, 480, 640
    pred = rng.normal(0, 0.05, (n, 2, 48, 64)).astype(np.float32)
    gt = rng.normal(0, 0.05, (n, 2, gh, gw)).astype(np.float32)
    gt[rng.rand(n, 2, gh, gw) < 0.02] = np.nan
    rs = ev._Resampler(48, 64, gh, gw, (0, 0, gh, gw), torch.device("cuda"))
    got = rs.flow_sums(torch.from_numpy(pred).cuda(), torch.from_numpy(gt).cuda())
    assert torch.equal(got, ev.flow_epe_sums(materialise(pred, gh, gw, (0, 0, gh, gw)), gt))


def test_motion_errors_and_gt_div_match_host():
    rng = np.random.RandomState(21)
    n = 12
    gt = np.concatenate([rng.normal(0, 0.3, (n, 3)), rng.normal(0, 1.0, (n, 3))], axis=1).astype(np.float32)
    pr = np.concatenate([rng.normal(0, 0.3, (n, 3)), rng.normal(0, 1.0, (n, 3))], axis=1).astype(np.float32)
    gt[1, 3:6] /= np.linalg.norm(gt[1, 3:6])        # a unit translation: gt_div 1
    gt[2, 0:3] = [1e-7, 0, 0]                        # below the 1e-6 angle rule
    gt[3, 0:3] = 0                                   # identical motions without rotation: d == 1 exactly, the d >= 1 branch
    pr[3] = gt[3]                                    # (with a rotation d sits within rounding of 1, where acos is ill conditioned)
    pr[4, 3:6] = [1e-8, 0, 0]                        # prediction too short to normalise
    gt[5, 4] = np.nan                                # NaN in the gt translation
    gt[6, 1] = np.nan                                # NaN in the gt rotation
    pr[7, 2] = np.nan                                # NaN in the prediction
    out, gt_div = ev.motion_errors(pr[:, 0:3], pr[:, 3:6], gt)
    out, gt_div = out.cpu().numpy(), gt_div.cpu().numpy()
    for i in range(n):
        want = ev.compute_motion_errors(pr[i], gt[i], True)
        np.testing.assert_allclose(out[i, 0:3], want, rtol=1e-12, atol=1e-12, equal_nan=True)
        t = np.array([1.0, 0.0, 0.0]) if np.isnan(gt[i]).any() else gt[i, 3:6].astype(np.float64)
        norm = np.sqrt((t * t).sum())
        assert gt_div[i] == np.float32(1.0 if np.isclose(1.0, norm) else norm)
        if np.isnan(gt[i]).any():
            assert np.isnan(out[i, 3])
        else:
            assert abs(out[i, 3] - np.linalg.norm(gt[i, 3:6].astype(np.float64))) <= 1e-12


def oracle_table(snaps, depth_gt, motion_gt, intrinsics, depthmask, crop, scaling='abs'):
    """The table of evaluate_to_xarray.evaluate composed from the stage-wise predictions, the numpy mask, scipy's zoom and
    the existing per-sample evaluate_depth / compute_flow_epe / compute_motion_errors."""
    n, gh, gw = depth_gt.shape
    intr = np.tile(np.array([ev.SUN3D_INTRINSICS], dtype=np.float32), (n, 1)) if intrinsics is None else intrinsics
    flow_gt = sops.depth_to_flow(depth_gt[:, None], intr, motion_gt[:, 0:3].copy(), motion_gt[:, 3:6].copy(),
                                 rotation_format="angleaxis3", inverse_depth=True, normalize_flow=True)
    gt = depth_gt.copy()
    if depthmask:
        ops = ev.visible_points_operands(motion_gt, intr, gh, gw)
        with np.errstate(divide='ignore'):
            absd = (np.float32(1) / gt).astype(np.float32)
        for i in range(n):
            gt[i][vt.visible_points_mask_numpy(absd[i], *[o[i] for o in ops], gw, gh) == 0] = np.nan
    window = ev.EIGEN_CROP if crop else (0, 0, gh, gw)
    y0, x0, oh, ow = window
    gt = gt[:, y0:y0 + oh, x0:x0 + ow]
    labels = sorted([str(k) for k in range(len(snaps))] + ['%d_refined' % k for k in range(len(snaps))], key=ev.iteration_sort_key)
    values = np.full((1, len(labels), n, 16, 2), np.nan)
    for k, s in enumerate(snaps):
        s = {key: v.cpu().numpy() for key, v in s.items()}
        for label, pred in ((str(k), s["predict_depth2"]), ('%d_refined' % k, s["predict_depth0"])):
            v = values[0, labels.index(label)]
            pm = materialise(pred[:n], gh, gw, window)[:, 0]
            for i in range(n):
                tgt = np.array([1., 0., 0.]) if np.isnan(motion_gt[i]).any() else motion_gt[i, 3:6]
                if not np.isnan(motion_gt[i]).any():
                    v[i, 15, :] = np.linalg.norm(tgt.astype(np.float64))
                e, es = ev.evaluate_depth(tgt, gt[i], pm[i], depth_scaling=scaling)
                for j, d in enumerate(ev.DISTANCES):
                    v[i, 3 + j] = (e[d], es[d])
                if label == str(k):
                    pmot = np.concatenate([s["predict_rotation"][i], s["predict_translation"][i]])
                    v[i, 0:3, :] = np.array(ev.compute_motion_errors(pmot, motion_gt[i], True))[:, None]
                    fpm = materialise(s["predict_flow2"][i:i + 1], gh, gw, (0, 0, gh, gw))[0]
                    v[i, 14, :] = ev.compute_flow_epe(fpm, flow_gt[i])
    return labels, values


def compare_tables(got, labels, want):
    assert got.coords['iteration'] == labels and got.coords['errors'] == ev.ERRORS
    depth = slice(3, 14)
    assert np.array_equal(got.values[..., depth, :], want[..., depth, :], equal_nan=True)
    np.testing.assert_allclose(got.values, want, rtol=1e-12, atol=1e-12, equal_nan=True)


def synthetic_gt(seed, n, gh, gw):
    rng = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:gh, 0:gw]
    inv = np.stack([(0.3 + 0.15 * np.sin(xx / (40.0 + 10 * i)) + 0.1 * np.cos(yy / 25.0)) for i in range(n)]).astype(np.float32)
    inv[rng.rand(n, gh, gw) < 0.02] = np.nan
    motion = np.concatenate([rng.normal(0, 0.05, (n, 3)), rng.normal(0, 0.4, (n, 3))], axis=1).astype(np.float32)
    intr = np.tile(np.array([[0.89, 1.19, 0.5, 0.5]], dtype=np.float32), (n, 1))
    return inv, motion, intr


@pytest.mark.parametrize("depthmask,crop", ((True, False), (False, True)))
def test_evaluator_table_equals_oracle_table(session, depthmask, crop):
    ip, i22 = random_inputs(31)
    inv, motion, intr = synthetic_gt(4, B, 480, 640)
    motion[1, 3] = np.nan if crop else motion[1, 3]      # a gt motion with a NaN: translation (1, 0, 0), no baseline
    evaluator = ev.Evaluator(session, B, ITER, depthmask=depthmask, eigen_crop_gt_and_pred=crop)
    got = evaluator.add(ip, inv, motion, intr, image2_2=i22)
    labels, want = oracle_table(stagewise(session, ip, i22), inv, motion, intr, depthmask, crop)
    compare_tables(got, labels, want)
    assert got.to_dict()['attrs']['depthmask'] == depthmask
    # a smaller last batch is padded and evaluated on its real samples only
    part = evaluator.add(ip[:1], inv[:1], motion[:1], intr[:1], image2_2=i22[:1])
    compare_tables(part, labels, want[:, :, :1])
    assert evaluator.result().coords['sample'] == ['0', '1', '2']


def test_sculpture_pair_with_its_ground_truth(session, sculpture, golden_dir):
    """The reference's example pair and examples/sculpture_depth1.npy (192x256 camera z, 0 = unknown) with the relative
    pose of the pair, evaluated with the visibility mask at the sun3d intrinsics."""
    from scipy.spatial.transform import Rotation
    import os
    depth = np.load(os.path.join(golden_dir, "sculpture_depth1.npy")).astype(np.float32)
    with np.errstate(divide='ignore'):
        inv = (np.float32(1) / depth)[None].astype(np.float32)
    Rt2 = sculpture["Rt2"]
    motion = np.concatenate([Rotation.from_matrix(Rt2[:, :3]).as_rotvec(), Rt2[:, 3]]).astype(np.float32)[None]
    ip = torch.from_numpy(sculpture["image_pair"]).cuda()
    i22 = torch.from_numpy(sculpture["image2_2"]).cuda()
    got = ev.Evaluator(session, 1, ITER, depthmask=True).add(ip, inv, motion, None, image2_2=i22)
    labels, want = oracle_table(stagewise(session, ip, i22), inv, motion, None, True, False)
    compare_tables(got, labels, want)
    assert 0 < got.sel('3', 'camera_baseline')[0] == pytest.approx(float(np.linalg.norm(Rt2[:, 3])), rel=1e-6)
    assert np.isfinite(got.sel('3_refined', 'depth_l1_inverse')).all()
