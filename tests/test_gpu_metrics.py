"""GPU: the device evaluation metrics (demon_b200/evaluation.py over csrc/metrics.cu) against golden vectors produced by
the REFERENCE's own functions (python/depthmotionnet/evaluation/metrics.py imported unmodified by
tests/golden/make_metrics_golden.py).  Floating point: 1e-5 relative (float32 pairwise sums there, double accumulation
here); pixel counts may differ by the few pixels whose log-ratio sits within an ulp of a threshold."""
import os

import numpy as np
import pytest
import torch

from oracle import metrics as om

pytestmark = pytest.mark.gpu

NAMES = ['l1', 'l1_inverse', 'scale_invariant', 'abs_relative', 'sq_relative', 'avg_log10', 'rmse_log', 'rmse',
         'ratio_threshold_1.25', 'ratio_threshold_1.5625', 'ratio_threshold_1.953125']
RTOL = 1e-5


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "metrics_golden.npz"))


def gt_div_of(t):
    norm = np.sqrt(t.dot(t))
    return None if np.isclose(1.0, norm) else np.array([norm])


def check(errs, want, account):
    """account: oracle/metrics.py's threshold_account of the same compute_errors call."""
    assert abs(errs['num_valid'] - want[0]) <= 0, (errs['num_valid'], want[0])
    for k, w in zip(NAMES, want[1:]):
        g = errs[k]
        if np.isnan(w):
            assert np.isnan(g), k
        elif k.startswith('ratio_threshold'):
            a = account[om.THRESHOLDS.index(float(k.split('_')[-1]))]
            borderline = len(set(a['ambiguous']) | set(a['disagree']))
            assert abs(round(g * want[0]) - round(w * want[0])) <= borderline, (k, g * want[0], w * want[0], a)
        else:
            assert abs(g - w) <= RTOL * abs(w) + 1e-9, (k, g, w)


@pytest.mark.parametrize("ci", (0, 1, 2))
@pytest.mark.parametrize("scaling", ("abs", "log", "inv"))
def test_evaluate_depth_matches_reference(golden, ci, scaling):
    from demon_b200 import evaluation as ev
    gt, pred, t = golden["gt_%d" % ci], golden["pred_%d" % ci], golden["t_%d" % ci]
    errs, errs_scaled = ev.evaluate_depth(t, gt, pred, depth_scaling=scaling)
    check(errs, golden["errs_%d_%s" % (ci, scaling)], om.threshold_account(pred[None], gt[None], True, gt_div_of(t)))
    check(errs_scaled, golden["errs_scaled_%d_%s" % (ci, scaling)], om.threshold_account(pred[None], gt[None], True, gt_div_of(t), scaling))


@pytest.mark.parametrize("ci", (0, 1, 2))
def test_compute_errors_and_flow_epe_match_reference(golden, ci):
    from demon_b200 import evaluation as ev
    dpred, dgt = golden["dpred_%d" % ci], golden["dgt_%d" % ci]
    check(ev.compute_errors(dpred, dgt), golden["errs_plain_%d" % ci], om.threshold_account(dpred[None], dgt[None]))
    epe = ev.compute_flow_epe(golden["f1_%d" % ci], golden["f2_%d" % ci])
    assert abs(epe - float(golden["epe_%d" % ci])) <= RTOL * float(golden["epe_%d" % ci])


def test_all_invalid_and_motion_errors(golden):
    from demon_b200 import evaluation as ev
    e = ev.compute_errors(np.full((4, 4), np.nan, np.float32), np.ones((4, 4), np.float32))
    assert e['num_valid'] == 0 and all(np.isnan(e[k]) for k in NAMES)
    assert np.isnan(ev.compute_flow_epe(np.zeros((2, 3, 3), np.float32), np.zeros((2, 3, 3), np.float32)))
    m, want = golden["motions"], golden["motion_errors"]
    i = 0
    for a in range(0, 6, 2):
        for nt in (True, False):
            np.testing.assert_allclose(ev.compute_motion_errors(m[a], m[a + 1], nt), want[i], rtol=1e-9, atol=1e-9)
            i += 1


def test_batched_sums_are_deterministic_and_per_sample(golden):
    """evaluate_depth_batch keeps everything on the device: a batch of different samples gives each sample's own sums,
    and two runs are bit identical (fixed reduction order)."""
    from demon_b200 import evaluation as ev
    gt = torch.from_numpy(np.stack([golden["gt_0"], golden["gt_0"][::-1].copy(), golden["gt_0"] * 2])).cuda()
    pred = torch.from_numpy(np.stack([golden["pred_0"], golden["pred_0"][::-1].copy(), golden["pred_0"]])).cuda()
    t = np.tile(golden["t_0"], (3, 1))
    s1, s1s, sc1 = ev.evaluate_depth_batch(t, gt, pred)
    s2, s2s, sc2 = ev.evaluate_depth_batch(t, gt, pred)
    torch.cuda.synchronize()
    assert torch.equal(s1, s2) and torch.equal(s1s, s2s) and torch.equal(sc1, sc2)
    want = golden["errs_0_abs"]
    assert int(s1[0, 0].item()) == int(want[0])
    assert abs(s1[0, 1].item() / s1[0, 0].item() - want[1]) <= RTOL * want[1]
    assert abs(s1[1, 1].item() - s1[0, 1].item()) <= 1e-9 * abs(s1[0, 1].item())       # flipped rows: same sums up to order
    assert not torch.equal(s1[2], s1[0])
