"""CPU: the multi-view reader oracle (oracle/datareader.py) checked for geometric self-consistency, independently of its
own flip algebra, and the host side of demon_b200.datareader: drawing the augmentation and refusing bad parameters."""
import math

import numpy as np
import pytest

from demon_b200 import datareader as dr
from demon_b200.dataset_tools import View
from oracle import datareader as od
from oracle import ops as oops

# training/v2/training.py:96-108, verbatim (the duplicate 'builder_threads' key included)
TRAINING_PARAMS = {
    'batch_size': 32,
    'test_phase': False,
    'motion_format': 'ANGLEAXIS6',
    'inverse_depth': True,
    'builder_threads': 1,
    'scaled_width': 256,
    'scaled_height': 192,
    'norm_trans_scale_depth': True,
    'top_output': ('IMAGE_PAIR', 'MOTION', 'DEPTH', 'INTRINSICS'),
    'scene_pool_size': 650,
    'builder_threads': 8,   # noqa: F601
}
COMBOS = ((False, False), (True, False), (False, True), (True, True))


def _prepared(n, h, w, sh, sw, seed, centred=False):
    return [od.prepare(img, d, K, R, t, m, w, h) for R, t, K, img, d, m in od.synthetic_views(n, sh, sw, seed, centred=centred)]


def _rotation_vector(fmt, m):
    if fmt == 'ANGLEAXIS6':
        return m[:3]
    if fmt == 'ANGLEAXIS7':
        return m[0] * m[1:4]
    w, v = m[0], m[1:4]
    n = np.linalg.norm(v)
    return v / n * 2 * math.atan2(n, w)


@pytest.mark.parametrize("fmt", ['ANGLEAXIS6', 'ANGLEAXIS7', 'QUATERNION'])
def test_oracle_flow_is_depth_to_flow_of_its_own_outputs(fmt):
    """FLOW equals lmbspecialops' depth_to_flow of the item's DEPTH, INTRINSICS and MOTION within 1e-3 px for every
    rot180 / mirror_x combination: the flips of images, cameras, flow and depth agree with each other."""
    views = _prepared(2, 24, 32, 48, 64, 3)
    params = dict(dr.reader_params({'batch_size': 4, 'motion_format': fmt}))
    out, used = od.build_batch(views, [(0, 1)] * 4, params, [c[0] for c in COMBOS], [c[1] for c in COMBOS], None)
    assert list(used) == [0, 1, 2, 3]
    for s in range(4):
        m = out['MOTION'][s].astype(np.float64)
        flow = oops.depth_to_flow(out['DEPTH'][s:s + 1].astype(np.float64), out['INTRINSICS'][s:s + 1].astype(np.float64),
                                  _rotation_vector(fmt, m)[None], m[-3:][None], rotation_format='angleaxis3')
        ref = out['FLOW'][s:s + 1].astype(np.float64)
        assert np.array_equal(np.isnan(flow), np.isnan(ref)), COMBOS[s]
        ok = ~np.isnan(ref)
        assert ok.mean() > 0.9
        assert np.abs(flow[ok] - ref[ok]).max() < 1e-3, (COMBOS[s], np.abs(flow[ok] - ref[ok]).max())


def test_oracle_fmatrix_is_the_epipolar_constraint_of_its_flow():
    """FMATRIX is built from the rotated cameras but the unrotated, unmirrored K (:1756-1761), so it describes the
    output's geometry where the principal point is centred and nothing is mirrored: there x2' F x1 = 0 within 1e-3 px."""
    views = _prepared(2, 24, 32, 48, 64, 4, centred=True)
    params = dict(dr.reader_params({'batch_size': 2, 'motion_format': 'FMATRIX'}))
    out, _ = od.build_batch(views, [(0, 1)] * 2, params, [False, True], [False, False], None)
    h, w = 24, 32
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    for s in range(2):
        F = np.append(out['MOTION'][s].astype(np.float64), 1.0).reshape(3, 3).T   # column major, F(2,2) = 1
        fl = out['FLOW'][s].astype(np.float64)
        x1 = np.stack([(xx + 0.5) / w, (yy + 0.5) / h, np.ones_like(xx)])
        x2 = np.stack([(xx + 0.5 + fl[0]) / w, (yy + 0.5 + fl[1]) / h, np.ones_like(xx)])
        l2 = np.einsum('ij,jhw->ihw', F, x1)
        dist = np.abs((x2 * l2).sum(0)) / np.hypot(l2[0], l2[1]) * w
        ok = np.isfinite(dist)
        assert ok.mean() > 0.9 and dist[ok].max() < 1e-3, dist[ok].max()


def test_draw_augmentation_test_phase_counts():
    rng = np.random.default_rng(0)
    a = dr.draw_augmentation({'test_phase': True, 'augment_rot180': 0.25, 'augment_mirror_x': 0.5}, 8, rng)
    assert list(a.rot180) == [True, True] + [False] * 6
    assert list(a.mirror_x) == [True] * 4 + [False] * 4
    assert a.colour is None


def test_draw_augmentation_bernoulli_rates_and_colour():
    rng = np.random.default_rng(1)
    n = 20000
    a = dr.draw_augmentation({'augment_rot180': 0.3, 'augment_mirror_x': 0.7}, n, rng)
    assert abs(a.rot180.mean() - 0.3) < 0.015 and abs(a.mirror_x.mean() - 0.7) < 0.015
    assert a.colour is None   # no aug_* key: the colour step does not run (:653)
    b = dr.draw_augmentation({'aug_gamma': {'uniform': {'a': 0.5, 'b': 2.0}}, 'aug_hsv_hue': {'normal': {'mean': 0, 'stddev': 10}}},
                             n, rng)
    assert b.colour.shape == (n, 6) and b.colour.dtype == np.float32
    assert np.all(b.colour[:, [1, 2, 4]] == 0) and np.all(b.colour[:, 3] == 1)   # absent keys at the reader's defaults
    assert 0.5 <= b.colour[:, 5].min() and b.colour[:, 5].max() <= 2.0 and abs(b.colour[:, 5].mean() - 1.25) < 0.02
    assert abs(b.colour[:, 0].std() - 10) < 0.3


def test_parameters():
    p = dr.reader_params(TRAINING_PARAMS)
    assert p['batch_size'] == 32 and p['motion_format'] == 'ANGLEAXIS6' and p['depthmask_border1'] == 3
    with pytest.raises(ValueError, match="unknown"):
        dr.reader_params({'batch_sise': 4})
    with pytest.raises(ValueError):
        dr.reader_params({'motion_format': 'EULER'})
    with pytest.raises(ValueError):
        dr.reader_params({'top_output': ('IMAGE_PAIR', 'NORMALS')})


def test_refusals_before_the_device():
    pool = dr.ViewPool(256, 192)
    R, t, K, img, d, m = od.synthetic_views(1, 120, 160, 0)[0]
    with pytest.raises(ValueError, match="upscale"):
        pool.add([View(R, t, K, img, d, m)])
    with pytest.raises(ValueError, match="K must be"):
        dr.ViewPool(32, 24).add([View(R, t, K + np.eye(3)[::-1], img, d, m)])
    aug = dr.draw_augmentation({}, 1, np.random.default_rng(0))
    with pytest.raises(ValueError, match="out of range"):
        dr.build_batch(pool, [(0, 1)], {'batch_size': 1}, aug)
    with pytest.raises(ValueError, match="scaled_width"):
        dr.build_batch(pool, [(0, 1)], {'batch_size': 1, 'scaled_width': 640}, aug)


def test_oracle_area_scaling_is_opencvs():
    """cv::resize(INTER_AREA) as the oracle restates it: at 640x480 -> 256x192 (factor 2.5) every value is the exact
    area mean k/25 rounded (the 2x-upsampled image's 5x5 block sums over 25); at factor 2 a tie rounds up; at factor 3
    the value is float(sum) * (1.f / 9), rounded half to even."""
    rng = np.random.default_rng(5)
    img = rng.integers(0, 256, (480, 640, 3), dtype=np.uint8)
    out = od.area_downscale(img, 192, 256)
    up = img.repeat(2, 0).repeat(2, 1).astype(np.int64)
    sums = up.reshape(192, 5, 256, 5, 3).sum((1, 3))
    assert np.array_equal(out, np.rint(sums / 25).astype(np.uint8))
    tie = np.array([[[1, 2, 0], [2, 3, 0]], [[1, 2, 0], [2, 3, 0]]], np.uint8)   # means 1.5, 2.5, 0
    assert list(od.area_downscale(tie, 1, 1)[0, 0]) == [2, 3, 0]
    block = rng.integers(0, 256, (3, 3, 3), dtype=np.uint8)
    s = block.astype(np.int64).sum((0, 1))
    assert np.array_equal(od.area_downscale(block, 1, 1)[0, 0], np.rint(s.astype(np.float32) * (np.float32(1) / np.float32(9))))
