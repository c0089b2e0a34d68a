"""GPU: demon_b200.datareader against the numpy restatement of the reference's multi-view reader (oracle/datareader.py).

The prepared pool and IMAGE_PAIR, DEPTH, FLOW, DEPTHMASKS and INTRINSICS are compared bit for bit, NaN sign included;
MOTION within one float32 ulp of the float64 oracle.  The pose math is checked against a restatement of Eigen's
algorithms (quaternion, angle-axis, 4x4 determinant), not against Eigen itself, which is not available here."""
import numpy as np
import pytest
import torch

from demon_b200 import datareader as dr
from demon_b200.dataset_tools import View
from oracle import datareader as od

pytestmark = pytest.mark.gpu

COMBOS = ((False, False), (True, False), (False, True), (True, True))


def _bits(a):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else a
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _spoil_depths(views, seed):
    """zero, negative, NaN (both signs) and +-inf depths in every view"""
    rng = np.random.default_rng(seed)
    out = []
    for R, t, K, img, d, m in views:
        d = d.copy()
        flat = d.reshape(-1)
        for v in (0, -1.5, np.nan, -np.nan, np.inf, -np.inf, -0.0):
            flat[rng.integers(0, flat.size, flat.size // 50)] = v
        out.append((R, t, K, img, d, m))
    return out


def _colour(b, seed):
    """gamma below and above 1, brightness pushing values negative (fast_powf's overflow path), hues that wrap"""
    rng = np.random.default_rng(seed)
    c = np.stack([rng.uniform(-400, 400, b), rng.uniform(-0.3, 0.3, b), rng.uniform(-0.3, 0.3, b), rng.uniform(0.5, 1.6, b),
                  rng.uniform(-0.9, 0.3, b), rng.uniform(0.4, 1.6, b)], 1).astype(np.float32)
    c[0, 4] = -0.95   # most of item 0's values negative
    return c


def _check_pool(pool, idx, raw, h, w):
    prepared = [od.prepare(img, d, K, R, t, m, w, h) for R, t, K, img, d, m in raw]
    images, depths = pool.images[idx].cpu().numpy(), pool.depths[idx]
    for i, (img, d, cam) in enumerate(prepared):
        assert np.array_equal(images[i], img), "pool image %d" % i
        assert np.array_equal(_bits(depths[i]), _bits(d)), "pool depth %d" % i
        assert np.array_equal(pool.cameras[idx[i]], cam)
    return prepared


def _compare(pool, prepared_all, pairs, params, aug):
    p = dr.reader_params(params)
    got = dr.build_batch(pool, pairs, params, aug)
    ref, used = od.build_batch(prepared_all, pairs, p, aug.rot180, aug.mirror_x, aug.colour)
    assert list(got) == list(p['top_output'])
    assert list(got.used) == list(used)
    for k in p['top_output']:
        g = got[k]
        assert g.is_cuda and g.dtype == torch.float32 and tuple(g.shape) == ref[k].shape, k
        if k == 'MOTION':
            gm = g.cpu().numpy()
            ulp = np.spacing(np.abs(ref[k]).astype(np.float32))
            assert np.all(np.abs(gm.astype(np.float64) - ref[k].astype(np.float64)) <= ulp), k
        else:
            gb, rb = _bits(g), _bits(ref[k])
            bad = np.argwhere(gb != rb)
            assert bad.size == 0, (k, len(bad), bad[:3].tolist(), gb[tuple(bad[0])] if bad.size else None,
                                   rb[tuple(bad[0])] if bad.size else None)
    return got


def _aug(b, colour, seed):
    rot = np.array([COMBOS[i % 4][0] for i in range(b)])
    mir = np.array([COMBOS[i % 4][1] for i in range(b)])
    return dr.Augmentation(rot, mir, _colour(b, seed) if colour else None)


@pytest.fixture(scope="module")
def training_pool():
    raw = _spoil_depths(od.synthetic_views(8, 480, 640, 11), 1)
    pool = dr.ViewPool(256, 192)
    idx = pool.add([View(*v) for v in raw])
    return pool, _check_pool(pool, idx, raw, 192, 256)


@pytest.mark.parametrize("colour", [False, True])
def test_training_configuration(training_pool, colour):
    """training.py's reader: batch 32, 640x480 -> 256x192, ANGLEAXIS6, inverse depth, normalised translation; all six
    outputs, every rot180 / mirror_x combination."""
    pool, prepared = training_pool
    rng = np.random.default_rng(2)
    pairs = [tuple(rng.choice(8, 2, replace=False)) for _ in range(32)]
    params = {'batch_size': 32, 'motion_format': 'ANGLEAXIS6', 'inverse_depth': True, 'norm_trans_scale_depth': True,
              'scaled_width': 256, 'scaled_height': 192, 'top_output': dr.OUTPUTS}
    _compare(pool, prepared, pairs, params, _aug(32, colour, 3))


@pytest.mark.parametrize("fmt", sorted(dr.MOTION_SIZES))
@pytest.mark.parametrize("colour", [False, True])
def test_odd_sizes_ray_length_half_depth_pair(fmt, colour):
    """97x131 -> 61x83 with skew, float16 ray-length depths, depth_pair, min/max depth, every motion format."""
    raw = _spoil_depths(od.synthetic_views(4, 97, 131, 21, skew=0.7, depth_dtype=np.float16, depth_metric='ray_length'), 2)
    pool = dr.ViewPool(61, 83)
    idx = pool.add([View(*v) for v in raw])
    prepared = _check_pool(pool, idx, raw, 83, 61)
    params = {'batch_size': 8, 'motion_format': fmt, 'depth_pair': True, 'min_depth': 2.0, 'max_depth': 3.8,
              'depthmask_border1': 2, 'depthmask_border2': 4, 'image_range_min': -1.0, 'image_range_max': 1.5,
              'norm_trans_scale_depth': fmt != 'QUATERNION'}
    _compare(pool, prepared, [(0, 1), (1, 2), (2, 3), (3, 0), (0, 2), (1, 3), (2, 0), (3, 1)], params, _aug(8, colour, 4))


@pytest.mark.parametrize("colour", [False, True])
def test_integer_factor_ties_round_up_and_equal_size(colour):
    """128x96 -> 64x48 (factor 2, OpenCV's 2x2 path: ties round up) with constructed ties, and 64x48 -> 64x48, in one
    pool with a 131x97 source."""
    raw = od.synthetic_views(3, 96, 128, 31)
    img = raw[0][3]
    img[0:2, 0:2] = [[[1, 2, 3], [2, 3, 3]], [[1, 2, 4], [2, 3, 4]]]   # means 1.5, 2.5, 3.5 -> 2, 3, 4 (ties up)
    img[2:4, 0:2] = 0
    img[2, 0] = [2, 2, 2]                                               # mean 0.5 -> 1
    raw += od.synthetic_views(2, 48, 64, 32) + od.synthetic_views(1, 97, 131, 33)
    pool = dr.ViewPool(64, 48)
    idx = pool.add([View(*v) for v in raw])
    prepared = _check_pool(pool, idx, raw, 48, 64)
    assert list(pool.images[0, 0, 0].cpu().numpy()) == [2, 3, 4] and list(pool.images[0, 1, 0].cpu().numpy()) == [1, 1, 1]
    assert np.array_equal(pool.images[3].cpu().numpy(), raw[3][3])   # equal size: a copy
    params = {'batch_size': 8, 'motion_format': 'ANGLEAXIS7', 'inverse_depth': True}
    _compare(pool, prepared, [(0, 1), (1, 2), (3, 4), (4, 3), (0, 5), (5, 1), (2, 0), (3, 5)], params, _aug(8, colour, 5))


def test_pool_grows_and_keeps_earlier_views():
    raw = od.synthetic_views(20, 60, 80, 41)
    pool = dr.ViewPool(40, 30)
    a = pool.add([View(*v) for v in raw[:3]])
    b = pool.add([View(*v) for v in raw[3:]])   # past the first capacity
    assert list(a) == [0, 1, 2] and list(b) == list(range(3, 20)) and len(pool) == 20
    _check_pool(pool, np.arange(20), raw, 30, 40)


def test_skipped_pairs():
    """t12 = 0 (a view paired with itself) is skipped in every format; a forward motion with equal rotations has
    F(2,2) = 0 and is skipped for FMATRIX only; the next pair fills the slot, and too few pairs raise."""
    raw = od.synthetic_views(3, 48, 64, 51)
    R, t, K, img, d, m = raw[0]
    raw.append((R, t + np.array([0.0, 0.0, 0.4]), K, img, d, m))   # view 3: view 0 moved along its optical axis
    pool = dr.ViewPool(64, 48)
    idx = pool.add([View(*v) for v in raw])
    prepared = _check_pool(pool, idx, raw, 48, 64)
    pairs = [(0, 0), (0, 3), (0, 1), (2, 2), (1, 2), (2, 0)]
    aug = _aug(3, False, 0)
    g = _compare(pool, prepared, pairs, {'batch_size': 3, 'motion_format': 'FMATRIX'}, aug)
    assert list(g.used) == [2, 4, 5]
    g = _compare(pool, prepared, pairs, {'batch_size': 3, 'motion_format': 'ANGLEAXIS6'}, aug)
    assert list(g.used) == [1, 2, 4]
    with pytest.raises(ValueError, match="too few"):
        dr.build_batch(pool, pairs, {'batch_size': 4, 'motion_format': 'FMATRIX'}, _aug(4, False, 0))


def test_batch_feeds_ground_truth_and_network(training_pool):
    """A training batch goes into v2.losses.prepare_ground_truth_tensors and DemonPipelineV2.forward as it is."""
    from demon_b200.v2 import losses, weights as W2
    from demon_b200.v2.networks import DemonPipelineV2, Session
    pool, _ = training_pool
    params = {'batch_size': 2, 'motion_format': 'ANGLEAXIS6', 'inverse_depth': True, 'top_output': ('IMAGE_PAIR', 'MOTION', 'DEPTH', 'INTRINSICS')}
    b = dr.build_batch(pool, [(0, 1), (2, 3)], params, dr.draw_augmentation({'aug_gamma': {'uniform': {'a': 0.8, 'b': 1.2}}}, 2,
                                                                             np.random.default_rng(0)))
    gt = losses.prepare_ground_truth_tensors(b['DEPTH'], b['MOTION'][:, :3], b['MOTION'][:, 3:], b['INTRINSICS'])
    assert gt['flow0'].shape == (2, 2, 192, 256)
    s = Session()
    s.load_weights(W2.synthetic_weights(0))
    out = DemonPipelineV2(s, batch_size=2).forward(b['IMAGE_PAIR'])
    torch.cuda.synchronize()
    assert all(torch.isfinite(v).all() for v in out.values())
