"""CPU: the host side of the device evaluation run (demon_b200/evaluation.py): the nearest-neighbour index tables against
scipy, the numpy restatement of compute_visible_points_mask against the reference's own Cython (oracle/view_tools.py;
stored digests where the reference tree is absent), the R / K / P2 construction, and the result table's labels and
layout."""
import json
import math

import numpy as np
import pytest
import scipy.ndimage

from demon_b200 import evaluation as ev
from oracle import view_tools as vt


def zoom_index(n_in, n_out):
    """The input index skimage.transform.resize(order=0) reads: scipy.ndimage.zoom on an index ramp (0 = cval)."""
    ramp = np.arange(1, n_in + 1, dtype=np.float64)[:, None]
    z = scipy.ndimage.zoom(ramp, (n_out / n_in, 1), order=0, grid_mode=True, mode='grid-constant', cval=0)
    assert z.shape[0] == n_out
    return z[:, 0].astype(np.int64) - 1


@pytest.mark.parametrize("n_in", list(range(1, 40)) + [48, 64, 192, 256, 480, 640])
def test_nearest_index_matches_scipy_zoom(n_in):
    for n_out in list(range(1, 40)) + [48, 64, 192, 256, 436, 480, 588, 640, 1000]:
        assert np.array_equal(ev.nearest_index(n_in, n_out), zoom_index(n_in, n_out)), (n_in, n_out)


def test_nearest_index_ties_round_up():
    """192 -> 480 has exact .5 ties in 96 rows; they go to the upper source row."""
    o = np.arange(480)
    c = (o + 0.5) * 192 / 480 - 0.5
    ties = np.flatnonzero(c - np.floor(c) == 0.5)
    assert len(ties) == 96
    assert np.array_equal(ev.nearest_index(192, 480)[ties], np.floor(c[ties]).astype(np.int64) + 1)


@pytest.mark.parametrize("case", range(len(vt.edge_cases())))
def test_numpy_mask_matches_reference_cython(case):
    if not vt.available():
        pytest.skip("neither the reference tree nor the stored digests are present")
    depth, K1, R1, t1, K2, R2, t2, bx, by = vt.edge_cases()[case]
    ref = vt.reference_mask(depth, K1, R1, t1, K2, R2, t2, bx, by)
    mine = vt.visible_points_mask_numpy(depth, *vt.operands(K1, R1, t1, K2, R2, t2), depth.shape[1], depth.shape[0], bx, by)
    if isinstance(ref, vt.Recorded):
        assert ref.matches(mine)
    else:
        assert np.array_equal(mine, ref)


def test_mask_edge_cases_cover_what_they_claim():
    cases = vt.edge_cases()
    assert any(np.isnan(c[0]).any() and (c[0] == 0).any() and (c[0] < 0).any() for c in cases)
    assert any(c[0].shape == (480, 640) for c in cases)
    assert any(not np.array_equal(c[2], np.eye(3)) and np.any(c[3] != 0) for c in cases)
    # the border case: every point lands exactly on u = x, v = y, and the strict tests drop x == border
    border = [c for c in cases if c[0].shape == (12, 10)]
    for depth, K1, R1, t1, K2, R2, t2, bx, by in border:
        m = vt.visible_points_mask_numpy(depth, *vt.operands(K1, R1, t1, K2, R2, t2), 10, 12, bx, by)
        want = np.zeros((12, 10), dtype=np.uint8)
        want[by + 1:12 - by, bx + 1:10 - bx] = 1      # bx < x < 10 - bx and by < y < 12 - by
        assert np.array_equal(m, want)
    # points behind the second camera are dropped even though they are finite and positive
    behind = cases[8]
    m = vt.visible_points_mask_numpy(behind[0], *vt.operands(*behind[1:7]), 24, 16)
    ok = np.isfinite(behind[0]) & (behind[0] > 0)
    assert m.sum() < ok.sum() and (m <= ok).all()


def rodrigues(aa):
    aa = np.asarray(aa, dtype=np.float64)
    th = np.linalg.norm(aa)
    k = aa / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + math.sin(th) * Kx + (1 - math.cos(th)) * Kx.dot(Kx)


def test_rotation_K_and_P2_construction():
    rng = np.random.RandomState(3)
    for _ in range(20):
        aa = rng.normal(0, 0.7, 3)
        R = ev.angleaxis_to_rotation_matrix(aa)
        np.testing.assert_allclose(R, rodrigues(aa), rtol=0, atol=1e-14)
        np.testing.assert_allclose(R.dot(R.T), np.eye(3), rtol=0, atol=1e-14)
    # the 1e-6 angle rule: below it the rotation is exactly the identity
    assert np.array_equal(ev.angleaxis_to_rotation_matrix([3e-7, 0, 4e-7]), np.eye(3))
    assert not np.array_equal(ev.angleaxis_to_rotation_matrix([3e-6, 0, 4e-6]), np.eye(3))
    R, t = ev.motion_vector_to_Rt(np.array([0.1, -0.2, 0.3, 1.0, 2.0, 3.0], dtype=np.float32))
    assert t.dtype == np.float64 and np.array_equal(t, np.array([1.0, 2.0, 3.0]))
    K = ev.intrinsics_vector_to_K(np.array([0.891, 1.188, 0.5, 0.5], dtype=np.float32), 640, 480)
    want = np.array([[np.float64(np.float32(0.891)) * 640, 0, 320], [0, np.float64(np.float32(1.188)) * 480, 240], [0, 0, 1]])
    assert K.dtype == np.float64 and np.array_equal(K, want)
    P2 = ev.projection_matrix(K, R, t)
    Rt32 = np.concatenate([R, t[:, None]], axis=1).astype(np.float32)
    assert P2.dtype == np.float32 and np.array_equal(P2, K.dot(Rt32).astype(np.float32))


def test_visible_points_operands_match_the_views_of_invalidate():
    """evaluate_to_xarray.py:110-119: view 1 at the origin, view 2 at the motion, K of the intrinsics (sun3d if None)."""
    motion = np.array([[0.05, -0.1, 0.02, 0.4, 0.1, -0.2], [0.0, 0.0, 0.0, 1.0, 0.0, 0.0]], dtype=np.float32)
    intr = np.array([[0.9, 1.2, 0.48, 0.52], [0.891, 1.188, 0.5, 0.5]], dtype=np.float32)
    for intrinsics in (intr, None):
        K1, R1, t1, P2 = ev.visible_points_operands(motion, intrinsics, 48, 64)
        for i in range(2):
            R, t = ev.motion_vector_to_Rt(motion[i])
            K = ev.intrinsics_vector_to_K(intr[i] if intrinsics is not None else np.array([ev.SUN3D_INTRINSICS], dtype=np.float32), 64, 48)
            want = vt.operands(K, np.eye(3), np.zeros(3), K, R, t)
            for a, b in zip((K1[i], R1[i], t1[i], P2[i]), want):
                assert a.dtype == np.float32 and np.array_equal(a, b)


def test_iteration_labels_and_error_names():
    labels = ['3_refined', '1', '0_refined', '2', '0', '3', '1_refined', '2_refined']
    assert sorted(labels, key=ev.iteration_sort_key) == ['0', '0_refined', '1', '1_refined', '2', '2_refined', '3', '3_refined']
    assert ev.ERRORS == ['rot_err', 'tran_err', 'tran_angle_err', 'depth_l1', 'depth_l1_inverse', 'depth_scale_invariant',
                         'depth_abs_relative', 'depth_sq_relative', 'depth_avg_log10', 'depth_rmse_log', 'depth_rmse',
                         'depth_ratio_threshold_1.25', 'depth_ratio_threshold_1.5625', 'depth_ratio_threshold_1.953125',
                         'flow_epe', 'camera_baseline']
    assert ev.EIGEN_CROP == (23, 27, 436, 588)


def test_to_dict_layout_is_xarrays(tmp_path):
    """xarray.DataArray.to_dict(): dims, attrs, data, coords {name: {dims, attrs, data}}, name."""
    labels = ['0', '0_refined', '1', '1_refined']
    values = np.arange(1 * 4 * 3 * 16 * 2, dtype=np.float64).reshape(1, 4, 3, 16, 2)
    values[0, 1, :, 0:3, :] = np.nan
    r = ev.EvaluationResult(values, ['snapshot_1'], labels, ['0', '1', '2'], {'depthmask': True, 'depth_scaling': 'abs',
                                                                             'depth_pred_max': 'inf'})
    d = r.to_dict()
    assert list(d) == ['dims', 'attrs', 'data', 'coords', 'name']
    assert d['dims'] == ('snapshot', 'iteration', 'sample', 'errors', 'scaled') and d['name'] is None
    assert list(d['coords']) == list(d['dims'])
    for dim, want in (('snapshot', ['snapshot_1']), ('iteration', labels), ('sample', ['0', '1', '2']), ('errors', ev.ERRORS),
                      ('scaled', [False, True])):
        assert d['coords'][dim] == {'dims': (dim,), 'attrs': {}, 'data': want}
    assert d['attrs']['depth_pred_max'] == 'inf'
    assert np.array_equal(np.array(d['data']), values, equal_nan=True)
    assert r.sel('1', 'depth_l1', True)[2] == values[0, 2, 2, 3, 1]
    path = tmp_path / "eval.json"
    ev.write_xarray_json(r, str(path))
    back = json.load(open(path))
    assert np.array_equal(np.array(back['data'], dtype=np.float64), values, equal_nan=True)
    assert back['coords']['scaled']['data'] == [False, True]
    both = ev.EvaluationResult.concatenate([r, r])
    assert both.values.shape == (1, 4, 6, 16, 2) and both.coords['sample'] == [str(i) for i in range(6)]
