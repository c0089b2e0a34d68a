"""CPU: the oracles of the device dataset tools (demon_b200/dataset_tools.py, csrc/dataset_tools.cu) against the reference:
the pairwise-variance restatement of measure_sharpness against numpy / scipy / Pillow (and the reference's helpers where
its tree is present), the numpy restatement of compute_depth_ratios against the reference's own Cython or its stored
digests, the host side of check_depth_consistency against the reference's function, and the host grouping of
create_samples_from_sequence against the reference's on the synthetic SUN3D sequence (tests/golden/sun3d_groups.json)."""
import os

import numpy as np
import pytest
import scipy.ndimage
from PIL import Image

from demon_b200 import dataset_tools as dt
from oracle import dataset_tools as odt
from oracle import view_tools as vt

SHAPES = [(1, 1), (1, 7), (1, 8), (8, 16), (1, 129), (3, 43), (37, 53), (192, 256), (480, 640), (2, 2), (1, 9)]


def sharp_images(h, w, seed=0):
    rng = np.random.RandomState(seed + h * 1000 + w)
    yield rng.randint(0, 256, (h, w, 3)).astype(np.uint8)
    yield np.full((h, w, 3), 77, dtype=np.uint8)                                    # constant: variance 0
    yy, xx = np.mgrid[0:h, 0:w]
    yield np.repeat((((yy + xx) % 2) * 255).astype(np.uint8)[:, :, None], 3, axis=2)  # checkerboard


def numpy_sharpness(img):
    """helpers.measure_sharpness restated with the libraries it calls."""
    return np.var(scipy.ndimage.laplace(np.array(Image.fromarray(img).convert('L'), dtype=np.float32)))


@pytest.mark.parametrize("shape", SHAPES)
def test_sharpness_numpy_is_numpy_scipy_pillow_bit_for_bit(shape):
    for img in sharp_images(*shape):
        want = numpy_sharpness(img)
        got = odt.sharpness_numpy(img)
        assert got.dtype == np.float32 and want.dtype == np.float32
        assert got.tobytes() == want.tobytes(), (shape, got, want)


def test_sharpness_pairwise_schedule_matters_and_batches():
    """A plain float32 running sum differs from numpy's pairwise one, so the restatement is not trivially right; and the
    vectorised form gives every frame of a batch its own value."""
    rng = np.random.RandomState(1)
    imgs = rng.randint(0, 256, (4, 480, 640, 3)).astype(np.uint8)
    batch = odt.sharpness_numpy(imgs)
    for i in range(4):
        assert batch[i].tobytes() == numpy_sharpness(imgs[i]).tobytes()
    # the Laplacian's own sum is an exact integer; the squared deviations' is not
    lap = odt.laplace_reflect(odt.grey_pillow(imgs[0])).astype(np.float32).reshape(-1)
    sq = (lap - np.float32(lap.mean())) ** 2
    assert np.cumsum(sq, dtype=np.float32)[-1] != odt.pairwise_sum_f32(sq)


def test_grey_matches_pillow():
    rng = np.random.RandomState(2)
    img = rng.randint(0, 256, (64, 64, 3)).astype(np.uint8)
    assert np.array_equal(odt.grey_pillow(img), np.array(Image.fromarray(img).convert('L')))


@pytest.mark.skipif(not odt.have_reference(), reason="the reference tree is absent")
@pytest.mark.parametrize("shape", [(1, 7), (37, 53), (480, 640)])
def test_sharpness_numpy_is_the_references_helper(shape):
    helpers = odt.reference()[0]
    for img in sharp_images(*shape):
        assert odt.sharpness_numpy(img).tobytes() == np.float32(helpers.measure_sharpness(Image.fromarray(img))).tobytes()


RATIO_CASES = odt.ratio_edge_cases()


@pytest.mark.parametrize("case", range(len(RATIO_CASES)))
def test_depth_ratios_numpy_matches_reference_cython(case):
    if not odt.ratios_available():
        pytest.skip("neither the reference tree nor the stored digests are present")
    d1, d2, K1, R1, t1, K2, R2, t2 = RATIO_CASES[case]
    ref = odt.reference_depth_ratios(*RATIO_CASES[case])
    mine, oob = odt.depth_ratios_numpy(d1, d2, *vt.operands(K1, R1, t1, K2, R2, t2))
    # the out-of-array pixels are NaN in both (excluded from the reference's side: its value there is undefined)
    assert np.isnan(mine[oob]).all()
    if isinstance(ref, odt.RecordedRatios):
        assert ref.matches(mine)
    else:
        assert np.array_equal(mine, ref, equal_nan=True)


def test_depth_ratio_cases_cover_what_they_claim():
    """Lists the out-of-array pixels per case and checks the traps are exercised: ties that half-away rounding would send
    elsewhere, x2 = w reading the next row, lookups past the array, denormal d2 (inf ratios), points behind camera 2."""
    oob_counts, ties, alias, infs = [], 0, 0, 0
    for d1, d2, K1, R1, t1, K2, R2, t2 in RATIO_CASES:
        ops = vt.operands(K1, R1, t1, K2, R2, t2)
        r, oob = odt.depth_ratios_numpy(d1, d2, *ops)
        oob_counts.append(int(oob.sum()))
        infs += int(np.isinf(r).sum())
    # the tie cases: u = x + 0.5 exactly
    d1, d2, K1, R1, t1, K2, R2, t2 = RATIO_CASES[6]
    h, w = d1.shape
    r, oob = odt.depth_ratios_numpy(d1, d2, *vt.operands(K1, R1, t1, K2, R2, t2))
    for y in range(h - 1):
        for x in range(w):
            x2 = min(w, int(np.rint(x + 0.5)))
            y2 = min(h, int(np.rint(y + 0.5)))
            ties += int(x2 != int(np.floor(x + 1.0)))   # half away from zero would give x + 1
            want = d2.reshape(-1)[y2 * w + x2] if y2 * w + x2 < h * w else np.nan
            assert r[y, x] == np.float32(1) / want or (np.isnan(want) and np.isnan(r[y, x]))
            alias += int(x2 == w and y2 < h - 1)
    assert ties > 0 and alias > 0 and infs > 0
    assert oob_counts[6] == w and oob_counts[8] == 0   # y2 = h on the last row (even h), none with v = y + 0.5 + 2 ty
    assert oob_counts == [7, 16, 0, 0, 1, 1, 10, 1, 0, 0, 0], oob_counts
    behind = RATIO_CASES[5]
    r, _ = odt.depth_ratios_numpy(behind[0], behind[1], *vt.operands(*behind[2:]))
    assert np.isfinite(r).sum() < (np.isfinite(behind[0]) & (behind[0] > 0)).sum()


def reference_check(dr, th=0.9, min_valid=0.5, min_consistent=0.7):
    """view_tools.check_depth_consistency's body for one ratio map (view_tools.py:82-92)."""
    lo, hi = min(th, 1 / th), max(th, 1 / th)
    valid = dr[np.isfinite(dr)]
    if valid.size / dr.size < min_valid:
        return False
    num = np.count_nonzero((valid > lo) & (valid < hi))
    if num / valid.size < min_consistent:
        return False
    return True


def counts_check(dr, th=0.9, min_valid=0.5, min_consistent=0.7):
    lo, hi = dt.ratio_thresholds(th)
    f = np.isfinite(dr)
    return dt.consistent_from_counts(f.sum(), (f & (dr > lo) & (dr < hi)).sum(), dr.size, min_valid, min_consistent)


def test_counts_logic_equals_check_depth_consistency():
    rng = np.random.RandomState(4)
    for th in (0.9, 1 / 0.9, 0.8, 0.95):
        lo, hi = dt.ratio_thresholds(th)
        assert lo.dtype == np.float32 and lo == np.float32(min(th, 1 / th)) and hi == np.float32(max(th, 1 / th))
        edges = np.array([lo, hi, np.nextafter(lo, np.float32(0)), np.nextafter(lo, np.float32(2)), np.nextafter(hi, np.float32(0)),
                          np.nextafter(hi, np.float32(2))], dtype=np.float32)
        for k in range(200):
            n = rng.randint(1, 60)
            dr = rng.choice(np.concatenate([edges, np.array([np.nan, np.inf, -np.inf, 1.0, 0.5, 2.0], dtype=np.float32)]), n)
            dr = dr.astype(np.float32)
            for mv, mc in ((0.5, 0.7), (0.4, 0.7), (0.0, 0.5), (0.2, 1.0)):
                with np.errstate(invalid='ignore'):
                    assert counts_check(dr, th, mv, mc) == reference_check(dr, th, mv, mc), (dr, th, mv, mc)
    # no finite ratio and min_valid_threshold <= 0: the reference divides np.int64(0) by 0, gets nan with a RuntimeWarning
    # (no ZeroDivisionError) and passes the pair; so does the counts logic
    dr = np.full((4, 4), np.nan, dtype=np.float32)
    with pytest.warns(RuntimeWarning):
        assert reference_check(dr, 0.9, 0.0) is True
    with pytest.warns(RuntimeWarning):
        assert counts_check(dr, 0.9, 0.0) is True
    assert counts_check(dr, 0.9, 0.4) is False


def test_float32_thresholds_are_numpys_comparison():
    """numpy 2 compares a float32 array with a Python float in float32, which the float32 thresholds reproduce; a float64
    comparison would differ where float32(th) rounds above th (r = float32(th) is then > th but not > float32(th))."""
    differs = 0
    for th in (0.9, 0.8, 0.95, 0.7, 0.85):
        lo, hi = dt.ratio_thresholds(th)
        plo, phi = min(th, 1 / th), max(th, 1 / th)
        x = np.array([np.nextafter(v, d) for v in (lo, hi) for d in (np.float32(0), np.float32(2))] + [lo, hi], dtype=np.float32)
        assert np.array_equal(x > plo, x > lo) and np.array_equal(x < phi, x < hi)
        differs += int(np.any((x.astype(np.float64) > plo) != (x > lo)) or np.any((x.astype(np.float64) < phi) != (x < hi)))
    assert differs > 0


def test_synthetic_sequence_golden_and_host_grouping(tmp_path):
    odt.write_sequence(str(tmp_path))
    sharp_golden, groups_golden = odt.golden()
    R, t, K, depth, ids = odt.sequence_inputs(str(tmp_path))
    # the golden sharpness is numpy's on the regenerated images
    seq_images = sorted(os.listdir(os.path.join(str(tmp_path), odt.SEQ_NAME, 'image')))
    sharp = np.array([numpy_sharpness(np.array(Image.open(os.path.join(str(tmp_path), odt.SEQ_NAME, 'image', f)).convert('RGB')))
                      for f in seq_images], dtype=np.float32)
    assert sharp.tobytes() == sharp_golden.tobytes()
    if odt.have_reference():
        s_ref, g_ref = odt.reference_groups(str(tmp_path))
        assert s_ref.tobytes() == sharp_golden.tobytes()
        assert [g['name'] for g in g_ref] == [g['name'] for g in groups_golden]
        for a, b in zip(g_ref, groups_golden):
            assert a['frames'] == b['frames'] and np.array_equal(a['viewpoint_pairs'], b['viewpoint_pairs'])
    # the host grouping with the consistency computed from the numpy ratio maps (and from the reference's Cython function
    # where it exists) gives the golden groups
    sharp_idx = dt.sharp_frames(sharp, odt.SHARPNESS_WINDOW)
    valid = np.count_nonzero(np.isfinite(depth) & (depth > 0), axis=(1, 2))
    size = depth.shape[1] * depth.shape[2]
    views = [vt.View(R=R[f], t=t[f], K=K, image=None, depth=depth[f], depth_metric='camera_z') for f in range(len(R))]

    def numpy_consistent(i1, i2):
        def one(a, b):
            r, _ = odt.depth_ratios_numpy(a.depth, b.depth, *vt.operands(a.K, a.R, a.t, b.K, b.R, b.t))
            return counts_check(r, 0.9, **{'min_valid': 0.4, 'min_consistent': 0.7})
        v1, v2 = views[sharp_idx[i1]], views[sharp_idx[i2]]
        return one(v1, v2) and one(v2, v1)
    checkers = [numpy_consistent]
    if odt.have_reference():
        view_tools = odt.reference()[2]
        checkers.append(lambda i1, i2: (view_tools.check_depth_consistency(views[sharp_idx[i1]], [views[sharp_idx[i2]]], **dt.SEQUENCE_CHECK)
                                        and view_tools.check_depth_consistency(views[sharp_idx[i2]], [views[sharp_idx[i1]]],
                                                                               **dt.SEQUENCE_CHECK)))
    for consistent in checkers:
        groups = dt.group_views(sharp_idx, R, t, valid, size, odt.BASELINE_RANGE, consistent, odt.MAX_VIEWS_NUM, ids)
        assert ['synthetic_lab.seq_1' + g['suffix'] for g in groups] == [g['name'] for g in groups_golden]
        for a, b in zip(groups, groups_golden):
            assert a['frames'] == b['frames'] and np.array_equal(a['viewpoint_pairs'], b['viewpoint_pairs'])
    # the quirks are exercised: a group of max_views_num + 1 views, and a name from the sharp-list position
    assert max(len(g['frames']) for g in groups_golden) == odt.MAX_VIEWS_NUM + 1
    assert any(int(g['name'][-7:]) != g['frames'][0] for g in groups_golden)


def test_read_depth_arithmetic_all_values():
    raw = np.arange(65536, dtype=np.uint32).astype(np.uint16)
    want = (((raw >> 3) | (raw << 13)) / 1000).astype(np.float32)
    s = ((raw.astype(np.uint32) >> 3) | (raw.astype(np.uint32) << 13)) & 0xffff
    assert np.array_equal(np.float32(s / 1000.0), want)
