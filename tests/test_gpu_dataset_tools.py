"""GPU: the dataset tools on the device (csrc/dataset_tools.cu, demon_b200/dataset_tools.py) bit for bit against the
numpy restatements (oracle/view_tools.py), the reference's Cython compute_depth_ratios where oracle/_ref holds it (its
stored digests otherwise) and the reference's groups of the synthetic SUN3D sequence (tests/golden/sun3d_groups.json)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from demon_b200 import dataset_tools as dt
from oracle import dataset_tools as odt
from oracle import view_tools as vt

SHAPES = [(1, 1), (1, 7), (1, 8), (8, 16), (1, 129), (3, 43), (37, 53), (192, 256), (480, 640), (2, 2), (1, 9)]


def bits(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float32)).view(np.uint32)


@pytest.mark.parametrize("shape", SHAPES)
def test_sharpness_equals_numpy(shape):
    h, w = shape
    rng = np.random.RandomState(h * 7 + w)
    yy, xx = np.mgrid[0:h, 0:w]
    imgs = np.stack([rng.randint(0, 256, (h, w, 3)).astype(np.uint8), np.full((h, w, 3), 200, dtype=np.uint8),
                     np.repeat((((yy + xx) % 2) * 255).astype(np.uint8)[:, :, None], 3, axis=2)])
    got = dt.sharpness(torch.from_numpy(imgs).cuda()).cpu().numpy()
    assert np.array_equal(bits(got), bits(odt.sharpness_numpy(imgs)))
    # the one-image API returns the reference's np.float32
    one = dt.measure_sharpness(imgs[0])
    assert isinstance(one, np.float32) and bits(one) == bits(odt.sharpness_numpy(imgs[0]))


def test_sharpness_batch_of_256_cropped_frames():
    rng = np.random.RandomState(11)
    big = torch.from_numpy(rng.randint(0, 256, (256, 500, 660, 3)).astype(np.uint8)).cuda()
    big[::3] = (big[::3] // 32) * 32   # coarser frames: other variances
    frames = big[:, 7:487, 13:653]     # strided: 480x640 windows of 500x660 frames
    got = dt.sharpness(frames).cpu().numpy()
    host = frames.cpu().numpy()
    want = np.concatenate([odt.sharpness_numpy(host[k:k + 32]) for k in range(0, 256, 32)])
    assert np.array_equal(bits(got), bits(want))


def test_sun3d_depth_all_values():
    raw = np.arange(65536, dtype=np.uint32).astype(np.uint16).reshape(2, 128, 256)
    depth, valid = dt.sun3d_depth(raw)
    want = (((raw >> 3) | (raw << 13)) / 1000).astype(np.float32)
    assert np.array_equal(bits(depth.cpu().numpy()), bits(want))
    assert valid.dtype == torch.int64
    assert valid.cpu().tolist() == [int(np.count_nonzero(np.isfinite(want[i]) & (want[i] > 0))) for i in range(2)]
    # a frame of 480x640 with zeros and a single frame
    rng = np.random.RandomState(3)
    r = rng.randint(0, 65536, (3, 480, 640)).astype(np.uint16)
    r[1, :200] = 0
    d, v = dt.sun3d_depth(torch.from_numpy(r.view(np.int16)).cuda())
    assert v.cpu().tolist() == [int(np.count_nonzero(x)) for x in r]
    d1, v1 = dt.sun3d_depth(r[2])
    assert d1.shape == (480, 640) and int(v1) == int(np.count_nonzero(r[2]))


CASES = odt.ratio_edge_cases()


@pytest.mark.parametrize("case", range(len(CASES)))
def test_depth_ratio_maps_equal_cython(case):
    d1, d2, K1, R1, t1, K2, R2, t2 = CASES[case]
    v1 = dt.View(R=R1, t=t1, K=K1, image=None, depth=d1, depth_metric='camera_z')
    v2 = dt.View(R=R2, t=t2, K=K2, image=None, depth=d2, depth_metric='camera_z')
    got = dt.compute_depth_ratios(v1, v2)
    want, oob = odt.depth_ratios_numpy(d1, d2, *vt.operands(K1, R1, t1, K2, R2, t2))
    assert np.isnan(got[oob]).all()
    assert np.array_equal(got, want, equal_nan=True)
    if odt.ratios_available():
        ref = odt.reference_depth_ratios(*CASES[case])
        assert ref.matches(got) if isinstance(ref, odt.RecordedRatios) else np.array_equal(got, ref, equal_nan=True)


def random_views(n, h, w, seed):
    from demon_b200.evaluation import angleaxis_to_rotation_matrix, intrinsics_vector_to_K
    rng = np.random.RandomState(seed)
    K = intrinsics_vector_to_K(np.array([0.891, 1.188, 0.5, 0.5]), w, h)
    views = []
    for i in range(n):
        d = rng.uniform(1.0, 4.0, (h, w)).astype(np.float32)
        d[rng.rand(h, w) < 0.05] = np.nan
        d[rng.rand(h, w) < 0.02] = 0.0
        views.append(dt.View(R=angleaxis_to_rotation_matrix(rng.normal(0, 0.03, 3)), t=rng.normal(0, 0.05, 3), K=K, image=None, depth=d,
                             depth_metric='camera_z'))
    return views


@pytest.mark.parametrize("n,h,w,npairs", [(3, 7, 9, 6), (6, 48, 64, 30), (5, 480, 640, 20), (4, 31, 17, 12)])
def test_fused_counts_equal_counts_over_maps(n, h, w, npairs):
    views = random_views(n, h, w, seed=n * 100 + h)
    K, R, t, P = dt.view_operands(views)
    depth = torch.from_numpy(np.stack([v.depth for v in views])).cuda()
    rng = np.random.RandomState(h)
    pairs = [(i, j) for i in range(n) for j in range(n) if i != j]
    pairs = [pairs[k] for k in rng.randint(0, len(pairs), npairs)]
    pairs += [(j, i) for i, j in pairs]   # both directions
    maps = dt.depth_ratios(depth, K, R, t, P, pairs).cpu().numpy()
    for th in (0.9, 0.97):
        counts = dt.consistency_counts(depth, K, R, t, P, pairs, th).cpu().numpy()
        lo, hi = dt.ratio_thresholds(th)
        for k, (i, j) in enumerate(pairs):
            f = np.isfinite(maps[k])
            assert counts[k, 0] == f.sum() and counts[k, 1] == (f & (maps[k] > lo) & (maps[k] < hi)).sum()
            want, _ = odt.depth_ratios_numpy(views[i].depth, views[j].depth, *vt.operands(views[i].K, views[i].R, views[i].t,
                                                                                         views[j].K, views[j].R, views[j].t))
            assert np.array_equal(maps[k], want, equal_nan=True)
        assert counts[:, 1].sum() > 0 and (counts[:, 1] < counts[:, 0]).any()
    # check_depth_consistency over several views in one launch equals the per-pair host logic
    for k in range(n):
        rest = [v for i, v in enumerate(views) if i != k]
        want = True
        for v in rest:
            r, _ = odt.depth_ratios_numpy(views[k].depth, v.depth, *vt.operands(views[k].K, views[k].R, views[k].t, v.K, v.R, v.t))
            fin = np.isfinite(r)
            lo, hi = dt.ratio_thresholds(0.9)
            if not dt.consistent_from_counts(fin.sum(), (fin & (r > lo) & (r < hi)).sum(), r.size):
                want = False
                break
        assert dt.check_depth_consistency(views[k], rest) == want


def test_sequence_groups_equal_golden(tmp_path):
    root = str(tmp_path)
    odt.write_sequence(root)
    sharp_golden, groups_golden = odt.golden()
    sharp = dt.compute_sharpness(root, odt.SEQ_NAME)
    assert np.array_equal(bits(sharp), bits(sharp_golden))
    groups = dt.sun3d_view_groups(root, odt.SEQ_NAME, odt.BASELINE_RANGE, sharp, sharpness_window=odt.SHARPNESS_WINDOW,
                                  max_views_num=odt.MAX_VIEWS_NUM)
    assert [g['name'] for g in groups] == [g['name'] for g in groups_golden]
    for a, b in zip(groups, groups_golden):
        assert a['frames'] == b['frames'] and np.array_equal(a['viewpoint_pairs'], b['viewpoint_pairs'])
    # the same through sequence_view_groups from arrays: raw uint16 depth per frame, and float32 camera z on the device
    R, t, K, depth, ids = odt.sequence_inputs(root)
    for d in (torch.from_numpy(depth).cuda(), depth):
        got = dt.sequence_view_groups(sharp, R, t, K, d, odt.BASELINE_RANGE, odt.SHARPNESS_WINDOW, odt.MAX_VIEWS_NUM, ids)
        assert ['synthetic_lab.seq_1' + g['suffix'] for g in got] == [g['name'] for g in groups_golden]
        for a, b in zip(got, groups_golden):
            assert a['frames'] == b['frames'] and np.array_equal(a['viewpoint_pairs'], b['viewpoint_pairs'])


def test_bad_arguments():
    frames = torch.zeros((2, 8, 8, 3), dtype=torch.uint8, device="cuda")
    with pytest.raises(ValueError):
        dt.sharpness(frames.cpu())                                  # not CUDA
    with pytest.raises(ValueError):
        dt.sharpness(frames.float())                                # wrong dtype
    with pytest.raises(ValueError):
        dt.sharpness(torch.zeros((1, 4096, 4096, 3), dtype=torch.uint8, device="cuda"))   # h*w = 2^24
    with pytest.raises(ValueError):
        dt.sharpness(frames.permute(0, 2, 1, 3))                    # pixel stride is not 3
    with pytest.raises(ValueError):
        dt.sun3d_depth(np.zeros((2, 4, 4), dtype=np.int32))         # wrong dtype
    views = random_views(2, 8, 8, seed=1)
    small = dt.View(R=views[1].R, t=views[1].t, K=views[1].K, image=None, depth=np.ones((8, 9), np.float32), depth_metric='camera_z')
    with pytest.raises(ValueError):
        dt.compute_depth_ratios(views[0], small)                    # size mismatch
    with pytest.raises(ValueError):
        dt.compute_depth_ratios(views[0], views[1]._replace(depth=views[1].depth.astype(np.float64)))
    K, R, t, P = dt.view_operands(views)
    depth = torch.from_numpy(np.stack([v.depth for v in views])).cuda()
    with pytest.raises(ValueError):
        dt.consistency_counts(depth, K, R, t, P, [(0, 2)])          # pair index out of range
    with pytest.raises(ValueError):
        dt.depth_ratios(torch.zeros((2, 4096, 4096), device="cuda"), K, R, t, P, [(0, 1)])   # h*w = 2^24
    # the C entries check their sizes themselves
    from demon_b200 import _lib
    lib = _lib.load()
    with pytest.raises(ValueError):
        _lib.check(lib.demon_sharpness_u8(frames.data_ptr(), 192, 24, 1, 4096, 4096, depth.data_ptr(), None))
    with pytest.raises(ValueError):
        _lib.check(lib.demon_sun3d_depth_u16(None, 70000, 4, 4, None, None, None))
