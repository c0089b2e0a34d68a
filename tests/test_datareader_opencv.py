"""CPU: the multi-view reader's two cv::resize calls as oracle/datareader.py restates them, held to OpenCV.

tests/golden/datareader_resize_digests.json holds OpenCV's results for every case of make_datareader_golden.py.  With cv2
importable the fixture is regenerated and compared, and the oracle is compared with cv2 on random sizes; without it the
oracle is still held to the committed digests.  The exact area mean (this project's earlier definition of INTER_AREA)
lives here only as a yardstick for the general path."""
import importlib.util
import json
import os

import numpy as np
import pytest

from oracle import datareader as od

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def golden_module():
    spec = importlib.util.spec_from_file_location("make_datareader_golden", os.path.join(GOLDEN, "make_datareader_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def committed():
    d = json.load(open(os.path.join(GOLDEN, "datareader_resize_digests.json")))
    d.pop("_opencv")
    return d


def oracle_area(images, h, w):
    return [od.area_downscale(im, h, w) for im in images]


def oracle_nearest(planes, h, w):
    return [p[od.nearest_indices(p.shape[0], h)][:, od.nearest_indices(p.shape[1], w)] for p in planes]


def exact_area_mean(img, h, w):
    """the exact area-weighted mean of the source cells each output cell covers, float64 [h, w, c]"""
    def overlap(n, m):   # [m, n]: output cell o = [o*n, (o+1)*n) against source cell i = [i*m, (i+1)*m), in 1/m cells
        o, i = np.arange(m)[:, None], np.arange(n)[None, :]
        return np.maximum(0, np.minimum((i + 1) * m, (o + 1) * n) - np.maximum(i * m, o * n)).astype(np.float64)
    sh, sw = img.shape[:2]
    wy, wx = overlap(sh, h), overlap(sw, w)
    return np.stack([wy @ img[:, :, c].astype(np.float64) @ wx.T for c in range(img.shape[2])], -1) / (sh * sw)


def test_digests_match_opencv():
    """Regenerates every digest with the installed OpenCV: the fixture was written with the version under "_opencv"."""
    cv2 = pytest.importorskip("cv2")
    d = json.load(open(os.path.join(GOLDEN, "datareader_resize_digests.json")))
    assert d["_opencv"] == "4.13.0"
    fresh = golden_module().opencv_digests()
    assert set(fresh) == set(committed()), cv2.__version__
    assert [k for k in fresh if fresh[k] != committed()[k]] == []


def test_oracle_matches_committed_digests():
    """Every case, the row and column scans included, through the oracle: bit for bit what OpenCV returned."""
    fresh = golden_module().digests(oracle_area, oracle_nearest)
    ref = committed()
    assert set(fresh) == set(ref)
    assert [k for k in fresh if fresh[k] != ref[k]] == []


def test_cases_cover_every_path():
    g = golden_module()
    paths = {}
    for name, sh, sw, h, w, _ in g.CASES:
        paths.setdefault(name.split("/")[0], set()).add(od.area_path(sh, sw, h, w))
    assert paths["2x2"] == {"2x2"} and paths["fast"] == {"fast"} and paths["divisible"] == {"general"}
    assert paths["near"] == paths["sliver"] == paths["train"] == {"general"} and paths["edge"] == {"fast", "general"}
    for name, sh, sw, h, w, _ in g.CASES:
        if name.startswith("divisible"):
            assert sh % h == 0 and sw % w == 0, name
    assert [od.area_path(sh, sw, *g.F16_SIZE) for _, sh, sw in g.F16] == ["general", "2x2", "fast"]


def test_oracle_matches_opencv_on_random_sizes():
    """Several hundred seeded (sh, sw, h, w) with sides up to 1100, both calls, every path."""
    cv2 = pytest.importorskip("cv2")
    g = golden_module()
    rng = np.random.default_rng(20)
    seen = set()
    for i in range(300):
        if i % 3 == 0:   # an integer factor on both axes (the fast paths), or one axis off by one
            h, w = rng.integers(1, 120, 2)
            ky, kx = rng.integers(1, 9, 2)
            sh, sw = h * ky + (i % 2), w * kx
        else:
            sh, sw = rng.integers(1, 1101, 2)
            h, w = rng.integers(1, sh + 1), rng.integers(1, sw + 1)
        sh, sw, h, w = int(sh), int(sw), int(h), int(w)
        seen.add(od.area_path(sh, sw, h, w))
        img = rng.integers(0, 256, (sh, sw, 3), dtype=np.uint8)
        ref = cv2.resize(img, (w, h), interpolation=cv2.INTER_AREA).reshape(h, w, 3)
        assert np.array_equal(od.area_downscale(img, h, w), ref), (sh, sw, h, w, od.area_path(sh, sw, h, w))
        d = g.depth(i, sh, sw)
        ref = cv2.resize(d, (w, h), interpolation=cv2.INTER_NEAREST).reshape(h, w)
        assert np.array_equal(oracle_nearest([d], h, w)[0].view(np.uint32), ref.view(np.uint32)), (sh, sw, h, w)
    assert seen == {"2x2", "fast", "general"}


def test_path_classifier_is_opencvs_test_for_every_pair_up_to_8192():
    """OpenCV's per-axis test |scale - cvRound(scale)| < DBL_EPSILON, scale = 1 / (m / (double)n), restated over every
    n -> m with m <= n <= 8192: an integral scale implies n divisible by m, and 4802 divisible pairs (98 -> 2, 147 -> 3,
    49 -> 1, ...) are not integral.  oracle.area_factor agrees with it on every divisible pair and on a sample of the rest."""
    fast_pairs, not_fast = set(), []
    for n in range(1, 8193):
        m = np.arange(1, n + 1)
        s = 1.0 / (m / float(n))
        fast = np.abs(s - np.rint(s)) < np.finfo(np.float64).eps
        assert np.all(n % m[fast] == 0), n
        fast_pairs.update((n, int(k)) for k in m[fast])
        div = m[(n % m == 0) & ~fast]
        not_fast += [(n, int(k)) for k in div]
    assert len(not_fast) == 4802
    assert {(98, 2), (147, 3), (49, 1)} <= set(not_fast)
    for n, m in not_fast:
        assert od.area_factor(n, m) is None, (n, m)
    for n, m in fast_pairs:
        assert od.area_factor(n, m) == n // m, (n, m)
    rng = np.random.default_rng(0)
    for n in rng.integers(2, 8193, 20000):
        m = int(rng.integers(1, n + 1))
        assert (od.area_factor(int(n), m) is not None) == ((int(n), m) in fast_pairs)
    assert od.area_path(4, 4, 2, 2) == "2x2" and od.area_path(4, 8, 2, 2) == "fast"
    assert od.area_path(4, 98, 2, 2) == "general" and od.area_path(5, 4, 2, 2) == "general"


def test_divisible_but_not_fast_takes_opencvs_general_path():
    """On the divisible pairs whose scale is not integral OpenCV's result is the general path's, and on some of them the
    integer path would give a different image."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(3)
    differs = 0
    for sw, w in ((98, 2), (147, 3), (49, 1), (196, 4), (198, 2), (8190, 35), (8190, 78), (93, 1), (1666, 98)):
        img = rng.integers(0, 256, (3, sw, 3), dtype=np.uint8)
        ref = cv2.resize(img, (w, 3), interpolation=cv2.INTER_AREA).reshape(3, w, 3)
        assert np.array_equal(od.area_downscale(img, 3, w), ref), (sw, w)
        k = sw // w
        blocks = img.reshape(3, w, k, 3).astype(np.int64).sum(2)
        differs += int((np.rint(blocks.astype(np.float32) * np.float32(1.0 / k)) != ref).sum())
    assert differs > 0


def test_integer_paths_rounding():
    """2x2 rounds a tie up, the other integer factors multiply by float(1/area) and round half to even, which at area 14
    is not the exact mean rounded."""
    tie = np.array([[[1, 2, 0], [2, 3, 0]], [[1, 2, 0], [2, 3, 0]]], np.uint8)   # means 1.5, 2.5, 0
    assert list(od.area_downscale(tie, 1, 1)[0, 0]) == [2, 3, 0]
    sums = np.arange(14 * 255 + 1)   # every block sum of 14 pixels
    row = (sums[:, None] // 14 + (np.arange(14)[None, :] < sums[:, None] % 14)).astype(np.uint8).reshape(1, -1, 1)
    out = od.area_downscale(np.repeat(row, 3, 2), 1, sums.size)[0, :, 0].astype(np.int64)
    assert np.array_equal(out, np.rint(sums.astype(np.float32) * np.float32(1.0 / 14)))
    assert np.count_nonzero(out != np.rint(sums / 14)) > 0


def test_general_path_stays_within_one_of_the_exact_mean():
    """The float weights and float accumulation of the general path move a value by less than 1 from the exact
    area mean, and at training.py's 640x480 -> 256x192 (every weight k/25) not at all from its rounding."""
    rng = np.random.default_rng(8)
    for sh, sw, h, w in ((480, 640, 192, 256), (480, 640, 160, 213), (97, 131, 83, 61), (481, 641, 240, 320), (300, 1, 7, 1),
                         (1, 8190, 1, 35), (1000, 999, 3, 997), (577, 769, 192, 256)):
        assert od.area_path(sh, sw, h, w) == "general"
        img = rng.integers(0, 256, (sh, sw, 3), dtype=np.uint8)
        out, exact = od.area_downscale(img, h, w).astype(np.float64), exact_area_mean(img, h, w)
        assert np.abs(out - exact).max() < 1.0, (sh, sw, h, w)
        if (sh, sw) == (480, 640) and (h, w) == (192, 256):
            assert np.array_equal(out, np.rint(exact))


def test_area_table_entries():
    """computeResizeAreaTab at 640 -> 213 (output 0 covers source cells 0..3, the last one in part) and at 1024 -> 1023,
    where output 0 overlaps source cell 1 by 1/1023 of a cell, below the table's 1e-3: that sliver gets no entry."""
    idx, wt = od.area_table(640, 213)
    scale = 640 / 213
    assert list(idx[0]) == [0, 1, 2, 3] and wt[0, 3] == np.float32((scale - 3) / scale)
    assert np.all(wt[0, :3] == np.float32(1 / scale))
    idx, wt = od.area_table(1024, 1023)
    assert list(idx[0]) == [0, 0] and list(wt[0]) == [np.float32(1023 / 1024), 0]
    assert list(idx[1]) == [1, 2] and wt[1, 0] == np.float32((2 - 1024 / 1023) / (1024 / 1023))
    for n, m in ((640, 213), (1024, 1023), (2049, 2048), (97, 83), (8190, 35)):
        idx, wt = od.area_table(n, m)
        assert np.allclose(wt.astype(np.float64).sum(1), 1.0, atol=1.5e-3), (n, m)
