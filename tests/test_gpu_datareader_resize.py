"""GPU: ViewPool.add's two cv::resize calls (csrc/datareader.cu prepare_kernel) against OpenCV's own results, bit for bit.

Every case of tests/golden/make_datareader_golden.py goes through ViewPool.add, and the pool's images (INTER_AREA) and
depths (INTER_NEAREST, compared as bits) must hash to the digests OpenCV gave (tests/golden/datareader_resize_digests.json).
Nothing here runs OpenCV: the fixture is what it returned."""
import importlib.util
import json
import os

import numpy as np
import pytest
import torch

from demon_b200 import datareader as dr
from demon_b200.dataset_tools import View
from oracle import datareader as od

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
EYE = np.eye(3)


def golden_module():
    spec = importlib.util.spec_from_file_location("make_datareader_golden", os.path.join(GOLDEN, "make_datareader_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def committed():
    d = json.load(open(os.path.join(GOLDEN, "datareader_resize_digests.json")))
    d.pop("_opencv")
    return d


def pool_area(images, h, w):
    """every image in one add (one launch), with zero depths"""
    pool = dr.ViewPool(w, h)
    idx = pool.add([View(EYE, np.zeros(3), EYE, im, np.zeros(im.shape[:2], np.float32), 'camera_z') for im in images])
    out = pool.images[idx].cpu().numpy()
    return [out[i] for i in range(len(images))]


def pool_nearest(planes, h, w):
    """every depth plane in one add (one launch), with zero images"""
    pool = dr.ViewPool(w, h)
    idx = pool.add([View(EYE, np.zeros(3), EYE, np.zeros(p.shape + (3,), np.uint8), p, 'camera_z') for p in planes])
    out = pool.depths[idx].cpu().numpy()
    return [out[i] for i in range(len(planes))]


def test_pool_matches_every_opencv_digest():
    """All three INTER_AREA paths at their edges (ties, areas 14..30, an area above 2^24, a wrapping int sum, divisible
    sides whose scale is not integral, slivers below 1e-3 of a cell, 1-pixel sources and outputs, equal size), the row
    and column scans of every width and height up to 2048, and INTER_NEAREST's bits with NaN of both signs, +-inf, -0."""
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    got = golden_module().digests(pool_area, pool_nearest)
    ref = committed()
    assert set(got) == set(ref)
    assert [k for k in got if got[k] != ref[k]] == []


def test_mixed_pool_runs_every_path_in_one_launch_with_float16_depths():
    """640x480 (general), 512x384 (2x2) and 4096x3072 (16x16) sources in one add to 256x192, each with a float16 depth:
    the images and depths are OpenCV's, whichever path each view takes, and a second add appends the same views again."""
    g = golden_module()
    cases = {name: (i, sh, sw, h, w, data) for i, (name, sh, sw, h, w, data) in enumerate(g.CASES)}
    names = ["train/640x480-256x192", "2x2/512x384-256x192", "fast/16x16/4096x3072-256x192"]
    f16 = ["f16/640x480", "f16/512x384", "f16/4096x3072"]
    views, paths = [], []
    for name, (j, (fname, fh, fw)) in zip(names, enumerate(g.F16)):
        i, sh, sw, h, w, data = cases[name]
        assert (sh, sw) == (fh, fw) and (h, w) == g.F16_SIZE
        paths.append(od.area_path(sh, sw, h, w))
        views.append(View(EYE, np.zeros(3), EYE, g.image(100 + i, sh, sw, h, w, data), g.depth16(500 + j, sh, sw), 'camera_z'))
    assert paths == ["general", "2x2", "fast"]
    h, w = g.F16_SIZE
    pool = dr.ViewPool(w, h)
    ref = committed()
    for rep in range(2):
        idx = pool.add(views)
        assert list(idx) == [3 * rep, 3 * rep + 1, 3 * rep + 2]
        images, depths = pool.images[idx].cpu().numpy(), pool.depths[idx].cpu().numpy()
        for k in range(3):
            assert g._entry([images[k]]) == ref["area/" + names[k]], names[k]
            assert g._entry([depths[k]]) == ref["nearest/" + f16[k]], f16[k]
