"""CPU: the adjust_intrinsics fixture is what Pillow computes, the kernel's window arithmetic (demon_b200.images.
intrinsics_window) equals the reference's, the device's LANCZOS weights cannot differ from Pillow's through CUDA's sin, and bad
arguments are refused before any device work."""
import ctypes
import importlib.util
import json
import os

import numpy as np
import pytest
import torch

from demon_b200 import _lib, build as dbuild, images
from oracle import intrinsics as oi

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
NET = images.intrinsics4(images.demon_intrinsics(), (), "K_new")


def golden_module():
    spec = importlib.util.spec_from_file_location("make_intrinsics_golden", os.path.join(GOLDEN, "make_intrinsics_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_intrinsics_digests_match_pillow():
    """Regenerates every digest with the installed Pillow (the fixture was written with the version under "_pillow")."""
    pytest.importorskip("PIL")
    committed = json.load(open(os.path.join(GOLDEN, "intrinsics_digests.json")))
    committed.pop("_pillow")
    fresh = golden_module().pillow_digests()
    assert set(fresh) == set(committed)
    assert [k for k in fresh if fresh[k] != committed[k]] == []


def test_demon_intrinsics():
    K = images.demon_intrinsics()
    assert K.dtype == np.float64 and K.shape == (3, 3)
    assert np.array_equal(K, [[0.89115971 * 256, 0, 128], [0, 1.18821287 * 192, 96], [0, 0, 1]])
    assert np.array_equal(images.demon_intrinsics(64, 48)[:2, 2], [32, 24])


def _window_cases():
    mod = golden_module()
    out = []
    for _, (_, n, h, w), view, calls in mod.cases():
        if view is not None:
            w, h = view[2], view[3]
        for K, knew, ow, oh in calls[::97]:
            out += [(k, knew, w, h, ow, oh) for k in K]
    rng = np.random.default_rng(5)
    for _ in range(2000):   # random cameras on random image sizes, to DeMoN's 256x192
        w, h = (int(v) for v in rng.integers(1, 4097, 2))
        f = rng.uniform(0.2, 3.0) * max(w, h)
        out.append(((f, f * rng.uniform(0.8, 1.25), rng.uniform(-0.2, 1.2) * w, rng.uniform(-0.2, 1.2) * h), NET, w, h, 256, 192))
    return out


def test_window_arithmetic_equals_the_reference():
    """intrinsics_window states the kernel's IEEE operations (trunc, rint); oracle.window states the reference's Python
    (int(), round()): equal on the fixture's cases, including round()'s ties and products just below an integer, and on
    random cameras.  A resize the reference cannot make is invalid (status 2)."""
    for K, knew, w, h, ow, oh in _window_cases():
        d = images.intrinsics_window(np.asarray(K, np.float64), np.asarray(knew, np.float64), w, h, ow, oh)
        rw, rh, x0, y0, bilinear = oi.window(K, knew, w, h)
        got = tuple(int(d[k]) for k in ("rw", "rh", "x0", "y0", "bilinear", "status"))
        if not (1 <= rw <= 8192 and 1 <= rh <= 8192):   # Pillow refuses an empty resize; the kernel fills the image
            assert got[-1] == 2, (K, knew, w, h)
            continue
        assert got == (rw, rh, x0, y0, int(bilinear), int(oi.leaves(rw, rh, x0, y0, ow, oh))), (K, knew, w, h)


def test_window_ties_and_truncation():
    d = lambda K, knew, w, h, ow, oh: images.intrinsics_window(np.asarray(K), np.asarray(knew), w, h, ow, oh)
    tie = d([[200.0, 200.0, 105.0, 95.0], [200.0, 200.0, 107.0, 93.0]], [100.0, 100.0, 50.0, 50.0], 320, 240, 64, 64)
    assert tie["x0"].tolist() == [2, 4] and tie["y0"].tolist() == [-2, -4]     # 2.5, 3.5, -2.5, -3.5: half to even
    below = d([1.0, 1.0, 0.0, 0.0], [np.nextafter(0.9375, 0), np.nextafter(0.75, 0), 0, 0], 320, 240, 299, 179)
    assert (int(below["rw"]), int(below["rh"])) == (299, 179)                   # 320 * 0.9375 would be 300
    assert (320 * np.nextafter(0.9375, 0), int(320 * np.nextafter(0.9375, 0))) == (299.99999999999994, 299)


def test_window_invalid_intrinsics():
    bad = [(np.nan, 500, 320, 240), (500, 0, 320, 240), (-500, 500, 320, 240), (500, np.inf, 320, 240), (500, 500, np.nan, 240),
           (500, 500, 320, -np.inf), (1e-3, 500, 320, 240), (1e6, 500, 320, 240), (500, 500, 1e12, 240)]
    d = images.intrinsics_window(np.asarray(bad, np.float64), NET, 640, 480, 256, 192)
    assert d["status"].tolist() == [2] * len(bad)
    assert d["rw"].tolist() == [0] * len(bad)


def _lanczos(x):
    with np.errstate(all="ignore"):
        def sinc(v):
            p = v * np.pi
            return np.where(v == 0.0, 1.0, np.sin(p) / p)
        return np.where((-3.0 <= x) & (x < 3.0), sinc(x) * sinc(x / 3), 0.0)


def lanczos_margins(n_in, n_out):
    """Pillow's LANCZOS coefficients for an axis resized from n_in to n_out samples (Resample.c precompute_coeffs, in its
    order of operations, the weight sum sequential) -> (distance of every fixed-point weight w * 2^22 from the nearest
    rounding boundary k + 0.5, the most its value can move when every sin moves by up to 2 ulp)."""
    scale = n_in / n_out
    fs = max(scale, 1.0)
    support, ss = 3.0 * fs, 1.0 / fs
    center = (np.arange(n_out) + 0.5) * scale
    lo = np.maximum(np.trunc(center - support + 0.5), 0).astype(np.int64)
    hi = np.minimum(np.trunc(center + support + 0.5), n_in).astype(np.int64)
    taps = int((hi - lo).max())
    j = lo[:, None] + np.arange(taps)[None, :]
    valid = j < hi[:, None]
    w = np.where(valid, _lanczos(((j - center[:, None]) + 0.5) * ss), 0.0)
    ww = np.zeros(n_out)
    for t in range(taps):
        ww = ww + w[:, t]
    q = np.where(ww[:, None] != 0.0, w / np.where(ww == 0.0, 1.0, ww)[:, None], w) * float(1 << 22)
    margin = np.abs(np.abs(q) % 1.0 - 0.5)
    # Each raw weight is a product of two sin values over exact operations: a sin moved by 2 ulp (CUDA's bound) moves it by
    # at most 2^-51 relative; np.sin, used here, may itself be an ulp from libm's, hence eta = 2 * 3 ulp plus the roundings
    # of the three operations after the sins.  w_j / ww then moves by at most eta (|w_j| + |w_j| sum|w_i| / |ww|) / |ww|.
    eta = 6 * 2.0 ** -52 + 3 * 2.0 ** -53
    absw = np.abs(w).sum(1)
    bound = float(1 << 22) * eta * np.abs(w) / np.abs(ww)[:, None] * (1 + absw / np.abs(ww))[:, None] + 8 * 2.0 ** -53 * (np.abs(q) + 1)
    return margin[valid], bound[valid]


def test_lanczos_weights_do_not_depend_on_the_last_ulps_of_sin():
    """Every quantised LANCZOS weight of every axis the fixture resizes with LANCZOS stays the same when every sin value
    moves by up to 2 ulp, CUDA's documented bound for its double sin: so the device's weights are Pillow's even though
    its sin is not correctly rounded."""
    pairs = golden_module().lanczos_pairs()
    assert len(pairs) > 6000
    worst, count = np.inf, 0
    for n_in, n_out in pairs:
        margin, bound = lanczos_margins(n_in, n_out)
        count += margin.size
        assert np.all(margin > bound), (n_in, n_out, int(np.argmin(margin - bound)))
        worst = min(worst, float(np.min(margin / bound)))
    assert count > 50_000_000 and worst > 1.0


def test_lanczos_restatement_equals_pillow():
    """The weights above are Pillow's: a one-row image whose only non-zero pixel is 255 resized with LANCZOS gives the
    fixed-point weights of every output sample, each clamped to uint8 as Pillow does."""
    from PIL import Image
    n_in, n_out = 37, 11
    for pos in range(n_in):
        row = np.zeros((1, n_in, 3), np.uint8)
        row[0, pos] = 255
        got = np.asarray(Image.fromarray(row).resize((n_out, 1), Image.Resampling.LANCZOS))[0, :, 0]
        scale = n_in / n_out
        center = (np.arange(n_out) + 0.5) * scale
        lo = np.maximum(np.trunc(center - 3 * scale + 0.5), 0).astype(np.int64)
        hi = np.minimum(np.trunc(center + 3 * scale + 0.5), n_in).astype(np.int64)
        exp = []
        for i in range(n_out):
            ws = _lanczos(((np.arange(lo[i], hi[i]) - center[i]) + 0.5) / scale)
            s = 0.0
            for v in ws:
                s += v
            k = {j: int(np.trunc(v / s * 2 ** 22 + (0.5 if v >= 0 else -0.5))) for j, v in zip(range(lo[i], hi[i]), ws)}
            exp.append(min(max(((1 << 21) + 255 * k.get(pos, 0)) >> 22, 0), 255))
        assert got.tolist() == exp, pos


@pytest.mark.parametrize("box", [(-5, -7, 20, 13), (0, -3, 20, 13), (-4, 0, 20, 13), (3, -2, 20, 13), (-3, 2, 20, 13), (6, 5, 30, 13),
                                 (10, 10, 40, 30)])   # boxes that leave the 30x24 image (the only ones it gets)
def test_crop_against_the_reference_safe_crop_image(box):
    """With x0 <= 0 and y0 <= 0 the reference's safe_crop_image returns the crop, and oracle.crop_with_fill (like the device)
    equals it; with x0 > 0 or y0 > 0 it pastes the whole image instead, and the two differ exactly as
    oracle.reference_safe_crop states (DESIGN.md section 7)."""
    from PIL import Image
    safe_crop_image = oi.reference_safe_crop_image()
    img = np.random.default_rng(1).integers(0, 256, (24, 30, 3), dtype=np.uint8)
    x0, y0, w, h = box
    ours = oi.crop_with_fill(img, x0, y0, w, h)
    crop = np.array([[img[y0 + v, x0 + u] if 0 <= y0 + v < 24 and 0 <= x0 + u < 30 else (127, 127, 127) for u in range(w)]
                     for v in range(h)], np.uint8)
    assert np.array_equal(ours, crop)
    restated = oi.reference_safe_crop(img, x0, y0, w, h)
    assert np.array_equal(ours, restated) == (x0 <= 0 and y0 <= 0)
    if safe_crop_image is None:
        pytest.skip("the reference tree (DEMON_REF_SRC) is absent or its dataset_tools/helpers.py does not import")
    ref = np.asarray(safe_crop_image(Image.fromarray(img), (x0, y0, x0 + w, y0 + h), (127, 127, 127)))
    assert np.array_equal(ref, restated)


def test_adjust_intrinsics_argument_errors():
    ok = torch.zeros(1, 48, 64, 3, dtype=torch.uint8)
    K = np.array([[60.0, 0, 32], [0, 60, 24], [0, 0, 1]])
    for args, kw in [
        ((ok.float(), K), {}),
        ((ok, K), {}),                                                     # a CPU tensor
        ((torch.zeros(1, 64, 48, 4, dtype=torch.uint8), K), {}),
        ((ok, np.zeros((2, 3))), {}),                                      # K shape
        ((ok, np.zeros((2, 3, 3))), {}),                                   # K for two images
        ((ok, K), {"width_new": 0}),
        ((ok, K), {"height_new": 8193}),
        ((ok, K), {"K_new": [[0.0, 0, 1], [0, 1, 1], [0, 0, 1]]}),         # zero target focal length
        ((ok, K), {"K_new": np.zeros(3)}),
    ]:
        with pytest.raises(ValueError):
            images.adjust_intrinsics(*args, **kw)


def test_host_intrinsics_are_checked_before_device_work():
    """A CPU image tensor would fail later; the intrinsics are refused first, before any device call."""
    x = torch.zeros(2, 48, 64, 3, dtype=torch.uint8)
    for bad in ([np.nan, 60, 32, 24], [0, 60, 32, 24], [60, -1, 32, 24], [60, 60, np.inf, 24], [1e-4, 60, 32, 24], [60, 60, 1e12, 24]):
        K = np.array([[60.0, 60, 32, 24], bad])
        with pytest.raises(ValueError, match="image 1"):
            images._device_intrinsics(K, (2,), "K", 64, 48, NET, 256, 192, x.device)
    with pytest.raises(ValueError, match="taller"):
        images._check_adjust_source(101, 1, "images")
    images._check_adjust_source(100, 1, "images")


def test_intrinsics4_forms():
    K33 = np.array([[[500.0, 0.5, 320], [0, 510, 240], [0, 0, 1]]] * 3)
    K4 = np.array([[500.0, 510, 320, 240]] * 3)
    assert np.array_equal(images.intrinsics4(K33, (3,), "K"), K4)                     # the skew is ignored
    assert np.array_equal(images.intrinsics4(K33[0], (3,), "K"), K4)                  # one K for all
    assert np.array_equal(images.intrinsics4(torch.from_numpy(K4).float(), (3,), "K"), K4)
    assert np.array_equal(images.intrinsics4(K33.reshape(3, 1, 3, 3).repeat(2, 1), (3, 2), "K"), np.repeat(K4[:, None], 2, 1))


def test_adjust_and_pipeline_args_reject_bad_arguments_before_any_device_work():
    dbuild.build()
    lib = _lib.load()
    buf = (ctypes.c_uint8 * 64)()
    p = ctypes.addressof(buf)
    calls = [
        (None, 24, 24, 1, 8, 8, p, 500.0, 500.0, 4.0, 4.0, p, 4, 4, p),        # null source
        (p, 24, 24, 1, 8, 8, None, 500.0, 500.0, 4.0, 4.0, p, 4, 4, p),        # null K
        (p, 24, 24, 1, 8, 8, p, 500.0, 500.0, 4.0, 4.0, p, 4, 4, None),        # null status
        (p, 24, 24, -1, 8, 8, p, 500.0, 500.0, 4.0, 4.0, p, 4, 4, p),          # n
        (p, -24, 24, 1, 8, 8, p, 500.0, 500.0, 4.0, 4.0, p, 4, 4, p),          # negative stride
        (p, 24, 24, 1, 0, 8, p, 500.0, 500.0, 4.0, 4.0, p, 4, 4, p),           # empty source
        (p, 24, 3, 1, 801, 8, p, 500.0, 500.0, 4.0, 4.0, p, 4, 4, p),          # more than 100 times taller than wide
        (p, 24, 24, 1, 8, 8, p, 0.0, 500.0, 4.0, 4.0, p, 4, 4, p),             # target focal length
        (p, 24, 24, 1, 8, 8, p, 500.0, float("nan"), 4.0, 4.0, p, 4, 4, p),
        (p, 24, 24, 1, 8, 8, p, 500.0, 500.0, float("inf"), 4.0, p, 4, 4, p),  # target principal point
        (p, 24, 24, 1, 8, 8, p, 500.0, 500.0, 4.0, 4.0, p, 0, 4, p),           # output size
        (p, 24, 24, 1, 8, 8, p, 500.0, 500.0, 4.0, 4.0, p, 4, 8193, p),
    ]
    for args in calls:
        assert lib.demon_adjust_intrinsics_u8(*args, None) == -1, args
    args = _lib.PipelineArgs(input=_lib.INPUT_VIEWS_U8, images=p, h=480, w=640, K=p, status=p, resample=3, image2_2_mode=1,
                             iterations=3)
    assert lib.demon_pipeline_run(None, args, None) == -1
