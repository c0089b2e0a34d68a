"""CPU: the float64 statements of flow_warp, flow_warp_grad, flow_out_of_frame and resample (oracle/flow_ops.py), pinned by
per-element loops, central differences, and the reference's own CPU kernels (oracle/flow_ops_ref.py, or their digests in
tests/golden/flow_ops_digests.json); and the Python layer's shape and dtype errors, raised before any device is needed."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import flow_ops as of
from oracle import flow_ops_ref as fref
from oracle.ref import Recorded

EPS = float(np.finfo(np.float32).eps)


def data(seed, shape, scale=3.0):
    rng = np.random.RandomState(seed)
    n, c, h, w = shape
    return (rng.randn(*shape).astype(np.float32), (rng.randn(n, 2, h, w) * scale).astype(np.float32),
            rng.randn(*shape).astype(np.float32))


def loop_warp(image, flow):
    image = image.astype(np.float64)
    n, c, h, w = image.shape
    out = np.zeros(image.shape)
    for b in range(n):
        for y in range(h):
            for x in range(w):
                x2, y2 = float(np.float32(x) + flow[b, 0, y, x]), float(np.float32(y) + flow[b, 1, y, x])
                if not (0 <= x2 < w and 0 <= y2 < h):
                    continue
                L, T = int(x2), int(y2)
                R, B = min(L + 1, w - 1), min(T + 1, h - 1)
                a, bb = x2 - L, y2 - T
                out[b, :, y, x] = ((1 - a) * (1 - bb) * image[b, :, T, L] + a * (1 - bb) * image[b, :, T, R]
                                   + (1 - a) * bb * image[b, :, B, L] + a * bb * image[b, :, B, R])
    return out


def test_warp_equals_loop():
    image, flow, _ = data(1, (2, 3, 7, 9))
    assert np.allclose(of.flow_warp(image, flow), loop_warp(image, flow), rtol=0, atol=1e-12)


def test_image_grad_is_the_adjoint():
    image, flow, g = data(2, (2, 3, 8, 11))
    ig, _ = of.flow_warp_grad(image, flow, g)
    lhs = (of.flow_warp(image, flow) * g).sum()
    assert abs(lhs - (ig * image).sum()) < 1e-9 * max(1.0, abs(lhs))


def test_flow_grad_central_differences_away_from_edges():
    image, flow, g = data(3, (1, 2, 12, 14), scale=1.5)
    _, fg = of.flow_warp_grad(image, flow, g)
    inside, L, T, R, B, a, b = of._cells(flow)
    h = 1e-3
    checked = 0
    for y in range(12):
        for x in range(14):
            if not inside[0, y, x] or R[0, y, x] == L[0, y, x] or B[0, y, x] == T[0, y, x]:
                continue
            if min(a[0, y, x], 1 - a[0, y, x], b[0, y, x], 1 - b[0, y, x]) < 2e-3:
                continue
            for comp in (0, 1):
                fp, fm = flow.astype(np.float64).copy(), flow.astype(np.float64).copy()
                fp[0, comp, y, x] += h
                fm[0, comp, y, x] -= h
                # the warp is bilinear in the position, so central differences are exact up to rounding; the statement's
                # positions are float32 sums, which moves (a, b) by ~1e-7
                d = ((warp64(image, fp) - warp64(image, fm)) * g)[0, :, y, x].sum() / (2 * h)
                assert abs(d - fg[0, comp, y, x]) < 2e-5 * max(1, abs(d)), (y, x, comp)
                checked += 1
    assert checked > 100


def warp64(image, flow):
    n, c, h, w = image.shape
    ys, xs = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    x2, y2 = xs + flow[:, 0], ys + flow[:, 1]
    inside = (x2 >= 0) & (y2 >= 0) & (x2 < w) & (y2 < h)
    L, T = np.where(inside, np.trunc(np.where(inside, x2, 0)), 0).astype(int), np.where(inside, np.trunc(np.where(inside, y2, 0)), 0).astype(int)
    R, B = np.minimum(L + 1, w - 1), np.minimum(T + 1, h - 1)
    a, b = (x2 - L)[:, None], (y2 - T)[:, None]
    gat = lambda X, Y: of._gather(image.astype(np.float64), X, Y)  # noqa: E731
    out = (1 - a) * (1 - b) * gat(L, T) + a * (1 - b) * gat(R, T) + (1 - a) * b * gat(L, B) + a * b * gat(R, B)
    return np.where(inside[:, None], out, 0.0)


def test_flow_grad_at_clamped_edge_is_the_references_formula():
    """at the last row B = T, so gy = T - y2 = -beta: the x component is -beta (TR - TL) + (1 + beta) (TR - TL), the
    derivative (TR - TL) only by accident of the sum; the y component uses gx = R - x2 likewise"""
    image, _, g = data(4, (1, 1, 4, 5))
    flow = np.zeros((1, 2, 4, 5), np.float32)
    flow[0, 1, 3, :] = 0.25          # last row, y2 = 3.25: in frame, B = T = 3
    _, fg = of.flow_warp_grad(image, flow, g)
    x = 1
    TL, TR = image[0, 0, 3, x].astype(np.float64), image[0, 0, 3, x + 1].astype(np.float64)
    gy = 3 - 3.25
    assert np.isclose(fg[0, 0, 3, x], g[0, 0, 3, x] * (gy * (TR - TL) + (1 - gy) * (TR - TL)))
    assert fg[0, 1, 3, x] == 0.0     # BL - TL and BR - TR vanish: no y gradient at the clamped row


def test_out_of_frame_rounding_and_specials():
    flow = np.zeros((1, 2, 1, 4), np.float32)
    flow[0, 0] = [-0.5, -1.4999, 1.4999, 0.5]   # x + f = -0.5 (out: rounds to -1), -0.4999 (0), 3.4999 (3), 3.5 (out: 4)
    occ = np.full((1, 1, 4), 0.25, np.float32)
    out = of.flow_out_of_frame(flow, occ)
    assert out.ravel().tolist() == [1.0, 0.25, 0.25, 1.0]
    flow[0, 0] = [np.nan, np.inf, 3e9, -np.inf]
    assert of.flow_out_of_frame(flow, occ).ravel().tolist() == [1.0] * 4
    occ[0, 0, 1] = np.nan
    assert np.isnan(of.flow_out_of_frame(flow, occ).ravel()[1])


def test_resample_statement():
    x = np.random.RandomState(5).randn(1, 1, 9, 12)
    assert np.allclose(of.resample(x, 12, 9, True, "LINEAR"), x)          # identity: the triangle weight 1 at d = 0
    assert np.allclose(of.resample(x, 12, 9, True, "CUBIC"), x)
    c = np.full((1, 1, 9, 12), 2.5)
    for t in ("LINEAR", "CUBIC", "NEAREST"):
        assert np.allclose(of.resample(c, 5, 4, True, t), 2.5)            # normalised weights keep constants
    xr, yr = of.resample_positions(64, 16, 8, 16)                        # fy = 8, fx = 1: x_in = x + 4 - 0.5
    assert xr.max() >= 16 and not fref.nearest_in_range(64, 16, 8, 16)


# ---- the reference's CPU kernels --------------------------------------------------------------------------------------------
def _ref_or_skip():
    if not fref.available():
        pytest.skip("neither oracle/_ref/libref_flow_ops.so nor tests/golden/flow_ops_digests.json is present")


CPU_WARP_CASES = [(11, (2, 3, 9, 13)), (12, (1, 5, 16, 7)), (13, (3, 1, 6, 33))]


@pytest.mark.parametrize("seed,shape", CPU_WARP_CASES)
@pytest.mark.parametrize("fill", ["zero", "not_a_number"])
def test_warp_against_reference_cpu(seed, shape, fill):
    _ref_or_skip()
    image, flow, _ = data(seed, shape)
    ref = fref.flow_warp_cpu(image, flow, fill)
    ours = of.flow_warp(image, flow, fill)
    if isinstance(ref, Recorded):
        assert ref.shape == ours.shape   # the digest pins the kernel's bits; the tolerance needs its values
        return
    assert np.array_equal(np.isnan(ref), np.isnan(ours))
    ok = ~np.isnan(ref)
    assert np.allclose(ref[ok], ours[ok], rtol=0, atol=4 * EPS * np.abs(image).max())


@pytest.mark.parametrize("seed,shape", CPU_WARP_CASES)
def test_image_grad_against_reference_cpu(seed, shape):
    _ref_or_skip()
    image, flow, g = data(seed, shape)
    ref = fref.flow_warp_grad_cpu(image, flow, g)
    if isinstance(ref, Recorded):
        assert ref.shape == image.shape
        return
    ig, _ = of.flow_warp_grad(image, flow, g)
    mag, _ = of.flow_warp_grad(image, flow, np.abs(g))
    k = 4 * image.shape[2] * image.shape[3]
    assert (np.abs(ref - ig) <= k * EPS * mag + 1e-30).all()


def test_out_of_frame_against_reference_cpu():
    _ref_or_skip()
    rng = np.random.RandomState(21)
    n, h, w = 2, 9, 13
    ys, xs = np.meshgrid(np.arange(h, dtype=np.float32), np.arange(w, dtype=np.float32), indexing="ij")
    f = (rng.randn(n, 2, h, w) * 4).astype(np.float32)
    pick = rng.randint(0, 6, f.shape)
    f = np.where(pick == 0, np.stack([-xs - 0.5, -ys - 0.5])[None], f)
    f = np.where(pick == 1, np.stack([w - 0.5 - xs, h - 0.5 - ys])[None], f)
    sp = np.array([np.nan, np.inf, -np.inf, 3e9, -3e9], np.float32)
    m = pick == 2
    f[m] = sp[rng.randint(0, len(sp), m.sum())]
    f = f.astype(np.float32)
    occ = rng.rand(n, h, w).astype(np.float32)
    m = rng.rand(n, h, w) < 0.1
    occ[m] = np.array([np.nan, np.inf, -np.inf], np.float32)[rng.randint(0, 3, m.sum())]
    ref = fref.flow_out_of_frame_cpu(f, occ)
    ours = of.flow_out_of_frame(f, occ)
    if isinstance(ref, Recorded):
        assert ref.matches(ours)
    else:
        assert np.array_equal(ref.view(np.uint32), ours.view(np.uint32))


# ---- the Python layer's argument checks (no device needed) ------------------------------------------------------------------
def test_python_shape_and_dtype_errors():
    from demon_b200 import lmbspecialops as ops
    img, fl = np.zeros((1, 3, 4, 5), np.float32), np.zeros((1, 2, 4, 5), np.float32)
    for fn in (ops.flow_warp, ops.flow_warp_grad, ops.flow_out_of_frame, ops.resample, ops.flow_warp_autograd):
        assert callable(fn)
    with pytest.raises(ValueError):
        ops.flow_warp(img[0], fl)
    with pytest.raises(ValueError):
        ops.flow_warp(img, fl[:, :, :3])
    with pytest.raises(ValueError):
        ops.flow_warp(img, np.zeros((2, 2, 4, 5), np.float32))
    with pytest.raises(ValueError):
        ops.flow_warp(img, np.zeros((1, 3, 4, 5), np.float32))
    with pytest.raises(ValueError):
        ops.flow_warp(img, fl, fill_parameter="one")
    with pytest.raises(TypeError):
        ops.flow_warp(img.astype(np.float64), fl)
    with pytest.raises(ValueError):
        ops.flow_warp_grad(img, fl, img[:, :2])
    with pytest.raises(TypeError):
        ops.flow_warp_grad(img, fl, img.astype(np.float64))
    with pytest.raises(ValueError):
        ops.flow_out_of_frame(np.zeros((1, 3, 4, 5), np.float32), np.zeros(20, np.float32))
    with pytest.raises(ValueError):
        ops.flow_out_of_frame(fl, np.zeros(19, np.float32))
    with pytest.raises(TypeError):
        ops.flow_out_of_frame(fl.astype(np.float64), np.zeros(20, np.float32))
    with pytest.raises(ValueError):
        ops.resample(img, 0, 3)
    with pytest.raises(ValueError):
        ops.resample(img, 3, 3, type="AREA")
    with pytest.raises(ValueError):
        ops.resample(img[0], 3, 3)
