"""ORACLE (test infrastructure): float64 statements of lmbspecialops' FlowWarp, FlowWarpGrad, FlowOutOfFrame and Resample
(flowwarp.cc, flow_out_of_frame.cc, resample_cuda.cu), written from the ops' definitions, not from their code.

Positions are formed as the reference forms them, in float32 (x + fx, and the resample source position with its swapped
half offsets); everything after that is float64.  tests/test_flow_ops.py pins these statements by per-element loops and
central differences, and against the reference's own CPU kernels.
"""
import numpy as np

NAN_FILL_BITS = 0xFFE00000   # the reference GPU kernel's fill for 'not_a_number' (flowwarp_cuda.cu: int nan = 0xFFE00000)


def _cells(flow):
    """-> in-frame mask, L, T, R, B, alpha, beta (float64) for flow [n,2,h,w]."""
    flow = np.asarray(flow, dtype=np.float32)
    n, _, h, w = flow.shape
    ys, xs = np.meshgrid(np.arange(h, dtype=np.float32), np.arange(w, dtype=np.float32), indexing="ij")
    with np.errstate(invalid="ignore", over="ignore"):
        x2 = (xs[None] + flow[:, 0]).astype(np.float32)
        y2 = (ys[None] + flow[:, 1]).astype(np.float32)
        inside = (x2 >= 0) & (y2 >= 0) & (x2 < w) & (y2 < h)
    L = np.where(inside, np.trunc(np.where(inside, x2, 0)), 0).astype(np.int64)
    T = np.where(inside, np.trunc(np.where(inside, y2, 0)), 0).astype(np.int64)
    R = np.minimum(L + 1, w - 1)
    B = np.minimum(T + 1, h - 1)
    a = np.where(inside, x2.astype(np.float64) - L, 0.0)
    b = np.where(inside, y2.astype(np.float64) - T, 0.0)
    return inside, L, T, R, B, a, b


def _gather(image, L, T):
    n, c = image.shape[:2]
    ni = np.arange(n)[:, None, None, None]
    ci = np.arange(c)[None, :, None, None]
    return image[ni, ci, T[:, None], L[:, None]]


def flow_warp(image, flow, fill_parameter="zero"):
    """warped[n,c,y,x] = bilinear interpolation of image at (x + fx, y + fy), corners L = floor, R = min(L+1, w-1) (and T,
    B), or the fill out of frame: 0, or for 'not_a_number' a NaN (the device writes the bits NAN_FILL_BITS)."""
    image = np.asarray(image, dtype=np.float64)
    inside, L, T, R, B, a, b = _cells(flow)
    a, b = a[:, None], b[:, None]
    with np.errstate(invalid="ignore", over="ignore"):
        out = ((1 - a) * (1 - b) * _gather(image, L, T) + a * (1 - b) * _gather(image, R, T)
               + (1 - a) * b * _gather(image, L, B) + a * b * _gather(image, R, B))
    fill = 0.0 if fill_parameter == "zero" else np.nan
    return np.where(inside[:, None], out, fill)


def flow_warp_grad(image, flow, gradient):
    """-> (image_grad, flow_grad) of the reference's FlowWarpGrad.  image_grad is the adjoint of flow_warp in the image;
    flow_grad is the reference's formula: for x, sum_c g (gy (TR - TL) + (1 - gy) (BR - BL)) with gy = B - y2, for y,
    sum_c g (gx (BL - TL) + (1 - gx) (BR - TR)) with gx = R - x2; away from the clamped last row and column this is the
    derivative of flow_warp in the flow.  Out-of-frame pixels give nothing."""
    image = np.asarray(image, dtype=np.float64)
    g = np.asarray(gradient, dtype=np.float64)
    n, c, h, w = image.shape
    inside, L, T, R, B, a, b = _cells(flow)
    flow32 = np.asarray(flow, dtype=np.float32)
    ys, xs = np.meshgrid(np.arange(h, dtype=np.float32), np.arange(w, dtype=np.float32), indexing="ij")
    with np.errstate(invalid="ignore", over="ignore"):
        x2 = (xs[None] + flow32[:, 0]).astype(np.float64)
        y2 = (ys[None] + flow32[:, 1]).astype(np.float64)
    gm = np.where(inside[:, None], g, 0.0)
    image_grad = np.zeros_like(image)
    ni = np.broadcast_to(np.arange(n)[:, None, None, None], gm.shape)
    ci = np.broadcast_to(np.arange(c)[None, :, None, None], gm.shape)
    A, Bt = a[:, None], b[:, None]
    for wgt, yy, xx in (((1 - A) * (1 - Bt), T, L), (A * (1 - Bt), T, R), ((1 - A) * Bt, B, L), (A * Bt, B, R)):
        np.add.at(image_grad, (ni, ci, np.broadcast_to(yy[:, None], gm.shape), np.broadcast_to(xx[:, None], gm.shape)), gm * wgt)
    TL, TR, BL, BR = _gather(image, L, T), _gather(image, R, T), _gather(image, L, B), _gather(image, R, B)
    gy = np.where(inside, B - y2, 0.0)[:, None]
    gx = np.where(inside, R - x2, 0.0)[:, None]
    with np.errstate(invalid="ignore", over="ignore"):
        fgx = (gm * (gy * (TR - TL) + (1 - gy) * (BR - BL))).sum(axis=1)
        fgy = (gm * (gx * (BL - TL) + (1 - gx) * (BR - TR))).sum(axis=1)
    flow_grad = np.stack([np.where(inside, fgx, 0.0), np.where(inside, fgy, 0.0)], axis=1)
    return image_grad, flow_grad


def flow_out_of_frame(flow, occ):
    """[n,1,h,w]: occ where the target (x + fx, y + fy), rounded half away from zero, lies in the image, else 1; a NaN occ
    stays.  A NaN, infinite or beyond-int32 target is out of frame (x86 converts it to INT_MIN)."""
    flow = np.asarray(flow, dtype=np.float32)
    n, _, h, w = flow.shape
    occ = np.asarray(occ, dtype=np.float32).reshape(n, 1, h, w)
    ys, xs = np.meshgrid(np.arange(h, dtype=np.float32), np.arange(w, dtype=np.float32), indexing="ij")

    def rint(f):
        d = np.where(f >= 0, f.astype(np.float64) + 0.5, f.astype(np.float64) - 0.5)
        ok = np.isfinite(d) & (np.abs(d) < 2.0 ** 31)
        return np.where(ok, np.trunc(np.where(ok, d, 0)), -(2.0 ** 31))

    with np.errstate(invalid="ignore", over="ignore"):
        x2 = rint((xs[None] + flow[:, 0]).astype(np.float32))
        y2 = rint((ys[None] + flow[:, 1]).astype(np.float32))
    inside = ((x2 >= 0) & (y2 >= 0) & (x2 < w) & (y2 < h))[:, None]
    return np.where(inside | np.isnan(occ), occ, np.float32(1.0)).astype(np.float32)


def _round_half_away(v):
    return np.sign(v) * np.floor(np.abs(v) + 0.5)


def resample_positions(in_h, in_w, out_h, out_w):
    """Source positions (float32, as the reference forms them: fma(x_out, fx, fy/2) - 0.5 and fma(y_out, fy, fx/2) - 0.5, the
    half offsets swapped) rounded half away from zero -> (x_round [out_w], y_round [out_h]) as int64."""
    xin, yin, _, _ = _positions(in_h, in_w, out_h, out_w)
    return _round_half_away(xin.astype(np.float64)).astype(np.int64), _round_half_away(yin.astype(np.float64)).astype(np.int64)


def _positions(in_h, in_w, out_h, out_w):
    f32 = np.float32
    fx, fy = f32(in_w) / f32(out_w), f32(in_h) / f32(out_h)
    xo, yo = np.arange(out_w, dtype=np.float32), np.arange(out_h, dtype=np.float32)
    # the reference's fma(x_out, fx, fy / 2): the float products are exact in float64, and the sum is rounded once to float32
    xin = ((xo.astype(np.float64) * fx + np.float64(fy * f32(0.5))).astype(np.float32) - f32(0.5)).astype(np.float32)
    yin = ((yo.astype(np.float64) * fy + np.float64(fx * f32(0.5))).astype(np.float32) - f32(0.5)).astype(np.float32)
    return xin, yin, fx, fy


def _bicubic(x):
    x = np.abs(x)
    return np.where(x <= 1, x * x * (1.5 * x - 2.5) + 1, np.where(x < 2, x * (x * (-0.5 * x + 2.5) - 4) + 2, 0.0))


def _triangle(x):
    return np.where((x >= -1) & (x < 0), x + 1, np.where((x >= 0) & (x <= 1), 1 - x, 0.0))


def _axis_weights(pos, n_in, f, scale, kernel_width, kern):
    """[n_out, n_in] weights scale k(scale (pos - i)) over the reference's window |i - round(pos)| <= r."""
    r = 2 if f < 1 else int(np.ceil(np.float32(kernel_width) / np.float32(scale)))
    pr = _round_half_away(pos.astype(np.float64))
    i = np.arange(n_in)[None, :]
    d = pos.astype(np.float64)[:, None] - i
    wgt = scale * kern(scale * d)
    return np.where(np.abs(i - pr[:, None]) <= r, wgt, 0.0)


def resample(input, width, height, antialias=True, type="LINEAR"):
    """Resample's output [n,c,height,width] in float64.  NEAREST: the pixel at the rounded source position, clamped to the
    image.  LINEAR / CUBIC: the normalised weighted sum over the reference's window with separable weights
    (scale k(scale d)) per axis, scale = 1/f on both axes when antialias and either axis downsamples, else 1; a zero
    weight sum gives 0."""
    a = np.asarray(input, dtype=np.float64)
    n, c, ih, iw = a.shape
    xin, yin, fx, fy = _positions(ih, iw, height, width)
    if type == "NEAREST":
        xr, yr = resample_positions(ih, iw, height, width)
        xr, yr = np.clip(xr, 0, iw - 1), np.clip(yr, 0, ih - 1)
        return a[:, :, yr[:, None], xr[None, :]]
    kern, kw = (_bicubic, 4) if type == "CUBIC" else (_triangle, 2)
    aa = bool(antialias) and (fx > 1 or fy > 1)
    sx = float(np.float32(1) / fx) if aa else 1.0
    sy = float(np.float32(1) / fy) if aa else 1.0
    Wx = _axis_weights(xin, iw, fx, sx, kw, kern)
    Wy = _axis_weights(yin, ih, fy, sy, kw, kern)
    num = np.matmul(np.matmul(Wy, a), Wx.T)
    den = np.outer(Wy.sum(axis=1), Wx.sum(axis=1))[None, None]
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(den == 0, 0.0, num / np.where(den == 0, 1.0, den))
