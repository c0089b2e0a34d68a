"""numpy oracle of resize_area (demon_b200.images.resize_area, area_planes_kernel in csrc/net.cu).

`resize_area` restates the project's definition of tf.image.resize_area(align_corners=False) for integer factors
fy = h / oh, fx = w / ow, operation for operation in float32: each source row's fx pixels summed left to right from +0,
the fy row sums summed top to bottom from +0, times float32(1 / (fy fx)).

`area_exact` is TF's area kernel with general (fractional) weights, evaluated in float64: output pixel (y, x) averages the
input over the box [y h/oh, (y+1) h/oh) x [x w/ow, (x+1) w/ow), each input pixel weighted by its overlap with the box.
For integer factors every weight is 1; the float32 oracle must stay within `error_bound` of it.
"""
import numpy as np


def resize_area(x, size):
    """x float32 [..., h, w], size (oh, ow) with h % oh == w % ow == 0 -> float32 [..., oh, ow]."""
    x = np.asarray(x, dtype=np.float32)
    h, w = x.shape[-2:]
    oh, ow = size
    if h % oh or w % ow:
        raise ValueError("not an integer factor: %dx%d -> %dx%d" % (h, w, oh, ow))
    fy, fx = h // oh, w // ow
    v = x.reshape(x.shape[:-2] + (oh, fy, ow, fx))
    total = np.zeros(x.shape[:-2] + (oh, ow), dtype=np.float32)
    for y in range(fy):
        row = np.zeros_like(total)
        for j in range(fx):
            row = row + v[..., :, y, :, j]
        total = total + row
    return total * (np.float32(1) / np.float32(fy * fx))


def _weights(n_in, n_out):
    """[n_out, n_in] float64: the overlap of input pixel i with output pixel o's box [o s, (o+1) s), s = n_in / n_out."""
    s = n_in / n_out
    wts = np.zeros((n_out, n_in))
    for o in range(n_out):
        lo, hi = o * s, (o + 1) * s
        for i in range(int(np.floor(lo)), min(int(np.ceil(hi)), n_in)):
            wts[o, i] = min(hi, i + 1.0) - max(lo, float(i))
    return wts


def area_exact(x, size):
    """TF's area average with general weights in float64: x [..., h, w] -> float64 [..., oh, ow]."""
    x = np.asarray(x, dtype=np.float64)
    h, w = x.shape[-2:]
    oh, ow = size
    wy, wx = _weights(h, oh), _weights(w, ow)
    return np.einsum("oi,...ij,pj->...op", wy, x, wx) / ((h / oh) * (w / ow))


def error_bound(x, size):
    """float64 [..., oh, ow]: a bound on |resize_area(x) - area_exact(x)| for finite x.  k = fy fx terms are summed with
    k - 1 rounded adds, and the scale's rounding and the final multiply add two more: gamma(k + 1) * sum |x| / k."""
    x = np.abs(np.asarray(x, dtype=np.float64))
    h, w = x.shape[-2:]
    oh, ow = size
    k = (h // oh) * (w // ow)
    u = 2.0 ** -24
    gamma = (k + 1) * u / (1 - (k + 1) * u)
    return gamma * x.reshape(x.shape[:-2] + (oh, h // oh, ow, w // ow)).sum(axis=(-3, -1)) / k
