"""ORACLE (test infrastructure) -- float64 numpy statement of lmbspecialops' Correlation, Correlation1D and their gradients,
written from the ops' definitions:

  top[n, tc, y, x] = sum_{j, i < K, c} f(P1[n, c, Y1 + j, X1 + i], P2[n, c, Y1 + dy + j, X1 + dx + i]) / (K K C)

with P1, P2 the inputs zero-padded by pad_size (columns both sides; rows too for the 2D op), (X1, Y1) = (x s1 + md, y s1 + mdy)
(mdy = md for 2D, 0 for 1D), displacement channel tc = dyi * gw + dxi, (dx, dy) = ((dxi + xshift) s2, (dyi - ry) s2) and
f = a b ('mult') or |a - b| ('subt').  Every read outside the padded input is 0 (for the 1D op's single_dir = -1 this is
where the reference reads before the start of a padded row).

Gradients: 'mult' is the adjoint of the forward op (the CPU tests pin <top(x1, x2), g> = <x1, grad1> = <x2, grad2>).
'subt' is the reference's gradient.  With E(q) = +1 where P1(q) >= P2(q) and -1 elsewhere (a NaN compares false), every top
element g that reads input1 at padded position q1 = (Y1 + j, X1 + i) and input2 at q1 + d adds g E(q1 + d) to input1_grad
at q1 and -g E(q1) to input2_grad at q1 + d: the sign is taken at ONE position for both inputs, as the reference's kernels
take it, not the derivative of |a - b|.

Only tests/ and tools/ may import this module.
"""
import numpy as np


def geometry(shape, max_displacement, kernel_size, stride1=1, stride2=1, pad_size=0, one_d=False, single_dir=0):
    """dict of the op's derived sizes; the top size is ceil in float32 as the reference computes it."""
    n, c, h, w = (int(s) for s in shape)
    ks, md, s1, s2, pad = int(kernel_size), int(max_displacement), int(stride1), int(stride2), int(pad_size)
    kr = (ks - 1) // 2
    f = np.float32
    tw = int(np.ceil(f(w + 2 * pad - 2 * (md + kr)) / f(s1)))
    if one_d:
        th = int(np.ceil(f(h - 2 * kr) / f(s1)))
    else:
        th = int(np.ceil(f(h + 2 * pad - 2 * (md + kr)) / f(s1)))
    r = md // s2
    if one_d:
        gw = r + 1 if single_dir != 0 else 2 * r + 1
        gh, ry = 1, 0
        xshift = -gw if single_dir == -1 else (0 if single_dir == 1 else -r)
    else:
        gw = gh = 2 * r + 1
        xshift, ry = -r, r
    return dict(n=n, c=c, h=h, w=w, ks=ks, md=md, s1=s1, s2=s2, pad=pad, pady=0 if one_d else pad, mdy=0 if one_d else md,
                tw=tw, th=th, gw=gw, gh=gh, xshift=xshift, ry=ry, tc=gw * gh, sumelems=ks * ks * c)


def _displacements(g):
    for dyi in range(g["gh"]):
        for dxi in range(g["gw"]):
            yield dyi * g["gw"] + dxi, (dxi + g["xshift"]) * g["s2"], (dyi - g["ry"]) * g["s2"]


def _margin(g):
    return g["md"] + (g["gw"] + 1) * g["s2"] + g["ks"] + 1


def _pad(x, g):
    """x in a zero array with the op's padding plus a margin M every read lands in; padded position (py, px) is [M+py, M+px]."""
    m = _margin(g)
    n, c, h, w = x.shape
    out = np.zeros((n, c, h + 2 * g["pady"] + 2 * m, w + 2 * g["pad"] + 2 * m), dtype=np.float64)
    out[:, :, m + g["pady"]:m + g["pady"] + h, m + g["pad"]:m + g["pad"] + w] = x
    return out


def _crop(xp, g):
    m = _margin(g)
    return xp[..., m + g["pady"]:m + g["pady"] + g["h"], m + g["pad"]:m + g["pad"] + g["w"]]


def _window(g, j, i, dy=0, dx=0):
    """index of the padded array holding (Y1 + dy + j, X1 + dx + i) for every top pixel"""
    m = _margin(g)
    r0 = m + g["mdy"] + dy + j
    c0 = m + g["md"] + dx + i
    return (slice(r0, r0 + g["s1"] * (g["th"] - 1) + 1, g["s1"]), slice(c0, c0 + g["s1"] * (g["tw"] - 1) + 1, g["s1"]))


def _shift(x, dy, dx):
    """y[..., r, c] = x[..., r + dy, c + dx], 0 outside"""
    y = np.zeros_like(x)
    H, W = x.shape[-2:]
    ys, yd = (slice(dy, H), slice(0, H - dy)) if dy >= 0 else (slice(0, H + dy), slice(-dy, H))
    xs, xd = (slice(dx, W), slice(0, W - dx)) if dx >= 0 else (slice(0, W + dx), slice(-dx, W))
    y[..., yd, xd] = x[..., ys, xs]
    return y


def correlation(input1, input2, one_d=False, corr_type="mult", normalize=True, **attrs):
    """top [N, tc, th, tw] in float64 (attrs: max_displacement, kernel_size, stride1, stride2, pad_size, single_dir for 1D;
    do_abs is accepted and ignored).  normalize=False leaves out the division by K K C."""
    attrs.pop("do_abs", None)
    a = np.asarray(input1, dtype=np.float64)
    g = geometry(a.shape, one_d=one_d, **attrs)
    p1, p2 = _pad(a, g), _pad(np.asarray(input2, dtype=np.float64), g)
    top = np.zeros((g["n"], g["tc"], g["th"], g["tw"]))
    for tc, dx, dy in _displacements(g):
        acc = np.zeros((g["n"], g["th"], g["tw"]))
        for j in range(g["ks"]):
            for i in range(g["ks"]):
                ra, ca = _window(g, j, i)
                rb, cb = _window(g, j, i, dy, dx)
                A, B = p1[:, :, ra, ca], p2[:, :, rb, cb]
                acc += (A * B).sum(axis=1) if corr_type == "mult" else np.abs(A - B).sum(axis=1)
        top[:, tc] = acc
    return top / g["sumelems"] if normalize else top


def correlation_grad(gradient, input1, input2, one_d=False, corr_type="mult", normalize=True, **attrs):
    """(input1_grad, input2_grad) in float64, see the module docstring."""
    attrs.pop("do_abs", None)
    a = np.asarray(input1, dtype=np.float64)
    g = geometry(a.shape, one_d=one_d, **attrs)
    gt = np.asarray(gradient, dtype=np.float64)
    p1, p2 = _pad(a, g), _pad(np.asarray(input2, dtype=np.float64), g)
    g1, g2 = np.zeros_like(p1), np.zeros_like(p2)
    if corr_type == "mult":
        for tc, dx, dy in _displacements(g):
            gg = gt[:, tc][:, None]
            for j in range(g["ks"]):
                for i in range(g["ks"]):
                    ra, ca = _window(g, j, i)
                    rb, cb = _window(g, j, i, dy, dx)
                    g1[:, :, ra, ca] += gg * p2[:, :, rb, cb]
                    g2[:, :, rb, cb] += gg * p1[:, :, ra, ca]
    else:
        with np.errstate(invalid="ignore"):
            e = np.where(p1 >= p2, 1.0, -1.0)
        for tc, dx, dy in _displacements(g):
            t = np.zeros(p1.shape[:1] + p1.shape[2:])      # gradient scattered over the input1 patches
            for j in range(g["ks"]):
                for i in range(g["ks"]):
                    ra, ca = _window(g, j, i)
                    t[:, ra, ca] += gt[:, tc]
            g1 += t[:, None] * _shift(e, dy, dx)
            g2 -= _shift(t[:, None] * e, -dy, -dx)
    g1, g2 = _crop(g1, g), _crop(g2, g)
    if normalize:
        g1, g2 = g1 / g["sumelems"], g2 / g["sumelems"]
    return np.ascontiguousarray(g1), np.ascontiguousarray(g2)
