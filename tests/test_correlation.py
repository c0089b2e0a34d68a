"""CPU: the float64 correlation oracle (oracle/correlation.py), the shape rules and argument errors of
demon_b200.lmbspecialops.correlation / correlation_1d, and the C ABI's refusal of bad attributes before any launch.

The oracle is pinned three ways: the top size against the reference's formulas (a ceil in float32, correlation.cc:62-77,
correlation_1d_cuda.cu:485-505); 'mult' by the adjoint identity <top(x1, x2), g> = <x1, grad1> = <x2, grad2> in float64 on
every attribute combination the GPU tests use; and both modes against a per-element loop statement of the reference's
gathers (the clamped top window of every input element, correlation_cuda.cu:191-245 and :274-317).
"""
import ctypes
import math

import numpy as np
import pytest

from oracle import correlation as oc

# (one_d, attrs) at small sizes: the settings tests/test_gpu_correlation.py runs, scaled down
COMBOS = [
    (False, dict(max_displacement=4, kernel_size=1, stride1=1, stride2=2, pad_size=4)),    # FlowNetC-like
    (True, dict(max_displacement=4, kernel_size=1, stride1=1, stride2=1, pad_size=4, single_dir=0)),
    (True, dict(max_displacement=4, kernel_size=1, stride1=1, stride2=1, pad_size=4, single_dir=1)),
    (True, dict(max_displacement=4, kernel_size=1, stride1=1, stride2=1, pad_size=4, single_dir=-1)),
    (False, dict(max_displacement=2, kernel_size=3, stride1=2, stride2=1, pad_size=3)),
    (True, dict(max_displacement=2, kernel_size=3, stride1=2, stride2=1, pad_size=3, single_dir=-1)),
    (False, dict(max_displacement=5, kernel_size=1, stride1=1, stride2=2, pad_size=5)),
    (False, dict(max_displacement=2, kernel_size=1, stride1=1, stride2=1, pad_size=0)),
    (True, dict(max_displacement=5, kernel_size=3, stride1=3, stride2=2, pad_size=1, single_dir=1)),
    (True, dict(max_displacement=3, kernel_size=1, stride1=1, stride2=2, pad_size=0, single_dir=-1)),
]


def _ids():
    return ["%s-%s" % ("1d" if d else "2d", "-".join("%s%d" % (k[:4], v) for k, v in a.items())) for d, a in COMBOS]


def _inputs(seed, shape=(2, 5, 9, 13)):
    rng = np.random.RandomState(seed)
    return rng.randn(*shape), rng.randn(*shape), rng


@pytest.mark.parametrize("one_d,attrs", COMBOS, ids=_ids())
def test_mult_adjoint_identity(one_d, attrs):
    x1, x2, rng = _inputs(1)
    top = oc.correlation(x1, x2, one_d=one_d, **attrs)
    g = rng.randn(*top.shape)
    g1, g2 = oc.correlation_grad(g, x1, x2, one_d=one_d, **attrs)
    ref = float((top * g).sum())
    assert math.isclose(float((x1 * g1).sum()), ref, rel_tol=1e-12, abs_tol=1e-12)
    assert math.isclose(float((x2 * g2).sum()), ref, rel_tol=1e-12, abs_tol=1e-12)


def _read(x, g, n, c, py, px):
    """padded read: 0 outside the input"""
    y, xx = py - g["pady"], px - g["pad"]
    return x[n, c, y, xx] if 0 <= y < g["h"] and 0 <= xx < g["w"] else 0.0


def _loops(one_d, attrs, corr_type, x1, x2, gt):
    """the reference's forward and gathers element by element (float64)"""
    g = oc.geometry(x1.shape, one_d=one_d, **attrs)
    kr2, s1 = g["ks"] - 1, g["s1"]
    top = np.zeros((g["n"], g["tc"], g["th"], g["tw"]))
    g1, g2 = np.zeros_like(x1), np.zeros_like(x2)
    f = (lambda a, b: a * b) if corr_type == "mult" else (lambda a, b: abs(a - b))
    r = g["md"] // g["s2"]
    if one_d:   # correlation_1d_cuda.cu: x_shift -R, 0 or -(R+1) for single_dir 0, 1, -1
        xs = {0: -r, 1: 0, -1: -(r + 1)}[attrs.get("single_dir", 0)]
        disp = [(o, (o + xs) * g["s2"], 0) for o in range(g["tc"])]
    else:       # correlation_cuda.cu: s2o = (tc % gw - R) s2, s2p = (tc / gw - R) s2
        disp = [(tc, (tc % g["gw"] - r) * g["s2"], (tc // g["gw"] - r) * g["s2"]) for tc in range(g["tc"])]
    for n in range(g["n"]):
        for tc, dx, dy in disp:
            for y in range(g["th"]):
                for x in range(g["tw"]):
                    X1, Y1 = x * s1 + g["md"], y * s1 + g["mdy"]
                    top[n, tc, y, x] = sum(f(_read(x1, g, n, c, Y1 + j, X1 + i), _read(x2, g, n, c, Y1 + dy + j, X1 + dx + i))
                                           for j in range(g["ks"]) for i in range(g["ks"]) for c in range(g["c"]))
        for c in range(g["c"]):
            for yy in range(g["h"]):
                for xx in range(g["w"]):
                    l, m = xx + g["pad"], yy + g["pady"]
                    for second in (False, True):
                        s = 0.0
                        for tc, dx, dy in disp:
                            sx, sy = (-dx, -dy) if second else (0, 0)
                            xmin, xmax = -((-(l - kr2 - g["md"] + sx)) // s1), (l - g["md"] + sx) // s1
                            ymin, ymax = -((-(m - kr2 - g["mdy"] + sy)) // s1), (m - g["mdy"] + sy) // s1
                            if not (xmax >= 0 and ymax >= 0 and xmin <= g["tw"] - 1 and ymin <= g["th"] - 1):
                                continue
                            py, px = (m - dy, l - dx) if second else (m + dy, l + dx)
                            if corr_type == "mult":
                                v = _read(x1 if second else x2, g, n, c, py, px)
                            else:
                                ge = _read(x1, g, n, c, py, px) >= _read(x2, g, n, c, py, px)
                                v = (-1.0 if ge else 1.0) if second else (1.0 if ge else -1.0)
                            for ty in range(max(0, ymin), min(g["th"] - 1, ymax) + 1):
                                for tx in range(max(0, xmin), min(g["tw"] - 1, xmax) + 1):
                                    s += gt[n, tc, ty, tx] * v
                        (g2 if second else g1)[n, c, yy, xx] = s
    return top, g1, g2


@pytest.mark.parametrize("corr_type", ["mult", "subt"])
@pytest.mark.parametrize("one_d,attrs", COMBOS[3:6] + COMBOS[7:], ids=_ids()[3:6] + _ids()[7:])
def test_oracle_equals_the_reference_loops(one_d, attrs, corr_type):
    x1, x2, rng = _inputs(2, (1, 2, 7, 10))
    x1[0, 0, 2, 3] = x2[0, 1, 4, 5]                       # ties of the 'subt' sign
    top = oc.correlation(x1, x2, one_d=one_d, corr_type=corr_type, normalize=False, **attrs)
    gt = rng.randn(*top.shape)
    g1, g2 = oc.correlation_grad(gt, x1, x2, one_d=one_d, corr_type=corr_type, normalize=False, **attrs)
    t_ref, g1_ref, g2_ref = _loops(one_d, attrs, corr_type, x1, x2, gt)
    np.testing.assert_allclose(top, t_ref, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(g1, g1_ref, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(g2, g2_ref, rtol=1e-12, atol=1e-12)


def _reference_top(shape, md, ks, s1, s2, pad, one_d, single_dir):
    """correlation.cc:62-77 / correlation_1d_cuda.cu:481-505, with C's float arithmetic"""
    n, c, h, w = shape
    f = np.float32
    kr = (ks - 1) // 2
    border = md + kr
    tw = math.ceil(f(w + 2 * pad - border * 2) / f(s1))
    th = math.ceil(f(h - kr * 2) / f(s1)) if one_d else math.ceil(f(h + 2 * pad - border * 2) / f(s1))
    r = md // s2
    gw = (r + 1 if single_dir != 0 else 2 * r + 1) if one_d else 2 * r + 1
    return (n, gw if one_d else gw * gw, th, tw)


@pytest.mark.parametrize("one_d", [False, True])
def test_top_shape_rules(one_d):
    from demon_b200.lmbspecialops import correlation_top_shape
    rng = np.random.RandomState(3)
    for _ in range(400):
        shape = (int(rng.randint(1, 4)), int(rng.randint(1, 70)), int(rng.randint(1, 60)), int(rng.randint(1, 90)))
        md, ks, s1, s2, pad = int(rng.randint(0, 21)), int(rng.choice([1, 3, 5])), int(rng.randint(1, 4)), int(rng.randint(1, 4)), int(rng.randint(0, 21))
        sd = int(rng.choice([-1, 0, 1])) if one_d else 0
        want = _reference_top(shape, md, ks, s1, s2, pad, one_d, sd)
        assert correlation_top_shape(shape, md, ks, s1, s2, pad, one_d, sd) == want
        g = oc.geometry(shape, md, ks, s1, s2, pad, one_d, sd)
        assert (g["n"], g["tc"], g["th"], g["tw"]) == want
    # the FlowNetC and DispNetC settings
    assert correlation_top_shape((8, 256, 48, 64), 20, 1, 1, 2, 20) == (8, 441, 48, 64)
    assert correlation_top_shape((8, 256, 48, 64), 40, 1, 1, 1, 40, True, 0) == (8, 81, 48, 64)


def test_shape_and_type_errors():
    from demon_b200 import lmbspecialops as ops
    a = np.zeros((1, 3, 8, 8), np.float32)
    with pytest.raises(ValueError):
        ops.correlation(a[0], a[0], 1, 1)
    with pytest.raises(ValueError):
        ops.correlation_1d(a, a[:, :2], 1, 1)
    with pytest.raises(ValueError):
        ops.correlation_grad(np.zeros((1, 9, 8, 8), np.float32), a, np.zeros((1, 3, 8, 9), np.float32), 1, 1)
    with pytest.raises(ValueError):
        ops.correlation(a, a, 1, 1, corr_type="div")
    with pytest.raises(TypeError):
        ops.correlation(a.astype(np.float64), a, 1, 1)
    with pytest.raises(TypeError):
        ops.correlation_1d(a, a.astype(np.float64), 1, 1)
    with pytest.raises(TypeError):
        ops.correlation_grad(np.zeros((1, 9, 8, 8)), a, a, 1, 1)


# (corr_type, kernel_size, max_displacement, stride1, stride2, pad_size, single_dir) on a [2,4,8,8] input
INVALID = [
    (1, 2, 1, 1, 1, 1, 0),     # even kernel_size
    (1, 0, 1, 1, 1, 1, 0),
    (1, 1, 1, 0, 1, 1, 0),     # stride1 < 1
    (2, 1, 1, 1, 0, 1, 0),     # stride2 < 1
    (1, 1, -2, 1, 1, 1, 0),    # negative max_displacement
    (1, 1, 1, 1, 1, -1, 0),    # negative pad_size
    (1, 1, 1, 1, 1, 1, 2),     # single_dir not in {-1, 0, 1}
    (1, 1, 1, 1, 1, 1, -2),
    (1, 1, 6, 1, 1, 0, 0),     # top width / height < 1
    (2, 5, 3, 1, 1, 0, 0),
    (3, 1, 1, 1, 1, 1, 0),     # unknown corr_type
]


@pytest.mark.parametrize("args", INVALID)
def test_invalid_arguments_refused_before_any_launch(args):
    from demon_b200 import _lib
    L = _lib.load()
    ct, ks, md, s1, s2, pad, sd = args
    buf = (ctypes.c_float * 4096)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    n0 = L.demon_launch_count()
    calls = [
        lambda: L.demon_correlation_1d_f32(p, p, p, 2, 4, 8, 8, ct, ks, md, s1, s2, pad, 0, sd, None),
        lambda: L.demon_correlation_1d_grad_f32(p, p, p, p, p, 2, 4, 8, 8, ct, ks, md, s1, s2, pad, 0, sd, None),
    ]
    if sd == 0:
        calls += [
            lambda: L.demon_correlation_f32(p, p, p, 2, 4, 8, 8, ct, ks, md, s1, s2, pad, 0, None),
            lambda: L.demon_correlation_grad_f32(p, p, p, p, p, 2, 4, 8, 8, ct, ks, md, s1, s2, pad, 0, None),
        ]
    for call in calls:
        assert call() == -1, "accepted %s" % (args,)          # DEMON_E_INVALID
    assert L.demon_launch_count() == n0
