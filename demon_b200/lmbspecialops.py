"""Mirror of the reference's op binding `lmbspecialops`
(lmbspecialops/python/lmbspecialops/__init__.py:45-58,296-308; signatures documented in
lmbspecialops/doc/lmbspecialops_doc.md) over the sm_90a kernels of libdemon_b200.so.

Same function names, keyword arguments, shape rules and error behaviour as the TensorFlow ops:

  * tensors are NCHW, trailing dims are (C,)H,W and all leading dims collapse into N;
  * depth_to_flow / flow_to_depth / scale_invariant_gradient always return rank 4
    (depthtoflow.cc:225-232, flowtodepth.cc:321-328, scaleinvariantgradient.cc:127-134),
    warp2d / median3x3_downsample / leaky_relu keep the input's rank (warp2d.cc:147,
    median3x3downsample.cc:89-95);
  * shape violations raise ValueError at call time (TF raises it at graph construction from the
    op's shape function, e.g. "Dimensions must be equal", test_FlowToDepth2.py:194-200).

Inputs may be torch CUDA tensors (zero copy) or anything numpy can convert (copied to cuda:0 and
back; the result is then a numpy array).  float32 and float64 are supported like in the reference.
There is no CPU implementation here.
"""
import ctypes
import warnings

import numpy as np
import torch

from . import _lib

_ROT = {"matrix": (0, 9), "quaternion": (1, 4), "angleaxis3": (2, 3)}


def _device():
    if not torch.cuda.is_available():
        raise RuntimeError("demon_b200 ops need a CUDA device (there is no CPU fallback)")
    return torch.device("cuda", torch.cuda.current_device())


def _as_cuda(x, dtype=None):
    """-> (contiguous cuda tensor, was_numpy)"""
    if isinstance(x, torch.Tensor):
        t = x
        was_np = False
        if not t.is_cuda:
            t = t.to(_device())
    else:
        a = np.asarray(x)
        if a.dtype not in (np.float32, np.float64):
            a = a.astype(np.float32 if dtype is None else {torch.float32: np.float32, torch.float64: np.float64}[dtype])
        t = torch.from_numpy(np.ascontiguousarray(a)).to(_device())
        was_np = True
    if dtype is not None and t.dtype != dtype:
        t = t.to(dtype)
    if t.dtype not in (torch.float32, torch.float64):
        raise TypeError("demon_b200 ops take float32 or float64 tensors, got %s" % t.dtype)
    return t.contiguous(), was_np


def _shp(x):
    return tuple(x.shape) if hasattr(x, "shape") else np.shape(x)


def _ret(t, was_np):
    return t.cpu().numpy() if was_np else t


def _sfx(t):
    return "_f32" if t.dtype == torch.float32 else "_f64"


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _prod(shape):
    n = 1
    for s in shape:
        n *= int(s)
    return n


def _call(name, *args):
    _lib.check(getattr(_lib.load(), name)(*args))


def warp2d(input, displacements, normalized=False, border_mode="clamp", border_value=0.0):
    """Warps `input` with the displacement field (warp2d.cc:25-113)."""
    ishape, dshape = _shp(input), _shp(displacements)
    if len(ishape) < 2:
        raise ValueError("Shape must be at least rank 2 but is rank %d" % len(ishape))
    if len(dshape) < 3:
        raise ValueError("Shape must be at least rank 3 but is rank %d" % len(dshape))
    if dshape[-3] != 2:
        raise ValueError("Dimension must be 2 but is %d" % dshape[-3])
    if tuple(dshape[-2:]) != tuple(ishape[-2:]):
        raise ValueError("Dimensions must be equal, but are %s and %s" % (tuple(ishape[-2:]), tuple(dshape[-2:])))
    if border_mode not in ("clamp", "value"):
        raise ValueError("border_mode must be 'clamp' or 'value'")
    h, w = ishape[-2:]
    c = ishape[-3] if len(ishape) >= 3 else 1
    n = _prod(ishape[:-3]) if len(ishape) > 3 else 1
    if _prod(dshape[:-3]) != n:
        raise ValueError("Dimensions must be equal, but are %d and %d" % (n, _prod(dshape[:-3])))
    inp, was_np = _as_cuda(input)
    disp, _ = _as_cuda(displacements, inp.dtype)
    out = torch.empty_like(inp)
    bv = (ctypes.c_float if inp.dtype == torch.float32 else ctypes.c_double)(border_value)
    _call("demon_warp2d" + _sfx(inp), inp.data_ptr(), disp.data_ptr(), out.data_ptr(), n, c, h, w,
          int(bool(normalized)), 1 if border_mode == "clamp" else 2, bv, _stream())
    return _ret(out, was_np)


def _pose(n, dtype, intrinsics, rotation, translation, rotation_format):
    """Validates the camera arguments on their shapes first (so that shape errors do not need a GPU)."""
    if rotation_format not in _ROT:
        raise ValueError("rotation_format must be one of %s" % sorted(_ROT))
    fmt, step = _ROT[rotation_format]
    ks, rs, ts = _shp(intrinsics), _shp(rotation), _shp(translation)
    if len(ks) < 1 or ks[-1] != 4:
        raise ValueError("Dimension must be 4 but is %s" % (ks[-1] if ks else None))
    if len(ts) < 1 or ts[-1] != 3:
        raise ValueError("Dimension must be 3 but is %s" % (ts[-1] if ts else None))
    if rotation_format == "matrix":
        if len(rs) < 2 or tuple(rs[-2:]) != (3, 3):
            raise ValueError("Dimension must be 3 but is %s" % (tuple(rs[-2:]),))
        rn = _prod(rs[:-2])
    else:
        if len(rs) < 1 or rs[-1] != step:
            raise ValueError("Dimension must be %d but is %s" % (step, rs[-1] if rs else None))
        rn = _prod(rs[:-1])
    for other in (_prod(ks[:-1]), rn, _prod(ts[:-1])):
        if other != n:
            raise ValueError("Dimensions must be equal, but are %d and %d" % (n, other))
    if dtype is None:
        return None
    k, _ = _as_cuda(intrinsics, dtype)
    r, _ = _as_cuda(rotation, dtype)
    t, _ = _as_cuda(translation, dtype)
    return k, r, t, fmt


def _validate_pose_only(n, intrinsics, rotation, translation, rotation_format):
    _pose(n, None, intrinsics, rotation, translation, rotation_format)


def depth_to_flow(depth, intrinsics, rotation, translation, rotation_format="angleaxis3", inverse_depth=False,
                  normalize_flow=False):
    """Optical flow from a depth map and the relative camera pose (depthtoflow.cc:29-153)."""
    dshape = _shp(depth)
    if len(dshape) < 2:
        raise ValueError("Shape must be at least rank 2 but is rank %d" % len(dshape))
    h, w = dshape[-2:]
    n = _prod(dshape[:-2])
    _validate_pose_only(n, intrinsics, rotation, translation, rotation_format)
    d, was_np = _as_cuda(depth)
    k, r, t, fmt = _pose(n, d.dtype, intrinsics, rotation, translation, rotation_format)
    out = torch.empty((n, 2, h, w), dtype=d.dtype, device=d.device)
    _call("demon_depth_to_flow" + _sfx(d), d.data_ptr(), k.data_ptr(), r.data_ptr(), t.data_ptr(), out.data_ptr(),
          n, h, w, fmt, int(bool(inverse_depth)), int(bool(normalize_flow)), _stream())
    return _ret(out, was_np)


def flow_to_depth2(flow, intrinsics, rotation, translation, rotation_format="angleaxis3", inverse_depth=False,
                   normalized_flow=False, name=None):
    """Depth from optical flow and the relative camera pose by linear triangulation (flowtodepth2.cc)."""
    fshape = _shp(flow)
    if len(fshape) < 3:
        raise ValueError("Shape must be at least rank 3 but is rank %d" % len(fshape))
    if fshape[-3] != 2:
        raise ValueError("Dimension must be 2 but is %d" % fshape[-3])
    h, w = fshape[-2:]
    n = _prod(fshape[:-3])
    _validate_pose_only(n, intrinsics, rotation, translation, rotation_format)
    f, was_np = _as_cuda(flow)
    k, r, t, fmt = _pose(n, f.dtype, intrinsics, rotation, translation, rotation_format)
    out = torch.empty((n, 1, h, w), dtype=f.dtype, device=f.device)
    _call("demon_flow_to_depth" + _sfx(f), f.data_ptr(), k.data_ptr(), r.data_ptr(), t.data_ptr(), out.data_ptr(),
          n, h, w, fmt, int(bool(inverse_depth)), int(bool(normalized_flow)), _stream())
    return _ret(out, was_np)


def flow_to_depth(flow, intrinsics, rotation, translation, rotation_format=None, inverse_depth=None,
                  normalized_flow=None, name=None, nowarning=False):
    """Deprecated op the DeMoN graph still uses (blocks_original.py:344; wrapper at
    lmbspecialops/__init__.py:296-308).  Numerically identical to flow_to_depth2 in the reference."""
    if not nowarning:
        warnings.warn("flow_to_depth has incorrect behaviour but is kept for compatibility. Please use flow_to_depth2",
                      DeprecationWarning, stacklevel=2)
    return flow_to_depth2(flow, intrinsics, rotation, translation,
                          "angleaxis3" if rotation_format is None else rotation_format,
                          bool(inverse_depth), bool(normalized_flow))


def leaky_relu(input, leak=0.1):
    """max(leak*x, x) (leakyrelu.cc:25-96)."""
    x, was_np = _as_cuda(input)
    out = torch.empty_like(x)
    lk = (ctypes.c_float if x.dtype == torch.float32 else ctypes.c_double)(np.float32(leak))
    _call("demon_leaky_relu" + _sfx(x), x.data_ptr(), out.data_ptr(), x.numel(), lk, _stream())
    return _ret(out, was_np)


def median3x3_downsample(input):
    """3x3 median filter evaluated at every second pixel (median3x3downsample.cc:26-184)."""
    if len(_shp(input)) < 2:
        raise ValueError("Shape must be at least rank 2 but is rank %d" % len(_shp(input)))
    x, was_np = _as_cuda(input)
    h, w = x.shape[-2:]
    z = _prod(x.shape[:-2])
    out = torch.empty(tuple(x.shape[:-2]) + ((h + 1) // 2, (w + 1) // 2), dtype=x.dtype, device=x.device)
    _call("demon_median3x3_downsample" + _sfx(x), x.data_ptr(), out.data_ptr(), z, h, w, _stream())
    return _ret(out, was_np)


def scale_invariant_gradient(input, deltas=(1,), weights=(1.0,), epsilon=0.001):
    """Scale invariant gradient of Eq. 6 of the DeMoN paper (scaleinvariantgradient.cc:26-93)."""
    if len(_shp(input)) < 2:
        raise ValueError("Shape must be at least rank 2 but is rank %d" % len(_shp(input)))
    deltas = [int(d) for d in deltas]
    weights = [float(v) for v in weights]
    if len(deltas) != len(weights):
        raise ValueError("The size of the deltas and weights vectors must be the same")
    if len(deltas) > 16:
        raise ValueError("at most 16 deltas are supported")
    x, was_np = _as_cuda(input)
    h, w = x.shape[-2:]
    z = _prod(x.shape[:-2])
    out = torch.empty((z, 2, h, w), dtype=x.dtype, device=x.device)
    cty = ctypes.c_float if x.dtype == torch.float32 else ctypes.c_double
    d_arr = (ctypes.c_int * max(1, len(deltas)))(*deltas)
    # weights and epsilon are float32 attributes converted to T (scaleinvariantgradient.cc:109-113)
    w_arr = (cty * max(1, len(weights)))(*[float(np.float32(v)) for v in weights])
    _call("demon_scale_invariant_gradient" + _sfx(x), x.data_ptr(), out.data_ptr(), z, h, w,
          ctypes.cast(d_arr, ctypes.c_void_p), ctypes.cast(w_arr, ctypes.c_void_p), len(deltas),
          cty(float(np.float32(epsilon))), _stream())
    return _ret(out, was_np)


# ---- training-side companions (SURVEY.md section 8 f4) ---------------------------------------------------------------
def scale_invariant_gradient_grad(gradients, input, deltas=(1,), weights=(1.0,), epsilon=0.001):
    """Gradient of scale_invariant_gradient with respect to its input: the ScaleInvariantGradientGrad op the reference
    registers for it (scaleinvariantgradient.cc:224-404; `_scale_invariant_gradient_grad`,
    lmbspecialops/python/lmbspecialops/__init__.py).  gradients [z,2,h,w], input [...,h,w] -> input's shape."""
    deltas = [int(d) for d in deltas]
    weights = [float(v) for v in weights]
    if len(deltas) != len(weights):
        raise ValueError("The size of the deltas and weights vectors must be the same")
    if len(deltas) > 16:
        raise ValueError("at most 16 deltas are supported")
    x, was_np = _as_cuda(input)
    g, _ = _as_cuda(gradients, x.dtype)
    h, w = x.shape[-2:]
    z = _prod(x.shape[:-2])
    if tuple(g.shape) != (z, 2, h, w):
        raise ValueError("Dimensions must be equal: gradients %s, expected %s" % (tuple(g.shape), (z, 2, h, w)))
    out = torch.empty_like(x)
    cty = ctypes.c_float if x.dtype == torch.float32 else ctypes.c_double
    d_arr = (ctypes.c_int * max(1, len(deltas)))(*deltas)
    w_arr = (cty * max(1, len(weights)))(*[float(np.float32(v)) for v in weights])
    _call("demon_scale_invariant_gradient_grad" + _sfx(x), g.data_ptr(), x.data_ptr(), out.data_ptr(), z, h, w,
          ctypes.cast(d_arr, ctypes.c_void_p), ctypes.cast(w_arr, ctypes.c_void_p), len(deltas),
          cty(float(np.float32(epsilon))), _stream())
    return _ret(out, was_np)


def leaky_relu_grad(gradients, input, leak=0.1):
    """LeakyReluLmbGrad (leakyrelu.cc:100-172): gradients where input >= leak*input, leak*gradients elsewhere."""
    x, was_np = _as_cuda(input)
    g, _ = _as_cuda(gradients, x.dtype)
    if tuple(g.shape) != tuple(x.shape):
        raise ValueError("Dimensions must be equal: gradients %s, input %s" % (tuple(g.shape), tuple(x.shape)))
    out = torch.empty_like(x)
    lk = (ctypes.c_float if x.dtype == torch.float32 else ctypes.c_double)(np.float32(leak))
    _call("demon_leaky_relu_grad" + _sfx(x), g.data_ptr(), x.data_ptr(), out.data_ptr(), x.numel(), lk, _stream())
    return _ret(out, was_np)


def replace_nonfinite(input, value=0.0):
    """Replaces NaN / inf by `value` (replacenonfinite.cc:26-93; used by the v2 losses, v2/losses.py:49)."""
    x, was_np = _as_cuda(input)
    out = torch.empty_like(x)
    v = (ctypes.c_float if x.dtype == torch.float32 else ctypes.c_double)(np.float32(value))
    _call("demon_replace_nonfinite" + _sfx(x), x.data_ptr(), out.data_ptr(), x.numel(), v, _stream())
    return _ret(out, was_np)


def depth_to_normals(depth, intrinsics, inverse_depth=False):
    """Normal map [N,3,H,W] (camera frame) of a depth map; leading dims collapse into N, `intrinsics` is [N,4] (or [4],
    broadcast) normalised (fx, fy, cx, cy).  Border pixels and pixels next to a non-positive / non-finite depth are NaN
    (depthtonormals.cc:29-238; shape rules :36-68)."""
    dshape = _shp(depth)
    if len(dshape) < 2:
        raise ValueError("Shape must be at least rank 2 but is rank %d" % len(dshape))
    kshape = _shp(intrinsics)
    if len(kshape) < 1:
        raise ValueError("Shape must be at least rank 1 but is rank 0")
    if kshape[-1] != 4:
        raise ValueError("Dimension must be 4 but is %d" % kshape[-1])
    h, w = dshape[-2:]
    n = _prod(dshape[:-2])
    d, was_np = _as_cuda(depth)
    k, _ = _as_cuda(intrinsics, d.dtype)
    k = k.reshape(-1, 4)
    if k.shape[0] == 1 and n != 1:
        k = k.expand(n, 4)
    if k.shape[0] != n:
        raise ValueError("Dimensions must be equal: %d depth maps, %d intrinsics" % (n, k.shape[0]))
    k = k.contiguous()
    out = torch.empty((n, 3, h, w), dtype=d.dtype, device=d.device)
    _call("demon_depth_to_normals" + _sfx(d), d.data_ptr(), k.data_ptr(), out.data_ptr(), n, h, w, int(bool(inverse_depth)), _stream())
    return _ret(out, was_np)


def replace_nonfinite_grad(gradients, input):
    """ReplaceNonfiniteGrad (replacenonfinite.cc:97-168): zero gradient where the input was not finite."""
    x, was_np = _as_cuda(input)
    g, _ = _as_cuda(gradients, x.dtype)
    if tuple(g.shape) != tuple(x.shape):
        raise ValueError("Dimensions must be equal: gradients %s, input %s" % (tuple(g.shape), tuple(x.shape)))
    out = torch.empty_like(x)
    _call("demon_replace_nonfinite_grad" + _sfx(x), g.data_ptr(), x.data_ptr(), out.data_ptr(), x.numel(), _stream())
    return _ret(out, was_np)


class _SIGFunction(torch.autograd.Function):
    """torch.autograd counterpart of the @ops.RegisterGradient("ScaleInvariantGradient") hook of the reference binding."""

    @staticmethod
    def forward(ctx, x, deltas, weights, epsilon):
        ctx.save_for_backward(x)
        ctx.attrs = (deltas, weights, epsilon)
        return scale_invariant_gradient(x, deltas, weights, epsilon)

    @staticmethod
    def backward(ctx, grad_out):
        (x,) = ctx.saved_tensors
        deltas, weights, epsilon = ctx.attrs
        return scale_invariant_gradient_grad(grad_out.contiguous(), x, deltas, weights, epsilon), None, None, None


def scale_invariant_gradient_autograd(input, deltas=(1,), weights=(1.0,), epsilon=0.001):
    """scale_invariant_gradient on a torch CUDA tensor with the reference's analytic gradient attached."""
    return _SIGFunction.apply(input, tuple(deltas), tuple(weights), float(epsilon))


# ---- FlowNet cost volumes (correlation.cc, correlation_1d.cc, correlation_cuda.cu, correlation_1d_cuda.cu) ----------------
_CORR_TYPES = {"mult": 1, "subt": 2}   # DEMON_CORR_MULT, DEMON_CORR_SUBT


def correlation_top_shape(shape, max_displacement, kernel_size, stride1=1, stride2=1, pad_size=0, one_d=False, single_dir=0):
    """[N, top_channels, top_h, top_w] of correlation (one_d False, correlation.cc:62-77) or correlation_1d
    (correlation_1d.cc:47-67): the top size is a ceil taken in float32, as the reference takes it."""
    n, _, h, w = (int(s) for s in shape)
    kr = (int(kernel_size) - 1) // 2
    f = np.float32
    tw = int(np.ceil(f(w + 2 * pad_size - 2 * (max_displacement + kr)) / f(stride1)))
    th = int(np.ceil(f(h - 2 * kr) / f(stride1))) if one_d else int(np.ceil(f(h + 2 * pad_size - 2 * (max_displacement + kr)) / f(stride1)))
    r = int(max_displacement) // int(stride2)
    if one_d:
        tc = r + 1 if single_dir != 0 else 2 * r + 1
    else:
        tc = (2 * r + 1) ** 2
    return (n, tc, th, tw)


def _corr_inputs(input1, input2):
    s1, s2 = _shp(input1), _shp(input2)
    if len(s1) != 4:
        raise ValueError("Shape must be rank 4 but is rank %d" % len(s1))
    if len(s2) != 4:
        raise ValueError("Shape must be rank 4 but is rank %d" % len(s2))
    if tuple(s1) != tuple(s2):
        raise ValueError("Dimensions must be equal, but are %s and %s" % (tuple(s1), tuple(s2)))
    _no_float64(input1)
    _no_float64(input2)
    a, was_np = _as_cuda(input1)
    b, _ = _as_cuda(input2, torch.float32)
    return a, b, was_np


def _no_float64(x):
    dt = x.dtype if isinstance(x, torch.Tensor) else np.asarray(x).dtype
    if dt in (torch.float64, np.float64):
        raise TypeError("correlation is registered for float32 only (T: {float}), got %s" % dt)


def _corr_type(corr_type):
    if corr_type not in _CORR_TYPES:
        raise ValueError("corr_type must be 'mult' or 'subt', got %r" % (corr_type,))
    return _CORR_TYPES[corr_type]


def _corr_forward(one_d, input1, input2, kernel_size, max_displacement, stride1, stride2, pad_size, do_abs, corr_type, single_dir):
    ct = _corr_type(corr_type)
    a, b, was_np = _corr_inputs(input1, input2)
    shape = correlation_top_shape(a.shape, max_displacement, kernel_size, stride1, stride2, pad_size, one_d, single_dir)
    out = torch.empty(tuple(max(0, s) for s in shape), dtype=torch.float32, device=a.device)
    n, c, h, w = a.shape
    args = [a.data_ptr(), b.data_ptr(), out.data_ptr(), n, c, h, w, ct, int(kernel_size), int(max_displacement), int(stride1),
            int(stride2), int(pad_size), int(bool(do_abs))]
    if one_d:
        _call("demon_correlation_1d_f32", *args, int(single_dir), _stream())
    else:
        _call("demon_correlation_f32", *args, _stream())
    return _ret(out, was_np)


def _corr_grad(one_d, gradient, input1, input2, kernel_size, max_displacement, stride1, stride2, pad_size, do_abs, corr_type,
               single_dir):
    ct = _corr_type(corr_type)
    _no_float64(gradient)
    a, b, was_np = _corr_inputs(input1, input2)
    g, _ = _as_cuda(gradient, torch.float32)
    shape = correlation_top_shape(a.shape, max_displacement, kernel_size, stride1, stride2, pad_size, one_d, single_dir)
    if tuple(g.shape) != tuple(shape):
        raise ValueError("Dimensions must be equal: gradient %s, output of the forward op %s" % (tuple(g.shape), tuple(shape)))
    g1, g2 = torch.empty_like(a), torch.empty_like(b)
    n, c, h, w = a.shape
    args = [a.data_ptr(), b.data_ptr(), g.data_ptr(), g1.data_ptr(), g2.data_ptr(), n, c, h, w, ct, int(kernel_size),
            int(max_displacement), int(stride1), int(stride2), int(pad_size), int(bool(do_abs))]
    if one_d:
        _call("demon_correlation_1d_grad_f32", *args, int(single_dir), _stream())
    else:
        _call("demon_correlation_grad_f32", *args, _stream())
    return _ret(g1, was_np), _ret(g2, was_np)


def correlation(input1, input2, max_displacement, kernel_size, stride1=1, stride2=1, pad_size=0, do_abs=False, corr_type="mult"):
    """Correlation (correlation.cc:25-104): for every K x K patch of input1 (NCHW, float32) its correlation with the patches
    of input2 displaced by (2R+1)^2 offsets, R = max_displacement // stride2 -> [N, (2R+1)^2, top_h, top_w].  'mult': mean
    of the products, 'subt': mean of the absolute differences.  do_abs has no effect, as in the reference."""
    return _corr_forward(False, input1, input2, kernel_size, max_displacement, stride1, stride2, pad_size, do_abs, corr_type, 0)


def correlation_1d(input1, input2, max_displacement, kernel_size, stride1=1, stride2=1, pad_size=0, do_abs=False,
                   corr_type="mult", single_dir=0):
    """Correlation1D (correlation_1d.cc): correlation along x only, pad_size columns each side and no vertical padding.
    single_dir 0: displacements -R..R times stride2; 1: 0..R; -1: the reference's -(R+1)..-1 (not -R..0), kept for
    drop-in compatibility.  The reference reads before the start of a padded row there; those reads are 0 here."""
    return _corr_forward(True, input1, input2, kernel_size, max_displacement, stride1, stride2, pad_size, do_abs, corr_type,
                         single_dir)


def correlation_grad(gradient, input1, input2, max_displacement, kernel_size, stride1=1, stride2=1, pad_size=0, do_abs=False,
                     corr_type="mult"):
    """CorrelationGrad (correlation.cc:106-128): (input1_grad, input2_grad) of `gradient` [N, top_c, top_h, top_w].  For
    'subt' this is the reference's gradient, which takes the sign of input1 - input2 at the displaced position for both
    inputs, not the derivative of the forward op."""
    return _corr_grad(False, gradient, input1, input2, kernel_size, max_displacement, stride1, stride2, pad_size, do_abs,
                      corr_type, 0)


def correlation_1d_grad(gradient, input1, input2, max_displacement, kernel_size, stride1=1, stride2=1, pad_size=0, do_abs=False,
                        corr_type="mult", single_dir=0):
    """Correlation1DGrad (correlation_1d.cc:95-118): (input1_grad, input2_grad); see correlation_1d and correlation_grad."""
    return _corr_grad(True, gradient, input1, input2, kernel_size, max_displacement, stride1, stride2, pad_size, do_abs,
                      corr_type, single_dir)


class _CorrelationFunction(torch.autograd.Function):
    """torch.autograd counterpart of the reference binding's registered Correlation / Correlation1D gradients."""

    @staticmethod
    def forward(ctx, input1, input2, one_d, attrs):
        ctx.save_for_backward(input1, input2)
        ctx.one_d, ctx.attrs = one_d, attrs
        return _corr_forward(one_d, input1, input2, *attrs)

    @staticmethod
    def backward(ctx, grad_out):
        input1, input2 = ctx.saved_tensors
        g1, g2 = _corr_grad(ctx.one_d, grad_out.contiguous(), input1, input2, *ctx.attrs)
        return g1, g2, None, None


def correlation_autograd(input1, input2, max_displacement, kernel_size, stride1=1, stride2=1, pad_size=0, do_abs=False,
                         corr_type="mult"):
    """correlation on torch CUDA tensors with the reference's gradient attached."""
    attrs = (int(kernel_size), int(max_displacement), int(stride1), int(stride2), int(pad_size), bool(do_abs), corr_type, 0)
    return _CorrelationFunction.apply(input1, input2, False, attrs)


def correlation_1d_autograd(input1, input2, max_displacement, kernel_size, stride1=1, stride2=1, pad_size=0, do_abs=False,
                            corr_type="mult", single_dir=0):
    """correlation_1d on torch CUDA tensors with the reference's gradient attached."""
    attrs = (int(kernel_size), int(max_displacement), int(stride1), int(stride2), int(pad_size), bool(do_abs), corr_type,
             int(single_dir))
    return _CorrelationFunction.apply(input1, input2, True, attrs)
