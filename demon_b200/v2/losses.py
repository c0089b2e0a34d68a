"""DeMoN v2's training losses (the reference's python/depthmotionnet/v2/losses.py) on the device.

Same function names, argument names, defaults and result keys as the reference module.  Tensors are NCHW float32 or
float64.  Torch CUDA tensors in give 0-d torch CUDA tensors out without a host synchronisation; numpy in gives numpy out.
Weights may be Python numbers or 0-d tensors.  Scalar arithmetic follows TF's float32 order: a product of two Python
numbers, such as `level5_factor * flow_weight`, is one constant rounded to the tensor's precision, then one multiply.  A
product that involves a tensor weight is a tensor op in that precision.

The kernels are in csrc/losses.cu.  Each block runs as one table of terms: two launches for the forward pass, plus one
launch per confidence map.  What they compute:
  * pointwise_l2_loss: per pixel t = sqrt_rn(sum_c d_c^2 + eps), d_c = replace_nonfinite(pr_c - gt_c), with the channels
    summed in ascending order.  A non-finite difference counts as 0; it is not excluded from the mean.  The mean is
    accumulated in double in an order fixed by the shape, rounded once to the input precision, then weighted.
    TF's float32 reduce_mean has an order that cannot be reproduced; the double sum is at least as accurate.
  * the SIG losses compute the prediction's 10-channel SIG (deltas 1, 2, 4, 8, 16, one op call per delta as
    losses.py:57-79 does) on the fly and never store it.  SIG collapses leading dimensions, so a flow [N,2,H,W] is 2N
    planes and its mean runs over 2N*H*W pixels.
  * compute_confidence_map evaluates exp in double and rounds once, so the host can reproduce it bit for bit.

Gradients: every loss is differentiable with respect to every pr_* argument through torch.autograd.Functions whose
backward runs the gradient kernels.  Those take the upstream gradients as device scalars, so a whole training step's loss
forward and backward can be captured in one CUDA graph.  Losses on one prediction sum into one gradient buffer in a fixed
order.  No gradient reaches a ground-truth argument.  None reaches the confidence target exp(-s|pr_flow - gt_flow|)
either, as pointwise_l2_loss stops the gradient of its `gt` (losses.py:48).  Weights get no gradient.  The summaries
training.py never adds to the loss, `*_unscaled` and `rot_transl_loss_ratio`, come back detached: at eps = 0 they have no
finite gradient at a zero difference anyway.
"""
import ctypes

import numpy as np
import torch

from .. import _lib
from .. import lmbspecialops as sops

SIG_DELTAS = (1, 2, 4, 8, 16)
_L2, _SIG, _L1 = 0, 1, 2   # DEMON_LOSS_*


class _Term(ctypes.Structure):
    """demon_loss_term (include/demon_b200.h)."""
    _fields_ = [("kind", ctypes.c_int), ("c", ctypes.c_int), ("h", ctypes.c_int), ("w", ctypes.c_int), ("gt_plane", ctypes.c_int),
                ("accumulate", ctypes.c_int), ("n", ctypes.c_int64), ("pr", ctypes.c_void_p), ("gt", ctypes.c_void_p),
                ("eps", ctypes.c_double), ("sig_eps", ctypes.c_double), ("gt_sig_eps", ctypes.c_double), ("weight", ctypes.c_double),
                ("weight_dev", ctypes.c_void_p), ("out", ctypes.c_void_p), ("out0", ctypes.c_void_p), ("terms", ctypes.c_void_p),
                ("grad_out", ctypes.c_void_p), ("grad", ctypes.c_void_p)]


def _is_np(*xs):
    return not any(isinstance(x, torch.Tensor) for x in xs if x is not None)


def _t(x, dtype=None):
    """A contiguous CUDA tensor of x (torch tensors keep their autograd history)."""
    if isinstance(x, torch.Tensor):
        t = x if x.is_cuda else x.to(sops._device())
        if dtype is not None and t.dtype != dtype:
            t = t.to(dtype)
        if t.dtype not in (torch.float32, torch.float64):
            raise TypeError("the losses take float32 or float64 tensors, got %s" % t.dtype)
        return t.contiguous()
    return sops._as_cuda(x, dtype)[0]


def _np(x):
    return x.detach().cpu().numpy()


def _sig_eps(eps):
    """The SIG op's epsilon is a float attribute converted to T (scaleinvariantgradient.cc:109-113)."""
    return float(np.float32(eps))


# ---- weights: Python numbers stay Python numbers (one constant); a tensor makes the product a tensor op -----------------
def _mulw(a, b):
    return a * b


def _divw(a, b):
    return a / b


def _weight(w, dtype, device):
    """(host weight, device T scalar or None)"""
    if isinstance(w, torch.Tensor):
        return 0.0, w.detach().to(device=device, dtype=dtype).reshape(()).contiguous()
    return float(w), None


class _Spec:
    """One demon_loss_term: prediction prs[pr] against gt."""

    def __init__(self, kind, pr, gt, shape, eps, weight=1.0, sig_eps=0.0, gt_plane=False, gt_sig_eps=0.0, terms=False):
        self.kind, self.pr, self.gt, self.eps, self.weight = kind, pr, gt, float(eps), weight
        self.sig_eps, self.gt_plane, self.gt_sig_eps, self.want_terms = float(sig_eps), bool(gt_plane), float(gt_sig_eps), terms
        if kind == _L2:
            if len(shape) != 4:
                raise ValueError("pointwise_l2_loss takes NCHW tensors, got rank %d" % len(shape))
            self.n, self.c, self.h, self.w = (int(s) for s in shape)
            if gt is not None and tuple(gt.shape) != tuple(shape):
                raise ValueError("Dimensions must be equal, but are %s and %s" % (tuple(shape), tuple(gt.shape)))
        elif kind == _SIG:
            if len(shape) < 2:
                raise ValueError("Shape must be at least rank 2 but is rank %d" % len(shape))
            self.h, self.w = int(shape[-2]), int(shape[-1])
            self.n, self.c = sops._prod(shape[:-2]), 1
            want = tuple(shape) if gt_plane else (self.n, 2 * len(SIG_DELTAS), self.h, self.w)
            if tuple(gt.shape) != want:
                raise ValueError("the ground-truth SIG must be %s, got %s" % (want, tuple(gt.shape)))
        else:
            self.n, self.c, self.h, self.w = 1, sops._prod(shape), 1, 1
            if gt is not None and tuple(gt.shape) != tuple(shape):
                raise ValueError("Dimensions must be equal, but are %s and %s" % (tuple(shape), tuple(gt.shape)))


def _table(specs, prs, dtype, outs=None, grads=None, grad_bufs=None):
    arr = (_Term * len(specs))()
    keep = []
    written = set()
    for k, s in enumerate(specs):
        t = arr[k]
        t.kind, t.c, t.h, t.w, t.n = s.kind, s.c, s.h, s.w, s.n
        t.gt_plane, t.eps, t.sig_eps, t.gt_sig_eps = int(s.gt_plane), s.eps, s.sig_eps, s.gt_sig_eps
        t.pr = prs[s.pr].data_ptr()
        t.gt = s.gt.data_ptr() if s.gt is not None else None
        t.weight, wdev = _weight(s.weight, dtype, prs[s.pr].device)
        if wdev is not None:
            keep.append(wdev)
            t.weight_dev = wdev.data_ptr()
        if outs is not None:
            t.out, t.out0 = outs[k][0].data_ptr(), outs[k][1].data_ptr()
            if outs[k][2] is not None:
                t.terms = outs[k][2].data_ptr()
        if grad_bufs is not None and grad_bufs[s.pr] is not None:
            g = grads[k]
            t.grad_out = g.data_ptr() if g is not None else None
            t.grad = grad_bufs[s.pr].data_ptr()
            t.accumulate = int(s.pr in written)
            written.add(s.pr)
    return arr, keep


def _workspace(arr, n, dtype, backward, device):
    elem = 4 if dtype == torch.float32 else 8
    nbytes = _lib.load().demon_loss_workspace_bytes(ctypes.cast(arr, ctypes.c_void_p), n, elem, int(backward))
    if nbytes < 0:
        _lib.check(-1)
    return torch.empty(max(1, nbytes), dtype=torch.uint8, device=device), nbytes


def _forward(specs, prs):
    dtype, device = prs[0].dtype, prs[0].device
    outs = []
    for s in specs:
        terms = torch.empty((s.n, s.h, s.w), dtype=dtype, device=device) if s.want_terms else None
        outs.append((torch.empty((), dtype=dtype, device=device), torch.empty((), dtype=dtype, device=device), terms))
    arr, keep = _table(specs, prs, dtype, outs=outs)
    ws, nbytes = _workspace(arr, len(specs), dtype, False, device)
    sops._call("demon_loss_forward" + sops._sfx(prs[0]), ctypes.cast(arr, ctypes.c_void_p), len(specs), ws.data_ptr(), nbytes,
               sops._stream())
    return outs


class _LossFunction(torch.autograd.Function):
    """All terms of one call: outputs (out_0, out0_0, out_1, out0_1, ...); the out0 (eps 0) summaries are detached."""

    @staticmethod
    def forward(ctx, specs, *prs):
        outs = _forward(specs, prs)
        ctx.specs = specs
        ctx.save_for_backward(*prs)
        ctx.set_materialize_grads(False)
        flat = []
        for o in outs:
            flat += [o[0], o[1]]
        ctx.mark_non_differentiable(*flat[1::2])
        return tuple(flat)

    @staticmethod
    def backward(ctx, *grads):
        prs = ctx.saved_tensors
        specs = ctx.specs
        dtype, device = prs[0].dtype, prs[0].device
        bufs = [torch.empty_like(p) if ctx.needs_input_grad[1 + i] else None for i, p in enumerate(prs)]
        gouts = [None if g is None else g.to(dtype).contiguous() for g in grads[0::2]]
        arr, keep = _table(specs, prs, dtype, grads=gouts, grad_bufs=bufs)
        ws, nbytes = _workspace(arr, len(specs), dtype, True, device)
        sops._call("demon_loss_backward" + sops._sfx(prs[0]), ctypes.cast(arr, ctypes.c_void_p), len(specs), ws.data_ptr(), nbytes,
                   sops._stream())
        return (None,) + tuple(bufs)


def _evaluate(specs, prs):
    """[(loss, loss with eps 0)] per spec, differentiable with respect to prs where autograd records."""
    if torch.is_grad_enabled() and any(p.requires_grad for p in prs):
        flat = _LossFunction.apply(specs, *prs)
        return [(flat[2 * k], flat[2 * k + 1]) for k in range(len(specs))]
    return [(o[0], o[1]) for o in _forward(specs, prs)]


def _out(d, was_np):
    return {k: (_np(v) if was_np else v) for k, v in d.items()}


# ---- the reference module's functions -------------------------------------------------------------------------------------
def l1_loss(x, epsilon):
    """sum(sqrt(x^2 + epsilon)) (losses.py:23-29)."""
    was_np = _is_np(x)
    xt = _t(x)
    (loss, _), = _evaluate([_Spec(_L1, 0, None, tuple(xt.shape), epsilon)], [xt])
    return _np(loss) if was_np else loss


def pointwise_l2_loss(inp, gt, epsilon, data_format='NCHW', reduction='mean'):
    """Mean over the pixels of sqrt(sum over the channels of replace_nonfinite(inp - gt)^2 + epsilon) (losses.py:32-53).
    gt gets no gradient.  reduction='none' (an extension) returns the per-pixel terms [N,H,W] instead, without gradient."""
    if data_format not in ('NCHW', 'NHWC'):
        raise ValueError("data_format must be 'NCHW' or 'NHWC'")
    if reduction not in ('mean', 'none'):
        raise ValueError("reduction must be 'mean' or 'none'")
    was_np = _is_np(inp, gt)
    p = _t(inp)
    g = _t(gt, p.dtype).detach()
    if data_format == 'NHWC':
        p, g = p.permute(0, 3, 1, 2).contiguous(), g.permute(0, 3, 1, 2).contiguous()
    if reduction == 'none':
        outs = _forward([_Spec(_L2, 0, g, tuple(p.shape), epsilon, terms=True)], [p.detach()])
        return _np(outs[0][2]) if was_np else outs[0][2]
    (loss, _), = _evaluate([_Spec(_L2, 0, g, tuple(p.shape), epsilon)], [p])
    return _np(loss) if was_np else loss


def scale_invariant_gradient(inp, deltas, weights, epsilon=0.001):
    """The per-delta SIG images concatenated along C (losses.py:57-79): [N', 2*len(deltas), H, W] with N' the product of
    the leading dimensions.  Differentiable through the mirror op's gradient."""
    assert len(deltas) == len(weights)
    if _is_np(inp):
        return np.concatenate([sops.scale_invariant_gradient(inp, deltas=[d], weights=[w], epsilon=epsilon)
                               for d, w in zip(deltas, weights)], axis=1)
    x = _t(inp)
    return torch.cat([sops.scale_invariant_gradient_autograd(x, [d], [w], epsilon) for d, w in zip(deltas, weights)], dim=1)


def scale_invariant_gradient_loss(inp, gt, epsilon):
    """The sum over the channel pairs (2i, 2i+1) of pointwise_l2_loss (losses.py:83-104), added in order."""
    num_channels_inp, num_channels_gt = _t(inp).shape[1], _t(gt).shape[1]
    assert num_channels_inp % 2 == 0
    assert num_channels_inp == num_channels_gt
    total = None
    for i in range(num_channels_inp // 2):
        li = pointwise_l2_loss(inp[:, i * 2:i * 2 + 2, :, :], gt[:, i * 2:i * 2 + 2, :, :], epsilon)
        total = li if total is None else total + li
    return total


def compute_confidence_map(predicted_flow, gt_flow, scale=1):
    """exp(-scale * |predicted_flow - gt_flow|) (losses.py:360-373): the product in the input precision, exp in double,
    rounded once.  A training target: it carries no gradient."""
    was_np = _is_np(predicted_flow, gt_flow)
    p = _t(predicted_flow).detach()
    g = _t(gt_flow, p.dtype).detach()
    if tuple(p.shape) != tuple(g.shape):
        raise ValueError("Dimensions must be equal, but are %s and %s" % (tuple(p.shape), tuple(g.shape)))
    out = torch.empty_like(p)
    sops._call("demon_confidence_map" + sops._sfx(p), p.data_ptr(), g.data_ptr(), out.data_ptr(), p.numel(), float(scale),
               sops._stream())
    return _np(out) if was_np else out


def flow_loss_block(gt_flow2, gt_flow5, gt_flow2_sig, pr_flow2, pr_flow5, pr_conf2, pr_conf5, flow_weight, conf_weight,
                    flow_sig_weight, conf_sig_weight, conf_diff_scale=1, level5_factor=0.5, loss_prefix=''):
    """The flow losses (losses.py:109-191); the keys depend on which optional arguments are None as in the reference."""
    was_np = _is_np(gt_flow2, pr_flow2, pr_flow5, pr_conf2, pr_conf5)
    epsilon = 0.00001
    f2 = _t(pr_flow2)
    dt = f2.dtype
    f5 = _t(pr_flow5, dt)
    g2, g5 = _t(gt_flow2, dt).detach(), _t(gt_flow5, dt).detach()
    prs = [f5, f2]
    specs = [_Spec(_L2, 0, g5, tuple(f5.shape), epsilon, _mulw(level5_factor, flow_weight)),
             _Spec(_L2, 1, g2, tuple(f2.shape), epsilon, flow_weight)]
    keys = [('loss_flow5', 'loss_flow5_unscaled'), ('loss_flow2', 'loss_flow2_unscaled')]
    conf2 = None
    if pr_conf5 is not None:
        c5 = _t(pr_conf5, dt)
        conf5 = compute_confidence_map(f5.detach(), g5, conf_diff_scale)
        prs.append(c5)
        specs.append(_Spec(_L2, len(prs) - 1, conf5, tuple(c5.shape), epsilon, _mulw(level5_factor, conf_weight)))
        keys.append(('loss_conf5', 'loss_conf5_unscaled'))
    if pr_conf2 is not None:
        c2 = _t(pr_conf2, dt)
        conf2 = compute_confidence_map(f2.detach(), g2, conf_diff_scale)
        prs.append(c2)
        i_c2 = len(prs) - 1
        specs.append(_Spec(_L2, i_c2, conf2, tuple(c2.shape), epsilon, conf_weight))
        keys.append(('loss_conf2', 'loss_conf2_unscaled'))
    sig_eps = _sig_eps(0.001)
    if flow_sig_weight is not None:
        gs = _t(gt_flow2_sig, dt).detach()
        specs.append(_Spec(_SIG, 1, gs, tuple(f2.shape), epsilon, flow_sig_weight, sig_eps=sig_eps))
        keys.append(('loss_flow2_sig', 'loss_flow2_sig_unscaled'))
    if conf_sig_weight is not None and pr_conf2 is not None:
        specs.append(_Spec(_SIG, i_c2, conf2, tuple(prs[i_c2].shape), epsilon, conf_sig_weight, sig_eps=sig_eps, gt_plane=True,
                           gt_sig_eps=sig_eps))
        keys.append(('loss_conf2_sig', 'loss_conf2_sig_unscaled'))
    vals = _evaluate(specs, prs)
    # the reference's insertion order: flow5, flow2, both unscaled, then conf5, conf2, flow2_sig, conf2_sig pairs
    losses = {}
    losses[keys[0][0]], losses[keys[1][0]] = vals[0][0], vals[1][0]
    losses[keys[0][1]], losses[keys[1][1]] = vals[0][1], vals[1][1]
    for (k, k0), (v, v0) in zip(keys[2:], vals[2:]):
        losses[k], losses[k0] = v, v0
    return _out({loss_prefix + k: losses[k] for k in losses}, was_np)


def _scaled_sum(factor, loss):
    """factor * loss as TF multiplies them: one multiply in the loss's precision."""
    if isinstance(factor, torch.Tensor):
        return factor.to(device=loss.device, dtype=loss.dtype) * loss
    return loss * float(factor)


def depthnormal_loss_block(gt_depth2, gt_depth2_sig, gt_normal2, gt_rotation, gt_translation, pr_depth2, pr_normal2, pr_rotation,
                           pr_translation, depth_weight, depth_sig_weight, normal_weight, rotation_weight, translation_weight,
                           translation_factor, loss_prefix=''):
    """The depth, normal and motion losses (losses.py:197-262)."""
    was_np = _is_np(gt_depth2, pr_depth2, pr_normal2, pr_rotation, pr_translation)
    epsilon = 0.00001
    d2 = _t(pr_depth2)
    dt = d2.dtype
    batch_size = int(d2.shape[0])
    n2, rot, tr = _t(pr_normal2, dt), _t(pr_rotation, dt), _t(pr_translation, dt)
    prs = [d2, n2, rot, tr]
    specs = [_Spec(_L2, 0, _t(gt_depth2, dt).detach(), tuple(d2.shape), epsilon, depth_weight),
             _Spec(_SIG, 0, _t(gt_depth2_sig, dt).detach(), tuple(d2.shape), epsilon, depth_sig_weight, sig_eps=_sig_eps(0.01)),
             _Spec(_L2, 1, _t(gt_normal2, dt).detach(), tuple(n2.shape), epsilon, normal_weight),
             _Spec(_L1, 2, _t(gt_rotation, dt).detach(), tuple(rot.shape), epsilon, _divw(rotation_weight, batch_size)),
             _Spec(_L1, 3, _t(gt_translation, dt).detach(), tuple(tr.shape), epsilon, _divw(translation_weight, batch_size))]
    vals = _evaluate(specs, prs)
    loss_rotation, loss_translation_no_factor = vals[3][0], vals[4][0]
    losses = {
        'loss_depth2': vals[0][0],
        'loss_depth2_sig': vals[1][0],
        'loss_depth2_sig_unscaled': vals[1][1],
        'loss_normal2': vals[2][0],
        'loss_rotation': loss_rotation,
        'loss_translation': _scaled_sum(translation_factor, loss_translation_no_factor),
        'loss_translation_no_factor': loss_translation_no_factor,
        'rot_transl_loss_ratio': (loss_rotation / loss_translation_no_factor).detach(),
    }
    return _out({loss_prefix + k: losses[k] for k in losses}, was_np)


def depth_refine_loss_block(gt_depth0, gt_depth0_sig, gt_normal0, pr_depth0, pr_normal0, depth_weight, depth_sig_weight, normal_weight,
                            loss_prefix=''):
    """The refinement losses (losses.py:265-308)."""
    was_np = _is_np(gt_depth0, pr_depth0, pr_normal0)
    epsilon = 0.00001
    d0 = _t(pr_depth0)
    dt = d0.dtype
    n0 = _t(pr_normal0, dt)
    specs = [_Spec(_L2, 0, _t(gt_depth0, dt).detach(), tuple(d0.shape), epsilon, depth_weight),
             _Spec(_SIG, 0, _t(gt_depth0_sig, dt).detach(), tuple(d0.shape), epsilon, depth_sig_weight, sig_eps=_sig_eps(0.01)),
             _Spec(_L2, 1, _t(gt_normal0, dt).detach(), tuple(n0.shape), epsilon, normal_weight)]
    vals = _evaluate(specs, [d0, n0])
    losses = {
        'loss_depth0': vals[0][0],
        'loss_depth0_sig': vals[1][0],
        'loss_depth0_sig_unscaled': vals[1][1],
        'loss_normal0': vals[2][0],
    }
    return _out({loss_prefix + k: losses[k] for k in losses}, was_np)


def prepare_ground_truth_tensors(depth, rotation, translation, intrinsics):
    """Ground truth at levels 0, 2 and 5 from an inverse depth map [N,1,H,W] (losses.py:312-356): six launches, each output
    bit for bit the composition of the mirror ops in the reference's order.  'depth0' is `depth` itself."""
    was_np = _is_np(depth)
    shape = sops._shp(depth)
    if len(shape) < 2:
        raise ValueError("Shape must be at least rank 2 but is rank %d" % len(shape))
    h, w = int(shape[-2]), int(shape[-1])
    n = sops._prod(shape[:-2])
    sops._validate_pose_only(n, intrinsics, rotation, translation, "angleaxis3")
    d = _t(depth).detach()
    k, r, t, _ = sops._pose(n, d.dtype, intrinsics, rotation, translation, "angleaxis3")
    sizes = [(h, w)]
    for _ in range(5):
        sizes.append(((sizes[-1][0] + 1) // 2, (sizes[-1][1] + 1) // 2))
    (h2, w2), (h5, w5) = sizes[2], sizes[5]

    def new(*s):
        return torch.empty(s, dtype=d.dtype, device=d.device)
    depth2 = new(*(tuple(shape[:-2]) + (h2, w2)))
    out = {'depth2': depth2, 'flow0': new(n, 2, h, w), 'flow2': new(n, 2, h2, w2), 'flow5': new(n, 2, h5, w5),
           'normal0': new(n, 3, h, w), 'normal2': new(n, 3, h2, w2), 'depth0_sig': new(n, 10, h, w), 'depth2_sig': new(n, 10, h2, w2),
           'flow2_sig': new(2 * n, 10, h2, w2)}
    lib = _lib.load()
    nbytes = lib.demon_loss_ground_truth_workspace_bytes(n, h, w, d.element_size())
    if nbytes < 0:
        _lib.check(-1)
    ws = torch.empty(max(1, nbytes), dtype=torch.uint8, device=d.device)
    sops._call("demon_loss_ground_truth" + sops._sfx(d), d.data_ptr(), k.data_ptr(), r.data_ptr(), t.data_ptr(), n, h, w,
               *[out[key].data_ptr() for key in ('depth2', 'flow0', 'flow2', 'flow5', 'normal0', 'normal2', 'depth0_sig', 'depth2_sig',
                                                 'flow2_sig')], ws.data_ptr(), nbytes, sops._stream())
    res = {'depth0': depth if not was_np else np.asarray(depth)}
    for key in ('depth0_sig', 'depth2', 'depth2_sig', 'flow0', 'flow2', 'flow2_sig', 'flow5', 'normal0', 'normal2'):
        res[key] = _np(out[key]) if was_np else out[key]
    order = ('depth0', 'depth0_sig', 'depth2', 'depth2_sig', 'flow0', 'flow2', 'flow2_sig', 'flow5', 'normal0', 'normal2')
    return {key: res[key] for key in order}
