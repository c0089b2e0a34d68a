"""ORACLE (test infrastructure) -- numpy restatement of DeMoN v2's training losses (python/depthmotionnet/v2/losses.py) in
this project's defined per-pixel order, float32 or float64, with the float64 gradients.

Per pixel: d_c = replace_nonfinite(pr_c - gt_c), s = ((0 + d_0^2) + d_1^2) + ..., t = sqrt(s + eps), all in the input
precision.  The mean is math.fsum of the terms over M, rounded once to the input precision, then multiplied by the weight
(a Python number, one constant in that precision).  The SIG stacks, the median chain, depth_to_flow and depth_to_normals
come from the C oracle (oracle/ops.py).  tests/golden/losses_golden.npz pins this restatement to the reference's own
losses.py (see oracle/losses_ref.py).
"""
import math

import numpy as np

from . import ops

SIG_DELTAS = (1, 2, 4, 8, 16)
EPS = 0.00001


def _sig_eps(eps):
    return float(np.float32(eps))


def sig_stack(x, eps):
    """The per-delta SIG images concatenated along C: [N', 10, H, W] (losses.py:57-79)."""
    return np.concatenate([ops.scale_invariant_gradient(x, [d], [1.0], eps) for d in SIG_DELTAS], axis=1)


def diffs(pr, gt):
    with np.errstate(invalid="ignore", over="ignore"):
        d = pr - gt
    return d


def terms(pr, gt, eps):
    """Per-pixel terms [N,H,W] of pointwise_l2_loss for NCHW pr, gt."""
    T = pr.dtype.type
    d = diffs(pr, gt)
    d = np.where(np.isfinite(d), d, T(0))
    s = np.zeros((pr.shape[0],) + pr.shape[2:], pr.dtype)
    for c in range(pr.shape[1]):
        s = s + d[:, c] * d[:, c]
    return np.sqrt(s + T(eps))


def mean(t):
    """The mean of the terms, rounded once to their precision."""
    return t.dtype.type(math.fsum(t.ravel().astype(np.float64).tolist()) / t.size)


def pointwise_l2_loss(pr, gt, eps, weight=1.0):
    T = pr.dtype.type
    return T(weight) * mean(terms(pr, gt, eps))


def l1_loss(x, eps, weight=1.0):
    T = x.dtype.type
    t = np.sqrt(x * x + T(eps))
    return T(weight) * T(math.fsum(t.ravel().astype(np.float64).tolist()))


def scale_invariant_gradient(inp, deltas, weights, epsilon=0.001):
    return np.concatenate([ops.scale_invariant_gradient(np.asarray(inp), [d], [w], epsilon) for d, w in zip(deltas, weights)], axis=1)


def scale_invariant_gradient_loss(inp, gt, epsilon):
    total = None
    for i in range(inp.shape[1] // 2):
        li = pointwise_l2_loss(np.asarray(inp[:, 2 * i:2 * i + 2]), np.asarray(gt[:, 2 * i:2 * i + 2]), epsilon)
        total = li if total is None else total + li
    return total


def compute_confidence_map(pr, gt, scale=1):
    T = pr.dtype.type
    with np.errstate(invalid="ignore", over="ignore"):
        a = T(-scale) * np.abs(diffs(pr, gt))
        return np.exp(a.astype(np.float64)).astype(pr.dtype)


def prepare_ground_truth_tensors(depth, rotation, translation, intrinsics):
    levels = [depth]
    for _ in range(5):
        levels.append(ops.median3x3_downsample(levels[-1]))
    depth2, depth5 = levels[2], levels[5]

    def flow(dm):
        return ops.depth_to_flow(dm, intrinsics, rotation, translation, inverse_depth=True, normalize_flow=True)
    flow2 = flow(depth2)
    return {'depth0': depth, 'depth0_sig': sig_stack(depth, 0.001), 'depth2': depth2, 'depth2_sig': sig_stack(depth2, 0.001),
            'flow0': flow(depth), 'flow2': flow2, 'flow2_sig': sig_stack(flow2, 0.001), 'flow5': flow(depth5),
            'normal0': ops.depth_to_normals(depth, intrinsics, inverse_depth=True),
            'normal2': ops.depth_to_normals(depth2, intrinsics, inverse_depth=True)}


def flow_loss_block(gt_flow2, gt_flow5, gt_flow2_sig, pr_flow2, pr_flow5, pr_conf2, pr_conf5, flow_weight, conf_weight,
                    flow_sig_weight, conf_sig_weight, conf_diff_scale=1, level5_factor=0.5, loss_prefix=''):
    L = {}
    L['loss_flow5'] = pointwise_l2_loss(pr_flow5, gt_flow5, EPS, level5_factor * flow_weight)
    L['loss_flow2'] = pointwise_l2_loss(pr_flow2, gt_flow2, EPS, flow_weight)
    L['loss_flow5_unscaled'] = pointwise_l2_loss(pr_flow5, gt_flow5, 0)
    L['loss_flow2_unscaled'] = pointwise_l2_loss(pr_flow2, gt_flow2, 0)
    conf2 = compute_confidence_map(pr_flow2, gt_flow2, conf_diff_scale)
    conf5 = compute_confidence_map(pr_flow5, gt_flow5, conf_diff_scale)
    if pr_conf5 is not None:
        L['loss_conf5'] = pointwise_l2_loss(pr_conf5, conf5, EPS, level5_factor * conf_weight)
        L['loss_conf5_unscaled'] = pointwise_l2_loss(pr_conf5, conf5, 0)
    if pr_conf2 is not None:
        L['loss_conf2'] = pointwise_l2_loss(pr_conf2, conf2, EPS, conf_weight)
        L['loss_conf2_unscaled'] = pointwise_l2_loss(pr_conf2, conf2, 0)
    if flow_sig_weight is not None:
        s = sig_stack(pr_flow2, 0.001)
        L['loss_flow2_sig'] = pointwise_l2_loss(s, gt_flow2_sig, EPS, flow_sig_weight)
        L['loss_flow2_sig_unscaled'] = pointwise_l2_loss(s, gt_flow2_sig, 0)
    if conf_sig_weight is not None and pr_conf2 is not None:
        s, g = sig_stack(pr_conf2, 0.001), sig_stack(conf2, 0.001)
        L['loss_conf2_sig'] = pointwise_l2_loss(s, g, EPS, conf_sig_weight)
        L['loss_conf2_sig_unscaled'] = pointwise_l2_loss(s, g, 0)
    return {loss_prefix + k: v for k, v in L.items()}


def depthnormal_loss_block(gt_depth2, gt_depth2_sig, gt_normal2, gt_rotation, gt_translation, pr_depth2, pr_normal2, pr_rotation,
                           pr_translation, depth_weight, depth_sig_weight, normal_weight, rotation_weight, translation_weight,
                           translation_factor, loss_prefix=''):
    T = pr_depth2.dtype.type
    batch_size = pr_depth2.shape[0]
    s = sig_stack(pr_depth2, 0.01)
    L = {'loss_depth2': pointwise_l2_loss(pr_depth2, gt_depth2, EPS, depth_weight),
         'loss_depth2_sig': pointwise_l2_loss(s, gt_depth2_sig, EPS, depth_sig_weight),
         'loss_depth2_sig_unscaled': pointwise_l2_loss(s, gt_depth2_sig, 0),
         'loss_normal2': pointwise_l2_loss(pr_normal2, gt_normal2, EPS, normal_weight)}
    rot = l1_loss(pr_rotation - gt_rotation, EPS, rotation_weight / batch_size)
    tnf = l1_loss(pr_translation - gt_translation, EPS, translation_weight / batch_size)
    L['loss_rotation'] = rot
    L['loss_translation'] = T(translation_factor) * tnf
    L['loss_translation_no_factor'] = tnf
    L['rot_transl_loss_ratio'] = rot / tnf
    return {loss_prefix + k: v for k, v in L.items()}


def depth_refine_loss_block(gt_depth0, gt_depth0_sig, gt_normal0, pr_depth0, pr_normal0, depth_weight, depth_sig_weight, normal_weight,
                            loss_prefix=''):
    s = sig_stack(pr_depth0, 0.01)
    L = {'loss_depth0': pointwise_l2_loss(pr_depth0, gt_depth0, EPS, depth_weight),
         'loss_depth0_sig': pointwise_l2_loss(s, gt_depth0_sig, EPS, depth_sig_weight),
         'loss_depth0_sig_unscaled': pointwise_l2_loss(s, gt_depth0_sig, 0),
         'loss_normal0': pointwise_l2_loss(pr_normal0, gt_normal0, EPS, normal_weight)}
    return {loss_prefix + k: v for k, v in L.items()}


# ---- float64 gradients of the weighted losses (scale = upstream gradient * weight) ------------------------------------------
def l2_grad(pr, gt, eps, scale=1.0):
    """d(scale * pointwise_l2_loss)/d pr: scale * d_c / (M t), 0 where d_c is not finite."""
    d = diffs(pr.astype(np.float64), gt.astype(np.float64))
    ok = np.isfinite(d)
    t = terms(pr.astype(np.float64), gt.astype(np.float64), eps)
    return np.where(ok, scale * np.where(ok, d, 0.0) / (t.size * t)[:, None], 0.0)


def l1_grad(x, eps, scale=1.0):
    x = x.astype(np.float64)
    return scale * x / np.sqrt(x * x + eps)


def sig_input_grad(x, g, eps):
    """Gradient of sum(g * sig_stack(x, eps)) with respect to x [Z,H,W] for g [Z,10,H,W]: each delta's SIG derivative
    (scaleinvariantgradient.cc:247-268), 0 at a non-finite x, terms with a non-finite neighbour skipped."""
    x = np.asarray(x, np.float64)
    Z, H, W = x.shape
    out = np.zeros_like(x)
    fin = np.isfinite(x)
    for i, dl in enumerate(SIG_DELTAS):
        for axis, ch in ((2, 2 * i), (1, 2 * i + 1)):
            n = x.shape[axis]
            if dl >= n:
                continue
            sl_c = [slice(None)] * 3
            sl_n = [slice(None)] * 3
            sl_c[axis], sl_n[axis] = slice(0, n - dl), slice(dl, n)
            c, nb, gg = x[tuple(sl_c)], x[tuple(sl_n)], g[:, ch][tuple(sl_c)]
            ok = fin[tuple(sl_c)] & fin[tuple(sl_n)]
            with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
                S = np.abs(c) + np.abs(nb) + eps
                dc = -1.0 / S + np.where(c < 0, 1.0, -1.0) * (nb - c) / (S * S)
                dn = 1.0 / S + np.where(nb < 0, 1.0, -1.0) * (nb - c) / (S * S)
            out[tuple(sl_c)] += np.where(ok, dc * gg, 0.0)
            out[tuple(sl_n)] += np.where(ok, dn * gg, 0.0)
    out[~fin] = 0.0
    out[~np.isfinite(out)] = 0.0
    return out


def sig_loss_grad(pr, gt_sig, eps, sig_eps, scale=1.0):
    """d(scale * pointwise_l2_loss(sig_stack(pr, sig_eps), gt_sig, eps))/d pr, pr [..,H,W] (float64)."""
    x = pr.astype(np.float64)
    s = sig_stack(x, sig_eps)
    g = l2_grad(s, gt_sig.astype(np.float64), eps, scale)
    return sig_input_grad(x.reshape((-1,) + x.shape[-2:]), g, _sig_eps(sig_eps)).reshape(pr.shape)
