"""ORACLE (test infrastructure) -- the loss gradient kernels of csrc/losses.cu restated in numpy, operation for operation.

Every function performs exactly the IEEE operations of its kernel, in the kernel's order, on arrays of the input
precision (float32 or float64): add, subtract, multiply, divide and sqrt, each correctly rounded, nothing upcast, every
constant a `dtype.type(...)`.  So the device's gradients must equal these bit for bit.

  scale   gs = g * T(w): the upstream gradient times the weight (a Python number rounded once to T, or a device scalar)
  L2      pointwise_grad_kernel: gs * d_c / (T(M) * sqrt(s + eps)), s = sum over c ascending of replace_nonfinite(d_c)^2,
          d_c = pr_c - gt_c; 0 where d_c is not finite
  L1      gs * x / sqrt(x * x + eps), x = pr - gt
  SIG     sig_u_kernel: U = the L2 gradient of the prediction's 10-channel SIG stack against the target stack (the C
          oracle's SIG, bit-exact to the device's); sig_gather_kernel: per pixel and delta, tmp = 0 plus, in this order,
          the centre-x term, the neighbour-x term at x - d, the centre-y term and the neighbour-y term at y - d, each
          sig_dcenter / sig_dneighbour times U, skipped where the neighbour is outside the image or not finite;
          diff = diff + tmp over deltas 1, 2, 4, 8, 16; 0 where the centre or diff is not finite
  table   the terms on one prediction: the first writes, the next add, in table order

The block helpers take the arguments of demon_b200.v2.losses' blocks plus one upstream scalar per loss output and build
the same term tables in the same order.  oracle/losses.py holds the independent float64 gradients this restatement is
checked against (tests/test_loss_grads.py), and the bounds below state how far the float32 restatement may lie from them.
"""
import numpy as np

from . import losses as OL

SIG_DELTAS = (1, 2, 4, 8, 16)
EPS = 0.00001
L2, SIG, L1 = 0, 1, 2
U32 = 2.0 ** -24


def sig_eps(eps):
    """The SIG op's epsilon is a float attribute (scaleinvariantgradient.cc:109-113)."""
    return float(np.float32(eps))


def grad_scale(g, weight, dtype):
    """fmul(g, T(w)); g None is a NULL grad_out, which reads as 0."""
    T = np.dtype(dtype).type
    return (T(0) if g is None else T(g)) * T(weight)


def l2_grad(pr, gt, eps, gs):
    """pointwise_grad_kernel's L2 branch for pr, gt [n,c,h,w]."""
    T = pr.dtype.type
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        d = pr - gt
        fin = np.isfinite(d)
        e = np.where(fin, d, T(0))
        s = np.zeros((pr.shape[0],) + pr.shape[2:], pr.dtype)
        for c in range(pr.shape[1]):
            s = s + e[:, c] * e[:, c]
        den = T(pr.shape[0] * pr.shape[2] * pr.shape[3]) * np.sqrt(s + T(eps))
        return np.where(fin, (T(gs) * d) / den[:, None], T(0))


def l1_grad(pr, gt, eps, gs):
    """pointwise_grad_kernel's L1 branch; gt None is a NULL gt (x = pr)."""
    T = pr.dtype.type
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        x = pr - gt if gt is not None else pr
        return (T(gs) * x) / np.sqrt(x * x + T(eps))


def sig_u(planes, gt, eps, s_eps, gs, gt_plane=False, gt_s_eps=0.0):
    """sig_u_kernel: U [Z,10,H,W] for the prediction planes [Z,H,W] against a target stack [Z,10,H,W] or, with gt_plane,
    the SIG stack of the target planes [Z,H,W]."""
    ps = OL.sig_stack(planes, s_eps)
    g = OL.sig_stack(gt.reshape(planes.shape), gt_s_eps) if gt_plane else gt.reshape(ps.shape)
    return l2_grad(ps, g, eps, gs)


def sig_dcenter(c, n, eps):
    T = c.dtype.type
    s = (np.abs(c) + np.abs(n)) + eps
    return T(-1) / s + (np.where(c < 0, T(1), T(-1)) * (n - c)) / (s * s)


def sig_dneighbour(c, n, eps):
    T = c.dtype.type
    s = (np.abs(c) + np.abs(n)) + eps
    return T(1) / s + (np.where(n < 0, T(1), T(-1)) * (n - c)) / (s * s)


def _pairs(shape):
    """(delta index, channel, lower slice, upper slice) of every neighbour pair in sig_gather_kernel's order: per delta
    the x pairs, then the y pairs.  The pair's SIG term sits at the lower pixel, its neighbour at the upper one."""
    Z, H, W = shape
    for i, dl in enumerate(SIG_DELTAS):
        for axis, ch, n in ((2, 2 * i, W), (1, 2 * i + 1, H)):
            if dl >= n:
                continue
            lo, hi = [slice(None)] * 3, [slice(None)] * 3
            lo[axis], hi[axis] = slice(0, n - dl), slice(dl, n)
            yield i, ch, tuple(lo), tuple(hi)


def sig_gather(x, U, s_eps):
    """sig_gather_kernel: the gradient [Z,H,W] of sum(U * SIG stack of x) for the planes x [Z,H,W]."""
    T = x.dtype.type
    eps = T(s_eps)
    pairs = list(_pairs(x.shape))
    diff = np.zeros_like(x)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        for i in range(len(SIG_DELTAS)):   # every delta adds its tmp, +0 where it has no pair (-0 + 0 is +0)
            tmp = np.zeros_like(x)
            for _, ch, lo, hi in (p for p in pairs if p[0] == i):
                left, right, u = x[lo], x[hi], U[:, ch][lo]
                t = tmp[lo]   # the centre term of the lower pixel, then the neighbour term of the upper pixel
                tmp[lo] = np.where(np.isfinite(right), t + sig_dcenter(left, right, eps) * u, t)
                t = tmp[hi]
                tmp[hi] = np.where(np.isfinite(left), t + sig_dneighbour(left, right, eps) * u, t)
            diff = diff + tmp
    return np.where(np.isfinite(x) & np.isfinite(diff), diff, T(0))


class Term:
    """One demon_loss_term of a table: prediction prs[pr] against gt."""

    def __init__(self, kind, pr, gt, eps, weight, s_eps=0.0, gt_plane=False, gt_s_eps=0.0):
        self.kind, self.pr, self.gt, self.eps, self.weight = kind, pr, gt, eps, weight
        self.s_eps, self.gt_plane, self.gt_s_eps = s_eps, gt_plane, gt_s_eps


def term_grad(t, x, g):
    """d(out)/d(pr) of one term for the upstream scalar g (None: 0)."""
    gs = grad_scale(g, t.weight, x.dtype)
    if t.kind == L2:
        return l2_grad(x, t.gt, t.eps, gs)
    if t.kind == L1:
        return l1_grad(x, t.gt, t.eps, gs)
    planes = x.reshape((-1,) + x.shape[-2:])
    U = sig_u(planes, t.gt, t.eps, t.s_eps, gs, t.gt_plane, t.gt_s_eps)
    return sig_gather(planes, U, t.s_eps).reshape(x.shape)


def table_grads(terms, prs, upstream):
    """Every prediction's gradient (None where no term acts on it): the terms on one prediction write, then add."""
    out = [None] * len(prs)
    for t, g in zip(terms, upstream):
        v = term_grad(t, prs[t.pr], g)
        out[t.pr] = v if out[t.pr] is None else out[t.pr] + v
    return out


# ---- the blocks of demon_b200/v2/losses.py: the same tables, one upstream scalar per loss output (absent: not used) -------
def flow_block_grads(gt_flow2, gt_flow5, gt_flow2_sig, pr_flow2, pr_flow5, pr_conf2, pr_conf5, flow_weight, conf_weight,
                     flow_sig_weight, conf_sig_weight, upstream, conf_diff_scale=1, level5_factor=0.5, conf2=None, conf5=None):
    """{pr name: gradient} of flow_loss_block.  conf2 / conf5 are the confidence targets (default: oracle/losses.py's
    compute_confidence_map, which in float64 may differ from CUDA's exp in the last bit)."""
    prs, names = [pr_flow5, pr_flow2], ["pr_flow5", "pr_flow2"]
    terms = [Term(L2, 0, gt_flow5, EPS, level5_factor * flow_weight), Term(L2, 1, gt_flow2, EPS, flow_weight)]
    keys = ["loss_flow5", "loss_flow2"]
    if pr_conf5 is not None:
        c5 = OL.compute_confidence_map(pr_flow5, gt_flow5, conf_diff_scale) if conf5 is None else conf5
        prs.append(pr_conf5), names.append("pr_conf5")
        terms.append(Term(L2, len(prs) - 1, c5, EPS, level5_factor * conf_weight))
        keys.append("loss_conf5")
    if pr_conf2 is not None:
        c2 = OL.compute_confidence_map(pr_flow2, gt_flow2, conf_diff_scale) if conf2 is None else conf2
        prs.append(pr_conf2), names.append("pr_conf2")
        i_c2 = len(prs) - 1
        terms.append(Term(L2, i_c2, c2, EPS, conf_weight))
        keys.append("loss_conf2")
    if flow_sig_weight is not None:
        terms.append(Term(SIG, 1, gt_flow2_sig, EPS, flow_sig_weight, sig_eps(0.001)))
        keys.append("loss_flow2_sig")
    if conf_sig_weight is not None and pr_conf2 is not None:
        terms.append(Term(SIG, i_c2, c2, EPS, conf_sig_weight, sig_eps(0.001), gt_plane=True, gt_s_eps=sig_eps(0.001)))
        keys.append("loss_conf2_sig")
    grads = table_grads(terms, prs, [upstream.get(k) for k in keys])
    return dict(zip(names, grads))


def depthnormal_block_grads(gt_depth2, gt_depth2_sig, gt_normal2, gt_rotation, gt_translation, pr_depth2, pr_normal2, pr_rotation,
                            pr_translation, depth_weight, depth_sig_weight, normal_weight, rotation_weight, translation_weight,
                            translation_factor, upstream):
    """{pr name: gradient} of depthnormal_loss_block.  loss_translation = loss_translation_no_factor * factor, so its
    upstream reaches the L1 term as g * T(factor), added to loss_translation_no_factor's own."""
    T = pr_depth2.dtype.type
    batch = pr_depth2.shape[0]
    parts = []
    if upstream.get("loss_translation") is not None:
        parts.append(T(upstream["loss_translation"]) * T(translation_factor))
    if upstream.get("loss_translation_no_factor") is not None:
        parts.append(T(upstream["loss_translation_no_factor"]))
    g_tr = None if not parts else (parts[0] if len(parts) == 1 else parts[0] + parts[1])
    terms = [Term(L2, 0, gt_depth2, EPS, depth_weight), Term(SIG, 0, gt_depth2_sig, EPS, depth_sig_weight, sig_eps(0.01)),
             Term(L2, 1, gt_normal2, EPS, normal_weight), Term(L1, 2, gt_rotation, EPS, rotation_weight / batch),
             Term(L1, 3, gt_translation, EPS, translation_weight / batch)]
    ups = [upstream.get(k) for k in ("loss_depth2", "loss_depth2_sig", "loss_normal2", "loss_rotation")] + [g_tr]
    grads = table_grads(terms, [pr_depth2, pr_normal2, pr_rotation, pr_translation], ups)
    return dict(zip(("pr_depth2", "pr_normal2", "pr_rotation", "pr_translation"), grads))


def depth_refine_block_grads(gt_depth0, gt_depth0_sig, gt_normal0, pr_depth0, pr_normal0, depth_weight, depth_sig_weight, normal_weight,
                             upstream):
    """{pr name: gradient} of depth_refine_loss_block."""
    terms = [Term(L2, 0, gt_depth0, EPS, depth_weight), Term(SIG, 0, gt_depth0_sig, EPS, depth_sig_weight, sig_eps(0.01)),
             Term(L2, 1, gt_normal0, EPS, normal_weight)]
    grads = table_grads(terms, [pr_depth0, pr_normal0], [upstream.get(k) for k in ("loss_depth0", "loss_depth0_sig", "loss_normal0")])
    return dict(zip(("pr_depth0", "pr_normal0"), grads))


# ---- the forward's per-pixel SIG terms (the partial kernel's t), for exact checks of the eps-0 mean -------------------------
def sig_terms(planes, gt, eps, s_eps, gt_plane=False, gt_s_eps=0.0):
    """t = sqrt(s + eps) per pixel [Z,H,W] of a SIG term, as loss_partial_kernel computes it."""
    ps = OL.sig_stack(planes, s_eps)
    g = OL.sig_stack(gt.reshape(planes.shape), gt_s_eps) if gt_plane else gt.reshape(ps.shape)
    return OL.terms(ps, g, eps)


# ---- first-order error bounds of the restatement in a precision of unit roundoff u, against the exact gradient ------------
def l2_grad_bound(pr, gt, eps, scale, dpr=0.0, dgt=0.0, u=U32):
    """(bound, gradient) per element for the L2 gradient of pr, gt [n,c,h,w] given in float64 (the values the low precision
    run sees), the exact scale g * w, and absolute errors dpr, dgt of the inputs (nonzero when they are computed SIG stacks).
    Propagated:
      d  = pr - gt:        dd  = dpr + dgt + u|d|  (cancellation makes the inputs' errors absolute, not relative to d)
      s  = sum_c e_c^2:    ds  = sum_c 2|e_c| dd_c + C u s  (one square and C - 1 additions)
      s + eps:             dse = ds + u eps (eps rounded to T) + u (s + eps)
      t  = sqrt(s + eps):  dt  = dse / (2t) + u t
      g  = gs d / (M t):   |g| (2u (w rounded, g * w) + 2u (multiply, divide) + dt / t + 2u (M rounded, M * t)) + |gs| dd / (M t)"""
    pr, gt = np.asarray(pr, np.float64), np.asarray(gt, np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        d = pr - gt
    fin = np.isfinite(d)
    e = np.where(fin, d, 0.0)
    dd = np.where(fin, dpr + dgt + u * np.abs(e), 0.0)
    C = pr.shape[1]
    s = (e * e).sum(axis=1)
    ds = (2 * np.abs(e) * dd).sum(axis=1) + C * u * s
    se = s + eps
    t = np.sqrt(se)
    dt = (ds + u * eps + u * se) / (2 * t) + u * t
    M = pr.shape[0] * pr.shape[2] * pr.shape[3]
    g = scale * e / (M * t)[:, None]
    bound = np.abs(g) * (6 * u + (dt / t)[:, None]) + abs(scale) * dd / (M * t)[:, None]
    return np.where(fin, bound, 0.0), np.where(fin, g, 0.0)


def l1_grad_bound(x, eps, scale, u=U32):
    """(bound, gradient) for the L1 gradient of x = pr - gt (x given exactly, float64): x rounds once (dx = u|x|), x^2 + eps
    as in l2_grad_bound with C = 1, then sqrt, multiply and divide."""
    x = np.asarray(x, np.float64)
    dx = u * np.abs(x)
    se = x * x + eps
    r = np.sqrt(se)
    dse = 2 * np.abs(x) * dx + u * x * x + u * eps + u * se
    g = scale * x / r
    return np.abs(g) * (6 * u + dse / (2 * se)) + abs(scale) * dx / r, g


def sig_grad_bound(planes, gt, eps, s_eps, scale, gt_plane=False, gt_s_eps=0.0, u=U32):
    """(bound, gradient, addend magnitude) per element [Z,H,W] for a SIG term's gradient.
      SIG stack values: 4 roundings (subtract, two adds, divide) -> 4u|sig| for the prediction's, and the target's in
        gt_plane mode; then U as l2_grad_bound with those input errors, all 10 channels in t
      each SIG derivative A + B, A = -+1/S, B = +-(n - c)/S^2: S 2u, A 3u, B 7u, the add u -> 8u (|A| + |B|)
      each addend D U: |dD| |U| + |D| dU + u |D U|
      the gather: at most 20 addends per pixel, each through at most 7 roundings -> 7u sum |D U|"""
    x = np.asarray(planes, np.float64)
    ps = OL.sig_stack(x, s_eps)
    dps = np.where(np.isfinite(ps), 4 * u * np.abs(ps), 0.0)
    if gt_plane:
        g = OL.sig_stack(np.asarray(gt, np.float64).reshape(x.shape), gt_s_eps)
        dg = np.where(np.isfinite(g), 4 * u * np.abs(g), 0.0)
    else:
        g, dg = np.asarray(gt, np.float64).reshape(ps.shape), 0.0
    bU, U = l2_grad_bound(ps, g, eps, scale, dps, dg, u)
    bound, grad, mag = np.zeros_like(x), np.zeros_like(x), np.zeros_like(x)
    fin = np.isfinite(x)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        for _, ch, lo, hi in _pairs(x.shape):
            c, n = x[lo], x[hi]
            ok = np.isfinite(c) & np.isfinite(n)
            s = np.abs(c) + np.abs(n) + s_eps
            a, b = 1.0 / s, (n - c) / (s * s)
            dD = 8 * u * (np.abs(a) + np.abs(b))
            uu, bu = U[:, ch][lo], bU[:, ch][lo]
            for sl, D in ((lo, -a - np.where(c < 0, -1.0, 1.0) * b), (hi, a - np.where(n < 0, -1.0, 1.0) * b)):
                du = np.where(ok, D * uu, 0.0)
                grad[sl] += du
                mag[sl] += np.abs(du)
                bound[sl] += np.where(ok, dD * np.abs(uu) + np.abs(D) * bu + u * np.abs(du), 0.0)
    bound = np.where(fin, bound + 7 * u * mag, 0.0)
    return bound, np.where(fin, grad, 0.0), np.where(fin, mag, 0.0)
