"""ORACLE (test infrastructure) -- numpy restatement of the evaluation metrics of depthmotionnet.evaluation.metrics
(compute_valid_depth_mask, compute_errors, evaluate_depth, compute_depth_scale_factor, compute_flow_epe) pixel by pixel,
in the 16-slot layout of the device sums (csrc/metrics.cu):

    0 count   1 |d|   2 |1/dp - 1/dg|   3 ld   4 ld^2   5 |d|/dg   6 d^2/dg   7 |log10 dp - log10 dg|   8 d^2
    9..11 |ld| < log t for t = 1.25, 1.5625, 1.953125   12, 13 dp^2, dp*dg   14, 15 (1/dp)^2, (1/dp)*(1/dg)

with d = dp - dg and ld = log dp - log dg.  Slots 12-15 are the least-squares scale factor's sums; they are taken over the
pixels valid before the prediction is scaled and where their own product is finite and > 0.

`promotion` names how numpy evaluates the reference's mixed scalar / array expressions:
- "legacy" is NumPy 1.x value-based casting: `depth_gt / translation_norm` and `depth_pred * scale` are float32 operations
  with the scalar rounded to float32, and `|log_diff| < np.log(t)` compares in float32 against float32(log t).  This is
  what the device implements.
- "nep50" is NumPy >= 2 (NEP 50): those scalars are float64, so the divide, the scaled product and the threshold compare
  are float64 (and everything downstream of a float64 array is float64).

The non-log terms are numpy's own correctly rounded IEEE operations, which the device performs bit for bit.  CUDA's
logf / log10f cannot be reproduced bit for bit, so for the log terms the oracle gives the float64 value of the exact
expression and a rigorous bound on the device's float32 result: logf within 1 ulp, log10f within 2 ulp (CUDA C
Programming Guide, maximum ulp errors), ½ ulp for the subtraction, and ld^2 to first order plus its rounding.  Each
threshold then sorts every pixel into certainly in, certainly out or ambiguous.  The "host" log terms are numpy's own
logs under the promotion rule: what the reference computes on the running numpy.
"""
import math

import numpy as np

THRESHOLDS = (1.25, 1.5625, 1.953125)
# float32(log t): the thresholds of the legacy compare.  numpy's own float32 log(1.5625f) is 0x3ee47fbf, one float above.
LEGACY_LOG_T = np.array([0x3e647fbe, 0x3ee47fbe, 0x3f2b5fcf], dtype=np.uint32).view(np.float32)
NON_LOG = (0, 1, 2, 5, 6, 8, 12, 13, 14, 15)
LOG = (3, 4, 7)
RATIO = (9, 10, 11)
DISTANCES = ['l1', 'l1_inverse', 'scale_invariant', 'abs_relative', 'sq_relative', 'avg_log10', 'rmse_log', 'rmse',
             'ratio_threshold_1.25', 'ratio_threshold_1.5625', 'ratio_threshold_1.953125']
THREADS, MAX_SLOTS = 256, 64
U = 2.0 ** -53


def slots(hw):
    """CTA slots per sample of the device reduction: one per 1024 pixels, 1..64."""
    return int(min(MAX_SLOTS, max(1, -(-int(hw) // (4 * THREADS)))))


def chain_length(hw):
    """The longest chain of double additions a term passes through on the device: its thread's strided steps, the
    5-level warp shuffle tree, the 8 warps of a CTA and the slots folded in order."""
    ns = slots(hw)
    return -(-int(hw) // (THREADS * ns)) + 5 + 8 + ns


def ulp32(y):
    """Spacing of float32 at |y|, taken in the upper binade where |y| is within rounding of a power of two."""
    y = np.abs(np.asarray(y, dtype=np.float64))
    with np.errstate(over="ignore"):
        return np.spacing(np.float32(1.0 + 2.0 ** -22) * y.astype(np.float32)).astype(np.float64)


def exact_sum(x):
    """Exact sums of the rows of x (float32 or float64, finite), rounded once to float64: equal to math.fsum of each
    row.  Every value is an integer mantissa M times 2^(e-b), b = 24 for float32 and 53 for float64.  The mantissas are
    summed per exponent in float64, exactly: a float32 mantissa is below 2^24, a float64 one is split into its high 26
    and low 27 bits, and rows are shorter than 2^26.  math.fsum adds the few per-exponent partials."""
    x = np.asarray(x)
    single = x.dtype == np.float32
    rows = x.astype(np.float64).reshape(-1, x.shape[-1]) if x.ndim else x.astype(np.float64).reshape(1, 1)
    assert np.isfinite(rows).all() and rows.shape[1] < 2 ** 26
    m, e = np.frexp(rows)
    e0, ne = int(e.min()), int(e.max() - e.min()) + 1
    key = (np.arange(rows.shape[0])[:, None] * ne + (e - e0)).ravel()
    if single:
        pieces = [(np.ldexp(m, 24), 24)]
    else:
        M = np.ldexp(m, 53)
        hi = np.trunc(np.ldexp(M, -27))
        pieces = [(hi, 26), (M - np.ldexp(hi, 27), 53)]
    out = np.zeros(rows.shape[0])
    sums = [(np.bincount(key, weights=v.ravel(), minlength=rows.shape[0] * ne).reshape(-1, ne), b) for v, b in pieces]
    for i in range(rows.shape[0]):
        out[i] = math.fsum(math.ldexp(float(s[i, k]), int(k) + e0 - b) for s, b in sums for k in np.flatnonzero(s[i]))
    return out.reshape(x.shape[:-1]) if x.ndim else out[0]


def _valid(a, b):
    with np.errstate(invalid="ignore"):
        return np.isfinite(a) & np.isfinite(b) & (a > 0) & (b > 0)


def depth_pixels(pred, gt, inverse_pred=False, inverse_gt=False, gt_div=None, pred_scale=None, promotion="legacy"):
    """Per-pixel masks and terms of the depth sums.  pred, gt: float32 [n, ...] (trailing dims are pixels); gt_div,
    pred_scale: [n] or None, the divisor of the ground truth (the translation norm) and the factor of the prediction.
    Under "nep50" their dtype is the reference's scalar's (float64 for the norm; the scale factor's own dtype).

    Returns a dict of [n, hw] arrays:
      valid0, valid     the mask before and after the scale and the second compute_valid_depth_mask
      terms [16, n, hw] every slot, 0 where masked; the log slots and 9..11 from numpy's own logs ("host")
      ld, l10           float64 exact ld and |log10 dp - log10 dg| of the float32 (or float64) operands
      ld_err, ld2_err, l10_err   bounds on the device's float32 slots 3, 4 and 7 around ld, ld^2, l10
      thr_in, thr_amb [3, n, hw] the device rule (legacy float32 thresholds) on the bounded ld: certainly in, ambiguous
    """
    if promotion not in ("legacy", "nep50"):
        raise ValueError(promotion)
    F = np.float32
    p = np.asarray(pred, dtype=F)
    n = p.shape[0]
    p = p.reshape(n, -1)
    g = np.asarray(gt, dtype=F).reshape(n, -1)
    one = F(1)
    with np.errstate(all="ignore"):
        valid0 = _valid(p, g)
        dp = np.reciprocal(p) if inverse_pred else p.copy()
        dg = np.reciprocal(g) if inverse_gt else g.copy()
        if gt_div is not None:
            gd = np.asarray(gt_div).reshape(n, 1)
            dg = dg / (gd.astype(F) if promotion == "legacy" else gd)
        pp, pg = dp * dp, dp * dg
        s1 = valid0 & np.isfinite(pg) & (pg > 0)
        ip, ig = one / dp, one / dg
        ipp, ipg = ip * ip, ip * ig
        s2 = valid0 & np.isfinite(ipg) & (ipg > 0)
        if pred_scale is not None:
            ps = np.asarray(pred_scale).reshape(n, 1)
            dp = dp * (ps.astype(F) if promotion == "legacy" else ps)
        valid = valid0 & _valid(dp, dg)
        d = dp - dg
        lp, lg = np.log(dp), np.log(dg)
        ld_host = lp - lg
        l10_host = np.abs(np.log10(dp) - np.log10(dg))
        T = LEGACY_LOG_T if promotion == "legacy" else np.array([math.log(t) for t in THRESHOLDS])
        terms = [np.ones_like(d), np.abs(d), np.abs(one / dp - one / dg), ld_host, np.square(ld_host), np.abs(d) / dg,
                 np.square(d) / dg, l10_host, np.square(d)] + [(np.abs(ld_host) < T[k]).astype(d.dtype) for k in range(3)]
        dt = np.result_type(*terms)
        terms = [np.where(valid, t, 0).astype(dt) for t in terms]
        terms += [np.where(s1, pp, 0).astype(dt), np.where(s1, pg, 0).astype(dt), np.where(s2, ipp, 0).astype(dt),
                  np.where(s2, ipg, 0).astype(dt)]
        # float64 references of the log terms and the device's bounds around them
        dp64, dg64 = dp.astype(np.float64), dg.astype(np.float64)
        Lp, Lg = np.log(dp64), np.log(dg64)
        ld = np.where(valid, Lp - Lg, 0.0)
        slack = 8 * U * (np.abs(Lp) + np.abs(Lg))
        e = ulp32(Lp) + ulp32(Lg) + slack
        e = np.where(valid, e + 0.5 * ulp32(np.abs(ld) + e), 0.0)
        ld2_err = np.where(valid, (2 * np.abs(ld) + e) * e + 0.5 * ulp32(np.square(np.abs(ld) + e)), 0.0)
        Tp, Tg = np.log10(dp64), np.log10(dg64)
        l10 = np.where(valid, np.abs(Tp - Tg), 0.0)
        e10 = 2 * ulp32(Tp) + 2 * ulp32(Tg) + 8 * U * (np.abs(Tp) + np.abs(Tg))
        l10_err = np.where(valid, e10 + 0.5 * ulp32(l10 + e10), 0.0)
    Tl = LEGACY_LOG_T.astype(np.float64)[:, None, None]
    a = np.abs(ld)[None]
    thr_in = valid[None] & (a + e[None] < Tl)
    thr_amb = valid[None] & ~thr_in & (a - e[None] < Tl)
    return dict(valid0=valid0, valid=valid, terms=np.stack(terms), ld=ld, ld_err=e, ld2_err=ld2_err, l10=l10,
                l10_err=l10_err, thr_in=thr_in, thr_amb=thr_amb, dtype=dt)


def threshold_account(pred, gt, inverse=False, gt_div=None, scaling=None):
    """Where the reference's ratio-threshold counts (NumPy 2, the golden vectors) and the device's (legacy) can differ,
    for one compute_errors call: evaluate_depth's when inverse (gt_div the float64 translation norm or None), its scaled
    pass when `scaling` names the scale factor (each rule with its own).  One dict per threshold:
      nep50        the NumPy 2 indicator, from numpy's own logs
      certain      the device rule's certainly-in pixels;  ambiguous: indices within the device's logf bound
      disagree     indices where the legacy and NEP 50 rules, both evaluated by numpy, differ
      unexplained  indices, not ambiguous, where the NEP 50 indicator differs from the device rule"""
    px = {}
    for rule in ("nep50", "legacy"):
        p = depth_pixels(pred, gt, inverse, inverse, gt_div, promotion=rule)
        if scaling is not None:
            s = scale_factor(depth_sums(p, "host"), scaling).astype(p["dtype"])
            p = depth_pixels(pred, gt, inverse, inverse, gt_div, s, promotion=rule)
        px[rule] = p
    out = []
    for k in range(3):
        nep = px["nep50"]["terms"][9 + k][0] > 0
        leg = px["legacy"]["terms"][9 + k][0] > 0
        certain, amb = px["legacy"]["thr_in"][k][0], px["legacy"]["thr_amb"][k][0]
        out.append(dict(nep50=nep, certain=certain, ambiguous=np.flatnonzero(amb), disagree=np.flatnonzero(nep != leg),
                        unexplained=np.flatnonzero((nep != certain) & ~amb)))
    return out


def depth_sums(px, logs="exact"):
    """[n, 16] float64 exact sums of the per-pixel terms.  logs="exact": slots 3, 4, 7 from the float64 ld, ld^2 and
    l10, slots 9..11 the certainly-in counts; logs="host": numpy's own log terms of depth_pixels."""
    t = list(px["terms"])
    if logs == "exact":
        t[3], t[4], t[7] = px["ld"], np.square(px["ld"]), px["l10"]
        t[9:12] = px["thr_in"].astype(np.float32)
    elif logs != "host":
        raise ValueError(logs)
    return np.stack([exact_sum(v) for v in t], axis=1)


def depth_sum_bounds(px):
    """[n, 16] bounds on |device sum - depth_sums(px, "exact")|: L 2^-53 sum|t| for the double accumulation (L =
    chain_length) plus, for the log slots, the summed per-pixel bounds.  Slots 9..11 hold the ambiguous counts: the
    device count lies in [certainly in, certainly in + ambiguous]."""
    t = np.abs(px["terms"].astype(np.float64))
    L = chain_length(t.shape[2])
    errs = {3: px["ld_err"], 4: px["ld2_err"], 7: px["l10_err"]}
    ref = {3: np.abs(px["ld"]), 4: np.square(px["ld"]), 7: px["l10"]}
    out = np.zeros((t.shape[1], 16))
    for k in range(16):
        if k in RATIO:
            out[:, k] = px["thr_amb"][k - 9].sum(axis=1)
        elif k in errs:
            out[:, k] = (L * U * (1 + 2.0 ** -40)) * (ref[k] + errs[k]).sum(axis=1) + errs[k].sum(axis=1) * (1 + 2.0 ** -40)
        else:
            out[:, k] = (L * U * (1 + 2.0 ** -40)) * t[k].sum(axis=1)
    return out


def epe_pixels(flow1, flow2):
    """flow [n, 2, ...] float32 -> (valid [n, hw], epe float32 [n, hw]): sqrt(dx^2 + dy^2) in float32 and its
    compute_valid_depth_mask."""
    a = np.asarray(flow1, dtype=np.float32)
    n = a.shape[0]
    a = a.reshape(n, 2, -1)
    b = np.asarray(flow2, dtype=np.float32).reshape(n, 2, -1)
    with np.errstate(all="ignore"):
        diff = a - b
        epe = np.sqrt(np.square(diff[:, 0]) + np.square(diff[:, 1]))
        valid = np.isfinite(epe) & (epe > 0)
    return valid, np.where(valid, epe, np.float32(0))


def epe_sums(flow1, flow2):
    """[n, 2] exact (sum of the valid end point errors, count)."""
    valid, epe = epe_pixels(flow1, flow2)
    return np.stack([exact_sum(epe), valid.sum(axis=1).astype(np.float64)], axis=1)


def scale_factor(sums, mode):
    """compute_depth_scale_factor from the sums, in float64: 'abs' s13/s12, 'log' exp(-s3/s0), 'inv' s14/s15; 1 where
    its denominator is not positive."""
    s = np.atleast_2d(np.asarray(sums, dtype=np.float64))
    with np.errstate(all="ignore"):
        if mode == "abs":
            return np.where(s[:, 12] > 0, s[:, 13] / s[:, 12], 1.0)
        if mode == "log":
            return np.where(s[:, 0] > 0, np.exp(-s[:, 3] / s[:, 0]), 1.0)
        if mode == "inv":
            return np.where(s[:, 14] > 0, 1.0 / (s[:, 15] / s[:, 14]), 1.0)
    raise ValueError(mode)


def distances(row, clamp=True):
    """compute_errors' dictionary from one row of sums.  clamp=True is the device's choice for scale_invariant:
    sqrt(max(0, s4/n - (s3/n)^2)); clamp=False keeps the reference's formula, which is NaN where rounding makes the
    variance negative."""
    s = [float(v) for v in row]
    num = s[0]
    out = {'num_valid': int(num)}
    if num == 0:
        out.update({k: float('nan') for k in DISTANCES})
        return out
    var = s[4] / num - (s[3] * s[3]) / (num * num)
    out.update({'l1': s[1] / num, 'l1_inverse': s[2] / num,
                'scale_invariant': math.sqrt(max(0.0, var)) if clamp or var >= 0 else float('nan'),
                'abs_relative': s[5] / num, 'sq_relative': s[6] / num, 'avg_log10': s[7] / num,
                'rmse_log': math.sqrt(s[4] / num), 'rmse': math.sqrt(s[8] / num)})
    for k, t in zip(RATIO, THRESHOLDS):
        out['ratio_threshold_%s' % t] = s[k] / num
    return out


def distance_intervals(row, bound):
    """[lo, hi] of every distance over the sums row +- bound (counts exact): the propagated bound of distances()."""
    s, b = np.asarray(row, dtype=np.float64), np.asarray(bound, dtype=np.float64)
    num = s[0]
    out = {}
    if num == 0:
        return out
    lo, hi = s - b, s + b
    for name, k in (('l1', 1), ('l1_inverse', 2), ('abs_relative', 5), ('sq_relative', 6), ('avg_log10', 7)):
        out[name] = (lo[k] / num, hi[k] / num)
    for name, k in (('rmse_log', 4), ('rmse', 8)):
        out[name] = (math.sqrt(max(0.0, lo[k]) / num), math.sqrt(hi[k] / num))
    sq = sorted((lo[3] * lo[3], hi[3] * hi[3]))
    sq_lo = 0.0 if lo[3] <= 0 <= hi[3] else sq[0]
    out['scale_invariant'] = (math.sqrt(max(0.0, lo[4] / num - sq[1] / (num * num))),
                              math.sqrt(max(0.0, hi[4] / num - sq_lo / (num * num))))
    for k, t in zip(RATIO, THRESHOLDS):
        out['ratio_threshold_%s' % t] = (s[k] / num, (s[k] + b[k]) / num)
    return out


def resample(pred, rows, cols):
    """pred [..., ph, pw] read through the row and column index tables (int, -1 reads 0, skimage's cval): [..., len(rows),
    len(cols)], the nearest-neighbour resize and crop the device reads through the same tables."""
    pred = np.asarray(pred)
    r, c = np.asarray(rows, dtype=np.int64), np.asarray(cols, dtype=np.int64)
    out = pred[..., np.maximum(r, 0)[:, None], np.maximum(c, 0)[None, :]]
    return np.where((r[:, None] >= 0) & (c[None, :] >= 0), out, pred.dtype.type(0))
