"""GPU: the metric reductions of csrc/metrics.cu (depth_sums_kernel and epe_sums_kernel, dense and ResampledPixels)
against oracle/metrics.py, an independent numpy statement of the same per-pixel arithmetic with exact sums.

- One pixel per sample turns the reduction into a per-pixel readout: every non-log term is bit-equal to numpy float32,
  the device's own ld is within the oracle's logf bound, and the ratio thresholds are the legacy (NumPy 1.x) float32
  compare of that ld against float32(log t).
- At the evaluation's sizes (up to 960x1280, the 64-slot grid of 480x640 at batch 64) the sums are within the double
  accumulation's bound of the exact sums; one-hot rows catch a dropped or doubled pixel bit for bit.
- The resampled entries are checked against numpy index tables, never against the dense kernel.
"""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from demon_b200 import _lib
from demon_b200 import evaluation as ev
from oracle import metrics as om

F = np.float32
SIZES = (1, 31, 255, 256, 257, 1023, 1024, 1025, 64511, 64512, 64513, 65536, 436 * 588, 480 * 640, 960 * 1280)


@pytest.fixture(scope="module", autouse=True)
def peak_memory():
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    torch.cuda.reset_peak_memory_stats()
    yield
    print("\ntest_gpu_metrics_oracle: peak device memory %.1f MB" % (torch.cuda.max_memory_allocated() / 2 ** 20))


# ---------------------------------------------------------------------------------------------------------------------
# device calls
# ---------------------------------------------------------------------------------------------------------------------
def dev_depth_sums(pred, gt, inverse_pred=False, inverse_gt=False, gt_div=None, pred_scale=None):
    return ev.depth_error_sums(pred, gt, inverse_pred, inverse_gt, gt_div, pred_scale).cpu().numpy()


def dev_epe_sums(f1, f2):
    return ev.flow_epe_sums(f1, f2).cpu().numpy()


def dev_scale(sums, mode):
    return ev.depth_scale_factor(torch.from_numpy(sums).cuda(), mode).cpu().numpy()


def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def ptr(t):
    return None if t is None else t.data_ptr()


def stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def dev_resampled_depth(pred, gt, gt_valid, window, rows, cols, gt_div, pred_scale=None):
    n, ph, pw = pred.shape
    gh, gw = gt.shape[1:]
    y0, x0, oh, ow = window
    lib = _lib.load()
    p, g, v = cuda(pred), cuda(gt), None if gt_valid is None else cuda(gt_valid)
    r, c = cuda(np.asarray(rows, np.int32)), cuda(np.asarray(cols, np.int32))
    gd, ps = cuda(np.asarray(gt_div, F)), None if pred_scale is None else cuda(np.asarray(pred_scale, F))
    sums = torch.empty((n, 16), dtype=torch.float64, device="cuda")
    ws = torch.empty(max(1, lib.demon_metric_workspace_bytes(n, oh * ow) // 8), dtype=torch.float64, device="cuda")
    _lib.check(lib.demon_depth_error_sums_resampled_f32(ptr(p), ph, pw, ptr(g), ptr(v), gh, gw, n, y0, x0, oh, ow, ptr(r), ptr(c),
                                                        1, 1, ptr(gd), ptr(ps), ptr(sums), ptr(ws), stream()))
    return sums.cpu().numpy()


def dev_resampled_flow(pred, gt, window, rows, cols):
    n, _, ph, pw = pred.shape
    gh, gw = gt.shape[2:]
    y0, x0, oh, ow = window
    lib = _lib.load()
    p, g = cuda(pred), cuda(gt)
    r, c = cuda(np.asarray(rows, np.int32)), cuda(np.asarray(cols, np.int32))
    sums = torch.empty((n, 2), dtype=torch.float64, device="cuda")
    ws = torch.empty(max(1, lib.demon_metric_workspace_bytes(n, oh * ow) // 8), dtype=torch.float64, device="cuda")
    _lib.check(lib.demon_flow_epe_sums_resampled_f32(ptr(p), ph, pw, ptr(g), gh, gw, n, y0, x0, oh, ow, ptr(r), ptr(c), ptr(sums),
                                                     ptr(ws), stream()))
    return sums.cpu().numpy()


# ---------------------------------------------------------------------------------------------------------------------
# assertions against the oracle
# ---------------------------------------------------------------------------------------------------------------------
def assert_sums_within(got, px, tag=""):
    """got [n,16] device sums of the pixels px (depth_pixels, legacy): counts exact, thresholds between certainly in and
    certainly in + ambiguous, every other slot within the bound of the exact sum."""
    want, bound = om.depth_sums(px), om.depth_sum_bounds(px)
    assert np.array_equal(got[:, 0], want[:, 0]), (tag, got[:, 0], want[:, 0])
    for k in om.RATIO:
        assert ((got[:, k] >= want[:, k]) & (got[:, k] <= want[:, k] + bound[:, k])).all(), (tag, k, got[:, k], want[:, k], bound[:, k])
    for k in om.NON_LOG + om.LOG:
        err = np.abs(got[:, k] - want[:, k])
        assert (err <= bound[:, k]).all(), (tag, k, err.max(), bound[:, k][np.argmax(err - bound[:, k])])


def assert_epe_within(got, f1, f2, tag=""):
    valid, epe = om.epe_pixels(f1, f2)
    want = om.epe_sums(f1, f2)
    assert np.array_equal(got[:, 1], want[:, 1]), tag
    bound = om.chain_length(valid.shape[1]) * om.U * (1 + 2.0 ** -40) * epe.astype(np.float64).sum(axis=1)
    assert (np.abs(got[:, 0] - want[:, 0]) <= bound).all(), tag


# ---------------------------------------------------------------------------------------------------------------------
# a. one pixel per sample
# ---------------------------------------------------------------------------------------------------------------------
def step(a, k):
    """a moved by k floats (a > 0)."""
    return (a.view(np.int32) + np.int32(k)).view(F)


def candidate_pairs():
    """(pred, gt) float32 pairs: log-uniform magnitudes, specials, and for each threshold the nearest float32 to t*b and
    its +-4-ulp neighbours against b, in both orders."""
    rng = np.random.RandomState(1)
    a = np.exp2(rng.uniform(-30, 30, 4000)).astype(F)
    b = np.exp2(rng.uniform(-30, 30, 4000)).astype(F)
    ps, gs = [a, b[:2000]], [b, a[:2000] * F(1.0000001)]
    sp = np.array([0.0, -0.0, 1e-45, 1e-40, 1.1754944e-38, 2.9e-39, 1e-39, -1.0, 0.5, 1.0, 2.0, 3.4e38, np.nan, np.inf, -np.inf], F)
    ps.append(np.repeat(sp, sp.size))
    gs.append(np.tile(sp, sp.size))
    for t in om.THRESHOLDS:
        ps.append(np.array([t, 1.0], F))
        gs.append(np.array([1.0, t], F))
        base = np.exp2(rng.uniform(-20, 20, 1000)).astype(F)
        near = (np.float64(t) * base.astype(np.float64)).astype(F)
        for k in range(-4, 5):
            x = step(near, k)
            ps += [x, base]
            gs += [base, x]
    p, g = np.concatenate(ps), np.concatenate(gs)
    assert p.size <= 65535
    return p, g


COMBOS = [(ip, ig, gd, sc) for ip in (False, True) for ig in (False, True) for gd in (False, True) for sc in (False, True)]


@pytest.mark.parametrize("inverse_pred,inverse_gt,with_div,with_scale", COMBOS)
def test_per_pixel_terms(inverse_pred, inverse_gt, with_div, with_scale):
    p, g = candidate_pairs()
    n = p.size
    rng = np.random.RandomState(2)
    gd = rng.uniform(0.5, 3.0, n).astype(F) if with_div else None
    if gd is not None:
        gd[::5] = 1.0
    sc = rng.uniform(0.3, 3.0, n).astype(F) if with_scale else None
    got = dev_depth_sums(p[:, None], g[:, None], inverse_pred, inverse_gt, gd, sc)
    px = om.depth_pixels(p[:, None], g[:, None], inverse_pred, inverse_gt, gd, sc)
    valid = px["valid"][:, 0]
    assert np.array_equal(got[:, 0], valid.astype(np.float64))
    for k in om.NON_LOG:     # NaN where both reciprocals overflow: |inf - inf|, as in numpy
        assert np.array_equal(got[:, k], px["terms"][k][:, 0].astype(np.float64), equal_nan=True), k
    # slot 3 is the device's own ld (a float32 converted to double)
    ld = got[:, 3].astype(F)
    assert np.array_equal(ld.astype(np.float64), got[:, 3])
    assert (np.abs(got[:, 3] - px["ld"][:, 0]) <= px["ld_err"][:, 0]).all()
    assert np.array_equal(got[:, 4], (ld * ld).astype(np.float64))
    assert (np.abs(got[:, 7] - px["l10"][:, 0]) <= px["l10_err"][:, 0]).all()
    hits = []
    for k in range(3):
        want = valid & (np.abs(ld) < om.LEGACY_LOG_T[k])
        assert np.array_equal(got[:, 9 + k], want.astype(np.float64)), (om.THRESHOLDS[k], np.flatnonzero(got[:, 9 + k] != want))
        hits.append(int((valid & (np.abs(ld) == om.LEGACY_LOG_T[k])).sum()))
    if not (inverse_pred or inverse_gt or with_div or with_scale):
        # the threshold compare is only tested where some |ld| equals float32(log t) exactly
        print("\nexact-threshold hits |ld| == float32(log t) for t = %s: %s" % (om.THRESHOLDS, hits))
        assert all(h > 0 for h in hits), hits
        # the pairs (t, 1): logf(1) = +0, so slot 3 is the device's logf(t) itself
        idx = [int(np.flatnonzero((p == F(t)) & (g == F(1)))[0]) for t in om.THRESHOLDS]
        print("device logf(t) for t = %s: %s (float32(log t): %s)" % (om.THRESHOLDS, [hex(v) for v in ld[idx].view(np.uint32)],
                                                                     [hex(v) for v in om.LEGACY_LOG_T.view(np.uint32)]))


def test_per_pixel_epe():
    rng = np.random.RandomState(3)
    n = 60000
    a = rng.standard_normal((n, 2, 1)).astype(F) * np.exp2(rng.uniform(-30, 30, (n, 2, 1))).astype(F)
    b = rng.standard_normal((n, 2, 1)).astype(F) * np.exp2(rng.uniform(-30, 30, (n, 2, 1))).astype(F)
    sp = np.array([0.0, -0.0, 1e-45, 1e-39, 2e19, 3.4e38, -3.4e38, np.nan, np.inf, -np.inf], F)
    k = sp.size
    a[:k * k, 0, 0], b[:k * k, 0, 0] = np.repeat(sp, k), np.tile(sp, k)
    a[k * k:2 * k * k, 1, 0], b[k * k:2 * k * k, 1, 0] = np.repeat(sp, k), np.tile(sp, k)
    b[2 * k * k:2 * k * k + 100] = a[2 * k * k:2 * k * k + 100]          # epe 0 is masked out
    got = dev_epe_sums(a, b)
    valid, epe = om.epe_pixels(a, b)
    assert np.array_equal(got[:, 1], valid[:, 0].astype(np.float64))
    assert np.array_equal(got[:, 0], epe[:, 0].astype(np.float64))


# ---------------------------------------------------------------------------------------------------------------------
# b. the reduction at the evaluation's sizes
# ---------------------------------------------------------------------------------------------------------------------
def sample_data(hw, n, seed):
    """Inverse depths [n, hw]: every sample its own range and error spread, ~5% NaN, zero and negative entries."""
    rng = np.random.RandomState(seed)
    lo = np.exp2(rng.uniform(-6, 2, (n, 1)))
    gt = (lo * np.exp2(rng.uniform(0, rng.uniform(1, 8, (n, 1)), (n, hw)))).astype(F)
    pred = (gt * np.exp(rng.normal(0, rng.uniform(0.02, 0.6, (n, 1)), (n, hw)))).astype(F)
    bad = rng.rand(n, hw)
    gt[bad < 0.02] = np.nan
    pred[(bad >= 0.02) & (bad < 0.035)] = 0
    gt[(bad >= 0.035) & (bad < 0.045)] = -gt[(bad >= 0.035) & (bad < 0.045)]
    pred[(bad >= 0.045) & (bad < 0.05)] = np.inf
    gd = rng.uniform(0.4, 2.5, n).astype(F)
    gd[0] = 1.0
    return pred, gt, gd


def checked_rows(n):
    """Samples compared with the oracle: all of a small batch, first, last and a few between of a large one (every sample
    of a batch is also compared bit for bit with its own single-sample run)."""
    return list(range(n)) if n <= 3 else sorted({0, 1, n // 2 + 1, n - 1})


def oracle_rows(pred, gt, gd, rows, pred_scale=None):
    return om.depth_pixels(pred[rows], gt[rows], True, True, gd[rows], None if pred_scale is None else pred_scale[rows])


CASES = [(hw, n) for hw in SIZES for n in ((8,) if hw == 960 * 1280 else (1, 3, 64))]


@pytest.mark.parametrize("hw,n", CASES)
def test_sums_at_real_sizes(hw, n):
    pred, gt, gd = sample_data(hw, n, hw + n)
    got = dev_depth_sums(pred, gt, True, True, gd)
    rows = checked_rows(n) if hw > 1 else list(range(n))
    assert_sums_within(got[rows], oracle_rows(pred, gt, gd, rows), (hw, n))
    again = dev_depth_sums(pred, gt, True, True, gd)
    assert np.array_equal(got, again, equal_nan=True)                       # run to run
    f1 = np.stack([pred, gt[::-1]], axis=1)
    f2 = np.stack([gt, pred[::-1]], axis=1) * F(0.5)
    fe = dev_epe_sums(f1, f2)
    assert_epe_within(fe[rows], f1[rows], f2[rows], (hw, n))


@pytest.mark.parametrize("hw", (257, 65536, 436 * 588, 480 * 640))
def test_batch_independence(hw):
    """A sample's sums do not depend on its batch: the slot count depends on hw only, so each sample of a batch of 64
    equals its own single-sample run bit for bit."""
    pred, gt, gd = sample_data(hw, 64, 7 * hw)
    batch = dev_depth_sums(pred, gt, True, True, gd)
    for i in range(64):
        alone = dev_depth_sums(pred[i:i + 1], gt[i:i + 1], True, True, gd[i:i + 1])
        assert np.array_equal(alone[0], batch[i]), i
    f1, f2 = np.stack([pred, gt], axis=1), np.stack([gt, pred], axis=1)
    fb = dev_epe_sums(f1, f2)
    for i in (0, 31, 63):
        assert np.array_equal(dev_epe_sums(f1[i:i + 1], f2[i:i + 1])[0], fb[i]), i


def one_hot_positions(hw):
    ns = om.slots(hw)
    stride = om.THREADS * ns
    pos = {0, hw - 1}
    for k in (1, 2, 3, 7, 11, 18):
        pos |= {k * stride, k * stride - 1, k * stride + 1}
    last = (hw - 1) // stride * stride                       # the last strided step, full or ragged
    pos |= {last, last - 1, last - stride, last - stride + om.THREADS * (ns - 1)}
    return sorted(p for p in pos if 0 <= p < hw)


@pytest.mark.parametrize("hw", [s for s in SIZES if s > 1])
def test_one_hot_rows(hw):
    """Each sample has one valid pixel: its sums are that pixel's terms bit for bit (the pixel's own single-pixel run),
    which catches a dropped or doubled pixel at the slot and stride boundaries."""
    pos = one_hot_positions(hw)
    n = len(pos)
    rng = np.random.RandomState(hw)
    pv = rng.uniform(0.1, 3.0, n).astype(F)
    gv = rng.uniform(0.1, 3.0, n).astype(F)
    gd = rng.uniform(0.5, 2.0, n).astype(F)
    pred = np.full((n, hw), 0.7, F)
    gt = np.full((n, hw), np.nan, F)
    gt[np.arange(n), pos], pred[np.arange(n), pos] = gv, pv
    got = dev_depth_sums(pred, gt, True, True, gd)
    want = dev_depth_sums(pv[:, None], gv[:, None], True, True, gd)
    assert np.array_equal(got, want), [pos[i] for i in np.flatnonzero((got != want).any(axis=1))]
    assert (got[:, 0] == 1).all()
    f1 = np.zeros((n, 2, hw), F)
    f2 = np.full((n, 2, hw), np.nan, F)
    f2[np.arange(n), 0, pos], f2[np.arange(n), 1, pos] = pv, gv
    got = dev_epe_sums(f1, f2)
    assert np.array_equal(got, dev_epe_sums(np.zeros((n, 2, 1), F), f2[np.arange(n), :, pos][:, :, None]))
    assert (got[:, 1] == 1).all()


# ---------------------------------------------------------------------------------------------------------------------
# c. scale factors
# ---------------------------------------------------------------------------------------------------------------------
def scale_bound(want, bound, mode):
    """Bound on |device scale - oracle scale| from the sum bounds, before the float32 rounding."""
    s, b = want, bound
    if mode == "abs":
        rel = b[:, 12] / s[:, 12] + b[:, 13] / np.abs(s[:, 13])
    elif mode == "log":
        rel = 2 * b[:, 3] / s[:, 0]
    else:
        rel = b[:, 14] / s[:, 14] + b[:, 15] / np.abs(s[:, 15])
    return 1.01 * rel * np.abs(om.scale_factor(s, mode))


@pytest.mark.parametrize("mode", ("abs", "log", "inv"))
def test_scale_factor_and_scaled_pass(mode):
    hw, n = 480 * 640, 64
    pred, gt, gd = sample_data(hw, n, 99)
    got = dev_depth_sums(pred, gt, True, True, gd)
    scale = dev_scale(got, mode)
    rows = checked_rows(n)
    px = oracle_rows(pred, gt, gd, rows)
    want, bound = om.depth_sums(px), om.depth_sum_bounds(px)
    ref = om.scale_factor(want, mode)
    assert (np.abs(scale[rows].astype(np.float64) - ref) <= scale_bound(want, bound, mode) + om.ulp32(ref)).all()
    assert np.array_equal(scale, om.scale_factor(got, mode).astype(F))              # float32 of the double formula
    scaled = dev_depth_sums(pred, gt, True, True, gd, scale)
    assert_sums_within(scaled[rows], oracle_rows(pred, gt, gd, rows, scale), mode)


# ---------------------------------------------------------------------------------------------------------------------
# d. resampled entries
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ph,pw", ((48, 64), (192, 256)))
@pytest.mark.parametrize("crop", (False, True))
@pytest.mark.parametrize("masked", (False, True))
def test_resampled_against_index_tables(ph, pw, crop, masked):
    n, gh, gw = 64, 480, 640
    rng = np.random.RandomState(ph + 4 * crop + 2 * masked)
    pred = rng.uniform(0.05, 2.0, (n, ph, pw)).astype(F) * np.exp2(rng.uniform(-2, 2, (n, 1, 1))).astype(F)
    pred[rng.rand(n, ph, pw) < 0.02] = np.nan
    gt = rng.uniform(0.05, 2.0, (n, gh, gw)).astype(F)
    gt[rng.rand(n, gh, gw) < 0.03] = np.nan
    gt[rng.rand(n, gh, gw) < 0.01] = 0
    valid = (rng.rand(n, gh, gw) > 0.2).astype(np.uint8) if masked else None
    window = ev.EIGEN_CROP if crop else (0, 0, gh, gw)
    y0, x0, oh, ow = window
    rows_t, cols_t = ev.nearest_index(ph, gh)[y0:y0 + oh], ev.nearest_index(pw, gw)[x0:x0 + ow]
    gd = rng.uniform(0.5, 2.0, n).astype(F)
    got = dev_resampled_depth(pred, gt, valid, window, rows_t, cols_t, gd)
    rows = [0, n // 2 + 1, n - 1]
    gw_ = gt[rows].copy()
    if masked:
        gw_[valid[rows] == 0] = np.nan
    gw_ = gw_[:, y0:y0 + oh, x0:x0 + ow]
    pm = om.resample(pred[rows], rows_t, cols_t)
    px = om.depth_pixels(pm, gw_, True, True, gd[rows])
    assert_sums_within(got[rows], px, (ph, crop, masked))
    scale = dev_scale(got, "abs")
    scaled = dev_resampled_depth(pred, gt, valid, window, rows_t, cols_t, gd, scale)
    assert_sums_within(scaled[rows], om.depth_pixels(pm, gw_, True, True, gd[rows], scale[rows]), (ph, crop, masked, "scaled"))
    if not masked:
        fp = rng.normal(0, 0.05, (n, 2, ph, pw)).astype(F)
        fg = rng.normal(0, 0.05, (n, 2, gh, gw)).astype(F)
        fg[rng.rand(n, 2, gh, gw) < 0.02] = np.nan
        fe = dev_resampled_flow(fp, fg, window, rows_t, cols_t)
        assert_epe_within(fe[rows], om.resample(fp[rows], rows_t, cols_t), fg[rows][:, :, y0:y0 + oh, x0:x0 + ow], (ph, crop))


def test_resampled_hand_made_tables():
    """Tables with -1 entries (cval 0) and non-monotone, repeated indices, through the C entries: a depth pixel that reads
    0 is invalid, a flow pixel that reads 0 contributes |gt|."""
    n, ph, pw, gh, gw = 3, 5, 7, 6, 9
    window = (1, 2, 4, 5)
    rows_t, cols_t = np.array([4, -1, 0, 4]), np.array([6, -1, 3, 3, 0])
    rng = np.random.RandomState(8)
    pred = rng.uniform(0.1, 2.0, (n, ph, pw)).astype(F)
    gt = rng.uniform(0.1, 2.0, (n, gh, gw)).astype(F)
    valid = (rng.rand(n, gh, gw) > 0.3).astype(np.uint8)
    gd = np.array([1.0, 1.7, 0.6], F)
    y0, x0, oh, ow = window
    for v in (None, valid):
        got = dev_resampled_depth(pred, gt, v, window, rows_t, cols_t, gd)
        g = gt.copy()
        if v is not None:
            g[v == 0] = np.nan
        g = g[:, y0:y0 + oh, x0:x0 + ow]
        pm = om.resample(pred, rows_t, cols_t)
        px = om.depth_pixels(pm, g, True, True, gd)
        assert not px["valid"].reshape(n, oh, ow)[:, 1].any() and not px["valid"].reshape(n, oh, ow)[:, :, 1].any()
        assert_sums_within(got, px)
        assert got[:, 0].tolist() == px["valid"].sum(axis=1).tolist()
    fp = rng.normal(0, 1, (n, 2, ph, pw)).astype(F)
    fg = rng.normal(0, 1, (n, 2, gh, gw)).astype(F)
    fe = dev_resampled_flow(fp, fg, window, rows_t, cols_t)
    fm, fgw = om.resample(fp, rows_t, cols_t), fg[:, :, y0:y0 + oh, x0:x0 + ow]
    assert_epe_within(fe, fm, fgw)
    _, epe = om.epe_pixels(fm, fgw)
    cval = np.sqrt(np.square(fgw[:, 0]) + np.square(fgw[:, 1]))
    assert np.array_equal(epe.reshape(n, oh, ow)[:, 1], cval[:, 1])        # row table -1: |gt|


# ---------------------------------------------------------------------------------------------------------------------
# e. bounds and refusals
# ---------------------------------------------------------------------------------------------------------------------
GUARD = 4096
SENTINEL = 0x5A


class Guarded:
    """`nbytes` of device memory inside a sentinel-filled block; intact() checks every guard byte."""

    def __init__(self, nbytes):
        self.nbytes = int(nbytes)
        self.block = torch.full((self.nbytes + 2 * GUARD,), SENTINEL, dtype=torch.uint8, device="cuda")
        self.ptr = self.block.data_ptr() + GUARD

    def intact(self):
        b = self.block.cpu().numpy()
        return (b[:GUARD] == SENTINEL).all() and (b[GUARD + self.nbytes:] == SENTINEL).all()

    def doubles(self, n):
        return self.block[GUARD:GUARD + 8 * n].cpu().numpy().view(np.float64)


def guarded_dense(pred, gt, n, hw, lib):
    sums, ws = Guarded(n * 16 * 8), Guarded(lib.demon_metric_workspace_bytes(n, hw))
    p, g = (cuda(pred), cuda(gt)) if hw else (None, None)
    rc = lib.demon_depth_error_sums_f32(ptr(p), ptr(g), n, hw, 1, 1, None, None, sums.ptr, ws.ptr, stream())
    torch.cuda.synchronize()
    return rc, sums, ws


@pytest.mark.parametrize("hw,n", ((1, 5), (1025, 3), (480 * 640, 64), (0, 3)))
def test_sums_and_workspace_stay_in_bounds(hw, n):
    lib = _lib.load()
    pred, gt, gd = sample_data(max(hw, 1), n, 5)
    rc, sums, ws = guarded_dense(pred[:, :hw], gt[:, :hw], n, hw, lib)
    assert rc == 0
    assert sums.intact() and ws.intact(), (hw, n, ws.nbytes)
    if hw == 0:
        # no pixels: zero sums and NaN distances
        assert (sums.doubles(n * 16) == 0).all()
        assert all(np.isnan(ev.errors_from_sums(r)[k]) for r in sums.doubles(n * 16).reshape(n, 16) for k in ev.DISTANCES)
    f = Guarded(n * 2 * 8)
    fw = Guarded(lib.demon_metric_workspace_bytes(n, hw))
    a, b = (cuda(np.stack([pred[:, :hw], gt[:, :hw]], 1)), cuda(np.stack([gt[:, :hw], pred[:, :hw]], 1))) if hw else (None, None)
    assert lib.demon_flow_epe_sums_f32(ptr(a), ptr(b), n, hw, f.ptr, fw.ptr, stream()) == 0
    torch.cuda.synchronize()
    assert f.intact() and fw.intact()
    if hw == 0:
        assert (f.doubles(2 * n) == 0).all()


def test_resampled_sums_stay_in_bounds():
    lib = _lib.load()
    n, ph, pw, gh, gw = 4, 48, 64, 480, 640
    y0, x0, oh, ow = ev.EIGEN_CROP
    rng = np.random.RandomState(6)
    p, g = cuda(rng.uniform(0.1, 2, (n, ph, pw)).astype(F)), cuda(rng.uniform(0.1, 2, (n, gh, gw)).astype(F))
    fp, fg = cuda(rng.normal(0, 1, (n, 2, ph, pw)).astype(F)), cuda(rng.normal(0, 1, (n, 2, gh, gw)).astype(F))
    r, c = cuda(ev.nearest_index(ph, gh)[y0:y0 + oh].copy()), cuda(ev.nearest_index(pw, gw)[x0:x0 + ow].copy())
    gd = cuda(np.ones(n, F))
    for oh_, ow_ in ((oh, ow), (0, ow)):
        sums, ws = Guarded(n * 16 * 8), Guarded(lib.demon_metric_workspace_bytes(n, oh_ * ow_))
        assert lib.demon_depth_error_sums_resampled_f32(ptr(p), ph, pw, ptr(g), None, gh, gw, n, y0, x0, oh_, ow_, ptr(r), ptr(c), 1, 1,
                                                        ptr(gd), None, sums.ptr, ws.ptr, stream()) == 0
        f, fw = Guarded(n * 2 * 8), Guarded(lib.demon_metric_workspace_bytes(n, oh_ * ow_))
        assert lib.demon_flow_epe_sums_resampled_f32(ptr(fp), ph, pw, ptr(fg), gh, gw, n, y0, x0, oh_, ow_, ptr(r), ptr(c), f.ptr,
                                                     fw.ptr, stream()) == 0
        torch.cuda.synchronize()
        assert sums.intact() and ws.intact() and f.intact() and fw.intact(), (oh_, ow_)


def test_refusals_launch_nothing():
    lib = _lib.load()
    n0 = lib.demon_launch_count()
    d = torch.ones(64, device="cuda")
    w = torch.zeros(1 << 20, dtype=torch.float64, device="cuda")
    s = torch.zeros(1 << 10, dtype=torch.float64, device="cuda")
    i = torch.zeros(64, dtype=torch.int32, device="cuda")
    P, W, S, I = d.data_ptr(), w.data_ptr(), s.data_ptr(), i.data_ptr()
    st = stream()
    # n = 0 launches nothing and succeeds
    assert lib.demon_depth_error_sums_f32(P, P, 0, 4, 0, 0, None, None, S, W, st) == 0
    assert lib.demon_flow_epe_sums_f32(P, P, 0, 4, S, W, st) == 0
    assert lib.demon_depth_error_sums_resampled_f32(P, 2, 2, P, None, 4, 4, 0, 0, 0, 4, 4, I, I, 1, 1, None, None, S, W, st) == 0
    assert lib.demon_flow_epe_sums_resampled_f32(P, 2, 2, P, 4, 4, 0, 0, 0, 4, 4, I, I, S, W, st) == 0
    assert lib.demon_depth_scale_factor(S, 0, 0, P, st) == 0
    refused = [
        lib.demon_depth_error_sums_f32(P, P, 65536, 1, 0, 0, None, None, S, W, st),
        lib.demon_flow_epe_sums_f32(P, P, 65536, 1, S, W, st),
        lib.demon_depth_error_sums_f32(P, P, -1, 1, 0, 0, None, None, S, W, st),
        lib.demon_depth_error_sums_f32(P, P, 1, -1, 0, 0, None, None, S, W, st),
        lib.demon_depth_error_sums_f32(None, P, 1, 4, 0, 0, None, None, S, W, st),
        lib.demon_depth_error_sums_f32(P, P, 1, 4, 0, 0, None, None, None, W, st),
        lib.demon_depth_error_sums_f32(P, P, 1, 4, 0, 0, None, None, S, None, st),
        lib.demon_flow_epe_sums_f32(P, None, 1, 4, S, W, st),
        lib.demon_depth_error_sums_resampled_f32(P, 2, 2, P, None, 4, 4, 65536, 0, 0, 4, 4, I, I, 1, 1, None, None, S, W, st),
        lib.demon_depth_error_sums_resampled_f32(P, 2, 2, P, None, 4, 4, 1, 1, 0, 4, 4, I, I, 1, 1, None, None, S, W, st),
        lib.demon_depth_error_sums_resampled_f32(P, 2, 2, P, None, 4, 4, 1, 0, 1, 4, 4, I, I, 1, 1, None, None, S, W, st),
        lib.demon_depth_error_sums_resampled_f32(P, 2, 2, P, None, 4, 4, 1, -1, 0, 2, 2, I, I, 1, 1, None, None, S, W, st),
        lib.demon_depth_error_sums_resampled_f32(P, 2, 2, P, None, 4, 4, 1, 0, 0, 2, 2, None, I, 1, 1, None, None, S, W, st),
        lib.demon_depth_error_sums_resampled_f32(P, 2, 2, None, None, 4, 4, 1, 0, 0, 2, 2, I, I, 1, 1, None, None, S, W, st),
        lib.demon_flow_epe_sums_resampled_f32(P, 2, 2, P, 4, 4, 65536, 0, 0, 4, 4, I, I, S, W, st),
        lib.demon_flow_epe_sums_resampled_f32(P, 2, 2, P, 4, 4, 1, 0, 0, 5, 4, I, I, S, W, st),
        lib.demon_flow_epe_sums_resampled_f32(P, 2, 2, P, 4, 4, 1, 0, 0, 4, 4, I, None, S, W, st),
        lib.demon_depth_scale_factor(S, 1, 3, P, st),
        lib.demon_depth_scale_factor(None, 1, 0, P, st),
    ]
    assert refused == [-1] * len(refused), refused
    assert lib.demon_launch_count() == n0


# ---------------------------------------------------------------------------------------------------------------------
# f. the evaluator's table against a table computed on the host
# ---------------------------------------------------------------------------------------------------------------------
B, ITER = 2, 1


@pytest.fixture(scope="module")
def session(synthetic_weights):
    from demon_b200.networks_original import Session
    s = Session()
    s.load_weights(synthetic_weights)
    return s


def scale_candidates(want, bound, mode):
    """Every float32 the device's scale factor can be, given the exact sums and their bounds."""
    ref = float(om.scale_factor(want[None], mode)[0])
    b = float(scale_bound(want[None], bound[None], mode)[0])
    lo, hi = F(ref - b), F(ref + b)
    lo = np.nextafter(lo, F(-np.inf)) if float(lo) > ref - b else lo
    out = [lo]
    while out[-1] < hi or float(out[-1]) < ref + b:
        out.append(np.nextafter(out[-1], F(np.inf)))
        assert len(out) < 64
    return out


def within(v, interval, rel=1e-14):
    lo, hi = interval
    return lo - rel * abs(lo) <= v <= hi + rel * abs(hi)


def check_depth_row(got, px_for_scale, n_valid, tag):
    """got: the table's 11 distances of one sample (unscaled or scaled); px_for_scale: the oracle pixels."""
    want, bound = om.depth_sums(px_for_scale), om.depth_sum_bounds(px_for_scale)
    assert want[0, 0] == n_valid
    iv = om.distance_intervals(want[0], bound[0])
    for j, name in enumerate(om.DISTANCES):
        if not within(got[j], iv[name]):
            return False, (tag, name, got[j], iv[name])
        if name.startswith('ratio'):
            c = got[j] * n_valid
            if abs(c - round(c)) > 1e-6:
                return False, (tag, name, c)
    return True, None


@pytest.mark.parametrize("depthmask,crop", ((True, False), (False, True)))
def test_evaluator_table_against_host(session, depthmask, crop):
    from demon_b200 import lmbspecialops as sops
    from oracle import view_tools as vt
    gh, gw = 480, 640
    g = torch.Generator().manual_seed(41)
    ip = (torch.rand(B, 6, 192, 256, generator=g) - 0.5).cuda()
    i22 = sops.median3x3_downsample(sops.median3x3_downsample(ip[:, 3:6].contiguous()))
    rng = np.random.RandomState(12)
    yy, xx = np.mgrid[0:gh, 0:gw]
    inv = np.stack([0.3 + 0.15 * np.sin(xx / (40.0 + 10 * i)) + 0.1 * np.cos(yy / 25.0) for i in range(B)]).astype(F)
    inv[rng.rand(B, gh, gw) < 0.02] = np.nan
    motion = np.concatenate([rng.normal(0, 0.05, (B, 3)), rng.normal(0, 0.4, (B, 3))], axis=1).astype(F)
    intr = np.tile(np.array([[0.89, 1.19, 0.5, 0.5]], F), (B, 1))
    evaluator = ev.Evaluator(session, B, ITER, depthmask=depthmask, eigen_crop_gt_and_pred=crop)
    got = evaluator.add(ip, inv, motion, intr, image2_2=i22)
    snaps = {k: v.cpu().numpy() for k, v in evaluator.pipeline.forward_snapshots(ip, i22).items()}
    # host: mask, gt_div, tables
    gt = inv.copy()
    if depthmask:
        ops = ev.visible_points_operands(motion, intr, gh, gw)
        with np.errstate(divide='ignore'):
            absd = (F(1) / gt).astype(F)
        for i in range(B):
            gt[i][vt.visible_points_mask_numpy(absd[i], *[o[i] for o in ops], gw, gh) == 0] = np.nan
    window = ev.EIGEN_CROP if crop else (0, 0, gh, gw)
    y0, x0, oh, ow = window
    gtw = gt[:, y0:y0 + oh, x0:x0 + ow]
    norm = np.sqrt((motion[:, 3:6].astype(np.float64) ** 2).sum(axis=1))
    gd = np.where(np.isclose(1.0, norm), 1.0, norm).astype(F)
    flow_gt = sops.depth_to_flow(inv[:, None], intr, motion[:, 0:3].copy(), motion[:, 3:6].copy(), rotation_format="angleaxis3",
                                 inverse_depth=True, normalize_flow=True)
    fh, fw = snaps["predict_flow2"].shape[-2:]
    fr, fc = ev.nearest_index(fh, gh), ev.nearest_index(fw, gw)
    for k in range(ITER + 1):
        for label, key in ((str(k), "predict_depth2"), ("%d_refined" % k, "predict_depth0")):
            pred = snaps[key][k, :B, 0]
            ph, pw = pred.shape[-2:]
            pm = om.resample(pred, ev.nearest_index(ph, gh)[y0:y0 + oh], ev.nearest_index(pw, gw)[x0:x0 + ow])
            for i in range(B):
                px = om.depth_pixels(pm[i:i + 1], gtw[i:i + 1], True, True, gd[i:i + 1])
                nv = int(px["valid"].sum())
                table = got.values[0, got.coords['iteration'].index(label), i]
                ok, why = check_depth_row(table[3:14, 0], px, nv, (label, i))
                assert ok, why
                want, bound = om.depth_sums(px), om.depth_sum_bounds(px)
                results = []
                for s in scale_candidates(want[0], bound[0], 'abs'):
                    pxs = om.depth_pixels(pm[i:i + 1], gtw[i:i + 1], True, True, gd[i:i + 1], np.array([s], F))
                    results.append(check_depth_row(table[3:14, 1], pxs, int(pxs["valid"].sum()), (label, i, float(s))))
                assert any(r[0] for r in results), [r[1] for r in results]
                if label == str(k):
                    pmot = np.concatenate([snaps["predict_rotation"][k, i], snaps["predict_translation"][k, i]])
                    np.testing.assert_allclose(table[0:3, 0], ev.compute_motion_errors(pmot, motion[i], True), rtol=1e-12, atol=1e-12)
                    f1 = om.resample(snaps["predict_flow2"][k, i:i + 1], fr, fc)
                    valid, epe = om.epe_pixels(f1, flow_gt[i:i + 1])
                    s = om.epe_sums(f1, flow_gt[i:i + 1])[0]
                    b = om.chain_length(gh * gw) * om.U * 1.01 * s[0]
                    assert within(table[14, 0], ((s[0] - b) / s[1], (s[0] + b) / s[1])), (label, i, table[14, 0], s[0] / s[1])
                assert abs(table[15, 0] - norm[i]) <= 1e-6 * norm[i]
