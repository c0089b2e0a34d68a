"""CPU: oracle/metrics.py, the numpy statement of the evaluation metrics, pinned to the reference's own results
(tests/golden/metrics_golden.npz, made by importing the reference's metrics.py under NumPy 2) and to hand-worked cases.
The GPU tests (tests/test_gpu_metrics_oracle.py) then hold csrc/metrics.cu to this oracle pixel by pixel."""
import math
import os

import numpy as np
import pytest

from oracle import metrics as om

NAMES = om.DISTANCES


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "metrics_golden.npz"))


def gt_div_of(t):
    """evaluate_depth's divisor of the ground truth: the float64 translation norm, or None where it is close to 1."""
    norm = np.sqrt(t.dot(t))
    return None if np.isclose(1.0, norm) else np.array([norm])


def assert_matches_golden(sums, want, tag):
    e = om.distances(sums, clamp=False)
    n = int(want[0])
    assert e['num_valid'] == n, tag
    for k, w in zip(NAMES, want[1:]):
        if k.startswith('ratio_threshold'):
            assert round(e[k] * n) == round(w * n), (tag, k, e[k] * n, w * n)      # counts exactly
        else:
            assert abs(e[k] - w) <= 1e-6 * abs(w), (tag, k, e[k], w)


def test_exact_sum_is_fsum():
    rng = np.random.RandomState(0)
    x = (rng.standard_normal((5, 3001)) * np.exp2(rng.randint(-60, 60, (5, 3001)))).astype(np.float32)
    x[0, ::7] = 0
    x[1] = np.float32(1e-45) * rng.randint(-3, 4, 3001)         # subnormals only
    y = rng.standard_normal((3, 257)) * np.exp2(rng.randint(-300, 300, (3, 257)))
    for a in (x, y):
        got = om.exact_sum(a)
        assert got.shape == (a.shape[0],)
        for i in range(a.shape[0]):
            assert got[i] == math.fsum(float(v) for v in a[i])
    assert om.exact_sum(np.zeros((2, 4))).tolist() == [0.0, 0.0]
    big = np.full((1, 70000), np.float32(16777215.0))           # 2^24 - 1 mantissas, many of one exponent
    assert om.exact_sum(big)[0] == 70000 * 16777215.0


@pytest.mark.parametrize("ci", (0, 1, 2))
@pytest.mark.parametrize("scaling", ("abs", "log", "inv"))
def test_nep50_reproduces_golden_evaluate_depth(golden, ci, scaling):
    gt, pred, t = golden["gt_%d" % ci][None], golden["pred_%d" % ci][None], golden["t_%d" % ci]
    gd = gt_div_of(t)
    px = om.depth_pixels(pred, gt, True, True, gd, promotion="nep50")
    sums = om.depth_sums(px, "host")
    assert_matches_golden(sums[0], golden["errs_%d_%s" % (ci, scaling)], (ci, scaling))
    # the reference's scale has the dtype of its operands: float32, or float64 behind a float64 divide
    assert px["dtype"] == (np.float32 if gd is None else np.float64)
    scale = om.scale_factor(sums, scaling).astype(px["dtype"])
    scaled = om.depth_sums(om.depth_pixels(pred, gt, True, True, gd, scale, promotion="nep50"), "host")
    assert_matches_golden(scaled[0], golden["errs_scaled_%d_%s" % (ci, scaling)], (ci, scaling, "scaled"))


@pytest.mark.parametrize("ci", (0, 1, 2))
def test_nep50_reproduces_golden_compute_errors_and_epe(golden, ci):
    px = om.depth_pixels(golden["dpred_%d" % ci][None], golden["dgt_%d" % ci][None], promotion="nep50")
    assert_matches_golden(om.depth_sums(px, "host")[0], golden["errs_plain_%d" % ci], (ci, "plain"))
    s = om.epe_sums(golden["f1_%d" % ci][None], golden["f2_%d" % ci][None])[0]
    want = float(golden["epe_%d" % ci])
    assert abs(s[0] / s[1] - want) <= 1e-6 * want


def golden_cases(golden):
    """(tag, pred, gt, gt_div, scaling or None, inverse) of every compute_errors call behind the golden vectors."""
    for ci in range(3):
        gt, pred, t = golden["gt_%d" % ci][None], golden["pred_%d" % ci][None], golden["t_%d" % ci]
        gd = gt_div_of(t)
        yield (ci, "unscaled"), pred, gt, gd, None, True
        for scaling in ("abs", "log", "inv"):
            yield (ci, scaling), pred, gt, gd, scaling, True
        yield (ci, "plain"), golden["dpred_%d" % ci][None], golden["dgt_%d" % ci][None], None, None, False


def test_legacy_and_nep50_account_for_every_borderline_pixel(golden):
    """Every pixel where the golden (NumPy 2) count and the device's (legacy) count can differ is either ambiguous under
    the device's log bound or one where the two promotion rules disagree.  On these golden vectors both lists are empty:
    no pixel lies within the bound of a threshold, so the device's counts must equal the golden counts exactly."""
    report = []
    for tag, pred, gt, gd, scaling, inverse in golden_cases(golden):
        for k, acc in enumerate(om.threshold_account(pred, gt, inverse, gd, scaling)):
            assert set(acc["unexplained"]) <= set(acc["disagree"]), (tag, k, acc["unexplained"], acc["disagree"])
            report.append((tag, om.THRESHOLDS[k], acc["disagree"].tolist(), acc["ambiguous"].tolist()))
            assert len(acc["disagree"]) == 0 and len(acc["ambiguous"]) == 0, report[-1]
    print("pixels where legacy and NEP 50 disagree / ambiguous under the device bound:",
          ["%s t=%s %s %s" % r for r in report if r[2] or r[3]] or "none")


def test_exact_threshold_ratios():
    """The pairs (t, 1) and (1, t): log(1) = +0 exactly, so |ld| is the float32 log of t itself.  numpy's float32 log
    gives float32(log t) for 1.25 and 1.953125 and one float above it for 1.5625.  Against the float64 log t (NEP 50)
    the pair at 1.25 counts as in, because float32(log 1.25) < log 1.25; against float32(log t) (legacy) no pair counts:
    |ld| < |ld| is false."""
    t = np.array(om.THRESHOLDS, dtype=np.float32)
    pred = np.concatenate([t, np.ones(3, np.float32)])[None]
    gt = np.concatenate([np.ones(3, np.float32), t])[None]
    ld32 = np.abs(np.log(t))
    assert ld32.view(np.uint32).tolist() == [0x3e647fbe, 0x3ee47fbf, 0x3f2b5fcf]
    assert [float(v) < math.log(x) for v, x in zip(om.LEGACY_LOG_T, om.THRESHOLDS)] == [True, True, False]
    nep = om.depth_pixels(pred, gt, promotion="nep50")["terms"]
    leg = om.depth_pixels(pred, gt, promotion="legacy")
    for k in range(3):
        own = [k, 3 + k]                                                     # the pixels whose ratio is t_k itself
        assert nep[9 + k][0][own].tolist() == ([1, 1] if k == 0 else [0, 0]), k
        assert leg["terms"][9 + k][0][own].tolist() == [0, 0], k
        # the device's logf(t) is only known within its bound: the oracle calls these pixels ambiguous, and the GPU
        # test decides them from the device's own ld
        assert leg["thr_amb"][k][0][own].all() and not leg["thr_in"][k][0][own].any()
        # every other pair is decided
        other = [i for i in range(6) if i not in own]
        assert not leg["thr_amb"][k][0][other].any()
        assert leg["thr_in"][k][0][other].tolist() == [om.THRESHOLDS[i % 3] < om.THRESHOLDS[k] for i in other]


def test_zero_variance_scale_invariant_is_clamped():
    """Three pixels with one ratio: the variance of ld is 0, but the reference's float32 sums make it negative and
    scale_invariant NaN.  The device evaluates sqrt(max(0, s4/n - (s3/n)^2)) in double over its sums: 0 here, never
    NaN; demon_b200.evaluation.errors_from_sums is that formula."""
    from demon_b200 import evaluation as ev
    gt = np.full((1, 3), 0.8, np.float32)
    pred = (gt * np.float32(1.1005085)).astype(np.float32)
    ld = np.log(pred[0]) - np.log(gt[0])
    with np.errstate(invalid="ignore"):
        ref = np.sqrt(np.sum(np.square(ld)) / 3.0 - np.square(np.sum(ld)) / np.square(3.0))     # metrics.py:148
    assert np.isnan(ref)
    sums = om.depth_sums(om.depth_pixels(pred, gt), "host")[0]
    assert math.isnan(om.distances(sums, clamp=False)['scale_invariant'])
    assert om.distances(sums)['scale_invariant'] == 0.0 == ev.errors_from_sums(sums)['scale_invariant']


def floats_around(x):
    """The float32 just below and just above each float64 x: both are within 1 ulp of x."""
    f = x.astype(np.float32)
    lo = np.where(f.astype(np.float64) > x, np.nextafter(f, np.float32(-np.inf)), f)
    hi = np.where(f.astype(np.float64) < x, np.nextafter(f, np.float32(np.inf)), f)
    return lo, hi


def test_log_bounds_cover_every_admissible_logf():
    """Any float32 log within 1 ulp (and log10 within 2 ulp) of the exact value, followed by float32 subtractions and
    the square, stays within the oracle's per-pixel bounds; the extreme choices are tried on log-uniform pairs.  (numpy's
    own float32 log is up to about 3.3 ulp off, so it is no stand-in for the device's logf.)"""
    rng = np.random.RandomState(3)
    a = np.exp2(rng.uniform(-30, 30, (1, 100000))).astype(np.float32)
    b = np.exp2(rng.uniform(-30, 30, (1, 100000))).astype(np.float32)
    b[0, :1000] = a[0, :1000] * np.float32(1.25)                   # cancellation: ld near log 1.25
    px = om.depth_pixels(a, b)
    assert px["valid"].all()
    la, lb = floats_around(np.log(a.astype(np.float64))), floats_around(np.log(b.astype(np.float64)))
    ta, tb = np.log10(a.astype(np.float64)), np.log10(b.astype(np.float64))
    for x in la:
        for y in lb:
            ld = x - y
            assert (np.abs(ld.astype(np.float64) - px["ld"]) <= px["ld_err"]).all()
            assert (np.abs((ld * ld).astype(np.float64) - np.square(px["ld"])) <= px["ld2_err"]).all()
    for sa in (-2, 2):
        for sb in (-2, 2):
            x = ta.astype(np.float32) + np.float32(sa / 2) * om.ulp32(ta).astype(np.float32)
            y = tb.astype(np.float32) + np.float32(sb / 2) * om.ulp32(tb).astype(np.float32)
            assert (np.abs(np.abs(x - y).astype(np.float64) - px["l10"]) <= px["l10_err"]).all()


def test_resample_tables():
    pred = np.arange(2 * 3 * 4, dtype=np.float32).reshape(2, 3, 4) + 1
    rows, cols = np.array([2, -1, 0, 0]), np.array([3, 1, -1])
    got = om.resample(pred, rows, cols)
    assert got.shape == (2, 4, 3) and got.dtype == np.float32
    for i in range(2):
        for r in range(4):
            for c in range(3):
                want = 0 if rows[r] < 0 or cols[c] < 0 else pred[i, rows[r], cols[c]]
                assert got[i, r, c] == want


def test_sum_bounds_cover_reordered_sums():
    """The bound L 2^-53 sum|t| holds for the device's reduction order, restated here in float64: strided per-thread
    sums, the warp tree, the CTA's warps and the slots in order."""
    rng = np.random.RandomState(4)
    for hw in (1, 257, 1025, 70000):
        t = (rng.standard_normal(hw) * np.exp2(rng.randint(-20, 20, hw))).astype(np.float32).astype(np.float64)
        ns = om.slots(hw)
        stride = ns * om.THREADS
        slot_sums = []
        for s in range(ns):
            acc = np.zeros(om.THREADS)
            base = s * om.THREADS
            for i in range(base, hw, stride):
                seg = t[i:min(i + om.THREADS, hw)]
                acc[:seg.size] += seg
            warps = acc.reshape(8, 32).copy()
            for o in (16, 8, 4, 2, 1):
                warps = warps + warps[:, np.arange(32) ^ o]
            v = 0.0
            for w in range(8):
                v += warps[w, 0]
            slot_sums.append(v)
        total = 0.0
        for v in slot_sums:
            total += v
        assert abs(total - om.exact_sum(t[None])[0]) <= om.chain_length(hw) * om.U * np.abs(t).sum()
