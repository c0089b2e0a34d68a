"""CPU tests of oracle/loss_grads.py, the kernel-order restatement of the loss gradient kernels (csrc/losses.cu) that
tests/test_gpu_loss_grads.py holds the device to bit for bit.

In float64 the restatement must agree with the independent float64 gradients of oracle/losses.py (l2_grad, l1_grad,
sig_loss_grad; themselves checked against finite differences in tests/test_losses.py) to about 1e-13 of each element's
own magnitude.  In float32 it must lie, element by element, within the first-order error bound that oracle/loss_grads.py
derives from its operation sequence (l2_grad_bound, l1_grad_bound, sig_grad_bound).  Cases: odd and tile-straddling
plane sizes, NaN and +-inf in prediction, target and neighbours, and targets so close to the prediction that d cancels.
"""
import numpy as np
import pytest

from oracle import loss_grads as LG
from oracle import losses as OL

U = 2.0 ** -24
SHAPES = [(1, 1, 1, 1), (2, 1, 17, 65), (3, 1, 33, 129), (2, 2, 15, 63), (1, 1, 16, 64), (2, 1, 1, 40), (1, 2, 23, 1)]


def _poison(rng, a, frac=0.03):
    m = rng.rand(*a.shape)
    a = a.copy()
    a[m < frac / 3] = np.nan
    a[(m >= frac / 3) & (m < 2 * frac / 3)] = np.inf
    a[(m >= 2 * frac / 3) & (m < frac)] = -np.inf
    return a


def _sig_case(shape, seed, mode):
    """(pr [..,H,W], target, gt_plane) in float64 holding float32 values.  mode 'stack': an unrelated target stack; 'close':
    the target is the SIG of the prediction plus 1e-4 noise, so d cancels; 'plane': a target plane taken on the fly."""
    rng = np.random.RandomState(seed)
    pr = rng.uniform(-2, 2, shape)
    pr[np.abs(pr) < 0.05] = 0.0
    pr = _poison(rng, pr).astype(np.float32).astype(np.float64)
    planes = pr.reshape((-1,) + shape[-2:])
    if mode == "plane":
        return pr, _poison(rng, rng.uniform(-2, 2, shape)).astype(np.float32).astype(np.float64), True
    if mode == "close":
        st = OL.sig_stack(planes.astype(np.float32), 0.01) + rng.normal(0, 1e-4, (planes.shape[0], 10) + shape[-2:]).astype(np.float32)
    else:
        st = OL.sig_stack(_poison(rng, rng.uniform(-2, 2, planes.shape)).astype(np.float32), 0.001)
    return pr, _poison(rng, st, 0.01).astype(np.float32).astype(np.float64), False


def _l2_case(shape, seed, close=False):
    rng = np.random.RandomState(seed)
    if close:   # large values a few ulp apart: d cancels
        pr = 1e4 + rng.uniform(-1, 1, shape)
        gt = (pr.astype(np.float32) + rng.randint(-3, 4, shape) * np.spacing(np.float32(1e4))).astype(np.float64)
    else:
        pr, gt = rng.normal(0, 1, shape), rng.normal(0, 1, shape)
    pr, gt = _poison(rng, pr), _poison(rng, gt)
    return pr.astype(np.float32).astype(np.float64), gt.astype(np.float32).astype(np.float64)


def _per_element(got, want, scale, rtol):
    """max |got - want| / (rtol * scale) over the elements; got is 0 exactly where scale is 0."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert np.isfinite(got).all() and np.isfinite(want).all()
    err = np.abs(got - want)
    zero = scale == 0
    assert (err[zero] == 0).all()
    return float((err[~zero] / (rtol * scale[~zero])).max()) if (~zero).any() else 0.0


SIG_CASES = [(s, m) for s in SHAPES for m in ("stack", "close", "plane")]


@pytest.mark.parametrize("shape,mode", SIG_CASES)
def test_float64_sig_restatement_equals_the_independent_oracle(shape, mode):
    pr, tgt, gt_plane = _sig_case(shape, sum(shape), mode)
    s_eps = LG.sig_eps(0.01)
    scale = 0.75 * 1500.0
    t = LG.Term(LG.SIG, 0, tgt, LG.EPS, 1500.0, s_eps, gt_plane=gt_plane, gt_s_eps=LG.sig_eps(0.001))
    got = LG.term_grad(t, pr, 0.75)
    stack = OL.sig_stack(tgt.reshape((-1,) + shape[-2:]), LG.sig_eps(0.001)) if gt_plane else tgt
    want = OL.sig_loss_grad(pr, stack, LG.EPS, s_eps, scale)
    planes = pr.reshape((-1,) + shape[-2:])
    _, _, mag = LG.sig_grad_bound(planes, tgt, LG.EPS, s_eps, scale, gt_plane, LG.sig_eps(0.001))
    assert _per_element(got, want, mag.reshape(shape), 1e-13) <= 1.0


@pytest.mark.parametrize("shape", [(32, 2, 6, 8), (2, 3, 17, 65), (3, 1, 33, 129), (1, 10, 7, 5)])
@pytest.mark.parametrize("close", [False, True])
def test_float64_l2_and_l1_restatements_equal_the_independent_oracle(shape, close):
    pr, gt = _l2_case(shape, sum(shape) + close, close)
    got = LG.term_grad(LG.Term(LG.L2, 0, gt, LG.EPS, 300.0), pr, -1.25)
    want = OL.l2_grad(pr, gt, LG.EPS, -1.25 * 300.0)
    assert _per_element(got, want, np.abs(want), 1e-13) <= 1.0
    x, xg = pr.reshape(shape[0], -1)[:, :3], gt.reshape(shape[0], -1)[:, :3]
    x, xg = np.where(np.isfinite(x), x, 0.5), np.where(np.isfinite(xg), xg, -0.5)
    got = LG.term_grad(LG.Term(LG.L1, 0, xg, LG.EPS, 160.0 / shape[0]), x, 0.75)
    want = OL.l1_grad(x - xg, LG.EPS, 0.75 * (160.0 / shape[0]))
    assert _per_element(got, want, np.abs(want), 1e-13) <= 1.0


def _ratio(got32, want, bound):
    err = np.abs(np.asarray(got32, np.float64) - want)
    assert np.isfinite(got32).all()
    zero = bound == 0
    assert (err[zero] == 0).all()
    r = float((err[~zero] / bound[~zero]).max()) if (~zero).any() else 0.0
    g = float(err.max() / (U * np.abs(want).max())) if np.abs(want).max() > 0 else 0.0
    return r, g


@pytest.mark.parametrize("shape,mode", SIG_CASES)
def test_float32_sig_gradient_within_its_per_element_bound(shape, mode):
    pr, tgt, gt_plane = _sig_case(shape, sum(shape), mode)
    s_eps = LG.sig_eps(0.01)
    t = LG.Term(LG.SIG, 0, tgt.astype(np.float32), LG.EPS, 1500.0, s_eps, gt_plane=gt_plane, gt_s_eps=LG.sig_eps(0.001))
    got = LG.term_grad(t, pr.astype(np.float32), -1.25)
    assert got.dtype == np.float32
    planes = pr.reshape((-1,) + shape[-2:])
    bound, want, _ = LG.sig_grad_bound(planes, tgt, LG.EPS, s_eps, -1.25 * 1500.0, gt_plane, LG.sig_eps(0.001))
    stack = OL.sig_stack(tgt.reshape(planes.shape), LG.sig_eps(0.001)) if gt_plane else tgt
    indep = OL.sig_loss_grad(pr, stack, LG.EPS, s_eps, -1.25 * 1500.0).reshape(planes.shape)
    np.testing.assert_allclose(want, indep, rtol=1e-9, atol=1e-12 * np.abs(indep).max())
    r, g = _ratio(got.reshape(planes.shape), indep, bound)
    print("SIG %s %s: largest err/bound %.3f, err/(u max|g|) %.2f" % (shape, mode, r, g))
    assert r <= 1.0


@pytest.mark.parametrize("shape,s_eps,gt_plane", [((32, 1, 192, 256), 0.01, False), ((32, 2, 48, 64), 0.001, False),
                                                   ((32, 2, 48, 64), 0.001, True)], ids=["depth0", "flow2", "conf2"])
def test_float32_sig_gradient_within_its_bound_at_training_shapes(shape, s_eps, gt_plane):
    """depth0 SIG [32,1,192,256], flow2 SIG on 64 planes of 48x64, and the confidence SIG against a target plane."""
    rng = np.random.RandomState(sum(shape))
    pr = _poison(rng, rng.uniform(0.2, 2, shape)).astype(np.float32)
    planes = pr.reshape((-1,) + shape[-2:])
    if gt_plane:
        tgt = rng.uniform(0.05, 1, shape).astype(np.float32)
    else:
        tgt = _poison(rng, OL.sig_stack(np.abs(planes + rng.normal(0, 0.05, planes.shape).astype(np.float32)), 0.001), 0.01)
    se = LG.sig_eps(s_eps)
    got = LG.term_grad(LG.Term(LG.SIG, 0, tgt, LG.EPS, 1500.0, se, gt_plane=gt_plane, gt_s_eps=se), pr, -1.25)
    bound, _, _ = LG.sig_grad_bound(planes.astype(np.float64), tgt.astype(np.float64), LG.EPS, se, -1.25 * 1500.0, gt_plane, se)
    stack = OL.sig_stack(tgt.reshape(planes.shape), se) if gt_plane else tgt
    want = OL.sig_loss_grad(pr.astype(np.float64), stack.astype(np.float64), LG.EPS, se, -1.25 * 1500.0).reshape(planes.shape)
    r, g = _ratio(got.reshape(planes.shape), want, bound)
    print("SIG %s: largest err/bound %.3f, err/(u max|g|) %.2f" % (shape, r, g))
    assert r <= 1.0


@pytest.mark.parametrize("shape", [(32, 2, 6, 8), (2, 3, 17, 65), (3, 1, 33, 129), (1, 10, 7, 5), (32, 3, 192, 256)])
@pytest.mark.parametrize("close", [False, True])
def test_float32_l2_and_l1_gradients_within_their_per_element_bounds(shape, close):
    pr, gt = _l2_case(shape, sum(shape) + close, close)
    got = LG.term_grad(LG.Term(LG.L2, 0, gt.astype(np.float32), LG.EPS, 0.5 * 1.7), pr.astype(np.float32), 0.75)
    bound, _ = LG.l2_grad_bound(pr, gt, LG.EPS, 0.75 * 0.5 * 1.7)
    r, g = _ratio(got, OL.l2_grad(pr, gt, LG.EPS, 0.75 * 0.5 * 1.7), bound)
    print("L2 %s: largest err/bound %.3f, err/(u max|g|) %.2f" % (shape, r, g))
    assert r <= 1.0
    x = np.where(np.isfinite(pr), pr, 0.25).reshape(shape[0], -1)[:, :3]
    got = LG.term_grad(LG.Term(LG.L1, 0, None, LG.EPS, 15.0 / shape[0]), x.astype(np.float32), -1.25)
    bound, _ = LG.l1_grad_bound(x, LG.EPS, -1.25 * (15.0 / shape[0]))
    r, _ = _ratio(got, OL.l1_grad(x, LG.EPS, -1.25 * (15.0 / shape[0])), bound)
    assert r <= 1.0


def test_gather_adds_every_delta_even_without_a_pair():
    """A plane narrower and lower than a delta still adds that delta's tmp = +0, which turns a -0 sum into +0."""
    x = np.array([[[1.0, 2.0]]], np.float32)
    U0 = np.zeros((1, 10, 1, 2), np.float32)
    U0[0, 0, 0, 0] = -0.0
    g = LG.sig_gather(x, U0, LG.sig_eps(0.01))
    assert g.dtype == np.float32 and not np.signbit(g).any()


def _block_inputs(seed, dtype, n=2, h=17, w=21):
    rng = np.random.RandomState(seed)

    def a(*s, lo=-1.0, hi=1.0, bad=True):
        v = rng.uniform(lo, hi, s)
        return (_poison(rng, v, 0.02) if bad else v).astype(dtype)
    return a, n, h, w


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_block_tables_equal_the_oracle_gradients_summed(dtype):
    """The block helpers' term tables (which prediction, which target, which weight) against oracle/losses.py's float64
    gradients of the same losses summed: 1e-13 of the element's magnitude in float64, the float32 bounds in float32."""
    a, n, h, w = _block_inputs(11, dtype)
    f64 = np.float64
    tol = 1e-12 if dtype == np.float64 else 3e-5
    up = {"loss_flow5": 0.75, "loss_flow2": -1.25, "loss_conf5": 0.5, "loss_conf2": 1.5, "loss_flow2_sig": -0.75, "loss_conf2_sig": 1.25}
    gf2, gf5, f2, f5 = a(n, 2, h, w), a(n, 2, 3, 4), a(n, 2, h, w), a(n, 2, 3, 4)
    c2, c5 = a(n, 2, h, w, lo=0.05, bad=False), a(n, 2, 3, 4, lo=0.05, bad=False)
    gsig = OL.sig_stack(a(2 * n, 1, h, w), 0.001)
    kw = dict(flow_weight=1.7, conf_weight=0.3, flow_sig_weight=2.5, conf_sig_weight=0.8)
    got = LG.flow_block_grads(gf2, gf5, gsig, f2, f5, c2, c5, upstream=up, conf_diff_scale=10, level5_factor=0.25, **kw)
    conf2, conf5 = OL.compute_confidence_map(f2, gf2, 10), OL.compute_confidence_map(f5, gf5, 10)
    want = {"pr_flow5": OL.l2_grad(f5, gf5, 1e-5, 0.75 * 0.25 * 1.7),
            "pr_flow2": OL.l2_grad(f2, gf2, 1e-5, -1.25 * 1.7) + OL.sig_loss_grad(f2, gsig, 1e-5, 0.001, -0.75 * 2.5),
            "pr_conf5": OL.l2_grad(c5, conf5, 1e-5, 0.5 * 0.25 * 0.3),
            "pr_conf2": OL.l2_grad(c2, conf2, 1e-5, 1.5 * 0.3)
            + OL.sig_loss_grad(c2, OL.sig_stack(conf2.astype(f64), 0.001), 1e-5, 0.001, 1.25 * 0.8)}
    assert sorted(got) == sorted(want)
    for k in want:
        assert got[k].dtype == dtype
        np.testing.assert_allclose(got[k], want[k], rtol=tol, atol=tol * np.abs(want[k]).max(), err_msg=k)
    up = {"loss_depth2": 0.75, "loss_depth2_sig": -1.25, "loss_normal2": 0.5, "loss_rotation": 1.5, "loss_translation": -0.75,
          "loss_translation_no_factor": 0.25}
    gd, d, gn, nn = a(n, 1, h, w, lo=0.1, hi=2), a(n, 1, h, w, lo=0.1, hi=2), a(n, 3, h, w), a(n, 3, h, w)
    gr, r, gt_, t_ = a(n, 3, bad=False), a(n, 3, bad=False), a(n, 3, bad=False), a(n, 3, bad=False)
    dsig = OL.sig_stack(gd, 0.001)
    got = LG.depthnormal_block_grads(gd, dsig, gn, gr, gt_, d, nn, r, t_, 300.0, 1500.0, 50.0, 160.0, 15.0, 1.3, up)
    want = {"pr_depth2": OL.l2_grad(d, gd, 1e-5, 0.75 * 300.0) + OL.sig_loss_grad(d, dsig, 1e-5, 0.01, -1.25 * 1500.0),
            "pr_normal2": OL.l2_grad(nn, gn, 1e-5, 0.5 * 50.0),
            "pr_rotation": OL.l1_grad(r.astype(f64) - gr, 1e-5, 1.5 * 160.0 / n),
            "pr_translation": OL.l1_grad(t_.astype(f64) - gt_, 1e-5, (0.25 + -0.75 * 1.3) * 15.0 / n)}
    for k in want:
        np.testing.assert_allclose(got[k], want[k], rtol=tol, atol=tol * np.abs(want[k]).max(), err_msg=k)
    up = {"loss_depth0": 0.75, "loss_depth0_sig": -1.25}   # loss_normal0 unused: its upstream reads as 0
    got = LG.depth_refine_block_grads(gd, dsig, gn, d, nn, 300.0, 1500.0, 100.0, up)
    want = OL.l2_grad(d, gd, 1e-5, 0.75 * 300.0) + OL.sig_loss_grad(d, dsig, 1e-5, 0.01, -1.25 * 1500.0)
    np.testing.assert_allclose(got["pr_depth0"], want, rtol=tol, atol=tol * np.abs(want).max())
    assert (got["pr_normal0"] == 0).all()


def test_weights_round_once_to_the_precision():
    """gs = g * T(w): a Python weight product such as level5_factor * flow_weight rounds once, like _Spec does."""
    assert LG.grad_scale(0.75, 0.3 * 1.7, np.float32) == np.float32(0.75) * np.float32(0.3 * 1.7)
    assert np.float32(0.3 * 1.7) != np.float32(0.3) * np.float32(1.7)
    assert LG.grad_scale(None, -3.0, np.float32) == 0 and np.signbit(LG.grad_scale(None, -3.0, np.float32))
    assert LG.grad_scale(-1.25, 160.0 / 32, np.float64) == -1.25 * 5.0
