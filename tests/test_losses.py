"""CPU tests of oracle/losses.py, the numpy restatement of DeMoN v2's training losses the device losses are checked against.

It is pinned to the reference's own python/depthmotionnet/v2/losses.py through tests/golden/losses_golden.npz (written by
tests/golden/make_losses_golden.py from that module, run unmodified in float64): every block, every combination of the
flow block's optional arguments and its key set, at N = 1 and 3 and odd sizes, with NaN / +-inf / 0 in ground truth and
prediction.  Where the reference tree is present (DEMON_REF_SRC) the golden results are regenerated and compared too.
"""
import importlib.util
import os

import numpy as np
import pytest

from oracle import losses as OL
from oracle import losses_ref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _gen():
    spec = importlib.util.spec_from_file_location("make_losses_golden", os.path.join(GOLDEN, "make_losses_golden.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


GEN = _gen()


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(GOLDEN, "losses_golden.npz")))


def _inputs(golden, ci):
    return {k: golden["c%d/in/%s" % (ci, k)] for k in ("depth", "intrinsics", "rotation", "translation")}


@pytest.fixture(scope="module")
def oracle_runs(golden):
    out = {}
    for ci in range(len(GEN.SIZES)):
        inp = _inputs(golden, ci)
        gt = OL.prepare_ground_truth_tensors(inp["depth"], inp["rotation"], inp["translation"], inp["intrinsics"])
        out[ci] = GEN.run(OL, ci, inp, {k: np.asarray(v) for k, v in gt.items()})
    return out


def _close(a, b, rtol=1e-12):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape
    same_nan = np.isnan(a) == np.isnan(b)
    assert same_nan.all()
    ok = np.isnan(a) | (a == b) | (np.abs(a - b) <= rtol * np.abs(b))
    assert ok.all(), "max rel %g" % np.max(np.abs(a - b)[~ok] / np.abs(b)[~ok])


@pytest.mark.parametrize("ci", [0, 1])
def test_ground_truth_equals_reference(golden, oracle_runs, ci):
    for key in ("depth0", "depth0_sig", "depth2", "depth2_sig", "flow0", "flow2", "flow2_sig", "flow5", "normal0", "normal2"):
        assert GEN.digest(oracle_runs[ci]["gt/" + key]) == str(golden["c%d/gt/%s" % (ci, key)]), key


@pytest.mark.parametrize("ci", [0, 1])
@pytest.mark.parametrize("j", range(len(GEN.flow_combos())))
def test_flow_loss_block_equals_reference(golden, oracle_runs, ci, j):
    r = oracle_runs[ci]
    assert list(r["flow%d/keys" % j]) == list(golden["c%d/flow%d/keys" % (ci, j)])
    _close(r["flow%d/values" % j], golden["c%d/flow%d/values" % (ci, j)])


@pytest.mark.parametrize("ci", [0, 1])
@pytest.mark.parametrize("block", ["dn", "refine"])
def test_depth_blocks_equal_reference(golden, oracle_runs, ci, block):
    r = oracle_runs[ci]
    assert list(r[block + "/keys"]) == list(golden["c%d/%s/keys" % (ci, block)])
    _close(r[block + "/values"], golden["c%d/%s/values" % (ci, block)])


@pytest.mark.parametrize("ci", [0, 1])
def test_small_functions_equal_reference(golden, oracle_runs, ci):
    r = oracle_runs[ci]
    _close(r["conf2"], golden["c%d/conf2" % ci], rtol=0)
    _close(r["l1"], golden["c%d/l1" % ci])
    _close(r["l2"], golden["c%d/l2" % ci])
    g = {k[3:]: v for k, v in r.items() if k.startswith("gt/")}
    _close(GEN.sig_loss_value(OL, ci, g), golden["c%d/sig_loss" % ci])


def test_key_sets_follow_the_optional_arguments(golden):
    for j, (c2, c5, fs, cs, _, _, prefix) in enumerate(GEN.flow_combos()):
        keys = {k[len(prefix):] for k in golden["c0/flow%d/keys" % j]}
        want = {"loss_flow5", "loss_flow2", "loss_flow5_unscaled", "loss_flow2_unscaled"}
        if c5:
            want |= {"loss_conf5", "loss_conf5_unscaled"}
        if c2:
            want |= {"loss_conf2", "loss_conf2_unscaled"}
        if fs:
            want |= {"loss_flow2_sig", "loss_flow2_sig_unscaled"}
        if cs and c2:
            want |= {"loss_conf2_sig", "loss_conf2_sig_unscaled"}
        assert keys == want, j


def test_level5_factor_zero_zeroes_the_level5_losses_only(golden):
    j = [i for i, c in enumerate(GEN.flow_combos()) if c[5] == 0.0][0]
    d = dict(zip(golden["c1/flow%d/keys" % j], golden["c1/flow%d/values" % j]))
    assert d["netFlow1_loss_flow5"] == 0 and d["netFlow1_loss_conf5"] == 0
    assert d["netFlow1_loss_flow5_unscaled"] > 0 and d["netFlow1_loss_flow2"] > 0


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_flow_sig_is_2n_rows_of_single_components(dtype):
    rng = np.random.RandomState(1)
    n, h, w = 3, 9, 13
    pr = rng.uniform(-1, 1, (n, 2, h, w)).astype(dtype)
    gt_sig = rng.uniform(-1, 1, (2 * n, 10, h, w)).astype(dtype)
    s = OL.sig_stack(pr, 0.001)
    assert s.shape == (2 * n, 10, h, w)
    # row 2i + c of the stack is the SIG of component c of sample i alone
    for i in range(n):
        for c in range(2):
            assert np.array_equal(s[2 * i + c], OL.sig_stack(pr[i:i + 1, c:c + 1], 0.001)[0])
    t = OL.terms(s, gt_sig, 1e-5)
    assert t.shape == (2 * n, h, w)
    assert OL.pointwise_l2_loss(s, gt_sig, 1e-5) == dtype(np.float64(t.astype(np.float64).sum()) / (2 * n * h * w))


def test_depth_blocks_take_the_prediction_sig_at_0_01():
    rng = np.random.RandomState(2)
    pr = rng.uniform(0.1, 2, (2, 1, 11, 17))
    gt_sig = OL.sig_stack(rng.uniform(0.1, 2, (2, 1, 11, 17)), 0.001)
    r = OL.depth_refine_loss_block(pr, gt_sig, np.zeros((2, 3, 11, 17)), pr, np.zeros((2, 3, 11, 17)), 1.0, 1.0, 1.0)
    assert r["loss_depth0_sig"] == OL.pointwise_l2_loss(OL.sig_stack(pr, 0.01), gt_sig, 1e-5)
    assert r["loss_depth0_sig"] != OL.pointwise_l2_loss(OL.sig_stack(pr, 0.001), gt_sig, 1e-5)


def test_nonfinite_differences_count_as_zero():
    pr = np.array([[[[1.0, np.nan, np.inf, 2.0]]]])
    gt = np.array([[[[1.5, 0.0, 1.0, -np.inf]]]])
    t = OL.terms(pr, gt, 1e-5)
    assert np.array_equal(t, np.sqrt(np.array([[[0.25, 0.0, 0.0, 0.0]]]) + 1e-5))
    np.testing.assert_allclose(OL.pointwise_l2_loss(pr, gt, 1e-5), np.mean(t), rtol=1e-15)
    g = OL.l2_grad(pr, gt, 1e-5)
    assert np.array_equal(g[0, 0, 0, 1:], [0.0, 0.0, 0.0])


def _numeric(f, x, h=1e-6):
    g = np.zeros_like(x)
    for i in range(x.size):
        xp, xm = x.copy(), x.copy()
        xp.flat[i] += h
        xm.flat[i] -= h
        g.flat[i] = (f(xp) - f(xm)) / (2 * h)
    return g


def test_oracle_gradients_match_finite_differences():
    rng = np.random.RandomState(3)
    pr = rng.uniform(0.2, 2, (2, 1, 5, 19))
    gt = rng.uniform(0.2, 2, (2, 1, 5, 19))
    gt_sig = OL.sig_stack(gt, 0.001)
    g = OL.sig_loss_grad(pr, gt_sig, 1e-5, 0.01, 2.0)
    num = _numeric(lambda x: 2.0 * OL.pointwise_l2_loss(OL.sig_stack(x, 0.01), gt_sig, 1e-5), pr)
    np.testing.assert_allclose(g, num, rtol=1e-5, atol=1e-9)
    n = rng.uniform(-1, 1, (2, 3, 4, 5))
    gn = rng.uniform(-1, 1, (2, 3, 4, 5))
    np.testing.assert_allclose(OL.l2_grad(n, gn, 1e-5, 0.5), _numeric(lambda x: 0.5 * OL.pointwise_l2_loss(x, gn, 1e-5), n),
                               rtol=1e-5, atol=1e-9)
    x = rng.uniform(-1, 1, (3, 3))
    np.testing.assert_allclose(OL.l1_grad(x, 1e-5, 3.0), _numeric(lambda v: 3.0 * OL.l1_loss(v, 1e-5), x), rtol=1e-5, atol=1e-9)


@pytest.mark.skipif(losses_ref.load() is None, reason="the reference tree (DEMON_REF_SRC) is absent")
@pytest.mark.parametrize("ci", [0, 1])
def test_regenerated_reference_results_equal_the_golden_file(golden, ci):
    ref = losses_ref.load()
    r = GEN.run(ref, ci, _inputs(golden, ci))
    for k, v in r.items():
        if k.startswith("gt/"):
            assert GEN.digest(v) == str(golden["c%d/%s" % (ci, k)]), k
        elif not k.startswith("pr/"):
            assert np.array_equal(np.asarray(v), golden["c%d/%s" % (ci, k)], equal_nan=v.dtype.kind == "f"), k
