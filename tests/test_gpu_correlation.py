"""GPU: correlation, correlation_1d and their gradients (csrc/correlation.cu) bit for bit against the reference's own CUDA
kernels (oracle/correlation_ref.py: oracle/_ref/libref_correlation.so, or the digests it recorded in
tests/golden/correlation_digests.json), NaN positions included, and against the float64 oracle (oracle/correlation.py)
for single_dir = -1, where the reference reads out of bounds and is never run.

Every row of ROWS runs the forward op and both gradients through the C ABI into outputs filled with SENTINEL (so an element
no kernel writes fails the comparison) and must launch three kernels.  Which ones is shown by a torch.profiler trace for four
small rows that reach all eight kernels of the file (the forward kernel's instantiation follows from the top width: 64
pixels per CTA above 32, else 32), taken in a child process so that this process starts no trace.
"""
import collections
import os
import re
import sys

import numpy as np
import pytest
import torch
from torch.profiler import ProfilerActivity, profile

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import correlation as oc
from oracle import correlation_ref as cref
from oracle.ref import Recorded, digest

SENTINEL = -1.5e38
CT = {"mult": 1, "subt": 2}
EPS = float(np.finfo(np.float32).eps)

# (name, one_d, shape, attrs, non-finite inputs)
ROWS = [
    ("flownetc_b2", False, (2, 256, 48, 64), dict(max_displacement=20, kernel_size=1, stride1=1, stride2=2, pad_size=20), False),
    ("dispnet_1d_md40", True, (1, 256, 48, 64), dict(max_displacement=40, kernel_size=1, stride1=1, stride2=1, pad_size=40), False),
    ("k3_s1_2", False, (2, 16, 21, 26), dict(max_displacement=4, kernel_size=3, stride1=2, stride2=1, pad_size=4), False),
    ("k3_s1_2_1d", True, (2, 16, 21, 26), dict(max_displacement=4, kernel_size=3, stride1=2, stride2=1, pad_size=4), False),
    ("md5_s2_2", False, (1, 8, 17, 40), dict(max_displacement=5, kernel_size=1, stride1=1, stride2=2, pad_size=5), False),
    ("md5_s2_2_1d", True, (1, 8, 17, 40), dict(max_displacement=5, kernel_size=1, stride1=1, stride2=2, pad_size=5), False),
    ("pad0", False, (1, 8, 16, 20), dict(max_displacement=3, kernel_size=1, stride1=1, stride2=1, pad_size=0), False),
    ("pad0_1d", True, (1, 8, 16, 20), dict(max_displacement=3, kernel_size=1, stride1=1, stride2=1, pad_size=0), False),
    ("c1", False, (1, 1, 12, 14), dict(max_displacement=2, kernel_size=1, stride1=1, stride2=1, pad_size=2), False),
    ("c3_1d", True, (1, 3, 12, 14), dict(max_displacement=2, kernel_size=3, stride1=1, stride2=1, pad_size=2), False),
    ("c33", False, (1, 33, 12, 40), dict(max_displacement=2, kernel_size=1, stride1=1, stride2=1, pad_size=2), False),
    ("c70_k3", False, (1, 70, 12, 14), dict(max_displacement=2, kernel_size=3, stride1=1, stride2=1, pad_size=2), False),
    ("c70_1d", True, (1, 70, 12, 40), dict(max_displacement=2, kernel_size=1, stride1=1, stride2=1, pad_size=2), False),
    ("top1x1", False, (1, 4, 5, 5), dict(max_displacement=2, kernel_size=1, stride1=1, stride2=1, pad_size=0), False),
    ("top1x1_k3", False, (1, 4, 7, 7), dict(max_displacement=2, kernel_size=3, stride1=1, stride2=1, pad_size=0), False),
    ("batch3", False, (3, 32, 10, 12), dict(max_displacement=3, kernel_size=1, stride1=1, stride2=1, pad_size=3), False),
    ("batch3_1d", True, (3, 32, 10, 12), dict(max_displacement=3, kernel_size=1, stride1=1, stride2=1, pad_size=3), False),
    ("nonfinite", False, (2, 40, 12, 36), dict(max_displacement=3, kernel_size=1, stride1=1, stride2=1, pad_size=2), True),
    ("nonfinite_k3_1d", True, (2, 40, 12, 16), dict(max_displacement=3, kernel_size=3, stride1=1, stride2=1, pad_size=2), True),
]
CASES = [(r, ct, sd) for r in ROWS for ct in ("mult", "subt") for sd in ((0, 1) if r[1] else (0,))]


@pytest.fixture(scope="module")
def ops():
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    from demon_b200 import lmbspecialops
    return lmbspecialops


@pytest.fixture(scope="module")
def lib(ops):
    from demon_b200 import _lib
    return _lib.load()


@pytest.fixture(scope="module")
def reference():
    if not cref.available():
        pytest.fail("neither oracle/_ref/libref_correlation.so nor tests/golden/correlation_digests.json is present")
    return cref


# ---- which kernels ran ----------------------------------------------------------------------------------------------------
_KERNEL_NAME = re.compile(r"demon::(?:\(anonymous namespace\)::)?(\w+(?:<[^()]*>)?)\(")


def traced(fn):
    """fn() under torch.profiler -> (result, Counter of the library's kernels, number of other device activities)"""
    prof = profile(activities=[ProfilerActivity.CUDA])
    with prof:
        out = fn()
        torch.cuda.synchronize()
    ours, other = collections.Counter(), 0
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            m = _KERNEL_NAME.search(e.name)
            if m:
                ours[m.group(1).replace(" ", "")] += 1
            else:
                other += 1
    return out, ours, other


# ---- inputs and calls -----------------------------------------------------------------------------------------------------
def make_inputs(shape, seed, special):
    rng = np.random.RandomState(seed)
    x1 = rng.randn(*shape).astype(np.float32)
    x2 = rng.randn(*shape).astype(np.float32)
    if special:
        vals = np.array([np.nan, np.inf, -np.inf, -0.0, 3e38, -3e38], np.float32)
        for x in (x1, x2):
            m = rng.rand(*shape) < 0.01
            x[m] = vals[rng.randint(0, len(vals), m.sum())]
    return x1, x2, rng


def sentinel(shape):
    return torch.full(tuple(shape), SENTINEL, dtype=torch.float32, device="cuda")


def abi_forward(lib, one_d, x1, x2, attrs, ct, sd, top_shape):
    a, b = torch.from_numpy(x1).cuda(), torch.from_numpy(x2).cuda()
    out = sentinel(top_shape)
    n, c, h, w = x1.shape
    args = [a.data_ptr(), b.data_ptr(), out.data_ptr(), n, c, h, w, CT[ct], attrs["kernel_size"], attrs["max_displacement"],
            attrs["stride1"], attrs["stride2"], attrs["pad_size"], 0]
    stream = torch.cuda.current_stream().cuda_stream
    rc = lib.demon_correlation_1d_f32(*args, sd, stream) if one_d else lib.demon_correlation_f32(*args, stream)
    assert rc == 0, lib.demon_last_error()
    return out


def abi_grad(lib, one_d, x1, x2, gt, attrs, ct, sd):
    a, b, g = (torch.from_numpy(v).cuda() for v in (x1, x2, gt))
    g1, g2 = sentinel(x1.shape), sentinel(x2.shape)
    n, c, h, w = x1.shape
    args = [a.data_ptr(), b.data_ptr(), g.data_ptr(), g1.data_ptr(), g2.data_ptr(), n, c, h, w, CT[ct], attrs["kernel_size"],
            attrs["max_displacement"], attrs["stride1"], attrs["stride2"], attrs["pad_size"], 0]
    stream = torch.cuda.current_stream().cuda_stream
    rc = lib.demon_correlation_1d_grad_f32(*args, sd, stream) if one_d else lib.demon_correlation_grad_f32(*args, stream)
    assert rc == 0, lib.demon_last_error()
    return g1, g2


def assert_bits(ours, ref, what):
    if isinstance(ref, Recorded):
        assert ref.matches(ours), "%s: differs from the reference kernel's stored digest" % what
        return
    assert ours.shape == ref.shape, what
    if digest(ours) != digest(ref):
        bad = ~((ours == ref) | (np.isnan(ours) & np.isnan(ref))) | (np.signbit(ours) != np.signbit(ref)) & ~np.isnan(ref)
        idx = np.argwhere(bad)
        raise AssertionError("%s: %d of %d elements differ from the reference kernel, first at %s: %r vs %r" % (
            what, len(idx), ours.size, tuple(idx[0]), ours[tuple(idx[0])], ref[tuple(idx[0])]))


# ---- bit equality with the reference's kernels ----------------------------------------------------------------------------
def case_data(ops, row, sd):
    name, one_d, shape, attrs, special = row
    x1, x2, rng = make_inputs(shape, 11, special)
    top_shape = ops.correlation_top_shape(shape, attrs["max_displacement"], attrs["kernel_size"], attrs["stride1"],
                                          attrs["stride2"], attrs["pad_size"], one_d, sd)
    gt = rng.randn(*top_shape).astype(np.float32)
    if special:
        m = rng.rand(*top_shape) < 0.01
        gt[m] = np.array([np.nan, np.inf, -np.inf], np.float32)[rng.randint(0, 3, m.sum())]
    return x1, x2, gt, top_shape


@pytest.fixture(scope="module")
def reference_results(ops, reference):
    """(forward, input1_grad, input2_grad) of the reference for every case"""
    calls = []
    for row, ct, sd in CASES:
        name, one_d, shape, attrs, special = row
        x1, x2, gt, _ = case_data(ops, row, sd)
        if one_d:
            kw = dict(attrs, corr_type=ct, single_dir=sd)
            calls += [("correlation_1d", (x1, x2), kw), ("correlation_1d_grad", (gt, x1, x2), kw)]
        else:
            kw = dict(attrs, corr_type=ct)
            calls += [("correlation", (x1, x2), kw), ("correlation_grad", (gt, x1, x2), kw)]
    results = [getattr(reference, name)(*args, **kwargs) for name, args, kwargs in calls]
    return {(row[0], ct, sd): (results[2 * i],) + tuple(results[2 * i + 1]) for i, (row, ct, sd) in enumerate(CASES)}


def test_reference_forward_is_deterministic(reference):
    """CorrelateData reads the lane partials without a barrier after the warp reconverges; its bits are a valid bar only if
    two identical calls agree."""
    if not reference.have_library():
        pytest.skip("needs oracle/_ref/libref_correlation.so (the stored digests were recorded from it)")
    x1, x2, _ = make_inputs((2, 256, 48, 64), 5, False)
    flownetc = dict(max_displacement=20, kernel_size=1, stride1=1, stride2=2, pad_size=20)
    dispnet = dict(max_displacement=40, kernel_size=1, pad_size=40)
    rec = os.environ.pop("DEMON_REF_RECORD", None)   # inputs of their own: nothing to store
    try:
        a, b = (reference.correlation(x1, x2, **flownetc) for _ in range(2))
        c, d = (reference.correlation_1d(x1, x2, **dispnet) for _ in range(2))
    finally:
        if rec is not None:
            os.environ["DEMON_REF_RECORD"] = rec
    assert digest(a) == digest(b), "two identical reference Correlation calls differ in %d elements" % int((a != b).sum())
    assert digest(c) == digest(d), "two identical reference Correlation1D calls differ in %d elements" % int((c != d).sum())


def run_abi(lib, row, ct, sd, x1, x2, gt, top_shape):
    """forward and both gradients through the C ABI into SENTINEL-filled outputs -> numpy arrays"""
    name, one_d, shape, attrs, special = row
    out = abi_forward(lib, one_d, x1, x2, attrs, ct, sd, top_shape)
    g1, g2 = abi_grad(lib, one_d, x1, x2, gt, attrs, ct, sd)
    return out.cpu().numpy(), g1.cpu().numpy(), g2.cpu().numpy()


def check_bits(reference_results, row, ct, sd, out, g1, g2):
    name = row[0]
    r_out, r_g1, r_g2 = reference_results[(name, ct, sd)]
    assert_bits(out, r_out, name + " forward")
    assert_bits(g1, r_g1, name + " input1_grad")
    assert_bits(g2, r_g2, name + " input2_grad")


@pytest.mark.parametrize("row,ct,sd", CASES, ids=["%s-%s-sd%d" % (r[0], ct, sd) for r, ct, sd in CASES])
def test_bits_equal_reference(ops, lib, reference_results, row, ct, sd):
    name, one_d, shape, attrs, special = row
    x1, x2, gt, top_shape = case_data(ops, row, sd)
    n0 = lib.demon_launch_count()
    out, g1, g2 = run_abi(lib, row, ct, sd, x1, x2, gt, top_shape)
    assert lib.demon_launch_count() - n0 == 3, "one forward and two gradient kernels"
    check_bits(reference_results, row, ct, sd, out, g1, g2)

    # the mirror: numpy in, numpy out, the same bits
    attrs_sd = dict(attrs, single_dir=sd) if one_d else attrs
    fn = ops.correlation_1d if one_d else ops.correlation
    gn = ops.correlation_1d_grad if one_d else ops.correlation_grad
    m_out = fn(x1, x2, corr_type=ct, **attrs_sd)
    assert isinstance(m_out, np.ndarray) and digest(m_out) == digest(out)
    m_g1, m_g2 = gn(gt, x1, x2, corr_type=ct, **attrs_sd)
    assert digest(m_g1) == digest(g1) and digest(m_g2) == digest(g2)


# rows of CASES whose top widths (40 and 14) select the two forward tilings, in both modes: together every kernel of the file
VARIANT_ROWS = [(r, ct, 0) for r in ROWS if r[0] in ("md5_s2_2", "pad0") for ct in ("mult", "subt")]


def trace_variant_rows(out_path):
    """child process: every VARIANT_ROWS row under its own torch.profiler trace -> pickle of (probe kernels, [(kernels,
    outputs)])"""
    import pickle
    from demon_b200 import _lib
    from demon_b200 import lmbspecialops
    lib = _lib.load()
    _, _, probe = traced(lambda: torch.ones(4096, device="cuda").mul_(3.0))
    rows = []
    for row, ct, sd in VARIANT_ROWS:
        x1, x2, gt, top_shape = case_data(lmbspecialops, row, sd)
        outs, kernels, _ = traced(lambda: run_abi(lib, row, ct, sd, x1, x2, gt, top_shape))
        rows.append((dict(kernels), outs))
    with open(out_path, "wb") as f:
        pickle.dump((probe, rows), f)


def test_rows_run_the_kernels_they_name_and_reach_every_instantiation(ops, reference_results, tmp_path):
    """a torch.profiler trace per row: exactly the forward instantiation its top width selects and the two gradient kernels
    of its mode, with the reference's bits; the rows together run all eight kernels of csrc/correlation.cu.  The traces run in
    a child process: a process that keeps running GPU work after a trace loses the CUDA records of later traces, which the
    test modules after this one need."""
    import pickle
    import subprocess
    import sys
    out = str(tmp_path / "traces.pkl")
    flags = ["-s"] if sys.flags.no_user_site else []
    subprocess.run([sys.executable] + flags + [__file__, out], check=True)
    with open(out, "rb") as f:
        probe, rows = pickle.load(f)
    assert probe > 0, "torch.profiler recorded no CUDA kernel of a probe torch op here, so the paths cannot be checked"
    seen = collections.Counter()
    for (row, ct, sd), (kernels, (o, g1, g2)) in zip(VARIANT_ROWS, rows):
        top_w = o.shape[3]
        subt = "true" if ct == "subt" else "false"
        want = {"correlation_fwd_kernel<%s,%d>" % (subt, 2 if top_w > 32 else 1): 1,
                "correlation_grad_kernel<%s,false>" % subt: 1, "correlation_grad_kernel<%s,true>" % subt: 1}
        assert kernels == want, "%s-%s: launched %s, must launch %s" % (row[0], ct, kernels, want)
        check_bits(reference_results, row, ct, sd, o, g1, g2)
        seen.update(kernels)
    every = {"correlation_fwd_kernel<%s,%d>" % (s, p) for s in ("false", "true") for p in (1, 2)}
    every |= {"correlation_grad_kernel<%s,%s>" % (s, t) for s in ("false", "true") for t in ("false", "true")}
    assert set(seen) == every, "rows ran %s, the file has %s" % (sorted(seen), sorted(every))


# ---- single_dir = -1: the float64 oracle ----------------------------------------------------------------------------------
LEFT = [
    ((2, 16, 9, 30), dict(max_displacement=4, kernel_size=1, stride1=1, stride2=1, pad_size=4)),
    ((1, 40, 11, 28), dict(max_displacement=5, kernel_size=3, stride1=2, stride2=2, pad_size=1)),
    ((2, 7, 6, 50), dict(max_displacement=3, kernel_size=1, stride1=1, stride2=1, pad_size=0)),
]


def _bounds(x1, x2, gt, attrs, ct):
    """float32 error bounds: (terms + 2) eps times the sum of the absolute terms, over K K C, plus a rounding of the result"""
    kw = dict(one_d=True, single_dir=-1, normalize=False, **attrs)
    if ct == "mult":
        f_abs = oc.correlation(np.abs(x1), np.abs(x2), corr_type="mult", **kw)
        g1_abs, g2_abs = oc.correlation_grad(np.abs(gt), np.abs(x1), np.abs(x2), corr_type="mult", **kw)
    else:
        f_abs = oc.correlation(x1, x2, corr_type="subt", **kw)
        z = np.zeros_like(x1)
        g1_abs, g2_abs = (np.abs(v) for v in oc.correlation_grad(np.abs(gt), z, z, corr_type="subt", **kw))
    g = oc.geometry(x1.shape, one_d=True, single_dir=-1, **attrs)
    nf, ng = g["ks"] ** 2 * g["c"] + 34, g["tc"] * g["ks"] ** 2 + 2
    return [nf * EPS * f_abs / g["sumelems"], ng * EPS * g1_abs / g["sumelems"], ng * EPS * g2_abs / g["sumelems"]]


@pytest.mark.parametrize("ct", ["mult", "subt"])
@pytest.mark.parametrize("shape,attrs", LEFT)
def test_single_dir_left_within_tolerance_of_oracle(ops, shape, attrs, ct):
    x1, x2, rng = make_inputs(shape, 21, False)
    top = ops.correlation_1d(x1, x2, corr_type=ct, single_dir=-1, **attrs)
    gt = rng.randn(*top.shape).astype(np.float32)
    g1, g2 = ops.correlation_1d_grad(gt, x1, x2, corr_type=ct, single_dir=-1, **attrs)
    ref = [oc.correlation(x1, x2, one_d=True, corr_type=ct, single_dir=-1, **attrs)]
    ref += list(oc.correlation_grad(gt, x1, x2, one_d=True, corr_type=ct, single_dir=-1, **attrs))
    for what, ours, want, tol in zip(("forward", "input1_grad", "input2_grad"), (top, g1, g2), ref, _bounds(x1, x2, gt, attrs, ct)):
        err = np.abs(ours.astype(np.float64) - want)
        assert ours.shape == want.shape
        assert np.all(err <= tol + EPS * np.abs(want)), "%s: max excess %g" % (what, (err - tol - EPS * np.abs(want)).max())


@pytest.mark.parametrize("ct", ["mult", "subt"])
@pytest.mark.parametrize("shape,attrs", LEFT)
def test_single_dir_left_exact_on_representable_data(ops, shape, attrs, ct):
    """small integers times powers of two: every sum is exact in float32 in any order, so the result is the exact sum
    divided once, in float32, by K K C"""
    rng = np.random.RandomState(31)
    x1 = (rng.randint(-8, 9, shape) * 0.125).astype(np.float32)
    x2 = (rng.randint(-8, 9, shape) * 0.25).astype(np.float32)
    top = ops.correlation_1d(x1, x2, corr_type=ct, single_dir=-1, **attrs)
    gt = (rng.randint(-8, 9, top.shape) * 0.0625).astype(np.float32)
    g1, g2 = ops.correlation_1d_grad(gt, x1, x2, corr_type=ct, single_dir=-1, **attrs)
    se = np.float32(oc.geometry(shape, one_d=True, single_dir=-1, **attrs)["sumelems"])
    kw = dict(one_d=True, corr_type=ct, single_dir=-1, normalize=False, **attrs)
    want = [oc.correlation(x1, x2, **kw)] + list(oc.correlation_grad(gt, x1, x2, **kw))
    for what, ours, w in zip(("forward", "input1_grad", "input2_grad"), (top, g1, g2), want):
        assert np.array_equal(w.astype(np.float32).astype(np.float64), w), "%s: the exact sum is not a float32" % what
        expect = w.astype(np.float32) / se
        assert np.array_equal(ours.view(np.int32), expect.view(np.int32)), "%s: %d elements differ" % (what, int((ours != expect).sum()))


# ---- autograd -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ct", ["mult", "subt"])
@pytest.mark.parametrize("one_d,sd", [(False, 0), (True, 0), (True, 1), (True, -1)])
def test_autograd_equals_correlation_grad(ops, one_d, sd, ct):
    x1, x2, rng = make_inputs((2, 24, 10, 20), 41, False)
    attrs = dict(max_displacement=3, kernel_size=3, stride1=1, stride2=1, pad_size=3)
    a = torch.from_numpy(x1).cuda().requires_grad_(True)
    b = torch.from_numpy(x2).cuda().requires_grad_(True)
    if one_d:
        y = ops.correlation_1d_autograd(a, b, corr_type=ct, single_dir=sd, **attrs)
        fwd = ops.correlation_1d(a.detach(), b.detach(), corr_type=ct, single_dir=sd, **attrs)
    else:
        y = ops.correlation_autograd(a, b, corr_type=ct, **attrs)
        fwd = ops.correlation(a.detach(), b.detach(), corr_type=ct, **attrs)
    assert torch.equal(y.detach(), fwd)
    g = torch.from_numpy(rng.randn(*y.shape).astype(np.float32)).cuda()
    y.backward(g)
    if one_d:
        g1, g2 = ops.correlation_1d_grad(g, a.detach(), b.detach(), corr_type=ct, single_dir=sd, **attrs)
    else:
        g1, g2 = ops.correlation_grad(g, a.detach(), b.detach(), corr_type=ct, **attrs)
    assert isinstance(g1, torch.Tensor) and g1.is_cuda
    assert torch.equal(a.grad.view(torch.int32), g1.view(torch.int32))
    assert torch.equal(b.grad.view(torch.int32), g2.view(torch.int32))


if __name__ == "__main__":
    trace_variant_rows(sys.argv[1])
