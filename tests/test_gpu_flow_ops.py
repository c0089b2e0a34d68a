"""GPU: flow_warp, flow_warp_grad, flow_out_of_frame and resample (csrc/flow_ops.cu) bit for bit against the reference's own
kernels (oracle/flow_ops_ref.py: oracle/_ref/libref_flow_ops.so, or the digests it recorded in
tests/golden/flow_ops_digests.json):
  * flow_warp and flow_warp_grad's flow_grad against the reference's GPU kernels;
  * flow_warp_grad's image_grad against the reference's CPU kernel (whose order it keeps), and within the rounding of the
    GPU kernel's atomic sums of the same products;
  * flow_out_of_frame against the reference's CPU kernel (the op has no GPU kernel);
  * resample, float32 and float64, against the reference's GPU kernels, except NEAREST where the reference reads outside
    its input: those rows are compared with the float64 oracle (oracle/flow_ops.py), and their clamped pixels are listed.
Every call goes through the C ABI into outputs filled with SENTINEL and must make the number of launches it names.  A
torch.profiler trace, taken in a child process, shows that the calls reach every kernel of the file.
"""
import collections
import gc
import os
import zlib
import re
import sys

import numpy as np
import pytest
import torch
from torch.profiler import ProfilerActivity, profile

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import flow_ops as of
from oracle import flow_ops_ref as fref
from oracle.ref import Recorded, digest

SENTINEL = -1.5e38
EPS = float(np.finfo(np.float32).eps)
FILL = {"zero": 1, "not_a_number": 2}
RTYPE = {"NEAREST": 1, "CUBIC": 2, "LINEAR": 3}

# (name, shape, flow kind, non-finite image and gradient values)
WARP_ROWS = [
    ("image_8x3x384x512", (8, 3, 384, 512), "random", False),
    ("feature_2x256x48x64", (2, 256, 48, 64), "random", False),
    ("c1_w45_edges", (1, 1, 20, 45), "edges", False),
    ("c33_w70_integers", (1, 33, 17, 70), "integers", False),
    ("c70_w37", (2, 70, 9, 37), "random", False),
    ("n3_edges", (3, 5, 13, 33), "edges", False),
    ("huge_nonfinite_flow", (1, 3, 16, 40), "huge", False),
    ("nonfinite_image", (2, 6, 12, 35), "random", True),
    ("collapse", (2, 4, 40, 52), "collapse", False),
    ("collapse_corner", (1, 3, 24, 33), "collapse_corner", False),
]


@pytest.fixture(scope="module")
def ops():
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    from demon_b200 import lmbspecialops
    return lmbspecialops


@pytest.fixture(scope="module", autouse=True)
def leave_the_device_idle():
    """The later modules (tests/test_gpu_op_paths.py) trace kernels with torch.profiler in this process: leave them an idle
    device with this module's buffers returned, not queued work or cached blocks."""
    yield
    if torch.cuda.is_available():
        torch.cuda.synchronize()
        gc.collect()
        torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def lib(ops):
    from demon_b200 import _lib
    return _lib.load()


@pytest.fixture(scope="module")
def reference():
    if not fref.available():
        pytest.fail("neither oracle/_ref/libref_flow_ops.so nor tests/golden/flow_ops_digests.json is present")
    return fref


# ---- inputs ---------------------------------------------------------------------------------------------------------------
def make_flow(shape, kind, rng):
    n, _, h, w = shape
    ys, xs = np.meshgrid(np.arange(h, dtype=np.float32), np.arange(w, dtype=np.float32), indexing="ij")
    if kind == "random":
        return (rng.randn(n, 2, h, w) * 4).astype(np.float32)
    if kind == "integers":
        return np.round(rng.randn(n, 2, h, w) * 3).astype(np.float32)
    if kind in ("collapse", "collapse_corner"):
        tx, ty = (w / 2 + 0.3, h / 2 + 0.6) if kind == "collapse" else (w - 0.5, h - 0.25)
        f = np.stack([np.float32(tx) - xs, np.float32(ty) - ys])[None]
        return np.repeat(f, n, axis=0).astype(np.float32)
    f = (rng.randn(n, 2, h, w) * 2).astype(np.float32)
    pick = rng.randint(0, 5, (n, 2, h, w))
    last = np.stack([w - 1 + rng.rand(h, w).astype(np.float32) * 0.999 - xs, h - 1 + rng.rand(h, w).astype(np.float32) * 0.999 - ys])
    f = np.where(pick == 0, last[None], f)                                          # into [w-1, w) / [h-1, h)
    f = np.where(pick == 1, np.round(f), f)                                         # exactly on integers
    f = np.where(pick == 2, -rng.rand(n, 2, h, w).astype(np.float32) * 1e-3, f)     # small negative: out at x = 0 / y = 0
    f = np.where(pick == 3, np.stack([w - 1 - xs, h - 1 - ys])[None], f)            # exactly the last column / row
    if kind == "huge":
        vals = np.array([np.nan, np.inf, -np.inf, 3e9, -3e9, 1e30, -0.0], np.float32)
        m = rng.rand(n, 2, h, w) < 0.3
        f[m] = vals[rng.randint(0, len(vals), m.sum())]
    return f.astype(np.float32)


def warp_data(row):
    name, shape, kind, special = row
    rng = np.random.RandomState(zlib.crc32(name.encode()) % 1000 + 3)
    image = rng.randn(*shape).astype(np.float32)
    grad = rng.randn(*shape).astype(np.float32)
    flow = make_flow(shape, kind, rng)
    if special:
        vals = np.array([np.nan, np.inf, -np.inf, -0.0], np.float32)
        for x in (image, grad):
            m = rng.rand(*shape) < 0.02
            x[m] = vals[rng.randint(0, len(vals), m.sum())]
    return image, flow, grad


def sentinel(shape, dtype=torch.float32):
    return torch.full(tuple(shape), SENTINEL, dtype=dtype, device="cuda")


def stream():
    return torch.cuda.current_stream().cuda_stream


def abi_warp(lib, image, flow, fill):
    a, f = torch.from_numpy(image).cuda(), torch.from_numpy(flow).cuda()
    out = sentinel(image.shape)
    n, c, h, w = image.shape
    before = lib.demon_launch_count()
    rc = lib.demon_flow_warp_f32(a.data_ptr(), f.data_ptr(), out.data_ptr(), n, c, h, w, FILL[fill], stream())
    assert rc == 0, lib.demon_last_error()
    assert lib.demon_launch_count() - before == 1
    return out.cpu().numpy()


def abi_grad(lib, image, flow, grad):
    a, f, g = (torch.from_numpy(v).cuda() for v in (image, flow, grad))
    ig, fg = sentinel(image.shape), sentinel(flow.shape)
    n, c, h, w = image.shape
    nbytes = lib.demon_flow_warp_grad_workspace_bytes(n, h, w)
    assert nbytes > 0, lib.demon_last_error()
    ws = torch.full((nbytes,), 0xA5, dtype=torch.uint8, device="cuda")
    before = lib.demon_launch_count()
    rc = lib.demon_flow_warp_grad_f32(a.data_ptr(), f.data_ptr(), g.data_ptr(), ig.data_ptr(), fg.data_ptr(), n, c, h, w,
                                      ws.data_ptr(), nbytes, stream())
    assert rc == 0, lib.demon_last_error()
    assert lib.demon_launch_count() - before == 4   # flow_grad, cells, bounds, image_grad (CUB's sort launches its own)
    return ig.cpu().numpy(), fg.cpu().numpy()


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


# ---- flow_warp / flow_warp_grad -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("row", WARP_ROWS, ids=[r[0] for r in WARP_ROWS])
def test_flow_warp_bits_equal_reference_gpu(lib, reference, row):
    image, flow, _ = warp_data(row)
    inside = of._cells(flow)[0]
    for fill in ("zero", "not_a_number"):
        ours = abi_warp(lib, image, flow, fill)
        assert_bits(ours, reference.flow_warp_gpu(image, flow, fill), "%s %s" % (row[0], fill))
        outside = np.broadcast_to(~inside[:, None], ours.shape)
        want = of.NAN_FILL_BITS if fill == "not_a_number" else 0
        assert (ours.view(np.uint32)[outside] == want).all(), "%s: fill bits" % row[0]
    if not row[3]:
        assert np.allclose(ours, of.flow_warp(image, flow, "not_a_number"), rtol=1e-5, atol=1e-5, equal_nan=True)


def _addend_bounds(flow, grad):
    """per image_grad element: number of addends k and the sum of their magnitudes (float64)"""
    ones = np.ones_like(grad)
    inside, L, T, R, B, a, b = of._cells(flow)
    n, c, h, w = grad.shape
    count = np.zeros(grad.shape)
    gm = np.where(inside[:, None], ones, 0.0)
    ni = np.broadcast_to(np.arange(n)[:, None, None, None], grad.shape)
    ci = np.broadcast_to(np.arange(c)[None, :, None, None], grad.shape)
    for yy, xx in ((T, L), (T, R), (B, L), (B, R)):
        np.add.at(count, (ni, ci, np.broadcast_to(yy[:, None], grad.shape), np.broadcast_to(xx[:, None], grad.shape)), gm)
    mag = of.flow_warp_grad(np.zeros_like(grad), flow, np.abs(grad))[0]
    return count, mag


@pytest.mark.parametrize("row", WARP_ROWS, ids=[r[0] for r in WARP_ROWS])
def test_flow_warp_grad_bits(lib, reference, row):
    image, flow, grad = warp_data(row)
    ig, fg = abi_grad(lib, image, flow, grad)
    ref_ig_gpu, ref_fg = reference.flow_warp_grad_gpu(image, flow, grad)
    assert_bits(fg, ref_fg, "%s flow_grad" % row[0])
    assert_bits(ig, reference.flow_warp_grad_cpu(image, flow, grad), "%s image_grad vs the CPU kernel" % row[0])
    ig2, fg2 = abi_grad(lib, image, flow, grad)
    assert ig2.tobytes() == ig.tobytes() and fg2.tobytes() == fg.tobytes(), "%s: two calls differ" % row[0]
    if isinstance(ref_ig_gpu, Recorded) or row[3]:
        return   # the atomic sums' bits depend on scheduling: only the compiled reference gives a value to bound
    k, mag = _addend_bounds(flow, grad)
    err = np.abs(ig.astype(np.float64) - ref_ig_gpu)
    assert (err <= np.maximum(k - 1, 0) * EPS * mag + 1e-300).all(), "%s: image_grad beyond the atomic sums' rounding" % row[0]
    few = k <= 2
    assert np.array_equal(ig[few].view(np.uint32), ref_ig_gpu[few].view(np.uint32)), "%s: k <= 2 not bit-equal" % row[0]


def test_flow_warp_grad_matches_float64_oracle(lib):
    image, flow, grad = warp_data(("oracle", (2, 5, 19, 27), "random", False))
    ig, fg = abi_grad(lib, image, flow, grad)
    oig, ofg = of.flow_warp_grad(image, flow, grad)
    k, mag = _addend_bounds(flow, grad)
    assert (np.abs(ig - oig) <= (k + 2) * EPS * mag + 1e-30).all()
    assert np.allclose(fg, ofg, rtol=1e-4, atol=1e-4)


def test_collapse_runs_linear(lib):
    """every pixel of a [1,2,256,320] image into one cell: finishes, equals the float64 oracle"""
    image, flow, grad = warp_data(("collapse_big", (1, 2, 256, 320), "collapse", False))
    ig, _ = abi_grad(lib, image, flow, grad)
    oig, _ = of.flow_warp_grad(image, flow, grad)
    k, mag = _addend_bounds(flow, grad)
    assert (np.abs(ig - oig) <= (k + 2) * EPS * mag + 1e-30).all()
    assert np.count_nonzero(k) == 4 * 2


# ---- flow_out_of_frame ----------------------------------------------------------------------------------------------------
def oof_data(seed, shape):
    rng = np.random.RandomState(seed)
    n, _, h, w = shape
    ys, xs = np.meshgrid(np.arange(h, dtype=np.float32), np.arange(w, dtype=np.float32), indexing="ij")
    f = (rng.randn(*shape) * 3).astype(np.float32)
    pick = rng.randint(0, 8, shape)
    f = np.where(pick == 0, np.stack([-xs - 0.5, -ys - 0.5])[None], f)                # ties at -0.5
    f = np.where(pick == 1, np.stack([w - 0.5 - xs, h - 0.5 - ys])[None], f)          # ties at size - 0.5
    f = np.where(pick == 2, np.stack([-xs + 0.4999, -ys - 0.4999])[None], f)
    specials = np.array([np.nan, np.inf, -np.inf, 3e9, -3e9, 2.0 ** 31, -2.0 ** 31], np.float32)
    m = pick == 3
    f[m] = specials[rng.randint(0, len(specials), m.sum())]
    occ = rng.rand(n, h, w).astype(np.float32)
    m = rng.rand(n, h, w) < 0.05
    occ[m] = np.array([np.nan, np.inf, -np.inf], np.float32)[rng.randint(0, 3, m.sum())]
    return f.astype(np.float32), occ


@pytest.mark.parametrize("shape", [(1, 2, 9, 13), (3, 2, 40, 70), (8, 2, 96, 128)])
def test_flow_out_of_frame_bits_equal_reference_cpu(lib, reference, shape):
    flow, occ = oof_data(shape[3], shape)
    n, _, h, w = shape
    f, o = torch.from_numpy(flow).cuda(), torch.from_numpy(occ).cuda()
    out = sentinel((n, 1, h, w))
    before = lib.demon_launch_count()
    assert lib.demon_flow_out_of_frame_f32(f.data_ptr(), o.data_ptr(), out.data_ptr(), n, h, w, stream()) == 0
    assert lib.demon_launch_count() - before == 1
    ours = out.cpu().numpy()
    assert_bits(ours, reference.flow_out_of_frame_cpu(flow, occ), "flow_out_of_frame %s" % (shape,))
    ref = of.flow_out_of_frame(flow, occ)
    assert np.array_equal(ours.view(np.uint32), ref.view(np.uint32))   # payloads of the NaN occ values included


# ---- resample -------------------------------------------------------------------------------------------------------------
RESAMPLE_SIZES = [
    ("identity", (1, 3, 24, 40), 24, 40),
    ("up4_flow", (8, 2, 96, 128), 384, 512),
    ("down4", (2, 3, 96, 128), 24, 32),
    ("nonint", (1, 3, 97, 131), 40, 53),
    ("one", (1, 2, 17, 23), 1, 1),
    ("aniso_y", (1, 2, 64, 16), 8, 16),
    ("aniso_x", (1, 2, 16, 64), 16, 8),
]
RESAMPLE_CASES = [(s, dt, t, aa) for s in RESAMPLE_SIZES for dt in ("float32", "float64") for t in ("NEAREST", "LINEAR", "CUBIC")
                  for aa in (True, False)]


def abi_resample(lib, x, oh, ow, aa, rtype):
    t = torch.from_numpy(x).cuda()
    n, c, ih, iw = x.shape
    out = sentinel((n, c, oh, ow), t.dtype)
    fn = lib.demon_resample_f32 if x.dtype == np.float32 else lib.demon_resample_f64
    before = lib.demon_launch_count()
    rc = fn(t.data_ptr(), out.data_ptr(), n, c, ih, iw, oh, ow, int(aa), RTYPE[rtype], stream())
    assert rc == 0, lib.demon_last_error()
    assert lib.demon_launch_count() - before == 1
    return out.cpu().numpy()


@pytest.mark.parametrize("case", RESAMPLE_CASES, ids=["%s-%s-%s-%s" % (c[0][0], c[1], c[2], "aa" if c[3] else "noaa") for c in RESAMPLE_CASES])
def test_resample_bits(lib, reference, case):
    (name, shape, oh, ow), dt, rtype, aa = case
    rng = np.random.RandomState(shape[2] * 7 + shape[3])
    x = rng.randn(*shape).astype(dt)
    ours = abi_resample(lib, x, oh, ow, aa, rtype)
    _, _, ih, iw = shape
    if rtype == "NEAREST" and not fref.nearest_in_range(ih, iw, oh, ow):
        xr, yr = of.resample_positions(ih, iw, oh, ow)
        clamped = [("x", i, int(v)) for i, v in enumerate(xr) if not 0 <= v < iw] + [("y", i, int(v)) for i, v in enumerate(yr) if not 0 <= v < ih]
        assert clamped, name
        print("%s: NEAREST clamps %s" % (name, clamped))
        assert np.array_equal(ours, of.resample(x, ow, oh, aa, rtype).astype(dt)), name
        return
    assert_bits(ours, reference.resample_gpu(x, ow, oh, aa, rtype), "resample %s %s %s aa=%s" % (name, dt, rtype, aa))
    if rtype != "NEAREST":
        tol = 1e-5   # the weights are float32 in both dtypes
        assert np.allclose(ours, of.resample(x, ow, oh, aa, rtype), rtol=tol, atol=tol), name


def test_resample_aniso_rows_are_the_out_of_range_ones():
    assert fref.nearest_in_range(24, 40, 24, 40) and fref.nearest_in_range(96, 128, 384, 512)
    assert not fref.nearest_in_range(64, 16, 8, 16)


# ---- autograd -------------------------------------------------------------------------------------------------------------
def test_flow_warp_autograd(ops):
    image, flow, grad = warp_data(("autograd", (2, 4, 11, 17), "edges", False))
    a = torch.from_numpy(image).cuda().requires_grad_(True)
    f = torch.from_numpy(flow).cuda().requires_grad_(True)
    out = ops.flow_warp_autograd(a, f)
    assert torch.equal(out, ops.flow_warp(a.detach(), f.detach()))
    g = torch.from_numpy(grad).cuda()
    torch.autograd.backward([out], [g])
    ig, fg = ops.flow_warp_grad(a.detach(), f.detach(), g)
    assert torch.equal(a.grad, ig) and torch.equal(f.grad, fg)


def test_python_ops_equal_abi(ops, lib):
    image, flow, grad = warp_data(("py", (1, 3, 10, 21), "random", False))
    assert np.array_equal(ops.flow_warp(image, flow, "not_a_number").view(np.uint32), abi_warp(lib, image, flow, "not_a_number").view(np.uint32))
    ig, fg = ops.flow_warp_grad(image, flow, grad)
    aig, afg = abi_grad(lib, image, flow, grad)
    assert np.array_equal(ig, aig) and np.array_equal(fg, afg)
    x = np.random.RandomState(1).randn(1, 2, 20, 30)
    assert np.array_equal(ops.resample(x, 7, 5, type="CUBIC"), abi_resample(lib, x, 5, 7, True, "CUBIC"))


def test_invalid_arguments_are_refused_before_any_launch(lib):
    before = lib.demon_launch_count()
    assert lib.demon_flow_warp_f32(None, None, None, 1, 1, 4, 4, 3, stream()) == -1
    assert lib.demon_resample_f32(None, None, 1, 1, 4, 4, 0, 4, 1, 3, stream()) == -1
    assert lib.demon_resample_f32(None, None, 1, 1, 4, 4, 4, 4, 1, 7, stream()) == -1
    assert lib.demon_flow_warp_grad_workspace_bytes(1 << 16, 1 << 8, 1 << 8) == -1
    t = torch.zeros(64, device="cuda")
    assert lib.demon_flow_warp_grad_f32(t.data_ptr(), t.data_ptr(), t.data_ptr(), t.data_ptr(), t.data_ptr(), 1, 1, 4, 4,
                                        t.data_ptr(), 4, stream()) == -1   # workspace too small
    assert lib.demon_launch_count() == before


# ---- which kernels ran ----------------------------------------------------------------------------------------------------
_KERNEL_NAME = re.compile(r"demon::(?:\(anonymous namespace\)::)?(\w+(?:<[^()]*>)?)\(")
EVERY_KERNEL = {"flow_warp_kernel", "flow_warp_flow_grad_kernel", "flow_warp_cells_kernel", "flow_warp_bounds_kernel",
                "flow_warp_image_grad_kernel", "flow_out_of_frame_kernel", "resample_kernel<float>", "resample_kernel<double>"}


def traced(fn):
    prof = profile(activities=[ProfilerActivity.CUDA])
    with prof:
        out = fn()
        torch.cuda.synchronize()
    ours = collections.Counter()
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            m = _KERNEL_NAME.search(e.name)
            if m:
                ours[m.group(1).replace(" ", "")] += 1
    return out, ours


def trace_rows(out_path):
    """child process: one call of each entry under its own trace -> pickle of [kernels]"""
    import pickle
    from demon_b200 import _lib
    lib = _lib.load()
    image, flow, grad = warp_data(WARP_ROWS[4])
    flow2, occ = oof_data(3, (1, 2, 9, 13))
    x = np.random.RandomState(0).randn(1, 2, 20, 30)
    calls = [lambda: abi_warp(lib, image, flow, "zero"), lambda: abi_grad(lib, image, flow, grad),
             lambda: lib.demon_flow_out_of_frame_f32(torch.from_numpy(flow2).cuda().data_ptr(), torch.from_numpy(occ).cuda().data_ptr(),
                                                    sentinel((1, 1, 9, 13)).data_ptr(), 1, 9, 13, stream()),
             lambda: abi_resample(lib, x.astype(np.float32), 9, 11, True, "LINEAR"), lambda: abi_resample(lib, x, 9, 11, True, "CUBIC")]
    rows = []
    for fn in calls:
        _, k = traced(fn)
        rows.append(dict(k))
    with open(out_path, "wb") as f:
        pickle.dump(rows, f)


def test_calls_run_the_kernels_they_name(ops, tmp_path):
    """a torch.profiler trace per call, in a child process (a process that keeps running GPU work after a trace loses the CUDA
    records of later traces): each call runs the kernels it names, and together they run every kernel of csrc/flow_ops.cu"""
    import pickle
    import subprocess
    out = str(tmp_path / "traces.pkl")
    flags = ["-s"] if sys.flags.no_user_site else []
    subprocess.run([sys.executable] + flags + [__file__, out], check=True)
    with open(out, "rb") as f:
        rows = pickle.load(f)
    want = [{"flow_warp_kernel": 1},
            {"flow_warp_flow_grad_kernel": 1, "flow_warp_cells_kernel": 1, "flow_warp_bounds_kernel": 1, "flow_warp_image_grad_kernel": 1},
            {"flow_out_of_frame_kernel": 1}, {"resample_kernel<float>": 1}, {"resample_kernel<double>": 1}]
    assert rows == want, "launched %s, must launch %s" % (rows, want)
    assert set().union(*rows) == EVERY_KERNEL


if __name__ == "__main__":
    trace_rows(sys.argv[1])
