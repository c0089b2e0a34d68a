"""GPU: every launch path of the standalone geometry and training ops of `demon_b200.lmbspecialops`, compared with the CPU
oracle, with a CUDA trace proving which kernels ran.

The launchers in csrc/geometry_ops.cu and csrc/training_ops.cu choose between a scalar kernel and a float4 ("v4") kernel from
the width, the 16-byte alignment of the pointers and the element count, and launch the plane-parallel ops in chunks of 32768
planes.  Which path a call took does not show in its result.  So every row of ROWS names the kernels it must launch and how
often, and test_row reads the kernels that ran from a torch.profiler CUDA trace and demands exactly those.
test_rows_reach_every_target checks that the rows together reach every kernel instantiation of the two files, the v4 kernel and
its scalar fallback at one width, more than one z-chunk of every chunked launch and every rotation format of both camera ops.

Oracles and tolerances are those of tests/test_gpu_ops.py and tests/test_gpu_training_ops.py:
  * bit for bit, NaN positions included: warp2d, median3x3_downsample, scale_invariant_gradient, leaky_relu and depth_to_flow
    with `matrix` or `quaternion` against oracle/ops.py; the training ops against the reference's own kernels (oracle/ref.py,
    or their stored digests);
  * depth_to_flow with `angleaxis3`: within 64 eps * max|ref| (sin and cos differ by a few ulp between glibc and CUDA's libm);
  * flow_to_depth(2), every rotation format: against the float64 oracle fed the same float inputs, relative error below 4e-7
    (float32) or 1e-9 (float64) where both are nonzero, and the same behind-camera pattern on at least 99.9 % of the pixels.
    f2d_camera works in double for every format, so test_flow_to_depth_matches_oracle's argument holds for all three.

Layouts: "aligned" is a fresh tensor.  "offset" holds the same data in a view one element into a buffer (`buf[1:].view(...)`):
the op's `.contiguous()` keeps the view, so its pointer is not 16-byte aligned.  "offset-disp" does that to warp2d's
displacements.  An offset row runs the aligned tensor too, and the two calls must give the same bits.

Every output is allocated in a block filled with SENTINEL just before the call (see `poisoned`), so an element no kernel writes
(a z-chunk launched at the wrong plane, say) fails the comparison even where the oracle's value is NaN.
"""
import collections
import os
import re
import time
import zlib
from typing import NamedTuple

import numpy as np
import pytest
import torch
from torch.profiler import ProfilerActivity, profile

pytestmark = pytest.mark.gpu

from oracle import ops as oops
from oracle import ref

F, D = np.float32, np.float64
CTYPE = {F: "float", D: "double"}
CHUNK = 32768                       # planes per launch of the chunked launchers
SENTINEL = -1.5e38                  # a value none of the ops computes from the data below
WINDOW_MARGIN_S = 0.005
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "demon_b200", "csrc")


@pytest.fixture(scope="module")
def ops():
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    from demon_b200 import lmbspecialops
    return lmbspecialops


@pytest.fixture(scope="module")
def lib(ops):
    from demon_b200 import _lib
    return _lib.load()


# ---- which kernels ran ----------------------------------------------------------------------------------------------------
_KERNEL_NAME = re.compile(r"demon::(?:\(anonymous namespace\)::)?(\w+(?:<[^()]*>)?)\(")


def device_kernels(prof):
    """(the library's kernels, every other device activity) of a profile, as Counters of names.  The library's kernels are named
    "name<targs>" without spaces, e.g. warp2d_kernel<float,true>."""
    ours, other = collections.Counter(), collections.Counter()
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            m = _KERNEL_NAME.search(e.name)
            if m:
                ours[m.group(1).replace(" ", "")] += 1
            else:
                other[e.name] += 1
    return ours, other


class Trace:
    """Runs calls under torch.profiler and counts the library's kernels they launched."""

    def __init__(self):
        self.kernels = collections.Counter()
        self.other = collections.Counter()

    def __call__(self, fn):
        prof = profile(activities=[ProfilerActivity.CUDA])
        try:
            with prof:
                # the profiler keeps only device activity inside its capture window, timed on the host's clock: keep the
                # calls clear of the window's edges, so that a small offset between the host and device clocks drops none
                torch.cuda.synchronize()
                time.sleep(WINDOW_MARGIN_S)
                out = fn()
                torch.cuda.synchronize()
                time.sleep(WINDOW_MARGIN_S)
        finally:
            ours, other = device_kernels(prof)
            self.kernels.update(ours)
            self.other.update(other)
        return out


@pytest.fixture(scope="module")
def profiler_records_kernels(ops):
    """Whether torch.profiler records CUDA kernels here at all, from a probe launch of a torch op.  The first row then shows that
    the library's own kernels, launched through ctypes, are recorded as well."""
    t = Trace()
    t(lambda: torch.ones(4096, device="cuda").mul_(3.0))
    return sum(t.other.values()) + sum(t.kernels.values()) > 0


def assert_kernels(trace, want, recorded, what):
    assert recorded, "torch.profiler recorded no CUDA kernel of a probe torch op here, so the path %s took cannot be checked" % what
    got = dict(trace.kernels)
    assert got == want, "%s: launched %s, must launch %s" % (what, got, want)


# ---- placing inputs and outputs -------------------------------------------------------------------------------------------
def place(a, layout="aligned"):
    """numpy -> CUDA tensor; "offset": a view one element into a buffer, so not 16-byte aligned."""
    t = torch.from_numpy(np.ascontiguousarray(a))
    if layout == "aligned":
        return t.cuda()
    buf = torch.empty(t.numel() + 1, dtype=t.dtype, device="cuda")
    v = buf[1:].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16 != 0
    return v


def poisoned(call, numel, dtype):
    """call() with the block its output of `numel` elements will get filled with SENTINEL first: the caching allocator hands
    a freed block to the next request of the same size.  Checked: the output must sit at that block."""
    block = torch.full((numel,), SENTINEL, dtype=torch.float32 if dtype == F else torch.float64, device="cuda")
    ptr = block.data_ptr()
    del block
    out = call()
    assert out.data_ptr() == ptr, "the output was not allocated in the poisoned block"
    return out.cpu().numpy()


# ---- comparisons ----------------------------------------------------------------------------------------------------------
def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32 if a.dtype == np.float32 else np.uint64)


def assert_bits(got, want, what):
    """Bit for bit, NaN positions included (NaN payloads are not compared); `want` may be a stored reference digest."""
    if isinstance(want, ref.Recorded):
        assert want.matches(got), "%s: differs from the reference kernel's stored result (shape %s, want %s)" % (
            what, got.shape, want.shape)
        return
    assert got.shape == want.shape and got.dtype == want.dtype, (what, got.shape, want.shape, got.dtype, want.dtype)
    nan_w = np.isnan(want)
    bad = (np.isnan(got) != nan_w) | (~nan_w & (_bits(got) != _bits(want)))
    if bad.any():
        i = tuple(int(v) for v in np.argwhere(bad)[0])
        pytest.fail("%s: %d of %d elements differ, first at %s: got %r, want %r" % (what, bad.sum(), bad.size, list(i), got[i], want[i]))


def assert_close(got, want, tol, what):
    """NaN and infinity positions equal, finite values within tol."""
    assert got.shape == want.shape and got.dtype == want.dtype, what
    fin = np.isfinite(want)
    assert np.array_equal(np.isnan(got), np.isnan(want)), "%s: NaN positions differ" % what
    assert np.array_equal(got[~fin & ~np.isnan(want)], want[~fin & ~np.isnan(want)]), "%s: infinities differ" % what
    assert np.isfinite(got[fin]).all(), "%s: non-finite value where the oracle's is finite" % what
    err = np.abs(got[fin].astype(np.float64) - want[fin])
    assert err.max() <= tol, "%s: max |err| %g > %g at %s" % (what, err.max(), tol, np.argwhere(fin)[err.argmax()].tolist())


# ---- the table ------------------------------------------------------------------------------------------------------------
class Row(NamedTuple):
    op: str
    dtype: type
    shape: tuple        # the op's input: warp2d [n,c,h,w]; depth_to_flow / flow_to_depth [n,h,w]; the others as passed
    layout: str         # "aligned", "offset" or "offset-disp"
    params: tuple       # per op, see the runners
    kernels: dict       # kernel -> launches (for an offset row: of both its calls)

    @property
    def id(self):
        p = "-".join(str(v) for v in self.params)
        return "%s-%s-%s-%s%s" % (self.op, CTYPE[self.dtype], "x".join(map(str, self.shape)), self.layout, "-" + p if p else "")

    def rng(self):
        return np.random.default_rng(zlib.crc32(self.id.encode()))


def tk(name, *targs):
    return "%s<%s>" % (name, ",".join(targs)) if targs else name


def b(v):
    return "true" if v else "false"


ROWS = []

# warp2d: params (normalized, border_mode).  v4: float, W % 4 == 0, W >= 128, aligned.  C = 1 and 2 sit below the 2 channels
# of the displacements that warp2d_fast's size guard counts with.
for c, w, normalized, mode in ((1, 128, False, "clamp"), (1, 130, False, "clamp"), (1, 128, True, "value"), (1, 126, True, "value"),
                               (2, 256, True, "clamp"), (2, 250, True, "clamp"), (2, 256, False, "value"), (2, 61, False, "value")):
    v4 = w % 4 == 0 and w >= 128
    ROWS.append(Row("warp2d", F, (2, c, 9, w), "aligned", (normalized, mode),
                    {tk("warp2d_v4_kernel", b(mode == "clamp"), "1") if v4 else tk("warp2d_kernel", "float", b(mode == "clamp")): 1}))
for c, layout, mode in ((3, "offset", "clamp"), (1, "offset-disp", "value")):
    ROWS.append(Row("warp2d", F, (2, c, 9, 256), layout, (False, mode),
                    {tk("warp2d_v4_kernel", b(mode == "clamp"), "1"): 1, tk("warp2d_kernel", "float", b(mode == "clamp")): 1}))
for c, mode in ((1, "clamp"), (2, "value")):
    ROWS.append(Row("warp2d", D, (2, c, 9, 128), "aligned", (True, mode), {tk("warp2d_kernel", "double", b(mode == "clamp")): 1}))

# depth_to_flow: params (rotation_format, inverse_depth, normalize_flow).  v4: float, W % 4 == 0, aligned.
FORMATS = ("matrix", "quaternion", "angleaxis3")
for fmt in FORMATS:
    for inv in (False, True):
        for nrm in (False, True):
            for w, layout in ((61, "aligned"), (250, "aligned"), (64, "offset"), (64, "aligned")):
                scalar = w % 4 != 0 or layout == "offset"
                k = {tk("depth_to_flow_kernel", "float"): 1} if scalar else {}
                if not scalar or layout == "offset":
                    k["depth_to_flow_v4_kernel"] = 1
                ROWS.append(Row("depth_to_flow", F, (3, 20 if w == 250 else 48, w), layout, (fmt, inv, nrm), k))
    ROWS.append(Row("depth_to_flow", D, (3, 48, 61), "aligned", (fmt, True, False), {tk("depth_to_flow_kernel", "double"): 1}))

# flow_to_depth / flow_to_depth2: params (rotation_format, inverse_depth, normalized_flow, entry).  One kernel.
for dt in (F, D):
    for fmt in ("matrix", "quaternion"):
        for i, (inv, nrm) in enumerate(((False, False), (False, True), (True, False), (True, True))):
            ROWS.append(Row("flow_to_depth", dt, (3, 48, 64), "aligned", (fmt, inv, nrm, ("flow_to_depth2", "flow_to_depth")[i % 2]),
                            {tk("flow_to_depth_kernel", CTYPE[dt]): 1}))
    ROWS.append(Row("flow_to_depth", dt, (3, 48, 64), "aligned", ("angleaxis3", True, True, "flow_to_depth2"),
                    {tk("flow_to_depth_kernel", CTYPE[dt]): 1}))

# median3x3_downsample.  v4: float, W % 8 == 0, W >= 256, aligned.  32769 planes: two launches, the second at plane 32768.
ROWS += [
    Row("median3x3_downsample", F, (3, 9, 256), "offset", (), {"median3x3_v4_kernel": 1, tk("median3x3_downsample_kernel", "float"): 1}),
    Row("median3x3_downsample", F, (CHUNK + 1, 2, 256), "aligned", (), {"median3x3_v4_kernel": 2}),
    Row("median3x3_downsample", F, (CHUNK + 1, 3, 5), "aligned", (), {tk("median3x3_downsample_kernel", "float"): 2}),
    Row("median3x3_downsample", D, (CHUNK + 1, 3, 5), "aligned", (), {tk("median3x3_downsample_kernel", "double"): 2}),
]

# scale_invariant_gradient.  v4: float, W % 4 == 0, W >= 128, aligned.
ROWS += [
    Row("scale_invariant_gradient", F, (2, 9, 128), "offset", (), {"sig_v4_kernel": 1, tk("sig_kernel", "float"): 1}),
    Row("scale_invariant_gradient", F, (CHUNK + 1, 2, 128), "aligned", (), {"sig_v4_kernel": 2}),
    Row("scale_invariant_gradient", F, (CHUNK + 1, 3, 5), "aligned", (), {tk("sig_kernel", "float"): 2}),
    Row("scale_invariant_gradient", D, (CHUNK + 1, 3, 5), "aligned", (), {tk("sig_kernel", "double"): 2}),
]

# leaky_relu: one kernel, vector and scalar loops inside; 2500003 elements reach the grid-stride loop
for dt, n in ((F, 2500003), (D, 100003)):
    ROWS.append(Row("leaky_relu", dt, (n,), "aligned", (), {tk("leaky_relu_kernel", CTYPE[dt]): 1}))
    ROWS.append(Row("leaky_relu", dt, (n,), "offset", (), {tk("leaky_relu_kernel", CTYPE[dt]): 2}))

# training ops: scale_invariant_gradient_grad on rows of one to three CTAs of 128 columns, with deltas that cross CTA edges and
# leave the row; 32769 planes of the chunked kernels
for dt in (F, D):
    for w in (127, 128, 129, 300):
        ROWS.append(Row("scale_invariant_gradient_grad", dt, (2, 1, 5, w), "aligned", (), {tk("sig_grad_kernel", CTYPE[dt]): 1}))
    ROWS.append(Row("scale_invariant_gradient_grad", dt, (CHUNK + 1, 1, 3, 5), "aligned", (), {tk("sig_grad_kernel", CTYPE[dt]): 2}))
    ROWS.append(Row("depth_to_normals", dt, (CHUNK + 1, 1, 4, 5), "aligned", (dt == D,), {tk("depth_to_normals_kernel", CTYPE[dt]): 2}))
    for op, k in (("leaky_relu_grad", "0"), ("replace_nonfinite", "1"), ("replace_nonfinite_grad", "2")):
        ROWS.append(Row(op, dt, (600001,), "aligned", (), {tk("elementwise_kernel", CTYPE[dt], k): 1}))

TRAINING = {"scale_invariant_gradient_grad", "depth_to_normals", "leaky_relu_grad", "replace_nonfinite", "replace_nonfinite_grad"}
SIG_DELTAS = (1, 2, 3, 4, 5, 8, 16, -1, -2, -4, -7, 127, 300)
SIG_WEIGHTS = tuple(1.0 / (1 + i) for i in range(len(SIG_DELTAS)))
GRAD_DELTAS = (1, 2, 3, -1, -5, 127, 128, 300)
GRAD_WEIGHTS = (1.0, 0.5, -0.75, 0.25, 2.0, -1.0, 0.125, 3.0)


# ---- data and references (CPU only, so that the reference digests can be recorded where the reference exists) ---------------
def _camera(rng, n, dt, fmt, small):
    """Intrinsics with fx != fy, and rotations in `fmt`: sample 0 is the identity, the quaternions are unnormalised."""
    K = np.array([[0.89115971, 1.18821287, 0.5, 0.5], [1.1, 0.9, 0.45, 0.55], [0.7, 0.75, 0.5, 0.4]], dt)[:n]
    aa = rng.uniform(-small, small, (n, 3))
    aa[0] = 0.0
    if fmt == "angleaxis3":
        rot = aa.astype(dt)
    elif fmt == "matrix":
        rot = oops.rotation_matrix(aa).astype(dt)
    else:
        ang = np.maximum(np.linalg.norm(aa, axis=1, keepdims=True), 1e-30)
        rot = (np.concatenate((np.cos(ang / 2), np.sin(ang / 2) * aa / ang), axis=1) * 1.7).astype(dt)
    return K, rot


def data(row):
    rng, dt, s = row.rng(), row.dtype, row.shape
    if row.op == "warp2d":
        n, c, h, w = s
        scale = 0.2 if row.params[0] else 9.0
        disp = rng.uniform(-scale, scale, (n, 2, h, w)).astype(dt)
        disp[0, 0, 0, :4] = [np.nan, np.inf, -np.inf, 1e30]
        disp[-1, 1, h - 1, :2] = [-3e9, 0.0]
        return {"img": rng.uniform(-1, 1, s).astype(dt), "disp": disp}
    if row.op == "depth_to_flow":
        n, h, w = s
        depth = rng.uniform(0.2, 4, (n, 1, h, w)).astype(dt)
        depth[0, 0, 0, :5] = [0, -1, np.inf, np.nan, 1e-30]
        K, rot = _camera(rng, n, dt, row.params[0], 0.2)
        if row.params[0] == "angleaxis3":
            rot[-1] = 1e-8                  # below angleaxis3's 1e-6 threshold: its identity branch
        return {"depth": depth, "K": K, "rot": rot, "t": rng.uniform(-1, 1, (n, 3)).astype(dt)}
    if row.op == "flow_to_depth":
        n, h, w = s
        fmt, inv, nrm, _ = row.params
        flow = rng.uniform(-0.08, 0.08, (n, 2, h, w))
        if not nrm:
            flow[:, 0] *= w
            flow[:, 1] *= h
        flow = flow.astype(dt)
        flow[0, :, 0, 0] = np.nan
        flow[1, 1, 5, 7] = np.nan
        K, rot = _camera(rng, n, dt, fmt, 0.05)
        t = (np.array([[1, 0, 0]]) + rng.uniform(-0.2, 0.2, (n, 3))).astype(dt)
        return {"flow": flow, "K": K, "rot": rot, "t": t}
    if row.op == "median3x3_downsample":
        if row.layout == "offset":      # ties, NaNs and signed zeros: which element the selection picks matters
            a = (np.round(rng.random(s) * 6) / 6 - 0.5).astype(dt)
            a[rng.random(s) < 0.1] = np.nan
            a[rng.random(s) < 0.05] = -0.0
            a[rng.random(s) < 0.05] = 0.0
        else:                           # every plane different
            a = rng.standard_normal(s).astype(dt)
            a[rng.random(s) < 0.02] = np.nan
        return {"x": a}
    if row.op == "scale_invariant_gradient":
        a = rng.uniform(-2, 2, s).astype(dt)
        a[..., 0, :3] = 0
        a.flat[rng.integers(0, a.size, 8)] = np.nan
        return {"x": a}
    if row.op == "leaky_relu":
        a = rng.uniform(-3, 3, s).astype(dt)
        a[:6] = [0.0, -0.0, np.nan, np.inf, -np.inf, 1e-30]
        return {"x": a}
    if row.op == "scale_invariant_gradient_grad":
        x = rng.uniform(-3, 3, s).astype(dt)
        x.flat[rng.integers(0, x.size, 12)] = [0.0, -0.0, np.nan, np.inf, -np.inf, 1e-30] * 2
        x[-1, 0, 1, 2] = np.nan         # in the last plane, i.e. the second z-chunk of the chunked row
        return {"x": x, "g": rng.uniform(-1, 1, (s[0], 2) + s[2:]).astype(dt)}
    if row.op == "depth_to_normals":
        z = s[0]
        d = rng.uniform(0.2, 4.0, s).astype(dt)
        for p in (3, CHUNK - 1, z - 1):     # invalid depths in the first chunk and in the second
            d[p, 0, 1, 1], d[p, 0, 2, 3] = (-1.0, np.nan) if p % 2 else (0.0, np.inf)
        K = np.stack((rng.uniform(0.7, 1.2, z), rng.uniform(0.7, 1.2, z), rng.uniform(0.4, 0.6, z), rng.uniform(0.4, 0.6, z)), 1)
        return {"depth": d, "K": K.astype(dt)}
    x = rng.uniform(-4, 4, s).astype(dt)           # the element-wise training ops
    x[:6] = [0.0, -0.0, np.nan, np.inf, -np.inf, 1e-30]
    return {"x": x, "g": rng.uniform(-1, 1, s).astype(dt)}


def reference(row, a):
    p = row.params
    if row.op == "warp2d":
        return oops.warp2d(a["img"], a["disp"], normalized=p[0], border_mode=p[1], border_value=0.25)
    if row.op == "depth_to_flow":
        return oops.depth_to_flow(a["depth"], a["K"], a["rot"], a["t"], *p)
    if row.op == "flow_to_depth":
        return oops.flow_to_depth2(*(a[k].astype(D) for k in ("flow", "K", "rot", "t")), p[0], p[1], p[2])
    if row.op == "median3x3_downsample":
        return oops.median3x3_downsample(a["x"])
    if row.op == "scale_invariant_gradient":
        return oops.scale_invariant_gradient(a["x"], SIG_DELTAS, SIG_WEIGHTS, 0.001)
    if row.op == "leaky_relu":
        return oops.leaky_relu(a["x"], 0.2)
    if row.op == "scale_invariant_gradient_grad":
        return ref.scale_invariant_gradient_grad(a["g"], a["x"], GRAD_DELTAS, GRAD_WEIGHTS, 0.001)
    if row.op == "depth_to_normals":
        return ref.depth_to_normals(a["depth"], a["K"], p[0])
    if row.op == "leaky_relu_grad":
        return ref.leaky_relu_grad(a["g"], a["x"], 0.2)
    if row.op == "replace_nonfinite":
        return ref.replace_nonfinite(a["x"], -7.5)
    return ref.replace_nonfinite_grad(a["g"], a["x"])


def device(ops, row, a, layout, trace):
    """The op on the device through lmbspecialops, its input in `layout`; returns the output as numpy."""
    dt, p = row.dtype, row.params
    first = "offset" if layout == "offset" else "aligned"
    if row.op == "warp2d":
        img, disp = place(a["img"], first), place(a["disp"], "offset" if layout == "offset-disp" else "aligned")
        return trace(lambda: poisoned(lambda: ops.warp2d(img, disp, normalized=p[0], border_mode=p[1], border_value=0.25), img.numel(), dt))
    if row.op in ("depth_to_flow", "flow_to_depth"):
        x = place(a["depth" if row.op == "depth_to_flow" else "flow"], first)
        K, rot, t = (place(a[k]) for k in ("K", "rot", "t"))
        n, h, w = row.shape
        if row.op == "depth_to_flow":
            return trace(lambda: poisoned(lambda: ops.depth_to_flow(x, K, rot, t, *p), n * 2 * h * w, dt))
        if p[3] == "flow_to_depth":
            call = lambda: ops.flow_to_depth(x, K, rot, t, p[0], p[1], p[2], nowarning=True)   # noqa: E731
        else:
            call = lambda: ops.flow_to_depth2(x, K, rot, t, p[0], p[1], p[2])                  # noqa: E731
        return trace(lambda: poisoned(call, n * h * w, dt))
    if row.op == "median3x3_downsample":
        x = place(a["x"], first)
        h, w = row.shape[-2:]
        return trace(lambda: poisoned(lambda: ops.median3x3_downsample(x), x.numel() // (h * w) * ((h + 1) // 2) * ((w + 1) // 2), dt))
    if row.op == "scale_invariant_gradient":
        x = place(a["x"], first)
        return trace(lambda: poisoned(lambda: ops.scale_invariant_gradient(x, SIG_DELTAS, SIG_WEIGHTS, 0.001), 2 * x.numel(), dt))
    if row.op == "leaky_relu":
        x = place(a["x"], first)
        return trace(lambda: poisoned(lambda: ops.leaky_relu(x, 0.2), x.numel(), dt))
    if row.op == "depth_to_normals":
        d, K = place(a["depth"]), place(a["K"])
        return trace(lambda: poisoned(lambda: ops.depth_to_normals(d, K, p[0]), 3 * d.numel(), dt))
    x, g = place(a["x"]), place(a["g"])
    if row.op == "scale_invariant_gradient_grad":
        call = lambda: ops.scale_invariant_gradient_grad(g, x, GRAD_DELTAS, GRAD_WEIGHTS, 0.001)   # noqa: E731
    elif row.op == "leaky_relu_grad":
        call = lambda: ops.leaky_relu_grad(g, x, 0.2)                                              # noqa: E731
    elif row.op == "replace_nonfinite":
        call = lambda: ops.replace_nonfinite(x, -7.5)                                              # noqa: E731
    else:
        call = lambda: ops.replace_nonfinite_grad(g, x)                                            # noqa: E731
    return trace(lambda: poisoned(call, x.numel(), dt))


def compare(row, got, want, what):
    if row.op == "depth_to_flow" and row.params[0] == "angleaxis3":
        fin = np.isfinite(want)
        assert_close(got, want, 64 * np.finfo(row.dtype).eps * np.abs(want[fin]).max(), what)
    elif row.op == "flow_to_depth":
        assert got.shape == want.shape and got.dtype == row.dtype, what
        assert (got[0, 0, 0, 0] == 0) and (got[1, 0, 5, 7] == 0), "%s: a NaN flow must give depth 0" % what
        flips = ((got != 0) != (want != 0)).mean()
        assert flips < 1e-3, "%s: behind-camera pattern differs on %.3g of the pixels" % (what, flips)
        both = (got != 0) & (want != 0)
        err = np.abs(got[both] - want[both]) / np.abs(want[both])
        assert err.max() < (4e-7 if row.dtype == F else 1e-9), "%s: relative error %g" % (what, err.max())
    elif row.op in TRAINING:
        assert_bits(got.reshape(want.shape), want, what)
    else:
        assert_bits(got, want, what)


# ---- the tests ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("row", ROWS, ids=[r.id for r in ROWS])
def test_row(ops, lib, row, profiler_records_kernels):
    if row.op in TRAINING and not ref.available():
        pytest.skip("neither oracle/_ref nor the stored reference results are present")
    a = data(row)
    want = reference(row, a)
    trace = Trace()
    got = device(ops, row, a, "aligned" if row.layout == "aligned" else row.layout, trace)
    compare(row, got, want, row.id)
    if row.layout != "aligned":     # the same data aligned: the other kernel, the same bits
        got_aligned = device(ops, row, a, "aligned", trace)
        compare(row, got_aligned, want, row.id + " (aligned copy)")
        assert_bits(got_aligned, got, "%s: the v4 kernel and the scalar fallback" % row.id)
    assert lib.demon_debug_tc_timeouts() == 0 and lib.demon_check_errors() == 0
    assert_kernels(trace, row.kernels, profiler_records_kernels, row.id)


def _zeros(*shape):
    return torch.zeros(shape, device="cuda")


# (case, the library's message, call): each launcher refuses a size its grid cannot hold before any launch
REFUSALS = [
    ("warp2d-n", "warp2d: n must be <= 65535", lambda o: o.warp2d(_zeros(65536, 1, 1, 1), _zeros(65536, 2, 1, 1))),
    ("warp2d-h", "warp2d: h must be <= 65535", lambda o: o.warp2d(_zeros(1, 1, 65536, 1), _zeros(1, 2, 65536, 1))),
    ("depth_to_flow-n", "depth_to_flow: n must be <= 65535",
     lambda o: o.depth_to_flow(_zeros(65536, 1, 1), _zeros(65536, 4), _zeros(65536, 3), _zeros(65536, 3))),
    ("flow_to_depth2-n", "flow_to_depth: n must be <= 65535",
     lambda o: o.flow_to_depth2(_zeros(65536, 2, 1, 1), _zeros(65536, 4), _zeros(65536, 3), _zeros(65536, 3))),
    ("median3x3_downsample-h", "median3x3_downsample: (h + 1) / 2 must be <= 65535", lambda o: o.median3x3_downsample(_zeros(1, 131071, 1))),
    ("scale_invariant_gradient-h", "scale_invariant_gradient: h must be <= 65535", lambda o: o.scale_invariant_gradient(_zeros(1, 65536, 1))),
    ("scale_invariant_gradient_grad-h", "scale_invariant_gradient_grad: h must be <= 65535",
     lambda o: o.scale_invariant_gradient_grad(_zeros(1, 2, 65536, 1), _zeros(1, 1, 65536, 1))),
    ("depth_to_normals-h", "depth_to_normals: h must be <= 65535", lambda o: o.depth_to_normals(_zeros(1, 1, 65536, 1), _zeros(1, 4))),
]


@pytest.mark.parametrize("message, call", [r[1:] for r in REFUSALS], ids=[r[0] for r in REFUSALS])
def test_refused_before_any_launch(ops, lib, message, call, profiler_records_kernels):
    launches = lib.demon_launch_count()
    trace = Trace()
    with pytest.raises(ValueError, match=re.escape(message)):
        trace(lambda: call(ops))
    assert lib.demon_launch_count() == launches
    assert lib.demon_check_errors() == 0
    assert_kernels(trace, {}, profiler_records_kernels, message)


# ---- coverage -------------------------------------------------------------------------------------------------------------
CHUNKED = {"median3x3_downsample", "scale_invariant_gradient", "scale_invariant_gradient_grad", "depth_to_normals"}


def features(row):
    """What a row reaches, from its declared kernels (test_row checks each row launches exactly those)."""
    f = {("kernel", k) for k in row.kernels}
    if row.layout != "aligned" and len(row.kernels) == 2:
        f.add(("v4 kernel and scalar fallback at the same width", row.op))
    if row.op in CHUNKED:
        planes = int(np.prod(row.shape[:-2]))
        if planes > CHUNK:
            f |= {("more than one z-chunk", k) for k, n in row.kernels.items() if n == -(-planes // CHUNK)}
    if row.op in ("depth_to_flow", "flow_to_depth"):
        f.add(("rotation format", row.op, row.params[0]))
    return f


def required_targets():
    ks = set()
    for name in ("warp2d_kernel", "depth_to_flow_kernel", "flow_to_depth_kernel", "leaky_relu_kernel", "median3x3_downsample_kernel",
                 "sig_kernel", "sig_grad_kernel", "depth_to_normals_kernel"):
        ks |= {tk(name, t) for t in ("float", "double")} if name != "warp2d_kernel" else {
            tk(name, t, c) for t in ("float", "double") for c in ("true", "false")}
    ks |= {tk("warp2d_v4_kernel", c, "1") for c in ("true", "false")}
    ks |= {"depth_to_flow_v4_kernel", "median3x3_v4_kernel", "sig_v4_kernel"}
    ks |= {tk("elementwise_kernel", t, o) for t in ("float", "double") for o in ("0", "1", "2")}
    t = {("kernel", k) for k in ks}
    t |= {("v4 kernel and scalar fallback at the same width", op)
          for op in ("warp2d", "depth_to_flow", "median3x3_downsample", "scale_invariant_gradient")}
    t |= {("more than one z-chunk", k) for k in ks if k.startswith(("median3x3", "sig", "depth_to_normals"))}
    t |= {("rotation format", op, fmt) for op in ("depth_to_flow", "flow_to_depth") for fmt in FORMATS}
    return t


def test_rows_reach_every_target():
    # every __global__ function of the two sources is among the required kernels
    defined = set()
    for f in ("geometry_ops.cu", "training_ops.cu"):
        with open(os.path.join(CSRC, f)) as fh:
            defined |= set(re.findall(r"__global__\s+void\s+(?:__launch_bounds__\(\d+\)\s+)?(\w+)\(", fh.read()))
    required = required_targets()
    required_names = {k.split("<")[0] for kind, *rest in required if kind == "kernel" for k in rest}
    assert defined == required_names, "kernels of the sources %s, required %s" % (sorted(defined), sorted(required_names))
    reached = set()
    for row in ROWS:
        reached |= features(row)
    missing = sorted(required - reached)
    assert not missing, "targets no row reaches: %s" % missing
