"""GPU: every variant of the tensor-core convolution, and every convolution layer of the network at its own batch, geometry and
channel slices, through the slice entry (demon_conv_slice_nhwc), compared with a float64 reference.

Every call reads its input from a channel slice of a wider buffer with one extra trailing image, all NaN outside the slice,
and writes its output slice into a buffer whose channels on both sides and trailing image hold a sentinel bit pattern, the
slice itself NaN before the call.  After each call every guard word is bit-unchanged, no NaN is left in the slice and no
pipeline wait of the kernel timed out (demon_check_errors).

On the exact datasets of tests/test_conv_variants.py, 3xTF32 (and on `int` also single-pass TF32 and the fp32 SIMT path)
equals float32(leaky(float64 reference)) bit for bit, so a mismatch names the variant and the element where it broke."""
import ctypes
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from demon_b200 import _lib
from test_conv_variants import (DATASETS, FP32, TF32, TC_PRECISIONS, VARIANTS, X3TF32, describe, exact_data, geometry, pitches,
                                tc_error_bound)

pytestmark = pytest.mark.gpu

SENTINEL = -0x5A5A5A5B   # 0xA5A5A5A5 as int32: a float no kernel computes here
PREC_NAME = {FP32: "fp32", X3TF32: "3xtf32", TF32: "tf32"}


def run_slice(x, in_off, in_pitch, k, b, Cout, out_off, out_pitch, geom, deconv, leaky, precision):
    """Runs the slice entry on x ([B,H,W,Cin] float32, device) placed at channel in_off of a NaN buffer of pitch in_pitch,
    checks the guards and returns the output slice ([B,Ho,Wo,Cout] float32, device)."""
    B, H, W, Cin = x.shape
    kh, kw, sy, sx = geom
    Ho, Wo = (2 * H, 2 * W) if deconv else (-(-H // sy), -(-W // sx))
    xin = torch.full((B + 1, H, W, in_pitch), float("nan"), device="cuda")
    xin[:B, :, :, in_off:in_off + Cin] = x
    out_bits = torch.full((B + 1, Ho, Wo, out_pitch), SENTINEL, dtype=torch.int32, device="cuda")
    out = out_bits.view(torch.float32)
    out[:B, :, :, out_off:out_off + Cout] = float("nan")
    kk = np.ascontiguousarray(k, np.float32)
    bb = np.ascontiguousarray(b, np.float32)
    lib = _lib.load()
    _lib.check(lib.demon_conv_slice_nhwc(xin.data_ptr() + 4 * in_off, in_pitch, out.data_ptr() + 4 * out_off, out_pitch, B, H, W, Cin,
                                         Cout, kh, kw, sy, sx, int(deconv), kk.ctypes.data, bb.ctypes.data, int(leaky), precision,
                                         ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    assert lib.demon_check_errors() == 0, "a pipeline wait timed out or a CUDA error is pending"
    guard = out_bits.clone()
    guard[:B, :, :, out_off:out_off + Cout] = SENTINEL
    bad = (guard != SENTINEL).nonzero()
    assert bad.shape[0] == 0, "%d guard words written, first at [n, y, x, channel] %s" % (bad.shape[0], bad[0].tolist())
    got = out[:B, :, :, out_off:out_off + Cout]
    nan = torch.isnan(got).nonzero()
    assert nan.shape[0] == 0, "%d output elements never written, first at %s" % (nan.shape[0], nan[0].tolist())
    return got


def ref64(x, k, b, geom, deconv):
    """float64 convolution on the device: caffe-padded conv2d with kernel [kh,kw,cin,cout], or the k4 s2 transposed conv
    (padding 1) with kernel [4,4,cout,cin]; NHWC in and out."""
    kh, kw, sy, sx = geom
    xx = x.double().permute(0, 3, 1, 2)
    kt = torch.from_numpy(np.ascontiguousarray(k, np.float64)).cuda().permute(3, 2, 0, 1)
    bt = torch.from_numpy(np.asarray(b, np.float64)).cuda()
    if deconv:
        y = F.conv_transpose2d(xx, kt, bt, stride=2, padding=1)
    else:
        y = F.conv2d(F.pad(xx, (kw // 2, kw // 2, kh // 2, kh // 2)), kt, bt, stride=(sy, sx))
    return y.permute(0, 2, 3, 1)


def expected_exact(y64, leaky):
    """float32(y64), then the kernel's leaky ReLU as its two float32 operations max(0.1f * y, y)."""
    y = y64.float()
    return torch.maximum(torch.tensor(0.1, dtype=torch.float32, device=y.device) * y, y) if leaky else y


def assert_bitwise(got, want, what):
    g = (got + 0.0).view(torch.int32)   # + 0.0: -0 and +0 compare as one value
    w = (want + 0.0).view(torch.int32)
    bad = (g != w).nonzero()
    if bad.shape[0]:
        i = tuple(bad[0].tolist())
        pytest.fail("%s: %d of %d elements differ, first at [n, y, x, channel] %s: got %r, want %r"
                    % (what, bad.shape[0], g.numel(), list(i), got[i].item(), want[i].item()))


def weight_shape(Cin, Cout, geom, deconv):
    kh, kw = geom[:2]
    return (4, 4, Cout, Cin) if deconv else (kh, kw, Cin, Cout)


def row_id(row):
    B, H, W, Cin, Cout, kh, kw, sy, sx, deconv, in_off, out_off = row
    op = "deconv" if deconv else "k%dx%ds%dx%d" % (kh, kw, sy, sx)
    return "B%d_%dx%d_%d-%d_%s_in%d_out%d" % (B, H, W, Cin, Cout, op, in_off, out_off)


# ---- every variant, exact data ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("dataset", DATASETS)
@pytest.mark.parametrize("row", VARIANTS, ids=[row_id(r) for r in VARIANTS])
def test_variant_exact(row, dataset):
    B, H, W, Cin, Cout, _, _, _, _, deconv, in_off, out_off = row
    geom = geometry(row)
    in_pitch, out_pitch = pitches(row)
    leaky = VARIANTS.index(row) % 2 == 0
    rng = np.random.default_rng([VARIANTS.index(row), DATASETS.index(dataset)])
    x, k, b = exact_data(dataset, (B, H, W, Cin), weight_shape(Cin, Cout, geom, deconv), Cout, rng)
    xd = torch.from_numpy(x).cuda()
    want = expected_exact(ref64(xd, k, b, geom, deconv), leaky)

    def run(prec):
        return run_slice(xd, in_off, in_pitch, k, b, Cout, out_off, out_pitch, geom, deconv, leaky, prec)

    plan = describe(row, X3TF32)["text"]
    assert_bitwise(run(X3TF32), want, "3xTF32, plan %s" % plan)
    assert_bitwise(run(FP32), want, "fp32 SIMT")
    got1 = run(TF32)
    if dataset == "int":
        assert_bitwise(got1, want, "TF32, plan %s" % describe(row, TF32)["text"])
    else:   # single pass truncates the 2^-11 parts away: the dataset does go through the lo terms
        assert not torch.equal(got1, want), "TF32 reproduced the %s dataset, which needs the 3xTF32 lo terms" % dataset


# ---- every variant, realistic data: a per-element bound from the arithmetic ---------------------------------------------
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    yield
    for prec, (ratio, bound_ratio, row) in sorted(WORST.items()):
        print("\nrealistic data, %s: largest |err| / S = %.3g (%.3g of the bound) at %s" % (PREC_NAME[prec], ratio, bound_ratio, row_id(row)))


def log_uniform(shape, rng):
    return (rng.choice((-1.0, 1.0), shape) * np.exp2(rng.uniform(-8, 8, shape))).astype(np.float32)


@pytest.mark.parametrize("precision", TC_PRECISIONS, ids=["3xtf32", "tf32"])
@pytest.mark.parametrize("row", VARIANTS, ids=[row_id(r) for r in VARIANTS])
def test_variant_realistic(row, precision):
    """Random signs, magnitudes log-uniform in 2^-8 .. 2^8 (x, w and bias), under the per-element bound |err| <= bound * S of
    tests/test_conv_variants.py: tc_error_bound (S = sum |x||w| + |b| over the terms of an output element).

    The split terms of that bound follow from the operand formats alone.  The accumulation terms do not: NVIDIA does not
    document how a wgmma rounds its internal sum, and "at most one float32 ulp of S per wgmma" is an assumption about Hopper's
    tensor cores that rests on measurement, not on a derivation.  On an H100 (seeds as below) the largest |err| / S was 4.7e-6
    for 3xTF32, under a tenth of its bound, where the accumulation terms dominate; and 1.8e-3 for TF32, 0.91 of its bound, where
    the operand truncation (a hard bound: a product of two truncated operands is never off by 2^-9 of itself) dominates.
    """
    B, H, W, Cin, Cout, kh, kw, _, _, deconv, in_off, out_off = row
    geom = geometry(row)
    in_pitch, out_pitch = pitches(row)
    leaky = VARIANTS.index(row) % 2 == 1
    rng = np.random.default_rng([VARIANTS.index(row), 7])
    x = log_uniform((B, H, W, Cin), rng)
    k = log_uniform(weight_shape(Cin, Cout, geom, deconv), rng)
    b = log_uniform((Cout,), rng)
    xd = torch.from_numpy(x).cuda()
    y = ref64(xd, k, b, geom, deconv)
    S = ref64(xd.abs(), np.abs(k), np.abs(b), geom, deconv)
    if leaky:
        y = torch.maximum(float(np.float32(0.1)) * y, y)
    got = run_slice(xd, in_off, in_pitch, k, b, Cout, out_off, out_pitch, geom, deconv, leaky, precision).double()
    d = describe(row, precision)
    bound = tc_error_bound(precision, Cin, kh, kw, deconv, d["ksplit"])
    ratio = ((got - y).abs() / S).max().item()
    if ratio > WORST.get(precision, (-1,))[0]:
        WORST[precision] = (ratio, ratio / bound, row)
    over = ((got - y).abs() > bound * S).nonzero()
    if over.shape[0]:
        i = tuple(over[0].tolist())
        pytest.fail("%d elements over the bound %.3g S, first at [n, y, x, channel] %s: got %r, float64 %r, S %r; plan %s"
                    % (over.shape[0], bound, list(i), got[i].item(), y[i].item(), S[i].item(), d["text"]))
    if precision == TF32:   # the bound has to separate the two modes, or it says nothing about the 3xTF32 lo terms
        assert ratio > 2.0 ** -19


# ---- the network's own layers ---------------------------------------------------------------------------------------
_LAYER_RE = re.compile(r"^(\S+)\s+(conv|deconv|dense) H (\d+) W (\d+) cin (\d+) cin_buf (\d+) in_pitch (\d+) in_off (\d+) cout (\d+) "
                       r"out_pitch (\d+) out_off (\d+) kh (\d+) kw (\d+) sy (\d+) sx (\d+) leaky (\d) scale (\d) : (.*)$")
_KEYS = ("H", "W", "cin", "cin_buf", "in_pitch", "in_off", "cout", "out_pitch", "out_off", "kh", "kw", "sy", "sx", "leaky", "scale")


def net_layers(batch, refine_hw, precision):
    """[(name, kind, geometry dict, plan text)] of every layer of a net, from demon_debug_describe_layers."""
    lib = _lib.load()
    ptr = ctypes.c_void_p()
    _lib.check(lib.demon_net_create(ctypes.byref(ptr), batch, refine_hw[0], refine_hw[1], precision))
    try:
        return describe_layers(ptr)
    finally:
        lib.demon_net_destroy(ptr)


def describe_layers(ptr):
    """net_layers of the net `ptr` (a demon_net*)."""
    lib = _lib.load()
    n = lib.demon_net_num_layers(ptr)
    buf = ctypes.create_string_buffer(1 << 20)
    lib.demon_debug_describe_layers(ptr, buf, 1 << 20)
    lines = buf.value.decode().splitlines()
    assert len(lines) == n
    out = []
    for line in lines:
        m = _LAYER_RE.match(line)
        assert m, line
        g = dict(zip(_KEYS, (int(v) for v in m.groups()[2:17])))
        out.append((m.group(1), m.group(2), g, m.group(18)))
    return out


# (batch, refinement block size, which layers): bench.py's three workloads
NET_CONFIGS = {"b64": (64, (192, 256), ""), "b1": (1, (192, 256), ""), "refine1024": (8, (768, 1024), "netRefine/")}


@pytest.mark.parametrize("config", sorted(NET_CONFIGS))
def test_network_layers_exact(config):
    """Every conv and transposed conv of the net, at the net's batch, geometry, pitches and offsets, on the `int` dataset:
    bit for bit at each precision the net runs it in (tensor-core layers at 3xTF32 and TF32, the others on the fp32 SIMT
    path, and every layer at fp32).  Input channels past cin (cin_buf > cin: 6 -> 8, 4 -> 8, 7/8/9 -> 32, 514 -> 576) hold
    finite nonzero values and get zero weights: padding channels must be finite, their weights are zero (conv.cuh).
    One exception: the slice entry has no per-image scale, so a layer with one (predict_depthnormal2/conv2, whose channel 0
    the net multiplies by the predicted scale; fp32 SIMT path) is checked as the plain convolution it is before that.
    Dense layers (motion_fc*) are not convolutions over an image and are left out."""
    batch, refine_hw, prefix = NET_CONFIGS[config]
    jobs = {}   # geometry -> (names, {precision: plan})
    for prec in (FP32, X3TF32, TF32):
        for name, kind, g, plan in net_layers(batch, refine_hw, prec):
            if kind == "dense" or not name.startswith(prefix):
                continue
            key = (kind,) + tuple(g[k] for k in _KEYS)
            names, precs = jobs.setdefault(key, (set(), {}))
            names.add(name)
            precs[prec if plan != "simt" or prec == FP32 else FP32] = plan
    assert any(p != "simt" for _, precs in jobs.values() for p in precs.values())
    gen = torch.Generator(device="cuda")
    for i, (key, (names, precs)) in enumerate(sorted(jobs.items())):
        deconv = key[0] == "deconv"
        g = dict(zip(_KEYS, key[1:]))
        geom = (g["kh"], g["kw"], g["sy"], g["sx"])
        cin, cb, cout = g["cin"], g["cin_buf"], g["cout"]
        gen.manual_seed(i)
        x = torch.randint(-1, 2, (batch, g["H"], g["W"], cb), generator=gen, device="cuda").float()
        if cb > cin:   # padding channels: finite, nonzero
            x[..., cin:] = torch.randint(0, 2, (batch, g["H"], g["W"], cb - cin), generator=gen, device="cuda").float() * 2 - 1
        rng = np.random.default_rng(i)
        k = rng.integers(-1, 2, weight_shape(cb, cout, geom, deconv)).astype(np.float32)
        if deconv:
            k[..., cin:] = 0
        else:
            k[:, :, cin:, :] = 0
        b = rng.integers(-2, 3, cout).astype(np.float32)
        want = expected_exact(ref64(x, k, b, geom, deconv), g["leaky"])
        for prec, plan in sorted(precs.items()):
            got = run_slice(x, g["in_off"], g["in_pitch"], k, b, cout, g["out_off"], g["out_pitch"], geom, deconv, g["leaky"], prec)
            assert_bitwise(got, want, "%s at %s (%s)" % (sorted(names), PREC_NAME[prec], plan))
        del x, want
