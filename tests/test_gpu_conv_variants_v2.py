"""GPU: every convolution of the v2 network at its own batch, geometry, pitches and offsets, through
demon_conv_slice_nhwc_same (TF 'same' padding) on integer data, bit for bit against float64 -- test_gpu_conv_variants.py's
test_network_layers_exact for v2.  The stride-2 layers read tap sets that v1 has not got (k3 s2: rows 0..2, k7 s2: -2..4,
k9 s2 in the 8-channel mode: -3..5), in the halo, per-tap and cin8 modes of the tensor-core kernel."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from demon_b200 import _lib
from test_conv_variants import FP32, TF32, X3TF32
from test_gpu_conv_variants import PREC_NAME, SENTINEL, assert_bitwise, expected_exact
from test_v2_plan import describe_plan

pytestmark = pytest.mark.gpu


def same_pads(n, k, s):
    out = -(-n // s)
    total = max((out - 1) * s + k - n, 0)
    return total // 2, total - total // 2


def ref64_same(x, k, b, geom):
    """float64 tf.nn.conv2d(padding='SAME') on the device, NHWC in and out, kernel [kh,kw,cin,cout]."""
    kh, kw, sy, sx = geom
    xx = x.double().permute(0, 3, 1, 2)
    py, px = same_pads(xx.shape[2], kh, sy), same_pads(xx.shape[3], kw, sx)
    kt = torch.from_numpy(np.ascontiguousarray(k, np.float64)).cuda().permute(3, 2, 0, 1)
    bt = torch.from_numpy(np.asarray(b, np.float64)).cuda()
    return F.conv2d(F.pad(xx, (px[0], px[1], py[0], py[1])), kt, bt, stride=(sy, sx)).permute(0, 2, 3, 1)


def run_slice_same(x, in_off, in_pitch, k, b, Cout, out_off, out_pitch, geom, leaky, precision):
    """test_gpu_conv_variants.run_slice through the 'same' entry: NaN around the input slice, sentinels around the output."""
    B, H, W, Cin = x.shape
    kh, kw, sy, sx = geom
    Ho, Wo = -(-H // sy), -(-W // sx)
    xin = torch.full((B + 1, H, W, in_pitch), float("nan"), device="cuda")
    xin[:B, :, :, in_off:in_off + Cin] = x
    out_bits = torch.full((B + 1, Ho, Wo, out_pitch), SENTINEL, dtype=torch.int32, device="cuda")
    out = out_bits.view(torch.float32)
    out[:B, :, :, out_off:out_off + Cout] = float("nan")
    kk, bb = np.ascontiguousarray(k, np.float32), np.ascontiguousarray(b, np.float32)
    lib = _lib.load()
    _lib.check(lib.demon_conv_slice_nhwc_same(xin.data_ptr() + 4 * in_off, in_pitch, out.data_ptr() + 4 * out_off, out_pitch, B, H, W,
                                              Cin, Cout, kh, kw, sy, sx, kk.ctypes.data, bb.ctypes.data, int(leaky), precision,
                                              ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    assert lib.demon_check_errors() == 0
    guard = out_bits.clone()
    guard[:B, :, :, out_off:out_off + Cout] = SENTINEL
    assert (guard != SENTINEL).sum().item() == 0, "guard words written"
    got = out[:B, :, :, out_off:out_off + Cout]
    assert not torch.isnan(got).any(), "output elements never written"
    return got


def plan_of(text):
    """The planner's part of a v2 describe line's tail ('tap0 dy dx : <plan>')."""
    return text.split(" : ", 1)[1] if text.startswith("tap0") else text


NET_CONFIGS = {"b64": (64, (192, 256), ""), "b1": (1, (192, 256), ""), "refine1024": (8, (768, 1024), "netRefine/"),
               "refine200x300": (2, (200, 300), "netRefine/")}


@pytest.mark.parametrize("config", sorted(NET_CONFIGS))
def test_v2_network_convs_exact(config):
    """Every v2 conv (the transposed convs are v1's and covered there) at each precision the net runs it in: tensor-core
    layers at 3xTF32 and TF32, the others on the fp32 SIMT path, and every layer at fp32.  Padding channels past cin hold
    finite nonzero values with zero weights.  predict_depthnormal2/conv2 is checked without its per-image scale."""
    batch, refine_hw, prefix = NET_CONFIGS[config]
    jobs = {}
    for prec in (FP32, X3TF32, TF32):
        for name, (g, tap0, text) in describe_plan(2, batch, refine_hw, prec).items():
            if g["kind"] != "conv" or not name.startswith(prefix):
                continue
            plan = plan_of(text)
            key = tuple(sorted((k, v) for k, v in g.items() if k != "kind"))
            names, precs = jobs.setdefault(key, (set(), {}))
            names.add(name)
            precs[prec if plan != "simt" or prec == FP32 else FP32] = plan
    assert sum(1 for _, precs in jobs.values() if any(p != "simt" for p in precs.values())) > 0
    gen = torch.Generator(device="cuda")
    for i, (key, (names, precs)) in enumerate(sorted(jobs.items())):
        g = dict(key)
        geom = (g["kh"], g["kw"], g["sy"], g["sx"])
        cin, cb, cout = g["cin"], g["cin_buf"], g["cout"]
        gen.manual_seed(i)
        x = torch.randint(-1, 2, (batch, g["H"], g["W"], cb), generator=gen, device="cuda").float()
        if cb > cin:
            x[..., cin:] = torch.randint(0, 2, (batch, g["H"], g["W"], cb - cin), generator=gen, device="cuda").float() * 2 - 1
        rng = np.random.default_rng(i)
        k = rng.integers(-1, 2, (g["kh"], g["kw"], cb, cout)).astype(np.float32)
        k[:, :, cin:, :] = 0
        b = rng.integers(-2, 3, cout).astype(np.float32)
        want = expected_exact(ref64_same(x, k, b, geom), g["leaky"])
        for prec, plan in sorted(precs.items()):
            got = run_slice_same(x, g["in_off"], g["in_pitch"], k, b, cout, g["out_off"], g["out_pitch"], geom, g["leaky"], prec)
            assert_bitwise(got, want, "%s at %s (%s)" % (sorted(names), PREC_NAME[prec], plan))
        del x, want


@pytest.mark.parametrize("k,s,n", [(3, 2, 12), (5, 2, 24), (7, 2, 96), (9, 2, 192), (3, 2, 13), (5, 1, 7), (3, 2, 50)])
def test_same_padding_tap_sets_exact(k, s, n):
    """Separable y and x convs with the stride-2 tap sets of v2, on even and odd sizes, 3xTF32 and fp32, bit for bit."""
    rng = np.random.default_rng(k * 100 + n)
    B, C, Cout = 2, 32, 32
    for geom, H, W in (((k, 1, s, 1), n, 16), ((1, k, 1, s), 16, n)):
        x = torch.from_numpy(rng.integers(-1, 2, (B, H, W, C)).astype(np.float32)).cuda()
        kk = rng.integers(-1, 2, geom[:2] + (C, Cout)).astype(np.float32)
        b = rng.integers(-2, 3, Cout).astype(np.float32)
        want = expected_exact(ref64_same(x, kk, b, geom), True)
        # the tensor-core path takes strided inputs whose size the stride divides; others run on the fp32 SIMT path only
        for prec in ((X3TF32, FP32) if n % s == 0 else (FP32,)):
            got = run_slice_same(x, 0, C, kk, b, Cout, 0, Cout, geom, True, prec)
            assert_bitwise(got, want, "k%d s%d n%d %s %s" % (k, s, n, geom, PREC_NAME[prec]))
