"""GPU: the convolution kernels through the C-ABI test entries, against torch-CPU float64 convolutions
of the same tensors (the definitionally correct result).  fp32 SIMT path: fp32 rounding only.  tensor-core
path: 3xTF32 must be fp32-grade, single-pass TF32 is the flagged fast mode (~1e-3)."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from demon_b200 import _lib

FP32, X3TF32, TF32 = 0, 1, 2


def run_conv(x_nhwc, k_tf, b, sy, sx, leaky, precision):
    lib = _lib.load()
    B, H, W, Cin = x_nhwc.shape
    kh, kw, _, Cout = k_tf.shape
    xin = torch.from_numpy(x_nhwc).cuda()
    Ho, Wo = -(-H // sy), -(-W // sx)
    out = torch.full((B, Ho, Wo, Cout), float("nan"), device="cuda")
    k = np.ascontiguousarray(k_tf, np.float32)
    bb = np.ascontiguousarray(b, np.float32)
    _lib.check(lib.demon_conv2d_nhwc(xin.data_ptr(), out.data_ptr(), B, H, W, Cin, Cout, kh, kw, sy, sx,
                                     k.ctypes.data, bb.ctypes.data, int(leaky), precision,
                                     ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    return out.cpu().numpy()


def ref_conv(x_nhwc, k_tf, b, sy, sx, leaky):
    x = torch.from_numpy(x_nhwc).double().permute(0, 3, 1, 2)
    k = torch.from_numpy(k_tf).double().permute(3, 2, 0, 1)
    kh, kw = k_tf.shape[:2]
    y = F.conv2d(F.pad(x, (kw // 2, kw // 2, kh // 2, kh // 2)), k, torch.from_numpy(b).double(), stride=(sy, sx))
    if leaky:
        y = torch.maximum(0.1 * y, y)
    return y.permute(0, 2, 3, 1).numpy()


def run_deconv(x_nhwc, k_tf, b, leaky, precision):
    lib = _lib.load()
    B, H, W, Cin = x_nhwc.shape
    Cout = k_tf.shape[2]
    xin = torch.from_numpy(x_nhwc).cuda()
    out = torch.full((B, 2 * H, 2 * W, Cout), float("nan"), device="cuda")
    k = np.ascontiguousarray(k_tf, np.float32)
    bb = np.ascontiguousarray(b, np.float32)
    _lib.check(lib.demon_deconv4x4s2_nhwc(xin.data_ptr(), out.data_ptr(), B, H, W, Cin, Cout, k.ctypes.data, bb.ctypes.data,
                                          int(leaky), precision, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    return out.cpu().numpy()


def ref_deconv(x_nhwc, k_tf, b, leaky):
    x = torch.from_numpy(x_nhwc).double().permute(0, 3, 1, 2)
    k = torch.from_numpy(k_tf).double().permute(3, 2, 0, 1)     # [kh,kw,cout,cin] -> [cin,cout,kh,kw]
    y = F.conv_transpose2d(x, k, torch.from_numpy(b).double(), stride=2, padding=1)
    if leaky:
        y = torch.maximum(0.1 * y, y)
    return y.permute(0, 2, 3, 1).numpy()


def rel_err(a, r):
    return np.abs(a - r).max() / np.abs(r).max()


# (B, H, W, Cin, Cout, kh, kw, sy, sx): every layer family of the DeMoN graphs, small spatial sizes
SIMT_CASES = [
    (2, 20, 24, 8, 32, 9, 1, 2, 1),     # conv1y (6 -> 8 padded channels)
    (2, 12, 40, 32, 32, 1, 9, 1, 2),    # conv1x
    (1, 13, 9, 12, 32, 3, 1, 1, 1),     # conv2_extra_inputsy, odd sizes
    (2, 6, 8, 64, 64, 1, 3, 1, 1),
    (2, 12, 16, 128, 256, 5, 1, 2, 1),  # conv4y
    (3, 6, 8, 512, 24, 3, 3, 1, 1),     # predict_flow5/conv1
    (3, 6, 8, 24, 4, 3, 3, 1, 1),       # predict_flow5/conv2
    (1, 16, 20, 4, 32, 3, 3, 1, 1),     # netRefine/conv0
    (1, 16, 20, 32, 64, 3, 3, 2, 2),    # netRefine/conv1
    (1, 10, 12, 16, 1, 3, 3, 1, 1),     # predict_depth0/conv2
    (2, 9, 150, 16, 1, 3, 3, 1, 1),     # same head, several pixel groups per CTA and a ragged last one
    (1, 7, 37, 32, 1, 3, 3, 1, 1),      # eight lanes per pixel
    (1, 8, 20, 16, 1, 3, 1, 1, 1),      # run-time tap loop of the lane-sharing kernel
    (2, 5, 70, 24, 4, 3, 3, 1, 1),      # 24 -> 4 head, wider than one CTA
    (5, 1, 1, 256, 7, 1, 1, 1, 1),      # dense as 1x1 conv
]


@pytest.mark.parametrize("case", SIMT_CASES)
def test_simt_conv_matches_float64(case):
    B, H, W, Cin, Cout, kh, kw, sy, sx = case
    rng = np.random.RandomState(sum(case))
    x = rng.uniform(-1, 1, (B, H, W, Cin)).astype(np.float32)
    k = (rng.standard_normal((kh, kw, Cin, Cout)) / np.sqrt(kh * kw * Cin)).astype(np.float32)
    b = rng.uniform(-0.1, 0.1, Cout).astype(np.float32)
    for leaky in (False, True):
        got = run_conv(x, k, b, sy, sx, leaky, FP32)
        ref = ref_conv(x, k, b, sy, sx, leaky)
        assert got.shape == ref.shape
        assert rel_err(got, ref) < 5e-6, rel_err(got, ref)     # fp32 accumulation over up to 4608 terms


@pytest.mark.parametrize("case", [(2, 6, 8, 512, 256), (1, 12, 16, 516, 128), (2, 5, 7, 4, 2), (1, 24, 32, 128, 32)])
def test_simt_deconv_matches_float64(case):
    B, H, W, Cin, Cout = case
    rng = np.random.RandomState(sum(case))
    x = rng.uniform(-1, 1, (B, H, W, Cin)).astype(np.float32)
    k = (rng.standard_normal((4, 4, Cout, Cin)) / np.sqrt(4 * Cin)).astype(np.float32)
    b = rng.uniform(-0.1, 0.1, Cout).astype(np.float32)
    got = run_deconv(x, k, b, True, FP32)
    ref = ref_deconv(x, k, b, True)
    assert got.shape == ref.shape and rel_err(got, ref) < 5e-6


# shapes the tensor-core path takes (Cin % 32 == 0, Cout >= 16)
TC_CASES = [
    (2, 32, 16, 8, 32, 9, 1, 2, 1),      # conv1y: 8-channel mode (4 taps per K step)
    (1, 32, 24, 8, 32, 3, 3, 1, 1),      # netRefine/conv0 (4 -> 8 padded channels)
    (2, 12, 40, 32, 32, 1, 9, 1, 2),     # conv1x
    (2, 24, 16, 32, 32, 7, 1, 2, 1),     # conv2y
    (2, 8, 16, 64, 64, 3, 1, 1, 1),      # conv2_1y
    (2, 8, 16, 64, 64, 1, 3, 1, 1),
    (2, 24, 32, 64, 128, 5, 1, 2, 1),    # conv3y
    (3, 12, 16, 128, 256, 1, 5, 1, 2),   # conv4x, 3 images (ragged tile)
    (3, 6, 8, 512, 512, 3, 1, 1, 1),     # conv5_1y, 6x8 images
    (3, 6, 8, 512, 24, 3, 3, 1, 1),      # predict_flow5/conv1 (Cout 24 -> N 32)
    (2, 12, 12, 128, 24, 3, 3, 1, 1),    # predict_*2/conv1
    (1, 16, 24, 32, 64, 3, 3, 2, 2),     # netRefine/conv1
    (1, 16, 24, 64, 64, 3, 3, 1, 1),     # netRefine/conv1_1
    (1, 24, 40, 64, 16, 3, 3, 1, 1),     # predict_depth0/conv1
    (1, 19, 21, 64, 64, 3, 3, 1, 1),     # sizes that do not divide the tile
]


@pytest.mark.parametrize("case", TC_CASES)
def test_tc_conv_3xtf32_is_fp32_grade(case):
    B, H, W, Cin, Cout, kh, kw, sy, sx = case
    rng = np.random.RandomState(sum(case) + 1)
    x = rng.uniform(-1, 1, (B, H, W, Cin)).astype(np.float32)
    k = (rng.standard_normal((kh, kw, Cin, Cout)) / np.sqrt(kh * kw * Cin)).astype(np.float32)
    b = rng.uniform(-0.1, 0.1, Cout).astype(np.float32)
    try:
        got = run_conv(x, k, b, sy, sx, True, X3TF32)
    except ValueError as e:
        pytest.skip("shape not on the tensor-core path: %s" % e)
    ref = ref_conv(x, k, b, sy, sx, True)
    simt = run_conv(x, k, b, sy, sx, True, FP32)
    assert got.shape == ref.shape
    assert not np.isnan(got).any()
    e_tc, e_simt = rel_err(got, ref), rel_err(simt, ref)
    assert e_tc < 5e-5, (e_tc, e_simt)      # 3xTF32: dropped lo*lo term and tf32 truncation of the lo parts, ~2^-21 per product
    got1 = run_conv(x, k, b, sy, sx, True, TF32)
    assert rel_err(got1, ref) < 5e-3
    assert _lib.load().demon_debug_tc_timeouts() == 0


# transposed convs: per-tap mode at low resolution (refine4/3/2 shapes; 17 chunks: a prime K loop that cannot be split, 18 chunks:
# the 576-channel concat4 of the pipeline, split-K at small batch), halo mode on whole 16x8 tiles (refine0: four stacked
# classes of N = 32; refine1: four classes of N = 64, three-instruction mode)
TC_DECONV_CASES = [(2, 6, 8, 512, 256), (1, 12, 16, 256, 128), (1, 24, 32, 128, 32), (2, 12, 16, 128, 64), (1, 12, 16, 544, 128),
                   (1, 12, 16, 576, 128), (2, 12, 16, 576, 128),
                   (3, 24, 32, 256, 64), (1, 32, 16, 128, 32), (2, 16, 24, 128, 64), (1, 16, 8, 32, 16)]


def test_split_k_plans_are_what_the_tests_exercise():
    """The halo planner splits the K loop of layers with few tiles (low resolution, small batch); the cases below and in
    TC_DECONV_CASES therefore run the two-pass path (partial sums + halo_splitk_reduce_kernel).  No device needed."""
    import ctypes
    lib = _lib.load()
    buf = ctypes.create_string_buffer(4096)

    def plan(B, H, W, Cin, Cout, kh, kw, sy, sx, deconv):
        lib.demon_debug_describe_conv(B, H, W, Cin, Cin, Cout, Cout, kh, kw, sy, sx, deconv, X3TF32, buf, 4096)
        return buf.value.decode()

    assert "ksplit 8" in plan(2, 6, 8, 512, 256, 4, 4, 2, 2, 1)        # refine4 at batch 2: 4 tiles, 160 steps
    assert "ksplit 1 " in plan(1, 12, 16, 544, 128, 4, 4, 2, 2, 1)     # 17 chunks: prime
    assert "ksplit 1 " not in plan(1, 12, 16, 576, 128, 4, 4, 2, 2, 1)
    assert "ksplit 1 " not in plan(3, 6, 8, 512, 24, 3, 3, 1, 1, 0)     # predict_flow5/conv1
    assert "ksplit 1 " in plan(64, 48, 64, 128, 24, 3, 3, 1, 1, 0)      # plenty of tiles: no split


@pytest.mark.parametrize("case", TC_DECONV_CASES)
def test_tc_deconv_3xtf32_is_fp32_grade(case):
    B, H, W, Cin, Cout = case
    rng = np.random.RandomState(sum(case) + 2)
    x = rng.uniform(-1, 1, (B, H, W, Cin)).astype(np.float32)
    k = (rng.standard_normal((4, 4, Cout, Cin)) / np.sqrt(4 * Cin)).astype(np.float32)
    b = rng.uniform(-0.1, 0.1, Cout).astype(np.float32)
    try:
        got = run_deconv(x, k, b, True, X3TF32)
    except ValueError as e:
        pytest.skip("shape not on the tensor-core path: %s" % e)
    ref = ref_deconv(x, k, b, True)
    assert got.shape == ref.shape and not np.isnan(got).any()
    assert rel_err(got, ref) < 2e-5, rel_err(got, ref)
    got1 = run_deconv(x, k, b, True, TF32)
    assert rel_err(got1, ref) < 5e-3
    assert _lib.load().demon_debug_tc_timeouts() == 0
