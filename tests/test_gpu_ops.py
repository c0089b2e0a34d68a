"""GPU: the sm_90a geometry-op kernels against the CPU oracle, through the C ABI (via the
lmbspecialops mirror).  Bit exact where the arithmetic is comparison / IEEE only, a few ulp where libm
(sin/cos) or a different least-squares solver is involved; tolerances are written at each assert."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import ops as oops

TYPES = (np.float32, np.float64)


@pytest.fixture(scope="module")
def ops():
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    from demon_b200 import lmbspecialops
    return lmbspecialops


def eps(dtype):
    return np.finfo(dtype).eps


# ---- median3x3_downsample: bit exact ------------------------------------------------------------
@pytest.mark.parametrize("dtype", TYPES)
def test_median_reference_kats(ops, dtype, golden_dir):
    z = np.load(os.path.join(golden_dir, "reference_kats.npz"))
    assert np.array_equal(ops.median3x3_downsample(z["median_in_single"].astype(dtype)), z["median_out_single"].astype(dtype))
    A = z["median_in_1d"].astype(dtype)
    assert np.array_equal(ops.median3x3_downsample(A), z["median_out_1d"].astype(dtype))
    assert np.array_equal(ops.median3x3_downsample(A.T.copy()), z["median_out_1d"].astype(dtype).T)


@pytest.mark.parametrize("dtype", TYPES)
@pytest.mark.parametrize("shape", [(10, 13), (3, 192, 256), (2, 3, 7, 5), (1, 1), (1, 9), (5, 2, 2, 1, 6)])
def test_median_bit_exact(ops, dtype, shape):
    rng = np.random.RandomState(sum(shape))
    A = rng.rand(*shape).astype(dtype)
    A = np.round(A * 8) / 8        # many ties
    assert np.array_equal(ops.median3x3_downsample(A), oops.median3x3_downsample(A))


def test_median_with_nans_selects_the_reference_element(ops):
    rng = np.random.RandomState(0)
    A = rng.rand(2, 31, 33).astype(np.float32)
    A[rng.rand(*A.shape) < 0.15] = np.nan
    g, r = ops.median3x3_downsample(A), oops.median3x3_downsample(A)
    assert np.array_equal(np.isnan(g), np.isnan(r)) and np.array_equal(g[~np.isnan(g)], r[~np.isnan(r)])


@pytest.mark.parametrize("shape", [(2, 32, 256), (1, 3, 33, 264), (3, 7, 512)])
def test_median_vector_path_bit_exact_with_nans_and_ties(ops, shape):
    """float, W a multiple of 8 and >= 256: the four-outputs-per-thread kernel (odd heights, NaNs, ties, signed zeros)."""
    rng = np.random.RandomState(sum(shape))
    A = (np.round(rng.rand(*shape) * 6) / 6 - 0.5).astype(np.float32)
    A[rng.rand(*shape) < 0.1] = np.nan
    A[rng.rand(*shape) < 0.05] = -0.0
    A[rng.rand(*shape) < 0.05] = 0.0
    g, r = ops.median3x3_downsample(A), oops.median3x3_downsample(A)
    assert g.shape == r.shape
    assert np.array_equal(np.isnan(g), np.isnan(r))
    m = ~np.isnan(r)
    assert np.array_equal(g[m].view(np.uint32), r[m].view(np.uint32))


@pytest.mark.parametrize("shape", [(2, 64, 256), (1, 2, 35, 512)])
def test_median_vector_path_min_max_network_bit_exact(ops, shape):
    """No NaN, no zero: the vector kernel takes its min/max network (sorted columns shared by the four windows) instead of
    the reference's selection passes; the selected VALUE, hence the bits, must be the same -- heavy ties, both signs."""
    rng = np.random.RandomState(7 + sum(shape))
    A = (np.round(rng.rand(*shape) * 5) / 5 + 0.1).astype(np.float32) * rng.choice([-1.0, 1.0], size=shape).astype(np.float32)
    assert not np.any(A == 0)
    g, r = ops.median3x3_downsample(A), oops.median3x3_downsample(A)
    assert np.array_equal(g.view(np.uint32), r.view(np.uint32))
    B = rng.standard_normal(shape).astype(np.float32) * 1e-3
    B[0, ..., :8] = np.float32(1e-42)   # subnormals compare and select like any other value
    g, r = ops.median3x3_downsample(B), oops.median3x3_downsample(B)
    assert np.array_equal(g.view(np.uint32), r.view(np.uint32))


def test_median_twice_at_benchmark_size_matches_oracle(ops):
    rng = np.random.RandomState(1)
    img = rng.uniform(-0.5, 0.5, (8, 3, 192, 256)).astype(np.float32)
    g = ops.median3x3_downsample(ops.median3x3_downsample(img))
    assert g.shape == (8, 3, 48, 64)
    assert np.array_equal(g, oops.median3x3_downsample(oops.median3x3_downsample(img)))


# ---- warp2d: IEEE ops in the oracle's order -> bit exact ------------------------------------------
@pytest.mark.parametrize("dtype", TYPES)
@pytest.mark.parametrize("normalized", (False, True))
@pytest.mark.parametrize("border_mode", ("clamp", "value"))
def test_warp2d_matches_oracle(ops, dtype, normalized, border_mode):
    rng = np.random.RandomState(11)
    img = rng.uniform(-1, 1, (3, 5, 37, 53)).astype(dtype)
    scale = 0.3 if normalized else 12.0
    disp = rng.uniform(-scale, scale, (3, 2, 37, 53)).astype(dtype)
    disp[0, 0, 3, 4] = np.nan
    disp[1, 1, 5, 6] = 1e30 if dtype == np.float32 else 1e300
    disp[2, 0, 7, 8] = -3e9
    g = ops.warp2d(img, disp, normalized=normalized, border_mode=border_mode, border_value=0.25)
    r = oops.warp2d(img, disp, normalized=normalized, border_mode=border_mode, border_value=0.25)
    assert g.shape == img.shape
    assert np.array_equal(np.isnan(g), np.isnan(r))
    m = ~np.isnan(r)
    assert np.array_equal(g[m], r[m]), np.abs(g[m] - r[m]).max()


@pytest.mark.parametrize("normalized", (False, True))
@pytest.mark.parametrize("border_mode", ("clamp", "value"))
@pytest.mark.parametrize("width", (128, 256, 260))
def test_warp2d_vector_path_matches_oracle(ops, normalized, border_mode, width):
    """float, W a multiple of 4 and >= 128: the four-pixels-per-thread kernel, edge cases included."""
    rng = np.random.RandomState(width)
    img = rng.uniform(-1, 1, (2, 3, 21, width)).astype(np.float32)
    scale = 0.2 if normalized else 9.0
    disp = rng.uniform(-scale, scale, (2, 2, 21, width)).astype(np.float32)
    disp[0, 0, 0, 0] = -0.5 / (width if normalized else 1)      # p2 in (-1, 0): truncation toward zero
    disp[0, 1, 0, 0] = -0.25 / (21 if normalized else 1)
    disp[0, 0, 3, 4:8] = [np.nan, np.inf, -np.inf, 1e30]
    disp[1, 1, 5, 8:12] = [np.nan, 3e9, -3e9, 0.0]
    disp[1, :, 20, width - 4:] = 0.0                             # last row / last columns, integer position
    g = ops.warp2d(img, disp, normalized=normalized, border_mode=border_mode, border_value=-0.75)
    r = oops.warp2d(img, disp, normalized=normalized, border_mode=border_mode, border_value=-0.75)
    assert np.array_equal(np.isnan(g), np.isnan(r))
    m = ~np.isnan(r)
    assert np.array_equal(g[m], r[m]), np.abs(g[m] - r[m]).max()


def test_warp2d_ranks_and_torch_io(ops):
    rng = np.random.RandomState(2)
    img = rng.rand(4, 5).astype(np.float32)
    assert ops.warp2d(img, np.zeros((2, 4, 5), np.float32)).shape == (4, 5)
    assert ops.warp2d(rng.rand(2, 4, 5).astype(np.float32), np.zeros((2, 4, 5), np.float32)).shape == (2, 4, 5)
    x = rng.rand(2, 2, 3, 4, 5).astype(np.float32)       # leading dims collapse (warp2d.cc:150-160)
    d = rng.uniform(-1, 1, (4, 2, 4, 5)).astype(np.float32)
    assert np.array_equal(ops.warp2d(x, d), oops.warp2d(x.reshape(4, 3, 4, 5), d).reshape(x.shape))
    t = ops.warp2d(torch.from_numpy(img).cuda(), torch.zeros(2, 4, 5, device="cuda"))
    assert isinstance(t, torch.Tensor) and t.is_cuda
    assert ops.warp2d(np.zeros((0, 3, 4, 5), np.float32), np.zeros((0, 2, 4, 5), np.float32)).shape == (0, 3, 4, 5)


def test_warp2d_config5_size_properties(ops):
    """BASELINE.json configs[4] size [8,3,768,1024]: matches the oracle on the whole tensor, and an integer
    shift is a pure copy."""
    rng = np.random.RandomState(3)
    img = torch.from_numpy(rng.rand(8, 3, 768, 1024).astype(np.float32)).cuda()
    disp = torch.zeros(8, 2, 768, 1024, device="cuda")
    disp[:, 0] = 3.0
    disp[:, 1] = -2.0
    out = ops.warp2d(img, disp, border_mode="clamp")
    assert torch.equal(out[:, :, 2:, :-3], img[:, :, :-2, 3:])
    d2 = torch.from_numpy(rng.uniform(-0.02, 0.02, (8, 2, 768, 1024)).astype(np.float32)).cuda()
    g = ops.warp2d(img, d2, normalized=True, border_mode="value").cpu().numpy()
    r = oops.warp2d(img.cpu().numpy(), d2.cpu().numpy(), normalized=True, border_mode="value")
    assert np.array_equal(g, r)


# ---- depth_to_flow -------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", TYPES)
@pytest.mark.parametrize("rotation_format", ("angleaxis3", "quaternion", "matrix"))
@pytest.mark.parametrize("inverse_depth", (False, True))
@pytest.mark.parametrize("normalize_flow", (False, True))
def test_depth_to_flow_matches_oracle(ops, dtype, rotation_format, inverse_depth, normalize_flow):
    rng = np.random.RandomState(5)
    n = 3
    depth = rng.uniform(0.2, 4, (n, 1, 48, 64)).astype(dtype)
    depth[0, 0, 0, :5] = [0, -1, np.inf, np.nan, 1e-30]
    K = np.tile(np.array([[0.89115971, 1.18821287, 0.5, 0.5]], dtype), (n, 1))
    aa = rng.uniform(-0.2, 0.2, (n, 3))
    aa[2] = 1e-8          # identity branch (rotation_format.h:69)
    t = rng.uniform(-1, 1, (n, 3)).astype(dtype)
    if rotation_format == "angleaxis3":
        rot = aa.astype(dtype)
    elif rotation_format == "matrix":
        rot = oops.rotation_matrix(aa.astype(np.float64)).astype(dtype)
    else:
        ang = np.linalg.norm(aa, axis=1, keepdims=True)
        rot = np.concatenate((np.cos(ang / 2), np.sin(ang / 2) * aa / ang), axis=1).astype(dtype) * 1.7   # unnormalized on purpose
    g = ops.depth_to_flow(depth, K, rot, t, rotation_format, inverse_depth, normalize_flow)
    r = oops.depth_to_flow(depth, K, rot, t, rotation_format, inverse_depth, normalize_flow)
    assert g.shape == (n, 2, 48, 64)
    assert np.array_equal(np.isnan(g), np.isnan(r))
    m = np.isfinite(r)
    # sin/cos differ by <= 2 ulp between glibc and CUDA libm in angleaxis mode; everything else is IEEE identical
    scale = np.abs(r[m]).max()
    assert np.abs(g[m] - r[m]).max() <= 64 * eps(dtype) * scale
    if rotation_format != "angleaxis3":
        assert np.array_equal(g[m], r[m])


# ---- flow_to_depth ---------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", TYPES)
@pytest.mark.parametrize("inverse_depth", (False, True))
@pytest.mark.parametrize("normalize_flow", (False, True))
def test_reference_round_trip_on_gpu(ops, dtype, inverse_depth, normalize_flow):
    """test_FlowToDepth2.py:37-70 with both ops on the GPU."""
    rng = np.random.RandomState(7)
    depth = rng.uniform(5, 10, (1, 1, 6, 12)).astype(dtype)
    if inverse_depth:
        depth = (1 / depth).astype(dtype)
    rotation = rng.uniform(0.0, 0.05, (1, 3)).astype(dtype)
    translation = (np.array([[1, 0, 0]]) + rng.uniform(-0.2, 0.2, (1, 3))).astype(dtype)
    K = np.array([[1, 1, 0.5, 0.5]]).astype(dtype)
    flow = ops.depth_to_flow(depth, K, rotation, translation, inverse_depth=inverse_depth, normalize_flow=normalize_flow)
    computed = ops.flow_to_depth2(flow, K, rotation, translation, inverse_depth=inverse_depth, normalized_flow=normalize_flow)
    np.testing.assert_allclose(depth, computed, rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("dtype", TYPES)
def test_flow_to_depth_matches_oracle(ops, dtype):
    """The triangulation is ill conditioned on some pixels (cond(A) up to 1e5 for arbitrary flows): the
    reference's float JacobiSVD carries cond * 6e-8 of noise there, and so does the float oracle (its own
    realisation of it -- the double oracle differs from the float oracle by up to 1e-3 on those pixels).  The
    kernel carries double from the float inputs to the solved point, so:
      * against the DOUBLE oracle (same float inputs) it must agree to float output rounding everywhere;
      * against the FLOAT oracle it must agree within the reference test's own 1e-4 (test_FlowToDepth2.py:70)
        except on the ill-conditioned pixels, where it must be no further than the float oracle's own noise."""
    rng = np.random.RandomState(9)
    n = 2
    flow = rng.uniform(-0.08, 0.08, (n, 2, 48, 64)).astype(dtype)
    flow[0, :, 0, 0] = np.nan
    K = np.tile(np.array([[0.89115971, 1.18821287, 0.5, 0.5]], dtype), (n, 1))
    r = rng.uniform(-0.05, 0.05, (n, 3)).astype(dtype)
    t = (np.array([[1, 0, 0]]) + rng.uniform(-0.2, 0.2, (n, 3))).astype(dtype)
    with pytest.warns(DeprecationWarning):
        g = ops.flow_to_depth(flow, K, r, t, normalized_flow=True, inverse_depth=True)
    ref_t = oops.flow_to_depth2(flow, K, r, t, normalized_flow=True, inverse_depth=True)
    ref_d = oops.flow_to_depth2(flow.astype(np.float64), K.astype(np.float64), r.astype(np.float64), t.astype(np.float64),
                                normalized_flow=True, inverse_depth=True)
    assert g.shape == (n, 1, 48, 64) and g[0, 0, 0, 0] == 0
    assert ((g != 0) != (ref_d != 0)).mean() < 1e-3          # behind-camera pattern (only ~infinite depths may flip)
    both = (g != 0) & (ref_d != 0)
    err_d = np.abs(g[both] - ref_d[both]) / np.abs(ref_d[both])
    assert err_d.max() < (4e-7 if dtype == np.float32 else 1e-9), err_d.max()     # cond(A) * 1e-16
    both_t = (g != 0) & (ref_t != 0) & (ref_d != 0)
    err_t = np.abs(g[both_t] - ref_t[both_t]) / np.abs(ref_t[both_t])
    noise = np.abs(ref_t[both_t] - ref_d[both_t]) / np.abs(ref_d[both_t])       # the float oracle's own noise
    assert (err_t > 1e-4).mean() < 0.01
    assert (err_t <= 1e-4 + 1.01 * noise).all()


def test_shapes_and_errors_on_gpu(ops):
    assert ops.flow_to_depth2(np.zeros((2, 6, 12), np.float32), np.array([1, 1, .5, .5], np.float32),
                              np.zeros(3, np.float32), np.array([1, 0, 0], np.float32)).shape == (1, 1, 6, 12)
    assert ops.depth_to_flow(np.ones((2, 3, 6, 12), np.float32), np.ones((6, 4), np.float32), np.zeros((6, 3), np.float32),
                             np.ones((6, 3), np.float32)).shape == (6, 2, 6, 12)
    for shape in ((8, 40, 31), (8, 1, 40, 31), (2, 2, 2, 40, 31)):
        assert ops.scale_invariant_gradient(np.ones(shape, np.float32)).shape == (8, 2, 40, 31)
        assert ops.leaky_relu(np.ones(shape, np.float32)).shape == shape
    assert ops.median3x3_downsample(np.zeros((0, 4, 4), np.float32)).shape == (0, 2, 2)
    assert ops.leaky_relu(np.zeros((0,), np.float32)).shape == (0,)


# ---- scale_invariant_gradient / leaky_relu ---------------------------------------------------------
@pytest.mark.parametrize("dtype", TYPES)
def test_sig_matches_oracle(ops, dtype):
    rng = np.random.RandomState(13)
    A = rng.uniform(-2, 2, (3, 2, 40, 31)).astype(dtype)
    A[0, 0, 0, 0] = 0
    deltas, weights = [1, 2, 4, 8, 16], [1, 0.5, 0.25, 0.125, 0.0625]       # v2/losses.py:339-343
    g = ops.scale_invariant_gradient(A, deltas, weights, 0.001)
    r = oops.scale_invariant_gradient(A, deltas, weights, 0.001)
    assert g.shape == (6, 2, 40, 31)
    assert np.array_equal(g, r)          # IEEE ops in the same order
    A4 = np.linspace(1, 2, num=16, dtype=dtype).reshape(4, 4)     # test_ScaleInvariantGradient.py:33
    assert np.array_equal(ops.scale_invariant_gradient(A4, [1, 2, 4], [1, 0.5, 0.25], 0.001),
                          oops.scale_invariant_gradient(A4, [1, 2, 4], [1, 0.5, 0.25], 0.001))


@pytest.mark.parametrize("shape", [(2, 1, 9, 128), (1, 3, 21, 256), (2, 7, 132)])
def test_sig_vector_path_matches_oracle_bit_for_bit(ops, shape):
    """float, W a multiple of 4 and >= 128: four pixels per thread, x neighbours taken out of aligned float4 groups.  Deltas of
    every residue mod 4, negative ones, one wider than the image, zeros and NaNs in the input."""
    rng = np.random.RandomState(sum(shape))
    A = rng.uniform(-2, 2, shape).astype(np.float32)
    A[..., 0, :5] = 0
    A[..., 3, 17] = np.nan
    deltas = [1, 2, 3, 4, 5, 8, 16, -1, -2, -4, -7, 127, 300]
    weights = [1.0 / (1 + i) for i in range(len(deltas))]
    g = ops.scale_invariant_gradient(A, deltas, weights, 0.001)
    r = oops.scale_invariant_gradient(A, deltas, weights, 0.001)
    assert g.shape == r.shape
    assert np.array_equal(np.isnan(g), np.isnan(r))
    m = ~np.isnan(r)
    assert np.array_equal(g[m].view(np.uint32), r[m].view(np.uint32))


@pytest.mark.parametrize("dtype", TYPES)
def test_leaky_relu_matches_oracle(ops, dtype):
    rng = np.random.RandomState(17)
    for n in (1, 7, 1024, 100003):
        x = rng.uniform(-3, 3, n).astype(dtype)
        assert np.array_equal(ops.leaky_relu(x, 0.2), oops.leaky_relu(x, 0.2))
        assert np.array_equal(ops.leaky_relu(x), oops.leaky_relu(x))
    x = torch.from_numpy(rng.uniform(-3, 3, 4099).astype(dtype)).cuda()[3:]     # unaligned view -> scalar path
    assert np.array_equal(ops.leaky_relu(x).cpu().numpy(), oops.leaky_relu(x.cpu().numpy()))
