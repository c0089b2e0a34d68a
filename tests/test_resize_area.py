"""CPU: the resize_area oracle (oracle/resize_area.py) against TF's area definition with general weights in float64 and
against torch's avg_pool2d in float64, and the argument checks of demon_b200.images.resize_area that need no device."""
import numpy as np
import pytest
import torch

from oracle import resize_area as ra

# (input shape, output size): training.py's image2_2 at batch 32 and 1, and the other integer factors
CASES = (((32, 3, 192, 256), (48, 64)), ((1, 3, 192, 256), (48, 64)), ((2, 3, 96, 128), (48, 64)), ((2, 3, 144, 192), (48, 64)),
         ((3, 2, 5, 256), (5, 1)), ((1, 1, 7, 9), (7, 3)))


def data(shape, seed):
    rng = np.random.RandomState(seed)
    x = rng.uniform(-0.5, 0.5, shape).astype(np.float32)
    x.reshape(-1)[rng.rand(x.size) < 0.01] *= np.float32(1e4)   # a few large values: cancellation inside a block
    return x


@pytest.mark.parametrize("shape,size", CASES)
def test_oracle_within_bound_of_general_area_definition(shape, size):
    x = data(shape, sum(shape))
    got = ra.resize_area(x, size)
    assert got.dtype == np.float32 and got.shape == shape[:-2] + size
    exact = ra.area_exact(x, size)
    bound = ra.error_bound(x, size)
    err = np.abs(got.astype(np.float64) - exact)
    assert (err <= bound).all(), float((err / np.maximum(bound, 1e-300)).max())
    # the general weights are exactly 1 for an integer factor: the float64 loop is the plain block mean
    fy, fx = shape[-2] // size[0], shape[-1] // size[1]
    assert np.array_equal(ra._weights(shape[-2], size[0]), np.kron(np.eye(size[0]), np.ones((1, fy))))
    assert np.array_equal(ra._weights(shape[-1], size[1]), np.kron(np.eye(size[1]), np.ones((1, fx))))


@pytest.mark.parametrize("shape,size", CASES)
def test_oracle_against_avg_pool2d_in_float64(shape, size):
    x = data(shape, 7 + sum(shape))
    fy, fx = shape[-2] // size[0], shape[-1] // size[1]
    pooled = torch.nn.functional.avg_pool2d(torch.from_numpy(x).double(), (fy, fx)).numpy()
    got = ra.resize_area(x, size).astype(np.float64)
    assert (np.abs(got - pooled) <= ra.error_bound(x, size) * (1 + 1e-9)).all()
    # on small integers every float32 sum is exact, and 1/16 is a power of two: bit equal for 4x4 blocks
    if (fy, fx) == (4, 4):
        ints = np.random.RandomState(3).randint(-1000, 1000, shape).astype(np.float32)
        ref = torch.nn.functional.avg_pool2d(torch.from_numpy(ints).double(), 4).numpy()
        assert np.array_equal(ra.resize_area(ints, size), ref.astype(np.float32))


def test_oracle_summation_order_and_specials():
    """The order is observable: rows left to right, then the row sums top to bottom, each from +0."""
    big, one = np.float32(2.0 ** 24), np.float32(1.0)
    x = np.zeros((1, 1, 2, 2), np.float32)
    x[0, 0] = [[big, one], [one, -big]]
    # row 0: (0 + 2^24) + 1 = 2^24 (ties to even); row 1: (0 + 1) - 2^24 = -(2^24 - 1); sum: 1; times 1/4
    assert ra.resize_area(x, (1, 1))[0, 0, 0, 0] == np.float32(0.25)
    x[0, 0] = [[-0.0, -0.0], [-0.0, -0.0]]
    r = ra.resize_area(x, (1, 1))[0, 0, 0, 0]
    assert r == 0 and not np.signbit(r)                     # +0 + -0 = +0
    x[0, 0] = [[np.inf, 1], [2, 3]]
    assert ra.resize_area(x, (1, 1))[0, 0, 0, 0] == np.inf
    x[0, 0] = [[np.inf, 1], [-np.inf, 3]]
    assert np.isnan(ra.resize_area(x, (1, 1))[0, 0, 0, 0])
    x[0, 0] = [[np.nan, 1], [2, 3]]
    assert np.isnan(ra.resize_area(x, (1, 1))[0, 0, 0, 0])
    # 3x3: the scale is float32(1/9), one rounded division, not 1/9 in float64
    y = np.ones((1, 1, 3, 3), np.float32)
    assert ra.resize_area(y, (1, 1))[0, 0, 0, 0] == np.float32(9) * (np.float32(1) / np.float32(9))


def test_resize_area_argument_checks_need_no_device():
    from demon_b200 import images
    x = np.zeros((2, 3, 192, 256), np.float32)
    for size in ((47, 64), (48, 65), (0, 64), (48, 0), (384, 256), (48,), "48x64", None):
        with pytest.raises(ValueError):
            images.resize_area(x, size)
    with pytest.raises(ValueError, match="float32"):
        images.resize_area(x.astype(np.float64), (48, 64))
    with pytest.raises(ValueError, match="float32"):
        images.resize_area(torch.zeros(2, 3, 192, 256, dtype=torch.float16), (48, 64))
    with pytest.raises(ValueError, match="N,C,h,w"):
        images.resize_area(np.zeros((192, 256), np.float32), (48, 64))
    with pytest.raises(ValueError, match="N,C,h,w"):
        images.resize_area(np.zeros((1, 1, 3, 192, 256), np.float32), (48, 64))
    with pytest.raises(ValueError, match="CUDA"):
        images.resize_area(torch.zeros(2, 3, 192, 256), (48, 64))
    with pytest.raises(ValueError, match="numpy"):
        images.resize_area([[[0.0]]], (1, 1))
