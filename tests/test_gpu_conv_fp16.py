"""GPU: the FP16 precision of the tensor-core convolution (DEMON_PREC_FP16, conv_tc_halo_kernel MODE 1), through the guarded
slice entries of tests/test_gpu_conv_variants.py (NaN around the input slice, sentinels around the output).

* Every variant (VARIANTS, FOLD_ROWS and FP16_ROWS) on data FP16 holds exactly: x, w in {-1, 0, 1} (`int`), or
  i + j 2^-10 in one operand (`a10`, `w10`), i, j in {-1, 0, 1}.  Every product is exact and every partial sum a multiple of
  2^-10 below 2^13, so the result equals float32(leaky(float64)) bit for bit.  On the 2^-11 datasets of
  tests/test_conv_variants.py (`alo`, `wlo`) FP16 must differ: 1 +- 2^-11 is not an FP16 value, so both operands really
  are converted.
* Log-uniform data under fp16_error_bound.
* An input of 1e5 (above FP16's 65504) gives non-finite outputs exactly in its receptive field.
* demon_net_finalize refuses a tensor-core layer's weight FP16 cannot hold.
* Every tensor-core layer of the v1 and v2 nets (b64, b1, refine1024) bit for bit on `int` data at its own batch, geometry
  and channel slice."""
import numpy as np
import pytest
import torch

from demon_b200 import weights as W1
from demon_b200.networks_original import _NetHandle
from demon_b200.v2 import weights as W2
from demon_b200.v2.networks import _NetHandleV2
from test_conv_variants import TF32, VARIANTS, describe, exact_data, geometry, pitches, tc_error_bound
from test_gpu_conv_fold import FOLD_ROWS
from test_gpu_conv_variants import (NET_CONFIGS, assert_bitwise, expected_exact, log_uniform, net_layers, ref64, row_id, run_slice,
                                    weight_shape)
from test_gpu_conv_variants_v2 import ref64_same, run_slice_same
from test_plans_fp16 import FP16, FP16_ROWS
from test_v2_plan import describe_plan

pytestmark = pytest.mark.gpu

ROWS = VARIANTS + FOLD_ROWS + FP16_ROWS
F16_DATASETS = ("int", "a10", "w10")


def exact16_data(name, xshape, wshape, nbias, rng):
    """(x, w, bias) float32 of an FP16-exact dataset (module docstring)."""
    def tern(shape):
        return rng.integers(-1, 2, shape).astype(np.float64)
    x, w = tern(xshape), tern(wshape)
    if name == "a10":
        x += tern(xshape) * 2.0 ** -10
    elif name == "w10":
        w += tern(wshape) * 2.0 ** -10
    b = rng.integers(-2, 3, nbias).astype(np.float64)
    out = tuple(a.astype(np.float32) for a in (x, w, b))
    for a in out[:2]:
        assert np.array_equal(a.astype(np.float16).astype(np.float32), a)
    return out


def fp16_error_bound(Cin, kh, kw, deconv, ksplit):
    """|err| <= bound * S for FP16 (S = sum |x||w| + |b|).  Both operands are rounded to nearest FP16, 2^-11 relative each,
    so a product is off by at most (2^-10 + 2^-22) of itself.  The accumulation terms are single-pass TF32's in
    tc_error_bound, (2 n8 + ksplit + 2) 2^-23: every wgmma rounds twice, at most one float32 ulp of a partial sum <= S each,
    plus split-K's and the epilogue's additions; an FP16 wgmma sums K = 16, so there are n8 / 2 of them, counted twice over."""
    return 2.0 ** -10 + 2.0 ** -22 + tc_error_bound(TF32, Cin, kh, kw, deconv, ksplit) - 2.0 ** -9


@pytest.mark.parametrize("dataset", F16_DATASETS + ("alo", "wlo"))
@pytest.mark.parametrize("row", ROWS, ids=[row_id(r) for r in ROWS])
def test_fp16_variant_exact(row, dataset):
    B, H, W, Cin, Cout, _, _, _, _, deconv, in_off, out_off = row
    geom = geometry(row)
    in_pitch, out_pitch = pitches(row)
    leaky = ROWS.index(row) % 2 == 0
    rng = np.random.default_rng([ROWS.index(row), (F16_DATASETS + ("alo", "wlo")).index(dataset), 16])
    shapes = ((B, H, W, Cin), weight_shape(Cin, Cout, geom, deconv), Cout, rng)
    x, k, b = exact16_data(dataset, *shapes) if dataset in F16_DATASETS else exact_data(dataset, *shapes)
    xd = torch.from_numpy(x).cuda()
    want = expected_exact(ref64(xd, k, b, geom, deconv), leaky)
    d = describe(row, FP16)
    assert d["mode"] == 1, d["text"]
    got = run_slice(xd, in_off, in_pitch, k, b, Cout, out_off, out_pitch, geom, deconv, leaky, FP16)
    if dataset in F16_DATASETS:
        assert_bitwise(got, want, "FP16, plan %s" % d["text"])
    else:
        assert not torch.equal(got, want), "FP16 reproduced the %s dataset, whose 2^-11 parts FP16 cannot hold" % dataset


WORST = {}


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    yield
    if WORST:
        ratio, share, row = WORST["fp16"]
        print("\nrealistic data, fp16: largest |err| / S = %.3g (%.3g of the bound) at %s" % (ratio, share, row_id(row)))


@pytest.mark.parametrize("row", ROWS, ids=[row_id(r) for r in ROWS])
def test_fp16_variant_realistic(row):
    """Random signs, magnitudes log-uniform in 2^-8 .. 2^8 (x, w and bias: FP16 normals), under fp16_error_bound."""
    B, H, W, Cin, Cout, kh, kw, _, _, deconv, in_off, out_off = row
    geom = geometry(row)
    in_pitch, out_pitch = pitches(row)
    leaky = ROWS.index(row) % 2 == 1
    rng = np.random.default_rng([ROWS.index(row), 17])
    x = log_uniform((B, H, W, Cin), rng)
    k = log_uniform(weight_shape(Cin, Cout, geom, deconv), rng)
    b = log_uniform((Cout,), rng)
    xd = torch.from_numpy(x).cuda()
    y = ref64(xd, k, b, geom, deconv)
    S = ref64(xd.abs(), np.abs(k), np.abs(b), geom, deconv)
    if leaky:
        y = torch.maximum(float(np.float32(0.1)) * y, y)
    got = run_slice(xd, in_off, in_pitch, k, b, Cout, out_off, out_pitch, geom, deconv, leaky, FP16).double()
    d = describe(row, FP16)
    bound = fp16_error_bound(Cin, kh, kw, deconv, d["ksplit"])
    ratio = ((got - y).abs() / S).max().item()
    if ratio > WORST.get("fp16", (-1,))[0]:
        WORST["fp16"] = (ratio, ratio / bound, row)
    over = ((got - y).abs() > bound * S).nonzero()
    if over.shape[0]:
        i = tuple(over[0].tolist())
        pytest.fail("%d elements over the bound %.3g S, first at [n, y, x, channel] %s: got %r, float64 %r, S %r; plan %s"
                    % (over.shape[0], bound, list(i), got[i].item(), y[i].item(), S[i].item(), d["text"]))
    assert ratio > 2.0 ** -19   # the operands are rounded: FP16 is not 3xTF32


@pytest.mark.parametrize("row", ROWS, ids=[row_id(r) for r in ROWS])
def test_fp16_out_of_range_input_is_non_finite_in_its_receptive_field(row):
    """One input value of 1e5 becomes +-inf in FP16; the outputs it reaches (nonzero weights everywhere) are non-finite,
    every other output is finite."""
    B, H, W, Cin, Cout, _, _, _, _, deconv, in_off, out_off = row
    geom = geometry(row)
    in_pitch, out_pitch = pitches(row)
    rng = np.random.default_rng([ROWS.index(row), 18])
    x = rng.uniform(-1, 1, (B, H, W, Cin)).astype(np.float32)
    k = (rng.choice((-1.0, 1.0), weight_shape(Cin, Cout, geom, deconv)) * rng.uniform(0.5, 1, weight_shape(Cin, Cout, geom, deconv))).astype(np.float32)
    b = rng.uniform(-1, 1, Cout).astype(np.float32)
    pos = (B - 1, H // 2, W // 3, Cin - 1)
    x[pos] = 1e5
    hit = np.zeros_like(x)
    hit[pos] = 1
    reach = ref64(torch.from_numpy(hit).cuda(), np.ones_like(k), np.zeros_like(b), geom, deconv) > 0
    got = run_slice(torch.from_numpy(x).cuda(), in_off, in_pitch, k, b, Cout, out_off, out_pitch, geom, deconv, True, FP16)
    assert reach.any()
    bad = (~torch.isfinite(got)) != reach
    assert not bad.any(), "%d outputs where non-finite != in the receptive field, first at %s; plan %s" % (
        int(bad.sum()), bad.nonzero()[0].tolist(), describe(row, FP16)["text"])


@pytest.mark.parametrize("variant", (1, 2), ids=["v1", "v2"])
def test_finalize_refuses_weights_fp16_cannot_hold(variant):
    handle, weights = (_NetHandle, W1.synthetic_weights(0)) if variant == 1 else (_NetHandleV2, W2.synthetic_weights(0))
    name = "netFlow1/conv2y/kernel"
    for bad in (65536.0, -7e4, float("inf"), float("nan")):
        w = dict(weights)
        w[name] = weights[name].copy()
        w[name].flat[5] = bad
        with pytest.raises(ValueError, match=name):
            handle(w, 1, (192, 256), "fp16")
        handle(w, 1, (192, 256), "3xtf32")   # the same weights are accepted where they are not converted
    w = dict(weights)
    w[name] = weights[name].copy()
    w[name].flat[5] = 65504.0   # FP16's largest finite value
    fc = "netDM1/motion_fc1/kernel"
    w[fc] = weights[fc].copy()
    w[fc].flat[0] = 1e6          # a dense layer runs in fp32 at every precision
    net = handle(w, 1, (192, 256), "fp16")
    assert net.uses_tensor_cores(name.rsplit("/", 1)[0]) and not net.uses_tensor_cores(fc.rsplit("/", 1)[0])


@pytest.mark.parametrize("config", sorted(NET_CONFIGS))
def test_fp16_network_layers_exact_v1(config):
    """Every tensor-core layer of the v1 net at FP16, at its batch, geometry, pitches and offsets, on `int` data (padding
    channels past cin finite and nonzero, with zero weights), bit for bit."""
    batch, refine_hw, prefix = NET_CONFIGS[config]
    jobs = {}
    for name, kind, g, plan in net_layers(batch, refine_hw, FP16):
        if kind != "dense" and name.startswith(prefix) and plan != "simt":
            assert " mode 1 " in plan, (name, plan)
            jobs.setdefault((kind,) + tuple(sorted(g.items())), []).append((name, plan))
    assert jobs
    gen = torch.Generator(device="cuda")
    for i, (key, names) in enumerate(sorted(jobs.items())):
        deconv = key[0] == "deconv"
        g = dict(key[1:])
        geom = (g["kh"], g["kw"], g["sy"], g["sx"])
        x, k, b = int_layer_data(g, batch, geom, deconv, gen, i)
        want = expected_exact(ref64(x, k, b, geom, deconv), g["leaky"])
        got = run_slice(x, g["in_off"], g["in_pitch"], k, b, g["cout"], g["out_off"], g["out_pitch"], geom, deconv, g["leaky"], FP16)
        assert_bitwise(got, want, "%s at fp16" % names)


@pytest.mark.parametrize("config", sorted(NET_CONFIGS))
def test_fp16_network_layers_exact_v2(config):
    batch, refine_hw, prefix = NET_CONFIGS[config]
    jobs = {}
    for name, (g, tap0, text) in describe_plan(2, batch, refine_hw, FP16).items():
        plan = text.split(" : ", 1)[1] if text.startswith("tap0") else text
        if g["kind"] == "conv" and name.startswith(prefix) and plan != "simt":
            assert " mode 1 " in plan, (name, plan)
            jobs.setdefault(tuple(sorted((k, v) for k, v in g.items() if k != "kind")), []).append((name, plan))
    assert jobs
    gen = torch.Generator(device="cuda")
    for i, (key, names) in enumerate(sorted(jobs.items())):
        g = dict(key)
        geom = (g["kh"], g["kw"], g["sy"], g["sx"])
        x, k, b = int_layer_data(g, batch, geom, False, gen, i)
        want = expected_exact(ref64_same(x, k, b, geom), g["leaky"])
        got = run_slice_same(x, g["in_off"], g["in_pitch"], k, b, g["cout"], g["out_off"], g["out_pitch"], geom, g["leaky"], FP16)
        assert_bitwise(got, want, "%s at fp16" % names)


def int_layer_data(g, batch, geom, deconv, gen, i):
    cin, cb, cout = g["cin"], g["cin_buf"], g["cout"]
    gen.manual_seed(i)
    x = torch.randint(-1, 2, (batch, g["H"], g["W"], cb), generator=gen, device="cuda").float()
    if cb > cin:
        x[..., cin:] = torch.randint(0, 2, (batch, g["H"], g["W"], cb - cin), generator=gen, device="cuda").float() * 2 - 1
    rng = np.random.default_rng(i)
    k = rng.integers(-1, 2, weight_shape(cb, cout, geom, deconv)).astype(np.float32)
    if deconv:
        k[..., cin:] = 0
    else:
        k[:, :, cin:, :] = 0
    b = rng.integers(-2, 3, cout).astype(np.float32)
    return x, k, b
