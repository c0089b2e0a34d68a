"""The fold mode of the tensor-core convolution (conv_tc_halo.cu): narrow 3x3 stride-1 layers with the filter taps in the
GEMM's N dimension.  CPU: which layers the planner folds.  GPU: the fold instantiations (FOLD 9 at N 144, FOLD 3 at N 72, both
precisions) on the exact datasets of tests/test_conv_variants.py, at the network's shapes and channel slices, through the same
guarded slice entry as tests/test_gpu_conv_variants.py."""
import ctypes
import importlib.util
import os
import re

import numpy as np
import pytest
import torch

from demon_b200 import _lib
from test_conv_variants import DATASETS, TC_PRECISIONS, TF32, VARIANTS, X3TF32, describe, exact_data, geometry, pitches, tc_error_bound
from test_gpu_conv_variants import assert_bitwise, expected_exact, log_uniform, ref64, row_id, run_slice, weight_shape

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (B, H, W, Cin, Cout, kh, kw, sy, sx, deconv, in_off, out_off), the VARIANTS format
FOLD_ROWS = [
    (1, 192, 256, 64, 16, 3, 3, 1, 1, 0, 32, 4),    # netRefine/predict_depth0/conv1 at batch 1: FOLD 9, resident weights,
                                                    # 256 tiles: a CTA runs a second tile
    (64, 24, 32, 64, 16, 3, 3, 1, 1, 0, 64, 32),    # FOLD 9 at batch 64, 256 tiles
    (1, 48, 64, 128, 24, 3, 3, 1, 1, 0, 128, 32),   # predict_flow2/conv1 at batch 1: FOLD 3, 12 weight blocks through the
                                                    # ring of 4
    (64, 48, 64, 128, 24, 3, 3, 1, 1, 0, 256, 4),   # ... at batch 64: 1024 tiles, 8 per CTA
    (2, 12, 16, 96, 20, 3, 3, 1, 1, 0, 0, 64),      # FOLD 3 with Cout 20 (columns 20 .. 23 of each tap zero), 3 chunks
]


def fold_of(text):
    return int(re.search(r" fold (\d+) ", text).group(1))


def test_planner_folds_the_narrow_heads_only():
    spec = importlib.util.spec_from_file_location("describe_plan", os.path.join(ROOT, "tools", "describe_plan.py"))
    tool = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tool)
    lib = _lib.load()
    buf = ctypes.create_string_buffer(8192)
    for B in (1, 64):
        for prec in TC_PRECISIONS:
            folded = {}
            for name, dec, H, W, Cin, ipitch, Cout, opitch, kh, kw, sy, sx in tool.SHAPES:
                lib.demon_debug_describe_conv(B, H, W, Cin, ipitch, Cout, opitch, kh, kw, sy, sx, dec, prec, buf, 8192)
                f = fold_of(buf.value.decode())
                if f:
                    folded[name] = f
            assert folded == {"predict2/conv1": 3, "R pd0/conv1": 9}, (B, prec)
    for row in VARIANTS:
        for prec in TC_PRECISIONS:
            assert fold_of(describe(row, prec)["text"]) == 0, row
    for row in FOLD_ROWS:
        for prec in TC_PRECISIONS:
            d = describe(row, prec)
            assert fold_of(d["text"]) == (9 if row[4] == 16 else 3) and d["kind"] == "halo" and (d["th"], d["tw"]) == (12, 16)
            assert d["ksplit"] == 1, d["text"]
    # what the fold mode refuses: 32 input channels, Cout 32, stride 2, 1 x 3 taps, images not made of whole 12 x 16 tiles
    for B, H, W, Cin, Cout, kh, kw, sy, sx in ((1, 48, 64, 32, 16, 3, 3, 1, 1), (1, 48, 64, 64, 32, 3, 3, 1, 1),
                                               (1, 96, 128, 64, 16, 3, 3, 2, 2), (1, 48, 64, 64, 16, 1, 3, 1, 1),
                                               (1, 40, 64, 64, 16, 3, 3, 1, 1), (1, 48, 72, 64, 16, 3, 3, 1, 1)):
        lib.demon_debug_describe_conv(B, H, W, Cin, Cin, Cout, Cout, kh, kw, sy, sx, 0, X3TF32, buf, 8192)
        assert fold_of(buf.value.decode()) == 0, (H, W, Cin, Cout, kh, kw, sy)


def test_fold_rows_reach_both_weight_layouts_and_several_tiles_per_cta():
    d = {(row, prec): describe(row, prec) for row in FOLD_ROWS for prec in TC_PRECISIONS}
    assert {v["wres"] for v in d.values()} == {0, 1}
    assert {v["mode"] for v in d.values()} == {0, 2}
    assert max(v["tiles"] for v in d.values()) > 132 * 2


@pytest.mark.gpu
@pytest.mark.parametrize("dataset", DATASETS)
@pytest.mark.parametrize("row", FOLD_ROWS, ids=[row_id(r) for r in FOLD_ROWS])
def test_fold_exact(row, dataset):
    B, H, W, Cin, Cout, _, _, _, _, deconv, in_off, out_off = row
    geom = geometry(row)
    in_pitch, out_pitch = pitches(row)
    leaky = FOLD_ROWS.index(row) % 2 == 0
    rng = np.random.default_rng([FOLD_ROWS.index(row), DATASETS.index(dataset), 11])
    x, k, b = exact_data(dataset, (B, H, W, Cin), weight_shape(Cin, Cout, geom, deconv), Cout, rng)
    xd = torch.from_numpy(x).cuda()
    want = expected_exact(ref64(xd, k, b, geom, deconv), leaky)

    def run(prec):
        return run_slice(xd, in_off, in_pitch, k, b, Cout, out_off, out_pitch, geom, deconv, leaky, prec)

    assert_bitwise(run(X3TF32), want, "3xTF32, plan %s" % describe(row, X3TF32)["text"])
    got1 = run(TF32)
    if dataset == "int":
        assert_bitwise(got1, want, "TF32, plan %s" % describe(row, TF32)["text"])
    else:
        assert not torch.equal(got1, want), "TF32 reproduced the %s dataset, which needs the 3xTF32 lo terms" % dataset


@pytest.mark.gpu
@pytest.mark.parametrize("precision", TC_PRECISIONS, ids=["3xtf32", "tf32"])
@pytest.mark.parametrize("row", FOLD_ROWS, ids=[row_id(r) for r in FOLD_ROWS])
def test_fold_realistic(row, precision):
    """Log-uniform data under tc_error_bound: the fold's epilogue adds up to nine per-tap sums, each of fewer wgmma than
    the bound counts, so the bound's accumulation terms still cover it."""
    B, H, W, Cin, Cout, kh, kw, _, _, deconv, in_off, out_off = row
    geom = geometry(row)
    in_pitch, out_pitch = pitches(row)
    leaky = FOLD_ROWS.index(row) % 2 == 1
    rng = np.random.default_rng([FOLD_ROWS.index(row), 13])
    x = log_uniform((B, H, W, Cin), rng)
    k = log_uniform(weight_shape(Cin, Cout, geom, deconv), rng)
    b = log_uniform((Cout,), rng)
    xd = torch.from_numpy(x).cuda()
    y = ref64(xd, k, b, geom, deconv)
    S = ref64(xd.abs(), np.abs(k), np.abs(b), geom, deconv)
    if leaky:
        y = torch.maximum(float(np.float32(0.1)) * y, y)
    got = run_slice(xd, in_off, in_pitch, k, b, Cout, out_off, out_pitch, geom, deconv, leaky, precision).double()
    bound = tc_error_bound(precision, Cin, kh, kw, deconv, describe(row, precision)["ksplit"])
    over = ((got - y).abs() > bound * S).nonzero()
    assert over.shape[0] == 0, "%d elements over the bound, first at %s" % (over.shape[0], over[0].tolist())
