"""CPU: the tiling plans the halo planner picks for the DeMoN layers (demon_debug_describe_conv needs no device).

These are the decisions DESIGN.md section 3.1 describes -- resident weights, split-K, the N tile, the 3xTF32 mode --
pinned here so that a planner change shows up as a test diff."""
import ctypes
import re

import pytest

from demon_b200 import _lib

X3TF32 = 1


@pytest.fixture(scope="module")
def plan():
    lib = _lib.load()
    buf = ctypes.create_string_buffer(8192)

    def f(B, H, W, Cin, Cout, kh, kw, sy, sx, deconv=0, in_pitch=None, out_pitch=None):
        lib.demon_debug_describe_conv(B, H, W, Cin, in_pitch or Cin, Cout, out_pitch or Cout, kh, kw, sy, sx, deconv, X3TF32, buf, 8192)
        text = buf.value.decode()
        d = {k: int(v) for k, v in re.findall(r"(n_tile|nbuf|mode|tiles|ksplit|wres|sa) (\d+)", text)}
        d["text"] = text
        return d
    return f


def test_resident_weights_for_the_narrow_single_n_tile_layers(plan):
    pd0 = plan(64, 192, 256, 64, 16, 3, 3, 1, 1)                 # netRefine/predict_depth0/conv1: 2 x 9 x 4 KB
    assert (pd0["n_tile"], pd0["mode"], pd0["wres"], pd0["ksplit"]) == (16, 2, 1, 1)
    conv1x = plan(64, 96, 256, 32, 32, 1, 9, 1, 2)               # 9 x 8 KB
    assert conv1x["wres"] == 1 and conv1x["sa"] >= 2
    p2 = plan(64, 48, 64, 128, 24, 3, 3, 1, 1)                   # predict_flow2/conv1: 4 x 9 x 8 KB = 288 KB -> ring
    assert (p2["n_tile"], p2["wres"]) == (32, 0)
    wide = plan(64, 48, 64, 128, 128, 3, 3, 1, 1)                # netRefine/conv2_1: tensor bound, ring
    assert (wide["n_tile"], wide["mode"], wide["wres"]) == (128, 2, 0)


def test_n_tile_and_split_k(plan):
    conv4x = plan(64, 12, 32, 256, 256, 1, 5, 1, 2)              # 96 pixel tiles x 2 N tiles of 128 fill the 132 SMs
    assert (conv4x["n_tile"], conv4x["tiles"]) == (128, 192)
    assert plan(64, 24, 64, 128, 128, 1, 5, 1, 2)["n_tile"] == 128      # conv3x
    assert plan(64, 6, 8, 128, 128, 3, 3, 1, 1)["n_tile"] == 64         # 24 pixel tiles: narrower N tiles for more CTAs
    pf5 = plan(64, 6, 8, 512, 24, 3, 3, 1, 1)                          # predict_flow5/conv1: 24 tiles, 144 steps each
    assert pf5["tiles"] == 24 and pf5["ksplit"] >= 2
    assert plan(64, 12, 16, 576, 128, 4, 4, 2, 2, deconv=1)["ksplit"] == 1   # refine3 at batch 64: the partial sums would cost more than the rounds save
    assert plan(1, 12, 16, 576, 128, 4, 4, 2, 2, deconv=1)["ksplit"] > 1     # ... at batch 1 they do not
    assert plan(1, 12, 16, 544, 128, 4, 4, 2, 2, deconv=1)["ksplit"] == 1    # 17 chunks: prime


def test_three_instruction_mode_and_register_accumulators(plan):
    conv1y = plan(64, 192, 256, 8, 32, 9, 1, 2, 1)                     # 8-channel input
    assert "cin8" in conv1y["text"] and conv1y["mode"] == 2
    # transposed convolutions: four classes of accumulators in registers, so at most N = 64 per class
    refine0 = plan(64, 96, 128, 128, 32, 4, 4, 2, 2, deconv=1)
    assert (refine0["mode"], refine0["n_tile"]) == (2, 32)
    refine1 = plan(64, 48, 64, 128, 64, 4, 4, 2, 2, deconv=1)
    assert (refine1["mode"], refine1["n_tile"]) == (2, 64)
    refine3 = plan(64, 12, 16, 576, 128, 4, 4, 2, 2, deconv=1)
    assert refine3["n_tile"] == 64 and "n_tile 64 x2" in refine3["text"]
