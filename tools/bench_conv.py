"""Runs ONE convolution shape of the DeMoN graphs at batch 64 through the C-ABI test entry (for ncu captures)."""
import ctypes
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from demon_b200 import _lib

SHAPES = {
    # name: (kind, B, H, W, Cin, Cout, kh, kw, sy, sx)
    "pd0_conv1": ("conv", 64, 192, 256, 64, 16, 3, 3, 1, 1),
    "refine_conv1_1": ("conv", 64, 96, 128, 64, 64, 3, 3, 1, 1),
    "refine_conv2_1": ("conv", 64, 48, 64, 128, 128, 3, 3, 1, 1),
    "refine0_upconv": ("deconv", 64, 96, 128, 128, 32),
    "conv1y": ("conv", 64, 192, 256, 8, 32, 9, 1, 2, 1),
    "conv1x": ("conv", 64, 96, 256, 32, 32, 1, 9, 1, 2),
    "conv2y": ("conv", 64, 96, 128, 32, 64, 7, 1, 2, 1),
    "predict2_conv1": ("conv", 64, 48, 64, 128, 24, 3, 3, 1, 1),
    "conv5_1y": ("conv", 64, 6, 8, 512, 512, 3, 1, 1, 1),
    "conv3x": ("conv", 64, 24, 64, 128, 128, 1, 5, 1, 2),
    "refine2_upconv": ("deconv", 64, 24, 32, 256, 64),
    "refine3_upconv": ("deconv", 64, 12, 16, 576, 128),   # netFlow2/refine3/upconv: the 514-channel concat4 padded to 18 chunks
    "refine4_upconv": ("deconv", 64, 6, 8, 512, 256),
    "conv2_1y": ("conv", 64, 48, 64, 64, 64, 3, 1, 1, 1),
    "conv4x": ("conv", 64, 12, 32, 256, 256, 1, 5, 1, 2),
    "conv5_1x": ("conv", 64, 6, 8, 512, 512, 1, 3, 1, 1),
}


def main():
    name = sys.argv[1]
    prec = int(sys.argv[2]) if len(sys.argv) > 2 else 1
    reps = int(sys.argv[3]) if len(sys.argv) > 3 else 2
    lib = _lib.load()
    spec = SHAPES[name]
    rng = np.random.RandomState(0)
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    timing = os.environ.get("TC_TIMING") == "1"
    if timing:
        lib.demon_debug_tc_timing(1, None, 0)
    if spec[0] == "conv":
        _, B, H, W, Cin, Cout, kh, kw, sy, sx = spec
        x = torch.rand(B, H, W, Cin, device="cuda") - 0.5
        out = torch.empty(B, -(-H // sy), -(-W // sx), Cout, device="cuda")
        k = (rng.standard_normal((kh, kw, Cin, Cout)) / np.sqrt(kh * kw * Cin)).astype(np.float32)
        b = np.zeros(Cout, np.float32)
        for _ in range(reps):
            _lib.check(lib.demon_conv2d_nhwc(x.data_ptr(), out.data_ptr(), B, H, W, Cin, Cout, kh, kw, sy, sx, k.ctypes.data, b.ctypes.data, 1, prec, stream))
    else:
        _, B, H, W, Cin, Cout = spec
        x = torch.rand(B, H, W, Cin, device="cuda") - 0.5
        out = torch.empty(B, 2 * H, 2 * W, Cout, device="cuda")
        k = (rng.standard_normal((4, 4, Cout, Cin)) / np.sqrt(4 * Cin)).astype(np.float32)
        b = np.zeros(Cout, np.float32)
        for _ in range(reps):
            _lib.check(lib.demon_deconv4x4s2_nhwc(x.data_ptr(), out.data_ptr(), B, H, W, Cin, Cout, k.ctypes.data, b.ctypes.data, 1, prec, stream))
    torch.cuda.synchronize()
    print(name, "done; timeouts", lib.demon_debug_tc_timeouts())
    print("  kernel time of the last call: %.4f ms" % lib.demon_debug_last_conv_ms())
    if timing:
        full = np.zeros((256, 16), np.int64)
        if lib.demon_debug_tc_timing(0, full.ctypes.data, 256) == 0:
            buf = full[:132]
            names = {0: "producer wait A_empty", 1: "producer wait W_empty", 3: "consumer wait W_full", 6: "consumer wait A_full",
                     8: "producer total", 9: "consumer total"}
            m = buf.mean(axis=0)
            for i, nm in names.items():
                print("  %-44s %12.0f cycles (avg per CTA)" % (nm, m[i]))

if __name__ == "__main__":
    main()
