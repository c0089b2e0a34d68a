"""Offline (no GPU): which kernel family and tiling plan every convolution shape of the DeMoN graphs gets at a batch size.
Usage: python tools/describe_plan.py [batch] [precision 0|1|2|3]"""
import ctypes
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from demon_b200 import _lib

# name: (deconv, H, W, Cin, in_pitch, Cout, out_pitch, kh, kw, sy, sx)   (input resolution)
SHAPES = [
    ("conv1y", 0, 192, 256, 8, 8, 32, 32, 9, 1, 2, 1), ("conv1x", 0, 96, 256, 32, 32, 32, 32, 1, 9, 1, 2),
    ("conv2y(32)", 0, 96, 128, 32, 32, 32, 64, 7, 1, 2, 1), ("conv2x(32)", 0, 48, 128, 32, 64, 32, 64, 1, 7, 1, 2),
    ("conv2y(64)", 0, 96, 128, 32, 32, 64, 64, 7, 1, 2, 1), ("conv2x(64)", 0, 48, 128, 64, 64, 64, 64, 1, 7, 1, 2),
    ("extra_y", 0, 48, 64, 32, 32, 32, 32, 3, 1, 1, 1), ("extra_x", 0, 48, 64, 32, 32, 32, 64, 1, 3, 1, 1),
    ("conv2_1y", 0, 48, 64, 64, 64, 64, 64, 3, 1, 1, 1), ("conv2_1x", 0, 48, 64, 64, 64, 64, 128, 1, 3, 1, 1),
    ("conv3y", 0, 48, 64, 64, 128, 128, 128, 5, 1, 2, 1), ("conv3x", 0, 24, 64, 128, 128, 128, 128, 1, 5, 1, 2),
    ("conv3_1y", 0, 24, 32, 128, 128, 128, 128, 3, 1, 1, 1), ("conv3_1x", 0, 24, 32, 128, 128, 128, 256, 1, 3, 1, 1),
    ("conv4y", 0, 24, 32, 128, 256, 256, 256, 5, 1, 2, 1), ("conv4x", 0, 12, 32, 256, 256, 256, 256, 1, 5, 1, 2),
    ("conv4_1y", 0, 12, 16, 256, 256, 256, 256, 3, 1, 1, 1), ("conv4_1x", 0, 12, 16, 256, 256, 256, 544, 1, 3, 1, 1),
    ("conv5y(k5)", 0, 12, 16, 256, 544, 512, 512, 5, 1, 2, 1), ("conv5x(k5)", 0, 6, 16, 512, 512, 512, 512, 1, 5, 1, 2),
    ("conv5y(k3)", 0, 12, 16, 256, 544, 512, 512, 3, 1, 2, 1), ("conv5x(k3)", 0, 6, 16, 512, 512, 512, 512, 1, 3, 1, 2),
    ("conv5_1y", 0, 6, 8, 512, 512, 512, 512, 3, 1, 1, 1), ("conv5_1x", 0, 6, 8, 512, 512, 512, 512, 1, 3, 1, 1),
    ("predict_flow5/conv1", 0, 6, 8, 512, 512, 24, 24, 3, 3, 1, 1), ("motion_conv1", 0, 6, 8, 512, 512, 128, 128, 3, 3, 1, 1),
    ("refine4", 1, 6, 8, 512, 512, 256, 544, 4, 4, 2, 2), ("refine3", 1, 12, 16, 544, 544, 128, 256, 4, 4, 2, 2),
    ("refine2", 1, 24, 32, 256, 256, 64, 128, 4, 4, 2, 2), ("predict2/conv1", 0, 48, 64, 128, 128, 24, 24, 3, 3, 1, 1),
    ("R conv0", 0, 192, 256, 8, 8, 32, 64, 3, 3, 1, 1), ("R conv1", 0, 192, 256, 32, 64, 64, 64, 3, 3, 2, 2),
    ("R conv1_1", 0, 96, 128, 64, 64, 64, 128, 3, 3, 1, 1), ("R conv2", 0, 96, 128, 64, 128, 128, 128, 3, 3, 2, 2),
    ("R conv2_1", 0, 48, 64, 128, 128, 128, 128, 3, 3, 1, 1), ("R refine1", 1, 48, 64, 128, 128, 64, 128, 4, 4, 2, 2),
    ("R refine0", 1, 96, 128, 128, 128, 32, 64, 4, 4, 2, 2), ("R pd0/conv1", 0, 192, 256, 64, 64, 16, 16, 3, 3, 1, 1),
]


def main():
    B = int(sys.argv[1]) if len(sys.argv) > 1 else 64
    prec = int(sys.argv[2]) if len(sys.argv) > 2 else 1
    lib = _lib.load()
    buf = ctypes.create_string_buffer(4096)
    for name, dec, H, W, Cin, ipitch, Cout, opitch, kh, kw, sy, sx in SHAPES:
        lib.demon_debug_describe_conv(B, H, W, Cin, ipitch, Cout, opitch, kh, kw, sy, sx, dec, prec, buf, 4096)
        print("%-20s %s" % (name, buf.value.decode()))


if __name__ == "__main__":
    main()
