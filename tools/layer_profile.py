"""Per-layer device time of the full pipeline at batch 64 (or argv[3]) (CUDA events around every layer launch through the
C ABI's demon_net_profile_* hooks).  Prints a table sorted by time and writes it as JSON."""
import ctypes
import json
import os
import sys

import torch

from benchkit import ROOT, span_ms
from demon_b200 import _lib, weights as W
from demon_b200.networks_original import Session, DemonPipeline


def main():
    precision = sys.argv[1] if len(sys.argv) > 1 else "3xtf32"
    out_path = sys.argv[2] if len(sys.argv) > 2 else os.path.join(ROOT, "gpurun_out", "layers_%s.json" % precision)
    B = int(sys.argv[3]) if len(sys.argv) > 3 else 64
    steps = 5
    lib = _lib.load()
    sess = Session(precision)
    sess.load_weights(W.synthetic_weights(0))
    pipe = DemonPipeline(sess, B, 3)
    g = torch.Generator().manual_seed(1234)
    x = (torch.rand(B, 6, 192, 256, generator=g) - 0.5).cuda()
    for _ in range(3):
        pipe.forward(x, None)
    torch.cuda.synchronize()
    _lib.check(lib.demon_net_profile_begin(pipe.net.ptr))
    total = span_ms(lambda: pipe.forward(x, None), steps, warmup=0)
    _lib.check(lib.demon_net_profile_end(pipe.net.ptr))
    lm = W.layer_macs()
    rows = []
    for i in range(lib.demon_net_num_layers(pipe.net.ptr)):
        name = lib.demon_net_layer_name(pipe.net.ptr, i).decode()
        t, calls, lpc, tc = ctypes.c_double(), ctypes.c_int64(), ctypes.c_int(), ctypes.c_int()
        lib.demon_net_layer_profile(pipe.net.ptr, i, ctypes.byref(t), ctypes.byref(calls), ctypes.byref(lpc), ctypes.byref(tc))
        if calls.value:
            ms = t.value / steps
            macs = lm[name] * B * calls.value / steps
            rows.append({"layer": name, "ms_per_step": ms, "calls_per_step": calls.value // steps, "tc": bool(tc.value),
                         "gmac_per_step": macs / 1e9, "tflops": 2 * macs / (ms / 1e3) / 1e12 if ms > 0 else 0})
    rows.sort(key=lambda r: -r["ms_per_step"])
    layer_sum = sum(r["ms_per_step"] for r in rows)
    print("precision %s  step %.2f ms (%.0f pairs/s)  sum of layer times %.2f ms  glue+gaps %.2f ms" % (
        precision, total, B / total * 1e3, layer_sum, total - layer_sum))
    print("%-44s %8s %6s %3s %9s %8s" % ("layer", "ms/step", "calls", "tc", "GMAC/step", "TFLOP/s"))
    for r in rows:
        print("%-44s %8.3f %6d %3s %9.2f %8.1f" % (r["layer"], r["ms_per_step"], r["calls_per_step"], "tc" if r["tc"] else "-",
                                                   r["gmac_per_step"], r["tflops"]))
    # group by layer basename across blocks
    json.dump({"precision": precision, "ms_per_step": total, "layers": rows}, open(out_path, "w"), indent=1)


if __name__ == "__main__":
    main()
