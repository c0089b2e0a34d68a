"""Times the v2 network on the device (README, DESIGN.md §0): the fused v2 pipeline (bootstrap + 3 iterations +
refinement) at batch 64 and batch 1, the v2 refinement block at 1024x768 batch 8, and dense5 alone at batch 1 (its 85 MB
weight read), all at 3xTF32 with synthetic v2 weights.  Appends JSON lines to --out (default profiles/h100_v2.jsonl).
GFLOP per pair are counted like demon_b200.weights.layer_macs counts v1's (2 x multiply-accumulates, no padding waste).

    python tools/bench_v2.py [--reps 20] [--out profiles/h100_v2.jsonl]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from demon_b200 import _lib                                   # noqa: E402
from demon_b200.v2 import weights as W2                        # noqa: E402
from demon_b200.v2.networks import DemonPipelineV2, RefinementNet, Session   # noqa: E402


def device_info():
    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        info["power_limit"], info["max_sm_clock"] = [s.strip() for s in q.split(",")]
    except Exception as e:   # the figure is still a measurement; say that the power limit could not be read
        info["power_limit"] = "unknown (%s)" % type(e).__name__
    return info


def time_ms(fn, reps, warmup=3):
    """Median, min and max per-call time over `reps` calls, each bracketed by CUDA events on the current stream."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times)), float(np.min(times)), float(np.max(times))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_v2.jsonl"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_v2 needs a CUDA device")
    info = device_info()
    lines = []
    s = Session("3xtf32")
    s.load_weights(W2.synthetic_weights(0))
    macs = W2.macs_per_pair()
    gflop_pair = 2 * macs["pipeline"] / 1e9
    g = torch.Generator().manual_seed(1234)
    for batch in (64, 1):
        pipe = DemonPipelineV2(s, batch_size=batch, iterations=3)
        x = (torch.rand(batch, 6, 192, 256, generator=g) - 0.5).cuda()
        med, lo, hi = time_ms(lambda: pipe.forward(x), args.reps)
        lines.append(dict(bench="v2_pipeline", batch=batch, iterations=3, precision="3xtf32", ms=med, ms_min=lo, ms_max=hi,
                          pairs_per_s=batch * 1000.0 / med, gflop_per_pair=gflop_pair, tflops=gflop_pair * batch / med,
                          launches=pipe.launches(), **info))
    # refinement block at 1024x768, batch 8
    rn = RefinementNet(s, "channels_first", 8, image_size=(768, 1024))
    im = (torch.rand(8, 3, 768, 1024, generator=g) - 0.5).cuda()
    d2 = (torch.rand(8, 1, 192, 256, generator=g) * 0.6 + 0.2).cuda()
    med, lo, hi = time_ms(lambda: rn.eval(im, d2, None), args.reps)
    gflop_ref = 2 * sum(v for k, v in W2.layer_macs((768, 1024)).items() if k.startswith("netRefine/")) / 1e9
    lines.append(dict(bench="v2_refine", batch=8, size=[768, 1024], precision="3xtf32", ms=med, ms_min=lo, ms_max=hi,
                      images_per_s=8 * 1000.0 / med, gflop_per_image=gflop_ref, **info))
    # dense5 at batch 1: per-layer CUDA events of the stage-wise bootstrap (demon_net_profile_*)
    lib = _lib.load()
    net = s.net(1)
    from demon_b200.v2.networks import BootstrapNet
    bn = BootstrapNet(s, "channels_first", 1)
    ip = (torch.rand(1, 6, 192, 256, generator=g) - 0.5).cuda()
    i22 = (torch.rand(1, 3, 48, 64, generator=g) - 0.5).cuda()
    for _ in range(3):
        bn.eval(ip, i22)
    torch.cuda.synchronize()
    _lib.check(lib.demon_net_profile_begin(net.ptr))
    for _ in range(args.reps):
        bn.eval(ip, i22)
    torch.cuda.synchronize()
    _lib.check(lib.demon_net_profile_end(net.ptr))
    for i in range(lib.demon_net_num_layers(net.ptr)):
        name = lib.demon_net_layer_name(net.ptr, i).decode()
        if name in ("netFlow1/dense5", "netDM1/dense5"):   # the two the bootstrap runs
            ms, calls = ctypes.c_double(), ctypes.c_int64()
            _lib.check(lib.demon_net_layer_profile(net.ptr, i, ctypes.byref(ms), ctypes.byref(calls), None, None))
            if calls.value == 0 or ms.value <= 0:
                raise RuntimeError("no device time recorded for %s (calls %d, ms %g)" % (name, calls.value, ms.value))
            per = ms.value / calls.value
            lines.append(dict(bench="v2_dense5", layer=name, batch=1, ms=per, weight_mb=4608 * 4608 * 4 / 1e6,
                              gb_per_s=4608 * 4608 * 4 / (per * 1e-3) / 1e9,
                              note="the dense kernel and its split-K reduction, without the gather / scatter copies", **info))
    with open(args.out, "a") as f:
        for ln in lines:
            f.write(json.dumps(ln) + "\n")
            print(json.dumps(ln))


if __name__ == "__main__":
    main()
