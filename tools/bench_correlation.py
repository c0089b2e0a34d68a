"""Device time of correlation / correlation_1d ('mult') and their gradients (csrc/correlation.cu) against the reference's own
CUDA kernels (oracle/_ref/libref_correlation.so) on the same card in the same call, at FlowNetC's correlation layer
(C 256 at 48x64, pad_size 20, kernel_size 1, max_displacement 20, stride2 2: 441 displacements; batch 8 and 64) and at
DispNetC's 1D layer (max_displacement 40, stride2 1, pad_size 40, C 256: 81 displacements; batch 8).

Ours: CUDA events around `--reps` back-to-back calls after warm-up.  The reference: the summed device time of every kernel
and memset one call of its Compute() launches (torch.profiler), so its host-side cudaMalloc and synchronisations are not
counted against it.  Both outputs are compared bit for bit at the timed size.  Operation counts come from the shapes:
forward = 2 N top_c top_h top_w K^2 C (one FMA per product); the gradient = twice that (each product is one FMA in each
input's gather).  Bytes: each tensor read or written once.  Share of peak = the larger of FLOP / 67 TFLOP/s and
bytes / 3.35 TB/s (H100 SXM data sheet, 700 W) over the measured time.  The card's name and power limit are read in the
same call.

    python tools/bench_correlation.py [--reps 20] [--out profiles/h100_correlation.jsonl]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from demon_b200 import lmbspecialops as ops
from oracle import correlation_ref as cref
from oracle.ref import digest

PEAK_FLOPS, PEAK_BYTES = 67e12, 3.35e12
ROWS = [
    ("flownetc", False, 8, dict(max_displacement=20, kernel_size=1, stride1=1, stride2=2, pad_size=20)),
    ("flownetc", False, 64, dict(max_displacement=20, kernel_size=1, stride1=1, stride2=2, pad_size=20)),
    ("dispnetc_1d", True, 8, dict(max_displacement=40, kernel_size=1, stride1=1, stride2=1, pad_size=40)),
]


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in out.split(","))
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception:
        return {"gpu": torch.cuda.get_device_name(), "power_limit": None, "max_sm_clock": None}


def event_ms(fn, reps, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def reference_device_ms(fn, reps):
    """mean summed device time (kernels and memsets) of one reference call"""
    fn()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    us = sum(e.device_time_total for e in prof.events()
             if e.device_type == torch.autograd.DeviceType.CUDA and "Memcpy" not in e.name)
    return us / 1e3 / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--ref-reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark measures the GPU"
    if not cref.have_library():
        sys.exit("oracle/_ref/libref_correlation.so is not built (build() with DEMON_REF_SRC set)")
    info = gpu_info()
    lines = []
    for name, one_d, n, attrs in ROWS:
        rng = np.random.RandomState(0)
        shape = (n, 256, 48, 64)
        x1 = rng.randn(*shape).astype(np.float32)
        x2 = rng.randn(*shape).astype(np.float32)
        a, b = torch.from_numpy(x1).cuda(), torch.from_numpy(x2).cuda()
        fwd = ops.correlation_1d if one_d else ops.correlation
        grad = ops.correlation_1d_grad if one_d else ops.correlation_grad
        rfwd = cref.correlation_1d if one_d else cref.correlation
        rgrad = cref.correlation_1d_grad if one_d else cref.correlation_grad
        top = fwd(a, b, **attrs)
        g = torch.from_numpy(rng.randn(*top.shape).astype(np.float32)).cuda()
        gnp = g.cpu().numpy()
        ours_g = grad(g, a, b, **attrs)
        same = (digest(top.cpu().numpy()) == digest(rfwd(x1, x2, **attrs))
                and all(digest(o.cpu().numpy()) == digest(r) for o, r in zip(ours_g, rgrad(gnp, x1, x2, **attrs))))
        fwd_ms = event_ms(lambda: fwd(a, b, **attrs), args.reps)
        grad_ms = event_ms(lambda: grad(g, a, b, **attrs), args.reps)
        ref_fwd_ms = reference_device_ms(lambda: rfwd(x1, x2, **attrs), args.ref_reps)
        ref_grad_ms = reference_device_ms(lambda: rgrad(gnp, x1, x2, **attrs), args.ref_reps)
        _, tc, th, tw = top.shape
        flop_f = 2.0 * n * tc * th * tw * attrs["kernel_size"] ** 2 * 256
        bytes_f = 4.0 * (2 * x1.size + top.numel())
        flop_g, bytes_g = 2 * flop_f, 4.0 * (4 * x1.size + top.numel())
        row = {"op": name, "batch": n, "shape": list(shape), "attrs": attrs, "top": list(top.shape), "corr_type": "mult",
               "bits_equal_reference": bool(same)}
        for what, ms, rms, flop, nbytes in (("forward", fwd_ms, ref_fwd_ms, flop_f, bytes_f), ("grad", grad_ms, ref_grad_ms, flop_g, bytes_g)):
            t_c, t_m = flop / PEAK_FLOPS, nbytes / PEAK_BYTES
            row[what] = {"ms": round(ms, 4), "reference_ms": round(rms, 4), "speedup": round(rms / ms, 2),
                         "gflop": round(flop / 1e9, 3), "tflops": round(flop / ms / 1e9, 2), "mbytes": round(nbytes / 1e6, 1),
                         "share_of_peak": round(max(t_c, t_m) * 1e3 / ms, 3), "bound": "fp32" if t_c >= t_m else "hbm"}
        row.update(info)
        lines.append(row)
        print(json.dumps(row), flush=True)
        del a, b, top, g, ours_g
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
