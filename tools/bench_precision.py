"""Times the tensor-core precisions against each other (README, DESIGN.md §3.1 and §4): fp16, tf32 and 3xtf32 on the v1
pipeline (bootstrap + 3 iterations + refinement) at batch 64 and batch 1, the v1 refinement block at 1024x768 batch 8 and
the v2 pipeline at batch 64, with synthetic weights.  In one process, the precisions alternate step by step (one timed step
of each in turn, `--reps` rounds), so clock and thermal drift fall on all three alike; each step is bracketed by CUDA
events.  A second, separate pass records one v1 batch-64 step per precision under torch.profiler and sums the device time
of conv_tc_halo_kernel by kind (halo-box modes: halo, 8-channel and fold; per-tap), and an FP16 cuBLAS GEMM (torch.matmul,
8192^3) gives the card's attainable FP16 tensor-core rate in the same run.  Appends JSON lines to --out (default
profiles/h100_precision.jsonl).

    python tools/bench_precision.py [--reps 20] [--out profiles/h100_precision.jsonl]
"""
import argparse
import json
import os
import re
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from demon_b200 import weights as W1                                             # noqa: E402
from demon_b200.networks_original import DemonPipeline, RefinementNet, Session   # noqa: E402
from demon_b200.v2 import weights as W2                                          # noqa: E402
from demon_b200.v2.networks import DemonPipelineV2, Session as SessionV2         # noqa: E402

PRECS = ("fp16", "tf32", "3xtf32")


def device_info():
    """The card's name and power limit, read in the same call as the timings."""
    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        info["power_limit"], info["max_sm_clock"] = [s.strip() for s in q.split(",")]
    except Exception as e:   # the figure is still a measurement; say that the power limit could not be read
        info["power_limit"] = "unknown (%s)" % type(e).__name__
    return info


def alternate(steps, reps, warmup=3):
    """steps: {precision: fn}.  Runs one step of each precision in turn, `reps` rounds after `warmup`; returns
    {precision: [ms per step]}."""
    for _ in range(warmup):
        for fn in steps.values():
            fn()
    torch.cuda.synchronize()
    times = {p: [] for p in steps}
    for _ in range(reps):
        for p, fn in steps.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            b.synchronize()
            times[p].append(a.elapsed_time(b))
    return times


def summary(ts):
    return dict(ms=float(np.median(ts)), ms_min=float(np.min(ts)), ms_max=float(np.max(ts)), steps=len(ts))


def kernel_kind(name):
    m = re.search(r"conv_tc_halo_kernel<(true|false)", name)
    return None if not m else ("per-tap" if m.group(1) == "true" else "halo")


def profile_conv_kernels(fn):
    """Device time of conv_tc_halo_kernel per kind over one call of fn, and every other kernel's, from torch.profiler."""
    fn()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {"halo": 0.0, "per-tap": 0.0, "other": 0.0}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        out[kernel_kind(ev.name) or "other"] += ev.device_time_total / 1000.0
    return out


def cublas_fp16_tflops(n=8192, reps=20):
    a = torch.randn(n, n, device="cuda", dtype=torch.float16)
    b = torch.randn(n, n, device="cuda", dtype=torch.float16)
    ts = alternate({"gemm": lambda: torch.matmul(a, b)}, reps)["gemm"]
    return 2.0 * n ** 3 / (float(np.median(ts)) * 1e-3) / 1e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_precision.jsonl"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_precision needs a CUDA device")
    info = device_info()
    lines = []
    g = torch.Generator().manual_seed(1234)
    s1 = {p: Session(p) for p in PRECS}
    s2 = {p: SessionV2(p) for p in PRECS}
    w1, w2 = W1.synthetic_weights(0), W2.synthetic_weights(0)
    for p in PRECS:
        s1[p].load_weights(w1)
        s2[p].load_weights(w2)

    def record(bench, times, per_step, unit, **extra):
        base = summary(times["3xtf32"])["ms"]
        for p in PRECS:
            sm = summary(times[p])
            lines.append(dict(bench=bench, precision=p, **sm, **{unit: per_step * 1000.0 / sm["ms"]},
                              speedup_vs_3xtf32=base / sm["ms"], speedup_vs_tf32=summary(times["tf32"])["ms"] / sm["ms"], **extra, **info))
            print(json.dumps(lines[-1]))

    for batch in (64, 1):
        x = (torch.rand(batch, 6, 192, 256, generator=g) - 0.5).cuda()
        pipes = {p: DemonPipeline(s1[p], batch_size=batch, iterations=3) for p in PRECS}
        record("v1_pipeline", alternate({p: (lambda q=pipes[p]: q.forward(x)) for p in PRECS}, args.reps), batch, "pairs_per_s",
               batch=batch, iterations=3)
        del pipes
    im = (torch.rand(8, 3, 768, 1024, generator=g) - 0.5).cuda()
    d2 = (torch.rand(8, 1, 192, 256, generator=g) * 0.6 + 0.2).cuda()
    nets = {p: RefinementNet(s1[p], "channels_first", 8, image_size=(768, 1024)) for p in PRECS}
    record("v1_refine", alternate({p: (lambda n=nets[p]: n.eval(im, d2)) for p in PRECS}, args.reps), 8, "images_per_s",
           batch=8, size=[768, 1024])
    del nets
    x = (torch.rand(64, 6, 192, 256, generator=g) - 0.5).cuda()
    pipes = {p: DemonPipelineV2(s2[p], batch_size=64, iterations=3) for p in PRECS}
    record("v2_pipeline", alternate({p: (lambda q=pipes[p]: q.forward(x)) for p in PRECS}, args.reps), 64, "pairs_per_s",
           batch=64, iterations=3)
    del pipes
    # separate pass: where the time of one v1 batch-64 step goes, per precision
    x = (torch.rand(64, 6, 192, 256, generator=g) - 0.5).cuda()
    tflops = cublas_fp16_tflops()
    for p in PRECS:
        pipe = DemonPipeline(s1[p], batch_size=64, iterations=3)
        k = profile_conv_kernels(lambda: pipe.forward(x))
        lines.append(dict(bench="v1_pipeline_kernels", precision=p, batch=64, conv_tc_halo_ms=k["halo"], conv_tc_per_tap_ms=k["per-tap"],
                          other_kernels_ms=k["other"], note="torch.profiler device time of one step, outside the timed runs",
                          **info))
        print(json.dumps(lines[-1]))
        del pipe
    gflop = 2 * W1.macs_per_pair()["pipeline"] / 1e9
    fp16_b64 = [ln for ln in lines if ln["bench"] == "v1_pipeline" and ln["precision"] == "fp16" and ln["batch"] == 64][0]
    lines.append(dict(bench="cublas_fp16_gemm", m=8192, n=8192, k=8192, tflops=tflops,
                      v1_b64_fp16_tflops=gflop * 64 / fp16_b64["ms"], v1_b64_fp16_share_of_cublas=gflop * 64 / fp16_b64["ms"] / tflops,
                      note="torch.matmul fp16 (cuBLAS), median of 20; the pipeline's rate counts 2 x its multiply-accumulates",
                      **info))
    print(json.dumps(lines[-1]))
    with open(args.out, "a") as f:
        for ln in lines:
            f.write(json.dumps(ln) + "\n")


if __name__ == "__main__":
    main()
