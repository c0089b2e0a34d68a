"""Device time of flow_warp, flow_warp_grad and resample (csrc/flow_ops.cu) against the reference's own CUDA kernels
(oracle/_ref/libref_flow_ops.so) on the same card in the same call: warp and warp-grad at FlowNet2's image size
[8,3,384,512] and at a feature warp [8,256,48,64]; resample x4 LINEAR up of a flow [8,2,96,128] -> 384x512, x4 CUBIC
antialiased down [8,3,384,512] -> 96x128, and NEAREST [8,3,384,512] -> 192x256.

Ours: CUDA events around `--reps` back-to-back calls of the Python op after warm-up, so output allocation and the ctypes
call are included (they dominate the shortest rows).  The reference: the summed device time of the kernels one call of
its Compute() launches (torch.profiler); its cudaMemsets, the harness's copies in and out and its host-side cudaMalloc
and synchronisations are not counted against it.  Bytes: each input and output read or written once; achieved bytes/s
against 3.35 TB/s (H100 SXM data sheet).  `equal` is the tests' equality: flow_warp, flow_grad and resample bit for bit with the reference's GPU
kernels; image_grad within (k-1) eps sum|addends| of its atomic sums.  The card's name and power limit are read in the
same call.

    python tools/bench_flow_ops.py [--reps 20] [--out profiles/h100_flow_ops.jsonl]
"""
import argparse
import os
import sys

import numpy as np
import torch

from benchkit import ROOT, Rows, device_events, span_ms
from demon_b200 import lmbspecialops as ops
from oracle import flow_ops as of
from oracle import flow_ops_ref as fref

PEAK_BYTES = 3.35e12
EPS = float(np.finfo(np.float32).eps)


def reference_ms(fn):
    fn()   # warm-up
    out, events = device_events(fn)
    return out, sum(e.device_time_total for e in events if not e.name.startswith(("Memcpy", "Memset"))) / 1e3


def bits_equal(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and bool(np.all((a == b) | (np.isnan(a) & np.isnan(b))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_flow_ops.jsonl"))
    args = ap.parse_args()
    if not fref.have_library():
        sys.exit("needs oracle/_ref/libref_flow_ops.so (build with DEMON_REF_SRC set)")
    rows = Rows(args.out)
    rng = np.random.RandomState(0)
    for name, shape in (("image", (8, 3, 384, 512)), ("feature", (8, 256, 48, 64))):
        image = rng.randn(*shape).astype(np.float32)
        flow = (rng.randn(shape[0], 2, shape[2], shape[3]) * 4).astype(np.float32)
        grad = rng.randn(*shape).astype(np.float32)
        ti, tf, tg = (torch.from_numpy(v).cuda() for v in (image, flow, grad))
        ours = ops.flow_warp(ti, tf)
        ref, ref_ms = reference_ms(lambda: fref.flow_warp_gpu(image, flow))
        ms = span_ms(lambda: ops.flow_warp(ti, tf), args.reps)
        nbytes = 4 * (2 * image.size + flow.size)
        rows.add(dict(op="flow_warp", shape=list(shape), ms=ms, ref_ms=ref_ms, bytes=nbytes,
                      bytes_per_s=nbytes / ms * 1e3, share_of_hbm=nbytes / ms * 1e3 / PEAK_BYTES,
                      equal=bits_equal(ours.cpu().numpy(), ref)))
        ig, fg = ops.flow_warp_grad(ti, tf, tg)
        (rig, rfg), ref_ms = reference_ms(lambda: fref.flow_warp_grad_gpu(image, flow, grad))
        ms = span_ms(lambda: ops.flow_warp_grad(ti, tf, tg), args.reps)
        mag = of.flow_warp_grad(np.zeros_like(image), flow, np.abs(grad))[0]
        ig = ig.cpu().numpy()
        inside, L, T, R, B, _, _ = of._cells(flow)
        k = np.zeros(shape)
        for yy, xx in ((T, L), (T, R), (B, L), (B, R)):
            for n in range(shape[0]):
                np.add.at(k[n], (slice(None), yy[n][inside[n]], xx[n][inside[n]]), 1.0)
        within = bool(np.all(np.abs(ig.astype(np.float64) - rig) <= np.maximum(k - 1, 0) * EPS * mag + 1e-300))
        nbytes = 4 * (3 * image.size + 2 * flow.size)
        rows.add(dict(op="flow_warp_grad", shape=list(shape), ms=ms, ref_ms=ref_ms, bytes=nbytes,
                      bytes_per_s=nbytes / ms * 1e3, share_of_hbm=nbytes / ms * 1e3 / PEAK_BYTES,
                      equal=bits_equal(fg.cpu().numpy(), rfg) and within))
    for label, shape, oh, ow, rtype in (("x4_linear_up", (8, 2, 96, 128), 384, 512, "LINEAR"),
                                        ("x4_cubic_aa_down", (8, 3, 384, 512), 96, 128, "CUBIC"),
                                        ("nearest_half", (8, 3, 384, 512), 192, 256, "NEAREST")):
        x = rng.randn(*shape).astype(np.float32)
        tx = torch.from_numpy(x).cuda()
        ours = ops.resample(tx, ow, oh, True, rtype)
        ref, ref_ms = reference_ms(lambda: fref.resample_gpu(x, ow, oh, True, rtype))
        ms = span_ms(lambda: ops.resample(tx, ow, oh, True, rtype), args.reps)
        nbytes = 4 * (x.size + shape[0] * shape[1] * oh * ow)
        rows.add(dict(op="resample_" + label, shape=list(shape), out=[oh, ow], ms=ms, ref_ms=ref_ms, bytes=nbytes,
                      bytes_per_s=nbytes / ms * 1e3, share_of_hbm=nbytes / ms * 1e3 / PEAK_BYTES,
                      equal=bits_equal(ours.cpu().numpy(), ref)))
    rows.save()


if __name__ == "__main__":
    main()
