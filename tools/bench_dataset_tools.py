"""Times the dataset tools on the device (demon_b200.dataset_tools, csrc/dataset_tools.cu; DESIGN.md §3, README): the
sharpness of 256 frames of 480x640 and the consistency counts of 512 pair-directions of 480x640 depth, against the
reference's host work for the same calls (numpy / scipy / Pillow per frame; the reference's Cython compute_depth_ratios
per pair from oracle/_ref, where it was built).  Appends JSON lines to --out (default profiles/h100_dataset_tools.jsonl).

    python tools/bench_dataset_tools.py [--reps 20] [--host-frames 8] [--host-pairs 8] [--out ...]
"""
import argparse
import os
import time

import numpy as np
import scipy.ndimage
import torch
from PIL import Image

from benchkit import ROOT, Rows, call_times, library_launches, summary
from demon_b200 import _lib
from demon_b200 import dataset_tools as dt
from oracle import view_tools as vt

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet


def views(n, h, w, seed=0):
    from demon_b200.evaluation import angleaxis_to_rotation_matrix, intrinsics_vector_to_K
    rng = np.random.RandomState(seed)
    K = intrinsics_vector_to_K(np.array([0.891, 1.188, 0.5, 0.5]), w, h)
    yy, xx = np.mgrid[0:h, 0:w]
    base = (2.0 + np.sin(xx / 50.0) + 0.5 * np.cos(yy / 30.0))
    out = []
    for i in range(n):
        d = (base * rng.uniform(0.97, 1.03) + rng.normal(0, 0.01, (h, w))).astype(np.float32)
        d[rng.rand(h, w) < 0.03] = np.nan
        out.append(dt.View(R=angleaxis_to_rotation_matrix(rng.normal(0, 0.02, 3)), t=rng.normal(0, 0.1, 3), K=K, image=None, depth=d,
                           depth_metric='camera_z'))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--host-frames", type=int, default=8)
    ap.add_argument("--host-pairs", type=int, default=8)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_dataset_tools.jsonl"))
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a GPU"
    rows = Rows(args.out)

    # sharpness: 256 frames of 480x640 RGB
    n, h, w = 256, 480, 640
    rng = np.random.RandomState(1)
    host = rng.randint(0, 256, (n, h, w, 3)).astype(np.uint8)
    frames = torch.from_numpy(host).cuda()
    tm = summary(call_times(lambda: dt.sharpness(frames), args.reps, warmup=3))
    med = tm["ms"]
    moved = 2 * n * h * w * 3 + 4 * n   # the frames read once per pass, the results
    line = {"bench": "sharpness", "frames": n, "size": [h, w], "device_ms": med, "device_ms_min": tm["ms_min"],
            "device_ms_max": tm["ms_max"], "reps": args.reps, "bytes_moved": moved, "achieved_GBps": moved / (med * 1e-3) / 1e9,
            "hbm_share": moved / (med * 1e-3) / HBM_BYTES_PER_S, "launches_per_call": library_launches(lambda: dt.sharpness(frames))}
    k = min(args.host_frames, n)
    if k > 0:
        t0 = time.perf_counter()
        for i in range(k):
            np.var(scipy.ndimage.laplace(np.array(Image.fromarray(host[i]).convert('L'), np.float32)))
        per = (time.perf_counter() - t0) * 1e3 / k
        line.update({"host_ms_per_frame": per, "host_ms_per_batch": per * n, "host_frames_timed": k,
                     "host_note": "measure_sharpness's numpy / scipy / Pillow calls, one host thread"})
    rows.add(line)

    # consistency counts: 512 pair-directions among 64 views of 480x640
    nv, npairs = 64, 256
    vs = views(nv, h, w)
    K, R, t, P = dt.view_operands(vs)
    depth = torch.from_numpy(np.stack([v.depth for v in vs])).cuda()
    prng = np.random.RandomState(2)
    fwd = [(int(i), int((i + 1 + prng.randint(nv - 1)) % nv)) for i in prng.randint(0, nv, npairs)]
    pairs = fwd + [(j, i) for i, j in fwd]
    pr = dt._pairs(pairs, nv)
    lo_t, hi_t = dt.ratio_thresholds(0.9)
    counts = torch.empty((len(pairs), 2), dtype=torch.int64, device="cuda")
    lib = _lib.load()

    def run():   # the C entry alone: the pairs and operands are on the device already
        _lib.check(lib.demon_depth_consistency_counts_f32(depth.data_ptr(), K.data_ptr(), R.data_ptr(), t.data_ptr(), P.data_ptr(), nv, h,
                                                          w, pr.data_ptr(), len(pairs), float(lo_t), float(hi_t), counts.data_ptr(),
                                                          dt._stream()))
    tm = summary(call_times(run, args.reps, warmup=3))
    med = tm["ms"]
    moved = len(pairs) * h * w * 4 * 2   # depth i streamed, depth j gathered (at least once per pair)
    line = {"bench": "consistency_counts", "pair_directions": len(pairs), "views": nv, "size": [h, w], "device_ms": med,
            "device_ms_min": tm["ms_min"], "device_ms_max": tm["ms_max"], "reps": args.reps, "bytes_moved": moved,
            "achieved_GBps": moved / (med * 1e-3) / 1e9, "hbm_share": moved / (med * 1e-3) / HBM_BYTES_PER_S,
            "launches_per_call": library_launches(run),
            "bytes_note": "two depth maps per pair direction; the 64 views' 79 MB mostly stay in L2, so this is L2-level traffic"}
    if vt.have_module() and args.host_pairs > 0:
        m = vt.module()
        k = min(args.host_pairs, len(pairs))
        t0 = time.perf_counter()
        for i, j in pairs[:k]:
            dr = m.compute_depth_ratios(vs[i], vs[j])
            valid = dr[np.isfinite(dr)]
            np.count_nonzero((valid > 0.9) & (valid < 1 / 0.9))
        per = (time.perf_counter() - t0) * 1e3 / k
        line.update({"host_cython_ms_per_pair": per, "host_cython_ms_per_call": per * len(pairs), "host_pairs_timed": k,
                     "host_note": "reference Cython compute_depth_ratios (-O2) and check_depth_consistency's numpy, one host thread"})
    rows.add(line)
    rows.save()


if __name__ == "__main__":
    main()
