"""Times the point clouds on the device (demon_b200.vis.point_clouds, csrc/vis.cu; DESIGN.md §3, README): 64 views of
192x256 inverse depth with image colours, with and without normals, and 8 views of 768x1024, against the reference's
Cython (oracle/_ref/vis_cython.so, where it was built) on the host for the same work.  Appends JSON lines to --out
(default profiles/h100_pointcloud.jsonl).

    python tools/bench_pointcloud.py [--reps 50] [--host-views 4] [--out profiles/h100_pointcloud.jsonl]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_eval import device_info, time_ms   # noqa: E402
from demon_b200 import vis                    # noqa: E402
from oracle import vis as ov                  # noqa: E402

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet


def inputs(n, h, w, seed=0):
    """Inverse depth like the network's (about 2 % invalid), the float image, normals and the sun3d K."""
    rng = np.random.RandomState(seed)
    inv = rng.uniform(0.1, 2.0, (n, h, w)).astype(np.float32)
    inv[rng.rand(n, h, w) < 0.02] = 0.0
    img = rng.uniform(-0.5, 0.5, (n, 3, h, w)).astype(np.float32)
    nrm = rng.normal(0, 1, (n, 3, h, w)).astype(np.float32)
    return inv, img, nrm, vis.prediction_K(None, n, h, w)


def bytes_moved(n, h, w, valid, normals):
    """DRAM traffic the two launches need at least: the depth twice (count, scatter), the image (and normals) once, and
    12 + 3 (+ 12) bytes per emitted point."""
    px = n * h * w
    return 2 * 4 * px + 12 * px + (12 * px if normals else 0) + valid * (12 + 3 + (12 if normals else 0))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--host-views", type=int, default=4)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_pointcloud.jsonl"))
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a GPU"
    info = device_info()
    lines = []
    for n, h, w, normals in ((64, 192, 256, False), (64, 192, 256, True), (8, 768, 1024, False)):
        inv, img, nrm, K = inputs(n, h, w)
        dev = dict(d=torch.from_numpy(inv).cuda(), i=torch.from_numpy(img).cuda(), n=torch.from_numpy(nrm).cuda(),
                   K=torch.from_numpy(K).cuda(), R=torch.eye(3, device="cuda"), t=torch.zeros(3, device="cuda"))

        def run():
            return vis.point_clouds(dev['d'], dev['K'], dev['R'], dev['t'], normals=dev['n'] if normals else None, image=dev['i'],
                                    inverse_depth=True)
        med, lo, hi = time_ms(run, args.reps, warmup=5)
        valid = int(run()['counts'].sum())
        moved = bytes_moved(n, h, w, valid, normals)
        line = {"bench": "point_clouds", "views": n, "size": [h, w], "normals": normals, "colors": "image", "inverse_depth": True,
                "device_ms": med, "device_ms_min": lo, "device_ms_max": hi, "reps": args.reps, "points": valid,
                "bytes_moved": moved, "achieved_GBps": moved / (med * 1e-3) / 1e9,
                "hbm_share": moved / (med * 1e-3) / HBM_BYTES_PER_S, "launches_per_call": 2}
        if ov.have_module() and args.host_views > 0:
            # visualize_prediction's host work per view: 1/inverse depth, the uint8 colours, the reference's Cython
            m = ov.module()
            k = min(args.host_views, n)
            t0 = time.perf_counter()
            for i in range(k):
                with np.errstate(all='ignore'):
                    depth = 1 / inv[i]
                m.compute_point_cloud_from_depthmap(depth, K[i], np.eye(3), np.zeros(3), nrm[i] if normals else None,
                                                    ov.image_to_colors(img[i]))
            per_view = (time.perf_counter() - t0) * 1e3 / k
            line.update({"host_cython_ms_per_view": per_view, "host_cython_ms_per_batch": per_view * n, "host_views_timed": k,
                         "host_note": "reference Cython (-O2), one host thread, including 1/inverse depth and the uint8 cast"})
        line.update(info)
        lines.append(line)
        print(json.dumps(line), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "a") as f:
        for line in lines:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
