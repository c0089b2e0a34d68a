"""Times demon_b200.datareader (README, DESIGN.md §3.8): ViewPool.add of 64 views from 640x480 to 256x192, and build_batch
at training.py's batch 32 and at batch 8 (its setting from 4_iterative on) with all six outputs, colour augmentation on and
off; and, for comparison, the numpy oracle (oracle/datareader.py) building the same batch-8 batch on one host core.
Device times are CUDA events around whole calls (host pose math, the table upload and the launch included), the median
of --reps calls after a warm-up; bytes moved are computed from the shapes.  GPU name and power limit are read in the same
run.  Appends JSON lines to --out (default profiles/h100_datareader.jsonl).

    python tools/bench_datareader.py [--reps 20] [--out profiles/h100_datareader.jsonl]
"""
import os

for _v in ("OMP_NUM_THREADS", "OPENBLAS_NUM_THREADS", "MKL_NUM_THREADS"):   # the oracle runs on one host core
    os.environ[_v] = "1"

import argparse   # noqa: E402
import time       # noqa: E402

import numpy as np   # noqa: E402
import torch         # noqa: E402

from benchkit import ROOT, Rows, call_times, summary       # noqa: E402
from demon_b200 import datareader as dr                    # noqa: E402
from demon_b200.dataset_tools import View                  # noqa: E402
from oracle import datareader as od                        # noqa: E402


def batch_bytes(b, h, w, nd=1):
    """Bytes the batch kernel must move: two uint8 RGB views and the depths it reads, the four float32 planes outputs."""
    reads = b * h * w * (2 * 3 + 4 * nd)
    writes = b * h * w * 4 * (6 + 2 + nd + nd)
    return reads + writes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_datareader.jsonl"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_datareader needs a CUDA device")
    rows = Rows(args.out)
    raw = od.synthetic_views(64, 480, 640, 0)
    views = [View(*v) for v in raw]
    pool = dr.ViewPool(256, 192)
    pool.add(views)   # warm-up and the pool the batches read
    t = summary(call_times(lambda: dr.ViewPool(256, 192).add(views), args.reps))
    nbytes = 64 * (480 * 640 * (3 + 4) + 192 * 256 * (3 + 4))
    rows.add({"bench": "datareader_add", "views": 64, "source": [480, 640], "scaled": [192, 256], "ms": t["ms"], "ms_min": t["ms_min"],
              "ms_max": t["ms_max"], "bytes": nbytes, "gb_per_s": nbytes / (t["ms"] * 1e-3) / 1e9,
              "note": "whole call: host staging, one upload of the 640x480 sources, one launch, pool allocation"})

    rng = np.random.default_rng(1)
    colour_params = {'aug_hsv_hue': {'normal': {'mean': 0, 'stddev': 10}}, 'aug_contrast': {'uniform': {'a': 0.8, 'b': 1.2}},
                     'aug_brightness': {'normal': {'mean': 0, 'stddev': 0.1}}, 'aug_gamma': {'uniform': {'a': 0.8, 'b': 1.2}}}
    for b in (32, 8):
        pairs = [tuple(rng.choice(64, 2, replace=False)) for _ in range(b)]
        params = {'batch_size': b, 'motion_format': 'ANGLEAXIS6', 'inverse_depth': True, 'norm_trans_scale_depth': True,
                  'top_output': dr.OUTPUTS}
        for colour in (False, True):
            aug = dr.draw_augmentation(dict(params, **(colour_params if colour else {})), b, rng)
            t = summary(call_times(lambda: dr.build_batch(pool, pairs, params, aug), args.reps))
            nbytes = batch_bytes(b, 192, 256)
            rows.add({"bench": "datareader_build_batch", "batch": b, "colour": colour, "outputs": list(dr.OUTPUTS), "ms": t["ms"],
                      "ms_min": t["ms_min"], "ms_max": t["ms_max"], "bytes": nbytes, "gb_per_s": nbytes / (t["ms"] * 1e-3) / 1e9,
                      "note": "whole call: host pose math, one table upload, one launch, output allocation"})
        if b == 8:
            prepared = [od.prepare(img, d, K, R, t_, m, 256, 192) for R, t_, K, img, d, m in raw[:max(max(p) for p in pairs) + 1]]
            p = dr.reader_params(params)
            for colour in (False, True):
                aug = dr.draw_augmentation(dict(params, **(colour_params if colour else {})), b, rng)
                times = []
                for _ in range(3):
                    t0 = time.perf_counter()
                    od.build_batch(prepared, pairs, p, aug.rot180, aug.mirror_x, aug.colour)
                    times.append((time.perf_counter() - t0) * 1e3)
                rows.add({"bench": "datareader_oracle_build_batch", "batch": b, "colour": colour, "ms": float(np.median(times)),
                          "note": "numpy oracle on one host core (BLAS threads 1), median of 3"})
    rows.save()


if __name__ == "__main__":
    main()
