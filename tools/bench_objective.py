"""Times demon_b200.v2.objective, training/v2/training.py's objective for a v2 checkpoint on one batch, per evolution at
training.py's batch sizes: 32 for 0_flow1 .. 3_dm2, and 8 new + 24 earlier samples for 4_iterative and 5_refine (netFlow1
and netDM1 on the 8, netFlow2 onwards on all 32; the earlier predictions are netDM1's for those 24 samples, made once
before timing).  The batch comes from datareader.build_batch over synthetic views with every rot180 / mirror_x pair, the
weights are v2.weights.synthetic_weights (no trained v2 weights are published).

Each row: milliseconds per call (median of CUDA-event timed calls, after warm-up) and the library's kernel launches per
call (its own launch counter; torch's own small ops of the composition are not counted), with the card's name and power
limit read in the same run.  One JSON line per evolution:
    python tools/bench_objective.py [--steps K] [--warmup W] [--precision 3xtf32] [--out profiles/h100_objective.jsonl]
"""
import argparse
import os
import sys

import numpy as np
import torch

from benchkit import Rows, call_times, library_launches, summary
from demon_b200 import datareader as dr
from demon_b200 import images
from demon_b200.dataset_tools import View
from demon_b200.v2 import blocks, objective
from demon_b200.v2 import weights as W2
from demon_b200.v2.networks import Session
from oracle.datareader import synthetic_views

BATCH, NEW = 32, 8   # training.py:92-94 and its queue of _simulated_iterations - 1 = 3 earlier batches


def training_batch(b, seed):
    pool = dr.ViewPool(256, 192)
    pool.add([View(*v) for v in synthetic_views(8, 480, 640, seed)])
    rng = np.random.default_rng(seed)
    pairs = [tuple(int(i) for i in rng.choice(8, 2, replace=False)) for _ in range(b)]
    params = {'batch_size': b, 'motion_format': 'ANGLEAXIS6', 'inverse_depth': True, 'norm_trans_scale_depth': True,
              'scaled_width': 256, 'scaled_height': 192, 'top_output': ('IMAGE_PAIR', 'MOTION', 'DEPTH', 'INTRINSICS')}
    aug = dr.Augmentation(np.arange(b) % 2 == 1, (np.arange(b) // 2) % 2 == 1)
    return dr.build_batch(pool, pairs, params, aug)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--precision", default="3xtf32")
    ap.add_argument("--out", default=os.path.join("profiles", "h100_objective.jsonl"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_objective needs a CUDA device")
    rows = Rows(args.out)
    session = Session(precision=args.precision)
    session.load_weights(W2.synthetic_weights(0))
    batch = training_batch(BATCH, 3)
    ip = batch['IMAGE_PAIR']
    # the earlier iterations' predictions for rows NEW.. : netDM1 on them, as the queue holds them at the start
    i22 = images.resize_area(ip[NEW:, 3:6], (48, 64))
    fc2 = blocks.flow_block(ip[NEW:], scope='netFlow1', session=session)['predict_flowconf2']
    earlier = blocks.depthmotion_block(ip[NEW:], i22, fc2[:, 0:2], fc2, scope='netDM1', session=session)
    session.kernel_l2()   # once per load_weights, not part of a call
    for evo in objective.EVOLUTIONS:
        prev = earlier if evo >= '4_iterative' else None

        def call(evo=evo, prev=prev):
            return objective.objective(session, batch, evo, prev)
        res = call()
        torch.cuda.synchronize()
        ms = summary(call_times(call, args.steps, args.warmup, sync_each=False))["ms"]
        rows.add({"row": "objective", "evolution": evo, "batch": BATCH, "new_samples": NEW if prev is not None else BATCH,
                  "precision": args.precision, "ms": round(ms, 3), "library_launches": library_launches(call),
                  "total": float(res["total"]), "finite": bool(all(torch.isfinite(v).item() for v in res.values()))})
    rows.save()
    if not all(r["finite"] for r in rows):
        sys.exit("a loss is not finite")


if __name__ == "__main__":
    main()
