"""Times demon_b200.v2.objective, training/v2/training.py's objective for a v2 checkpoint on one batch, per evolution at
training.py's batch sizes: 32 for 0_flow1 .. 3_dm2, and 8 new + 24 earlier samples for 4_iterative and 5_refine (netFlow1
and netDM1 on the 8, netFlow2 onwards on all 32; the earlier predictions are netDM1's for those 24 samples, made once
before timing).  The batch comes from datareader.build_batch over synthetic views with every rot180 / mirror_x pair, the
weights are v2.weights.synthetic_weights (no trained v2 weights are published).

Each row: milliseconds per call (median of CUDA-event timed calls, after warm-up) and the library's kernel launches per
call (demon_launch_count; torch's own small ops of the composition are not counted), with the card's name and power
limit read in the same run.  One JSON line per evolution:
    python tools/bench_objective.py [--steps K] [--warmup W] [--precision 3xtf32] [--out profiles/h100_objective.jsonl]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from demon_b200 import _lib                     # noqa: E402
from demon_b200 import datareader as dr        # noqa: E402
from demon_b200 import images                  # noqa: E402
from demon_b200.dataset_tools import View      # noqa: E402
from demon_b200.v2 import blocks, objective    # noqa: E402
from demon_b200.v2 import weights as W2        # noqa: E402
from demon_b200.v2.networks import Session     # noqa: E402
from oracle.datareader import synthetic_views  # noqa: E402

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


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
    for a, b in ev:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    return float(np.median([a.elapsed_time(b) for a, b in ev]))


def launches(fn):
    """Kernels the library launches in one call (its own counter, demon_launch_count); the torch ops of the composition
    (contiguous copies of channel slices, concatenations, scalar adds) come on top."""
    lib = _lib.load()
    n0 = lib.demon_launch_count()
    fn()
    return int(lib.demon_launch_count() - n0)


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                         timeout=30, check=True).stdout.strip().splitlines()[0]
    name, limit = (s.strip() for s in out.split(","))
    return name, limit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--precision", default="3xtf32")
    ap.add_argument("--out", default=os.path.join("profiles", "h100_objective.jsonl"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_objective needs a CUDA device")
    name, limit = gpu_info()
    session = Session(precision=args.precision)
    session.load_weights(W2.synthetic_weights(0))
    batch = training_batch(BATCH, 3)
    ip = batch['IMAGE_PAIR']
    # the earlier iterations' predictions for rows NEW.. : netDM1 on them, as the queue holds them at the start
    i22 = images.resize_area(ip[NEW:, 3:6], (48, 64))
    fc2 = blocks.flow_block(ip[NEW:], scope='netFlow1', session=session)['predict_flowconf2']
    earlier = blocks.depthmotion_block(ip[NEW:], i22, fc2[:, 0:2], fc2, scope='netDM1', session=session)
    session.kernel_l2()   # once per load_weights, not part of a call
    rows = []
    for evo in objective.EVOLUTIONS:
        prev = earlier if evo >= '4_iterative' else None

        def call(evo=evo, prev=prev):
            return objective.objective(session, batch, evo, prev)
        res = call()
        torch.cuda.synchronize()
        rec = {"row": "objective", "evolution": evo, "batch": BATCH, "new_samples": NEW if prev is not None else BATCH,
               "precision": args.precision, "ms": round(timed(call, args.steps, args.warmup), 3), "library_launches": launches(call),
               "total": float(res["total"]), "finite": bool(all(torch.isfinite(v).item() for v in res.values())),
               "gpu": name, "power_limit": limit}
        print(json.dumps(rec), flush=True)
        rows.append(rec)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            for r in rows:
                fh.write(json.dumps(r) + "\n")
    if not all(r["finite"] for r in rows):
        sys.exit("a loss is not finite")


if __name__ == "__main__":
    main()
