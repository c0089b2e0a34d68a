"""Times the v2 pipeline's input paths (README, DESIGN.md §3.6) with synthetic v2 weights at 3xTF32, batch 64, 3 iterations:
forward_images on 640x480 uint8 photos (bicubic, image2_2 'resize') and forward_views on the same photos with their
intrinsics, each next to forward on the prepared float pair in the same window; forward_snapshots with refinement plus
evaluate_batch at a 480x640 ground truth with the visibility mask (tools/bench_eval.py's v1 rows); the standalone
images.resize_area at [32,3,192,256] -> 48x64.  CUDA events, median of --reps calls; GPU name and power limit are read in
the same run.  Appends JSON lines to --out (default profiles/h100_v2_inputs.jsonl).

    python tools/bench_v2_inputs.py [--reps 20] [--out profiles/h100_v2_inputs.jsonl]
"""
import argparse
import os

import numpy as np
import torch

from benchkit import ROOT, Rows, call_times, summary
from demon_b200 import evaluation as ev, images
from demon_b200.v2 import weights as W2
from demon_b200.v2.networks import DemonPipelineV2, Session


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_v2_inputs.jsonl"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_v2_inputs needs a CUDA device")
    B, reps = args.batch, args.reps
    rows = Rows(args.out)
    s = Session("3xtf32")
    s.load_weights(W2.synthetic_weights(0))
    pipe = DemonPipelineV2(s, batch_size=B, iterations=3)
    rng = np.random.default_rng(0)
    photos = torch.from_numpy(rng.integers(0, 256, (B, 2, 480, 640, 3), dtype=np.uint8)).cuda()
    f = rng.uniform(500, 560, (B, 2))
    K = torch.from_numpy(np.stack([f, f, np.full((B, 2), 320.0), np.full((B, 2), 240.0)], -1)).cuda()
    prepared = images.prepare_input_data(photos[:, 0], photos[:, 1])
    pipe.stage(prepared["image_pair"], prepared["image2_2"])
    # each input path alternates with forward on the prepared floats in one window, so that drift hits both alike
    for name, call in (("forward_images", lambda: pipe.forward_images(photos, "bicubic", "resize")),
                       ("forward_views", lambda: pipe.forward_views(photos, K, "bicubic", "resize"))):
        t_fwd = summary(call_times(lambda: pipe.forward_staged(use_image2_2=True), reps))
        t_in = summary(call_times(call, reps))
        t_fwd2 = summary(call_times(lambda: pipe.forward_staged(use_image2_2=True), reps))
        fwd = min(t_fwd["ms"], t_fwd2["ms"])
        rows.add({"bench": "v2_" + name, "batch": B, "source": [480, 640], "resample": "bicubic", "image2_2": "resize", "iterations": 3,
                  "precision": "3xtf32", "ms": t_in["ms"], "ms_min": t_in["ms_min"], "ms_max": t_in["ms_max"],
                  "pairs_per_s": B * 1000.0 / t_in["ms"], "forward_on_prepared_floats_ms": fwd,
                  "forward_ms_runs": [[t["ms"], t["ms_min"], t["ms_max"]] for t in (t_fwd, t_fwd2)], "over_forward_ms": t_in["ms"] - fwd,
                  "launches": pipe.launches()})

    # forward_snapshots with refinement and evaluate_batch at 480x640 with the mask, as tools/bench_eval.py's v1 rows
    ip = prepared["image_pair"]
    t_snap = summary(call_times(lambda: pipe.forward_snapshots(ip, refine=True), reps))
    preds = {k: v.clone() for k, v in pipe.forward_snapshots(ip, refine=True).items()}
    n, gh, gw = B, 480, 640
    r = np.random.RandomState(1)
    yy, xx = np.mgrid[0:gh, 0:gw]
    inv = np.stack([(0.3 + 0.15 * np.sin(xx / (40.0 + i)) + 0.1 * np.cos(yy / 25.0)) for i in range(n)]).astype(np.float32)
    inv[r.rand(n, gh, gw) < 0.02] = np.nan
    motion = np.concatenate([r.normal(0, 0.05, (n, 3)), r.normal(0, 0.4, (n, 3))], axis=1).astype(np.float32)
    intr = np.tile(np.array([[0.89, 1.19, 0.5, 0.5]], dtype=np.float32), (n, 1))
    inv_d, motion_d = torch.from_numpy(inv).cuda(), torch.from_numpy(motion).cuda()
    t_eval = summary(call_times(lambda: ev.evaluate_batch(preds, inv_d, motion_d, intr, depthmask=True), max(5, reps // 2)))["ms"]
    rows.add({"bench": "v2_forward_snapshots_evaluate", "batch": B, "iterations": 3, "precision": "3xtf32", "gt": [gh, gw],
              "depthmask": True, "snapshots_refined_ms": t_snap["ms"], "snapshots_refined_ms_min": t_snap["ms_min"],
              "evaluate_batch_ms": t_eval, "total_ms": t_snap["ms"] + t_eval, "launches_snapshots_refined": pipe.snapshot_launches(),
              "evaluate_batch_note": "whole call: host operand construction, launches, one copy, host table"})

    # the standalone resize_area: one pass over 32 x 3 x 192 x 256 floats
    x = (torch.rand(32, 3, 192, 256, generator=torch.Generator().manual_seed(2)) - 0.5).cuda()
    out = torch.empty(32, 3, 48, 64, device="cuda")
    t_area = summary(call_times(lambda: images._resize_area_into(x, out), max(reps, 100)))
    nbytes = (x.numel() + out.numel()) * 4
    rows.add({"bench": "v2_resize_area", "shape": list(x.shape), "size": [48, 64], "ms": t_area["ms"], "ms_min": t_area["ms_min"],
              "ms_max": t_area["ms_max"], "bytes": nbytes, "gb_per_s": nbytes / (t_area["ms"] * 1e-3) / 1e9,
              "note": "one launch; time includes the launch and the event pair around it"})
    rows.save()


if __name__ == "__main__":
    main()
