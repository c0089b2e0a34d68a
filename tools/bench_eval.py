"""Times the evaluation run on the device (DESIGN.md §3, README): forward_snapshots against forward at batch 64, the
ground-truth work of a 64-sample 480x640 batch with the visibility mask, and the same evaluation per sample on the host
with numpy / scipy for comparison.  Appends JSON lines to --out (default profiles/h100_eval.jsonl).

    python tools/bench_eval.py [--batch 64] [--reps 20] [--host-samples 4] [--out profiles/h100_eval.jsonl]
"""
import argparse
import os
import time

import numpy as np
import scipy.ndimage
import torch

from benchkit import ROOT, Rows, call_times, summary
from demon_b200 import evaluation as ev
from demon_b200 import lmbspecialops as sops
from demon_b200 import weights as W
from demon_b200.networks_original import DemonPipeline, Session
from oracle import view_tools as vt


def median_ms(fn, reps):
    return summary(call_times(fn, reps))["ms"]


def host_errors(pred, gt):
    """The eleven distances and the abs scale factor of metrics.py:240-318 in numpy, for the host comparison."""
    valid = np.isfinite(pred) & np.isfinite(gt) & (pred > 0) & (gt > 0)
    p, g = 1 / pred[valid], 1 / gt[valid]
    s = (p * g).sum() / (p * p).sum()
    out = []
    for q in (p, p * s):
        d, ld = q - g, np.log(q) - np.log(g)
        out.append([np.abs(d).mean(), np.abs(1 / q - 1 / g).mean(), np.sqrt(max(0, (ld ** 2).mean() - ld.mean() ** 2)),
                    (np.abs(d) / g).mean(), (d * d / g).mean(), np.abs(np.log10(q) - np.log10(g)).mean(), np.sqrt((ld ** 2).mean()),
                    np.sqrt((d * d).mean())] + [(np.abs(ld) < np.log(t)).mean() for t in (1.25, 1.5625, 1.953125)])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--host-samples", type=int, default=4)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_eval.jsonl"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_eval needs a CUDA device")
    B, reps = args.batch, args.reps
    rows = Rows(args.out)
    sess = Session()
    sess.load_weights(W.synthetic_weights(0))
    pipe = DemonPipeline(sess, batch_size=B, iterations=3)
    g = torch.Generator().manual_seed(0)
    ip = (torch.rand(B, 6, 192, 256, generator=g) - 0.5).cuda()
    pipe.stage(ip)
    # alternate the three calls in one window so that drift on a shared host hits all of them alike
    t_fwd = summary(call_times(lambda: pipe.forward_staged(), reps))
    t_snap = median_ms(lambda: pipe.forward_snapshots(ip, refine=False), reps)
    t_snap_r = median_ms(lambda: pipe.forward_snapshots(ip, refine=True), reps)
    t_fwd2 = summary(call_times(lambda: pipe.forward_staged(), reps))
    fwd = min(t_fwd["ms"], t_fwd2["ms"])
    rows.add({"bench": "forward_snapshots", "batch": B, "iterations": 3, "precision": sess.precision, "forward_ms": fwd,
              "forward_ms_runs": [[t["ms"], t["ms_min"], t["ms_max"]] for t in (t_fwd, t_fwd2)],
              "snapshots_ms": t_snap, "snapshots_refined_ms": t_snap_r, "snapshots_refined_over_forward": t_snap_r / fwd,
              "launches_forward": pipe.launches(), "launches_snapshots_refined": pipe.snapshot_launches()})

    # ground truth of the batch: 480x640 inverse depth with holes, motions, intrinsics
    n, gh, gw = B, 480, 640
    rng = np.random.RandomState(1)
    yy, xx = np.mgrid[0:gh, 0:gw]
    inv = np.stack([(0.3 + 0.15 * np.sin(xx / (40.0 + i)) + 0.1 * np.cos(yy / 25.0)) for i in range(n)]).astype(np.float32)
    inv[rng.rand(n, gh, gw) < 0.02] = np.nan
    motion = np.concatenate([rng.normal(0, 0.05, (n, 3)), rng.normal(0, 0.4, (n, 3))], axis=1).astype(np.float32)
    intr = np.tile(np.array([[0.89, 1.19, 0.5, 0.5]], dtype=np.float32), (n, 1))
    preds = {k: v.clone() for k, v in pipe.forward_snapshots(ip, refine=True).items()}
    inv_d, motion_d, intr_d = torch.from_numpy(inv).cuda(), torch.from_numpy(motion).cuda(), torch.from_numpy(intr).cuda()
    ops = [torch.from_numpy(o).cuda() for o in ev.visible_points_operands(motion, intr, gh, gw)]
    mask = torch.empty((n, gh, gw), dtype=torch.uint8, device="cuda")
    lib = ev._lib.load()

    def run_mask():
        ev._lib.check(lib.demon_visible_points_mask_inverse_f32(inv_d.data_ptr(), *[o.data_ptr() for o in ops], n, gh, gw, gw, gh, 0, 0,
                                                               mask.data_ptr(), ev._stream()))

    def run_flow():
        return sops.depth_to_flow(inv_d.reshape(n, 1, gh, gw), intr_d, motion_d[:, 0:3].contiguous(), motion_d[:, 3:6].contiguous(),
                                  rotation_format="angleaxis3", inverse_depth=True, normalize_flow=True)
    flow = run_flow()
    rs2 = ev._Resampler(48, 64, gh, gw, (0, 0, gh, gw), torch.device("cuda"))
    rs0 = ev._Resampler(192, 256, gh, gw, (0, 0, gh, gw), torch.device("cuda"))
    _, gt_div = ev.motion_errors(preds["predict_rotation"][0], preds["predict_translation"][0], motion_d)

    def run_sums():
        for k in range(4):
            for rs, p in ((rs2, preds["predict_depth2"][k]), (rs0, preds["predict_depth0"][k])):
                s = rs.depth_sums(p, inv_d, mask, gt_div)
                rs.depth_sums(p, inv_d, mask, gt_div, ev.depth_scale_factor(s))
            rs2.flow_sums(preds["predict_flow2"][k], flow)

    def run_motion():
        for k in range(4):
            ev.motion_errors(preds["predict_rotation"][k], preds["predict_translation"][k], motion_d)
    t_mask, t_flow, t_sums, t_mot = (median_ms(f, reps) for f in (run_mask, run_flow, run_sums, run_motion))
    t_batch = median_ms(lambda: ev.evaluate_batch(preds, inv_d, motion_d, intr, depthmask=True), max(5, reps // 2))
    rows.add({"bench": "ground_truth_work", "samples": n, "gt": [gh, gw], "depthmask": True, "mask_ms": t_mask, "flow_gt_ms": t_flow,
              "sums_8_snapshots_ms": t_sums, "motion_ms": t_mot, "device_ms": t_mask + t_flow + t_sums + t_mot,
              "evaluate_batch_ms": t_batch, "evaluate_batch_note": "whole call: host operand construction, launches, one copy, host table"})

    # the same per sample on the host: numpy mask, scipy zoom of 8 depth snapshots and 4 flows, numpy errors
    hp = {k: v[:, :args.host_samples].cpu().numpy() for k, v in preds.items()}
    flow_h = flow[:args.host_samples].cpu().numpy()
    hops = ev.visible_points_operands(motion[:args.host_samples], intr[:args.host_samples], gh, gw)
    t0 = time.perf_counter()
    for i in range(args.host_samples):
        with np.errstate(all='ignore'):
            gt = inv[i].copy()
            m = vt.visible_points_mask_numpy(1 / gt, *[o[i] for o in hops], gw, gh)
            gt[m == 0] = np.nan
            for k in range(4):
                for pred in (hp["predict_depth2"][k, i, 0], hp["predict_depth0"][k, i, 0]):
                    z = scipy.ndimage.zoom(pred, (gh / pred.shape[0], gw / pred.shape[1]), order=0, grid_mode=True, mode='grid-constant')
                    host_errors(z, gt)
                f = np.stack([scipy.ndimage.zoom(c, (10, 10), order=0, grid_mode=True, mode='grid-constant') for c in hp["predict_flow2"][k, i]])
                epe = np.sqrt(((f - flow_h[i]) ** 2).sum(0))
                epe[np.isfinite(epe) & (epe > 0)].mean()
                ev.compute_motion_errors(np.concatenate([hp["predict_rotation"][k, i], hp["predict_translation"][k, i]]), motion[i], True)
    host_ms = (time.perf_counter() - t0) * 1000 / args.host_samples
    rows.add({"bench": "ground_truth_work_host", "samples_timed": args.host_samples, "per_sample_ms": host_ms,
              "per_64_samples_ms": host_ms * 64, "cpu": os.cpu_count(), "note": "numpy / scipy on one host thread per sample"})
    rows.save()


if __name__ == "__main__":
    main()
