"""Times DeMoN v2's training losses on the device (demon_b200.v2.losses) against the same computation composed from this
project's mirror ops and torch, in the same run, at training.py's shapes: batch 32, depth 192x256, levels 2 and 5.

Rows: ground-truth preparation; the forward pass of each block; forward + backward of the losses one '4_iterative' step
adds to the loss collection (netFlow2 and netDM2 blocks, training.py:354-427) and of one '5_refine' step (netRefine,
training.py:442-452).  Each row checks that both paths agree and reports milliseconds (median of CUDA-event timed
steps) and kernel launches per step (counted by torch.profiler).  One JSON line per row:
    python tools/bench_losses.py [--steps K] [--warmup W] [--out profiles/h100_losses.jsonl]
"""
import argparse
import os
import sys

import numpy as np
import torch

from benchkit import Rows, call_times, profiled_kernels, summary
from demon_b200 import lmbspecialops as sops
from demon_b200.v2 import losses as L

N, H, W = 32, 192, 256
FLOW = dict(flow_weight=1000.0, conf_weight=1000.0, flow_sig_weight=1000.0, conf_sig_weight=1000.0, conf_diff_scale=10, level5_factor=0)
DN = dict(depth_weight=300.0, depth_sig_weight=1500.0, normal_weight=100.0, rotation_weight=160.0, translation_weight=15.0,
          translation_factor=1)
REFINE = dict(depth_weight=300.0, depth_sig_weight=750.0, normal_weight=100.0)


# ---- the composition from the mirror ops and torch ---------------------------------------------------------------------------
def c_ground_truth(depth, rot, tr, k):
    lv = [depth]
    for _ in range(5):
        lv.append(sops.median3x3_downsample(lv[-1]))

    def flow(d):
        return sops.depth_to_flow(d, k, rot, tr, inverse_depth=True, normalize_flow=True)
    f2 = flow(lv[2])
    return {"depth0": depth, "depth0_sig": c_sig(depth, 0.001), "depth2": lv[2], "depth2_sig": c_sig(lv[2], 0.001), "flow0": flow(depth),
            "flow2": f2, "flow2_sig": c_sig(f2, 0.001), "flow5": flow(lv[5]), "normal0": sops.depth_to_normals(depth, k, True),
            "normal2": sops.depth_to_normals(lv[2], k, True)}


def c_sig(x, eps):
    return torch.cat([sops.scale_invariant_gradient_autograd(x, [d], [1.0], eps) for d in L.SIG_DELTAS], dim=1)


def c_l2(pr, gt, eps):
    d = pr - gt.detach()
    d = torch.where(torch.isfinite(d), d, torch.zeros_like(d))   # replace_nonfinite and its gradient
    return torch.sqrt((d * d).sum(1) + eps).mean()


def c_l1(x, eps):
    return torch.sqrt(x * x + eps).sum()


def c_flow_block(g, f2, f5, c2, c5, a):
    e = 0.00001
    conf2 = torch.exp(-a["conf_diff_scale"] * torch.abs(f2 - g["flow2"])).detach()
    conf5 = torch.exp(-a["conf_diff_scale"] * torch.abs(f5 - g["flow5"])).detach()
    return {"loss_flow5": (a["level5_factor"] * a["flow_weight"]) * c_l2(f5, g["flow5"], e), "loss_flow2": a["flow_weight"] * c_l2(f2, g["flow2"], e),
            "loss_conf5": (a["level5_factor"] * a["conf_weight"]) * c_l2(c5, conf5, e), "loss_conf2": a["conf_weight"] * c_l2(c2, conf2, e),
            "loss_flow2_sig": a["flow_sig_weight"] * c_l2(c_sig(f2, 0.001), g["flow2_sig"], e),
            "loss_conf2_sig": a["conf_sig_weight"] * c_l2(c_sig(c2, 0.001), c_sig(conf2, 0.001), e)}


def c_dn_block(g, rot_gt, tr_gt, d2, n2, rot, tr, a):
    e = 0.00001
    tnf = (a["translation_weight"] / N) * c_l1(tr - tr_gt, e)
    return {"loss_depth2": a["depth_weight"] * c_l2(d2, g["depth2"], e), "loss_depth2_sig": a["depth_sig_weight"] * c_l2(c_sig(d2, 0.01), g["depth2_sig"], e),
            "loss_normal2": a["normal_weight"] * c_l2(n2, g["normal2"], e), "loss_rotation": (a["rotation_weight"] / N) * c_l1(rot - rot_gt, e),
            "loss_translation": a["translation_factor"] * tnf}


def c_refine_block(g, d0, n0, a):
    e = 0.00001
    return {"loss_depth0": a["depth_weight"] * c_l2(d0, g["depth0"], e), "loss_depth0_sig": a["depth_sig_weight"] * c_l2(c_sig(d0, 0.01), g["depth0_sig"], e),
            "loss_normal0": a["normal_weight"] * c_l2(n0, g["normal0"], e)}


# ---- measurement ---------------------------------------------------------------------------------------------------------------
def agree(a, b, rtol):
    a, b = float(a.detach()), float(b.detach())
    return abs(a - b) <= rtol * max(abs(b), 1e-30)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=os.path.join("profiles", "h100_losses.jsonl"))
    args = ap.parse_args()
    torch.manual_seed(0)
    dev = "cuda"
    rng = np.random.RandomState(0)
    depth = rng.uniform(0.2, 2.0, (N, 1, H, W))
    depth[rng.rand(N, 1, H, W) < 0.03] = np.nan
    k = np.tile([0.89115971, 1.18821287, 0.5, 0.5], (N, 1))
    rot_gt = rng.uniform(-0.1, 0.1, (N, 3))
    tr_gt = rng.uniform(-0.5, 0.5, (N, 3)) + np.array([0.5, 0.0, 0.1])
    depth, k, rot_gt, tr_gt = (torch.from_numpy(a).float().to(dev) for a in (depth, k, rot_gt, tr_gt))
    g = L.prepare_ground_truth_tensors(depth, rot_gt, tr_gt, k)

    def noisy(t, s):
        return (torch.nan_to_num(t, nan=0.5, posinf=0.5, neginf=0.5) + s * torch.randn_like(t)).contiguous()
    pr = {"f2": noisy(g["flow2"], 0.01), "f5": noisy(g["flow5"], 0.01), "c2": torch.rand_like(g["flow2"]), "c5": torch.rand_like(g["flow5"]),
          "d2": noisy(g["depth2"], 0.05).abs() + 0.01, "n2": noisy(g["normal2"], 0.1), "rot": noisy(rot_gt, 0.01), "tr": noisy(tr_gt, 0.05),
          "d0": noisy(g["depth0"], 0.05).abs() + 0.01, "n0": noisy(g["normal0"], 0.1)}
    leaf = {key: v.clone().requires_grad_(True) for key, v in pr.items()}
    flow_sel = ("loss_flow5", "loss_flow2", "loss_flow2_sig", "loss_conf5", "loss_conf2", "loss_conf2_sig")
    dn_sel = ("loss_depth2", "loss_depth2_sig", "loss_normal2", "loss_rotation", "loss_translation")

    def f_flow(p):
        return L.flow_loss_block(g["flow2"], g["flow5"], g["flow2_sig"], p["f2"], p["f5"], p["c2"], p["c5"], loss_prefix="", **FLOW)

    def f_dn(p):
        return L.depthnormal_loss_block(g["depth2"], g["depth2_sig"], g["normal2"], rot_gt, tr_gt, p["d2"], p["n2"], p["rot"], p["tr"], **DN)

    def f_refine(p):
        return L.depth_refine_loss_block(g["depth0"], g["depth0_sig"], g["normal0"], p["d0"], p["n0"], **REFINE)

    def c_flow(p):
        return c_flow_block(g, p["f2"], p["f5"], p["c2"], p["c5"], FLOW)

    def c_dn(p):
        return c_dn_block(g, rot_gt, tr_gt, p["d2"], p["n2"], p["rot"], p["tr"], DN)

    def c_refine(p):
        return c_refine_block(g, p["d0"], p["n0"], REFINE)

    def step(blocks, sel, p):
        def run():
            for v in p.values():
                v.grad = None
            total = None
            for blk, keys in zip(blocks, sel):
                r = blk(p)
                for key in keys:
                    total = r[key] if total is None else total + r[key]
            total.backward()
            return total
        return run

    rows = Rows(args.out)

    def timed(fn):
        return round(summary(call_times(fn, args.steps, args.warmup, sync_each=False))["ms"], 4)

    def row(name, fused, composed, check):
        with torch.no_grad() if "backward" not in name else torch.enable_grad():
            ok = check()
            rec = {"row": name, "batch": N, "depth_hw": [H, W], "fused_ms": timed(fused), "composed_ms": timed(composed),
                   "fused_launches": profiled_kernels(fused), "composed_launches": profiled_kernels(composed), "agree": bool(ok)}
        rec["speedup"] = round(rec["composed_ms"] / rec["fused_ms"], 2)
        rows.add(rec)

    row("prepare_ground_truth", lambda: L.prepare_ground_truth_tensors(depth, rot_gt, tr_gt, k), lambda: c_ground_truth(depth, rot_gt, tr_gt, k),
        lambda: all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in
                    zip(L.prepare_ground_truth_tensors(depth, rot_gt, tr_gt, k).values(), c_ground_truth(depth, rot_gt, tr_gt, k).values())))
    for name, f, c, keys in (("flow_loss_block_forward", f_flow, c_flow, flow_sel), ("depthnormal_loss_block_forward", f_dn, c_dn, dn_sel),
                             ("depth_refine_loss_block_forward", f_refine, c_refine, ("loss_depth0", "loss_depth0_sig", "loss_normal0"))):
        row(name, lambda f=f: f(pr), lambda c=c: c(pr), lambda f=f, c=c, keys=keys: all(agree(f(pr)[key], c(pr)[key], 1e-4) for key in keys))
    fused_it, comp_it = step((f_flow, f_dn), (flow_sel, dn_sel), leaf), step((c_flow, c_dn), (flow_sel, dn_sel), leaf)
    fused_rf, comp_rf = step((f_refine,), (("loss_depth0", "loss_depth0_sig", "loss_normal0"),), leaf), \
        step((c_refine,), (("loss_depth0", "loss_depth0_sig", "loss_normal0"),), leaf)

    def grads_agree(a, b, keys):
        a()
        ga = {key: leaf[key].grad.clone() for key in keys}
        b()
        return all(torch.allclose(ga[key], leaf[key].grad, rtol=1e-3, atol=1e-6 * float(leaf[key].grad.abs().max())) for key in keys)
    row("4_iterative_forward_backward", fused_it, comp_it, lambda: grads_agree(fused_it, comp_it, ("f2", "f5", "c2", "c5", "d2", "n2", "rot", "tr")))
    row("5_refine_forward_backward", fused_rf, comp_rf, lambda: grads_agree(fused_rf, comp_rf, ("d0", "n0")))
    rows.save()
    if not all(r["agree"] for r in rows):
        sys.exit("the fused and composed results disagree")


if __name__ == "__main__":
    main()
