"""Times the sparse TSDF volume (SparseTsdfVolume; README, DESIGN.md §3.9) beside the dense TsdfVolume, and appends JSON
lines to --out with the device name and power limit in every row.

1. orbit: tools/bench_sequence.py's orbit_frames (64 and 256 frames of 192x256, colour on and off) at the dense 256^3
   volume's voxel size and origin.  Dense: integrate into the volume, and mesh.  Sparse: the first integrate of a fresh
   volume (allocation, pool growth and integration), integrate again into the filled volume, and mesh.  Blocks and the
   bytes of state (pool and hash table for the sparse volume) for both.
2. corridor: a walk of 256 frames down a 3 x 2.5 x 40.5 m box (sequence_oracle.render_depth) at 5 mm voxels, whose
   bounding box is past the dense volume's 2^31-voxel limit, without colour (4 KB per block), integrated 64 frames per
   call: ms per frame of each call, blocks, skipped pixels and bytes, then the mesh.

Device times are CUDA events around the call after a warm-up call, median of --reps (the sparse integrate synchronises
once per call, so its time includes that host round trip).

    python tools/bench_sparse_tsdf.py [--reps 10] [--out profiles/h100_sparse_tsdf.jsonl]
"""
import argparse
import os

import numpy as np
import torch

from benchkit import ROOT, Rows, call_times, summary
from bench_sequence import orbit_frames
from demon_b200 import sequence
import sequence_oracle as so


def corridor_frames(n, h=192, w=256):
    """n depth maps of a camera walking down the inside of a long box, swaying sideways and looking ahead."""
    K = so.K_pixels(so.NETWORK_INTRINSICS, w, h)
    box = ((-1.5, -1.25, -0.5), (1.5, 1.25, 40.0))
    Rs, ts, ds = [], [], []
    for k, z in enumerate(np.linspace(0.5, 30.0, n)):
        c = np.array([0.6 * np.sin(0.05 * k), 0.2 * np.sin(0.031 * k), z])
        R, t = so.look_at(c, c + np.array([0.3 * np.sin(0.023 * k), 0.05, 1.0]), up=(0, 1, 0))
        Rs.append(R)
        ts.append(t)
        ds.append(so.render_depth(R, t, K, h, w, box=box))
    img = np.random.RandomState(1).randint(0, 256, (n, h, w, 3)).astype(np.uint8)
    return np.array(ds, np.float32), K.astype(np.float32), np.array(Rs, np.float32), np.array(ts, np.float32), img, box


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_sparse_tsdf.jsonl"))
    args = ap.parse_args()
    rows = Rows(args.out)
    dims, origin, vs = (256, 256, 256), (-1.25, -1.25, -1.25), 2.5 / 255
    d, K, R, t, img = orbit_frames(256)
    dev = {k: torch.from_numpy(v).cuda() for k, v in dict(d=d, K=K, R=R, t=t, img=img).items()}
    for n in (64, 256):
        for color in (False, True):
            fr = (dev["d"][:n], dev["K"], dev["R"][:n], dev["t"][:n], dev["img"][:n] if color else None)
            dense = sequence.TsdfVolume(dims, origin, vs, color=color)
            tm = summary(call_times(lambda: dense.integrate(*fr), args.reps, warmup=1))
            dense = sequence.TsdfVolume(dims, origin, vs, color=color).integrate(*fr)
            mesh_ms = summary(call_times(dense.mesh, args.reps, warmup=1))["ms"]
            nbytes = sum(x.numel() * x.element_size() for x in (dense.tsdf, dense.weight, dense.color) if x is not None)
            rows.add({"bench": "orbit", "volume": "dense", "frames": n, "color": color, "voxel_size": vs, "dims": dims,
                      "integrate_ms": tm["ms"], "integrate_ms_min": tm["ms_min"], "integrate_ms_max": tm["ms_max"], "mesh_ms": mesh_ms,
                      "triangles": int(dense.mesh()[2].shape[0]), "voxels": int(np.prod(dims)), "state_bytes": nbytes})
            del dense
            first = summary(call_times(lambda: sequence.SparseTsdfVolume(vs, origin, color=color).integrate(*fr), args.reps, warmup=1))
            sp = sequence.SparseTsdfVolume(vs, origin, color=color).integrate(*fr)
            again = summary(call_times(lambda: sp.integrate(*fr), args.reps, warmup=1))
            sp = sequence.SparseTsdfVolume(vs, origin, color=color).integrate(*fr)
            mesh_ms = summary(call_times(sp.mesh, args.reps, warmup=1))["ms"]
            m = int(sp.blocks.shape[0])
            rows.add({"bench": "orbit", "volume": "sparse", "frames": n, "color": color, "voxel_size": vs,
                      "integrate_first_ms": first["ms"], "integrate_first_ms_min": first["ms_min"],
                      "integrate_first_ms_max": first["ms_max"], "integrate_again_ms": again["ms"],
                      "integrate_again_ms_min": again["ms_min"], "integrate_again_ms_max": again["ms_max"], "mesh_ms": mesh_ms,
                      "triangles": int(sp.mesh()[2].shape[0]), "blocks": m, "voxels": 512 * m, "capacity_blocks": sp.capacity,
                      "table_slots": sp.table_slots, "state_bytes": sp.nbytes, "skipped_pixels": sp.last_skipped_pixels})
            del sp
            torch.cuda.empty_cache()

    n, chunk, cvs = 256, 64, 0.005
    d, K, R, t, img, box = corridor_frames(n)
    extent = np.subtract(box[1], box[0])
    dense_voxels = int(np.prod(np.ceil(extent / cvs) + 1))
    dev = {k: torch.from_numpy(v).cuda() for k, v in dict(d=d, K=K, R=R, t=t, img=img).items()}
    vol = sequence.SparseTsdfVolume(cvs, box[0], color=False)
    for s in range(0, n, chunk):
        sl = slice(s, s + chunk)
        ms, = call_times(lambda: vol.integrate(dev["d"][sl], dev["K"], dev["R"][sl], dev["t"][sl]), 1, warmup=0)
        m = int(vol.blocks.shape[0])
        rows.add({"bench": "corridor_integrate", "frames": [s, s + chunk], "voxel_size": cvs, "box": box, "dense_voxels_of_box": dense_voxels,
                  "ms": ms, "ms_per_frame": ms / chunk, "blocks": m, "voxels": 512 * m, "state_bytes": vol.nbytes,
                  "skipped_pixels": vol.last_skipped_pixels, "pixels": chunk * d.shape[1] * d.shape[2]})
    tm = summary(call_times(vol.mesh, max(3, args.reps // 3), warmup=1))
    rows.add({"bench": "corridor_mesh", "frames": n, "voxel_size": cvs, "blocks": int(vol.blocks.shape[0]), "ms": tm["ms"],
              "ms_min": tm["ms_min"], "ms_max": tm["ms_max"], "triangles": int(vol.mesh()[2].shape[0]), "state_bytes": vol.nbytes})
    rows.save()


if __name__ == "__main__":
    main()
