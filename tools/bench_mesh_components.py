"""Times the connected components of an indexed mesh (mesh.components) and the removal of its small ones
(mesh.remove_small_components) on the device, checks both against tests/mesh_components_oracle.py, and times that
oracle (scipy's connected_components and numpy, on one host core) on the same mesh.  Appends JSON lines to --out with
the device name and power limit in every row.

Meshes:
1. orbit: tools/bench_sequence.py's 64-frame orbit fused into the dense 256^3 volume, with 1 % of each depth map's 2x2
   pixel cells at a random depth, so the indexed mesh has floaters.
2. corridor: tools/bench_sparse_tsdf.py's 5 mm corridor walk (256 frames, 64 per call, no colour): its indexed mesh.
3. strip: a triangle strip over 2^24 vertices with indices descending along it, where every union hooks a new smaller
   root (the deepest trees).

Each row: V, F, the component count C, the kept vertices and faces at --min-triangles, the median of --reps calls of
each function timed with CUDA events (each reads its counts back, so it synchronises), whether both equal the oracle bit
for bit, and the oracle's seconds for the components alone and with the filter.

    python tools/bench_mesh_components.py [--reps 10] [--min-triangles 200] [--out profiles/h100_mesh_components.jsonl]
"""
import argparse
import os
import time

import numpy as np
import torch

from benchkit import ROOT, Rows, call_times, summary
from bench_sequence import orbit_frames
from bench_sparse_tsdf import corridor_frames
import mesh_components_oracle as mco
from demon_b200 import mesh, sequence

KEYS = ("vertices", "normals", "colors", "faces")


def host(x):
    return None if x is None else x.cpu().numpy()


def same(a, b):
    if a is None or b is None:
        return a is None and b is None
    return a.shape == b.shape and a.tobytes() == b.tobytes()


def measure(rows, reps, m, min_triangles, **info):
    faces, nv = m["faces"], int(m["vertices"].shape[0])
    comp = summary(call_times(lambda: mesh.components(faces, nv), reps, warmup=2))
    rem = summary(call_times(lambda: mesh.remove_small_components(m, min_triangles=min_triangles), reps, warmup=2))
    got_c = {k: host(v) for k, v in mesh.components(faces, nv).items()}
    got_r = {k: host(v) for k, v in mesh.remove_small_components(m, min_triangles=min_triangles).items()}
    hm = {k: host(m.get(k)) for k in KEYS}
    t0 = time.perf_counter()
    want_c = mco.components(hm["faces"], nv)
    t1 = time.perf_counter()
    want_r = mco.remove_small_components(hm, min_triangles=min_triangles)
    t2 = time.perf_counter()
    equal = all(same(got_c[k], want_c[k]) for k in got_c) and all(same(got_r[k], want_r[k]) for k in KEYS)
    rows.add(dict(info, V=nv, F=int(faces.shape[0]), C=int(want_c["triangles"].size), min_triangles=min_triangles,
                  kept_V=int(want_r["vertices"].shape[0]), kept_F=int(want_r["faces"].shape[0]),
                  components_ms=comp["ms"], components_ms_min=comp["ms_min"], remove_ms=rem["ms"], remove_ms_min=rem["ms_min"],
                  equal_to_oracle=equal, oracle_components_s=t1 - t0, oracle_remove_s=t2 - t0, reps=reps))
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--min-triangles", type=int, default=200)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_mesh_components.jsonl"))
    args = ap.parse_args()
    torch.set_num_threads(1)
    rows = Rows(args.out)

    dims, origin, vs = (256, 256, 256), (-1.25, -1.25, -1.25), 2.5 / 255
    d, K, R, t, img = orbit_frames(64)
    rng = np.random.RandomState(0)
    cell = np.ones((1, 2, 2))
    n, h, w = d.shape
    out = np.kron(rng.rand(n, h // 2, w // 2) < 0.01, cell).astype(bool)
    d[out] = np.kron(rng.uniform(0.3, 4.0, (n, h // 2, w // 2)), cell).astype(np.float32)[out]
    d, K, R, t, img = (torch.from_numpy(x).cuda() for x in (d, K, R, t, img))
    dense = sequence.TsdfVolume(dims, origin, vs).integrate(d, K, R, t, img)
    measure(rows, args.reps, dense.indexed_mesh(), args.min_triangles, bench="orbit_outliers", volume="dense", dims=dims,
            voxel_size=vs, outlier_cells=0.01)
    del dense
    torch.cuda.empty_cache()

    n, chunk, cvs = 256, 64, 0.005
    d, K, R, t, _, box = corridor_frames(n)
    d, K, R, t = (torch.from_numpy(x).cuda() for x in (d, K, R, t))
    vol = sequence.SparseTsdfVolume(cvs, box[0], color=False)
    for s in range(0, n, chunk):
        vol.integrate(d[s:s + chunk], K, R[s:s + chunk], t[s:s + chunk])
    m = vol.indexed_mesh()
    del vol
    torch.cuda.empty_cache()
    measure(rows, max(3, args.reps // 3), m, args.min_triangles, bench="corridor", volume="sparse", voxel_size=cvs)
    del m
    torch.cuda.empty_cache()

    nv = 1 << 24
    f = torch.from_numpy(mco.strip(nv, "descending")).cuda()
    v = torch.zeros((nv, 3), dtype=torch.float32, device="cuda")
    measure(rows, max(3, args.reps // 3), {"vertices": v, "faces": f}, args.min_triangles, bench="strip_descending")
    rows.save()


if __name__ == "__main__":
    main()
