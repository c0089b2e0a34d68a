"""Times the triangle soup (mesh()) against the indexed mesh (indexed_mesh(), with and without normals) of the fused
volumes (README, DESIGN.md §3.9), and appends JSON lines to --out with the device name and power limit in every row.

Scenes:
1. orbit: tools/bench_sequence.py's orbit_frames, 64 frames of 192x256 fused into the dense 256^3 volume and into a
   sparse volume at the same voxel size and origin, with colour.
2. corridor: tools/bench_sparse_tsdf.py's 5 mm corridor walk, 256 frames fused 64 per call, without colour.
3. ring: tools/bench_sparse_stream.py's 512-frame ring walk at 5 mm without colour, fused with max_device_blocks at about
   1/4 and 1/16 of its blocks, so both meshes run over key-ordered chunks with host blocks.

Each row: V, T, V/T, the output bytes of each form (vertices 12 B, normals 12 B, colours 3 B per vertex, faces 12 B per
triangle) and the PLY bytes vis.write_ply would write, and the median of --reps calls timed with CUDA events (every call
reads its counts back, so it synchronises).  The indexed mesh of the budgeted ring is checked to equal the unbudgeted
volume's byte for byte.

    python tools/bench_mesh.py [--reps 10] [--out profiles/h100_mesh.jsonl]
"""
import argparse
import os

import torch

from benchkit import ROOT, Rows, call_times, summary
from bench_sequence import orbit_frames
from bench_sparse_stream import frames as ring_frames, VS as RING_VS, N as RING_N, CHUNK as RING_CHUNK
from bench_sparse_tsdf import corridor_frames
from demon_b200 import sequence


def ply_bytes(nv, nt, color, normals):
    """The size of vis.write_ply's file for nv vertices and nt triangles."""
    head = ["ply", "format binary_little_endian 1.0", "element vertex %d" % nv, "property float x", "property float y", "property float z"]
    head += ["property float nx", "property float ny", "property float nz"] if normals else []
    head += ["property uchar red", "property uchar green", "property uchar blue"] if color else []
    head += ["element face %d" % nt, "property list uchar int vertex_indices", "end_header"]
    return len("\n".join(head) + "\n") + nv * (12 + 12 * normals + 3 * color) + nt * 13


def measure(rows, reps, vol, color, **info):
    soup = summary(call_times(vol.mesh, reps, warmup=2))
    v, _, f = vol.mesh()
    t = int(f.shape[0])
    del v, f
    torch.cuda.empty_cache()
    out = {}
    for normals in (True, False):
        tm = summary(call_times(lambda: vol.indexed_mesh(normals=normals), reps, warmup=2))
        out[normals] = tm
    m = vol.indexed_mesh()
    nv = int(m["vertices"].shape[0])
    assert int(m["faces"].shape[0]) == t
    del m
    torch.cuda.empty_cache()
    rows.add(dict(info, V=nv, T=t, V_per_T=nv / t if t else None, soup_ms=soup["ms"], indexed_ms=out[True]["ms"],
                  indexed_no_normals_ms=out[False]["ms"], indexed_over_soup=out[True]["ms"] / soup["ms"],
                  soup_bytes=3 * t * (12 + 3 * color) + 12 * t, indexed_bytes=nv * (24 + 3 * color) + 12 * t,
                  indexed_no_normals_bytes=nv * (12 + 3 * color) + 12 * t, soup_ply_bytes=ply_bytes(3 * t, t, color, False),
                  indexed_ply_bytes=ply_bytes(nv, t, color, True), indexed_no_normals_ply_bytes=ply_bytes(nv, t, color, False),
                  reps=reps))


def same(a, b):
    for k in ("vertices", "normals", "colors", "faces"):
        x, y = a[k], b[k]
        if (x is None) != (y is None):
            return False
        if x is not None and not (x.shape == y.shape and torch.equal(x.view(torch.uint8) if x.dtype != torch.uint8 else x,
                                                                    y.view(torch.uint8) if y.dtype != torch.uint8 else y)):
            return False
    return True


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_mesh.jsonl"))
    args = ap.parse_args()
    rows = Rows(args.out)
    dims, origin, vs = (256, 256, 256), (-1.25, -1.25, -1.25), 2.5 / 255
    d, K, R, t, img = (torch.from_numpy(x).cuda() for x in orbit_frames(64))
    dense = sequence.TsdfVolume(dims, origin, vs).integrate(d, K, R, t, img)
    measure(rows, args.reps, dense, True, bench="orbit", volume="dense", dims=dims, voxel_size=vs)
    del dense
    torch.cuda.empty_cache()
    sp = sequence.SparseTsdfVolume(vs, origin).integrate(d, K, R, t, img)
    measure(rows, args.reps, sp, True, bench="orbit", volume="sparse", voxel_size=vs, blocks=int(sp.blocks.shape[0]))
    del sp
    torch.cuda.empty_cache()

    n, chunk, cvs = 256, 64, 0.005
    d, K, R, t, _, box = corridor_frames(n)
    d, K, R, t = (torch.from_numpy(x).cuda() for x in (d, K, R, t))
    vol = sequence.SparseTsdfVolume(cvs, box[0], color=False)
    for s in range(0, n, chunk):
        vol.integrate(d[s:s + chunk], K, R[s:s + chunk], t[s:s + chunk])
    measure(rows, max(3, args.reps // 3), vol, False, bench="corridor", volume="sparse", voxel_size=cvs, blocks=int(vol.blocks.shape[0]))
    del vol
    torch.cuda.empty_cache()

    dev = ring_frames()

    def ring(budget):
        v = sequence.SparseTsdfVolume(RING_VS, (0.0011, -0.0007, 0.0003), color=False, max_device_blocks=budget)
        for s in range(0, RING_N, RING_CHUNK):
            sl = slice(s, s + RING_CHUNK)
            v.integrate(dev["d"][sl], dev["K"], dev["R"][sl], dev["t"][sl])
        return v
    ref = ring(None)
    total = int(ref.blocks.shape[0])
    want = ref.indexed_mesh()
    measure(rows, 3, ref, False, bench="ring", volume="sparse", voxel_size=RING_VS, blocks=total, budget=None)
    del ref
    torch.cuda.empty_cache()
    for budget in (total // 4, total // 16):
        v = ring(budget)
        equal = same(v.indexed_mesh(), want)
        measure(rows, 3, v, False, bench="ring", volume="sparse", voxel_size=RING_VS, blocks=total, budget=budget,
                host_blocks=int(v.host["blocks"].shape[0]), equal_to_unbudgeted=equal)
        del v
        torch.cuda.empty_cache()
    rows.save()


if __name__ == "__main__":
    main()
