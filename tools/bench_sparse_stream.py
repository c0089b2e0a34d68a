"""Times a SparseTsdfVolume that streams its blocks to pinned host memory (max_device_blocks; README, DESIGN.md §3.9)
against one that keeps them all on the device, and appends JSON lines to --out with the device name and power limit in
every row.

The scene is a walk of 512 frames of 192x256, 1.3 times round a ring corridor (tests/sparse_stream_oracle.py: ring_walk,
an 8 x 8 m loop 1.5 m wide and 2.5 m high, whose pillar hides the far side), at 5 mm voxels without colour (4 KB per
block), integrated 64 frames per call.  Budgets: none, and about 1/4 and 1/16 of the unbudgeted volume's final blocks.
Rows per call: ms per frame (CUDA events around the call, which synchronises), device and host blocks, blocks moved in
and out, and torch.cuda.max_memory_allocated.  A second, profiled run of each budget gives the evict and restore kernels'
time and their achieved GB/s (bytes of the moved blocks over kernel time); its final state must equal the timed run's.
Then: ray casts at every 4th pose with far given (ms), the mesh (chunked with host blocks) against the unbudgeted mesh,
and whether the final states (device and host blocks, keyed by coordinates) equal the unbudgeted volume's.

    python tools/bench_sparse_stream.py [--out profiles/h100_sparse_stream.jsonl]
"""
import argparse
import os

import numpy as np
import torch

from benchkit import ROOT, Rows, call_times, device_events
from demon_b200 import sequence
import sparse_stream_oracle as ss
import sequence_oracle as so

VS, CHUNK, N = 0.005, 64, 512
BLOCK_BYTES = 2 * 512 * 4


def frames():
    K = so.K_pixels(so.NETWORK_INTRINSICS, 256, 192)
    d, _, R, t, _ = ss.ring_walk(N, loops=1.3, h=192, w=256, L=4.0, W=1.5, H=2.5, f=float(K[0, 0]))
    d = np.where(np.isfinite(d), d, np.nan).astype(np.float32)
    dev = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in dict(d=d, K=K.astype(np.float32), R=R, t=t).items()}
    return dev


def state(vol):
    """All blocks (device and host) sorted by key: coordinates, tsdf and weight on the device."""
    h = vol.host
    b = torch.cat([vol.blocks, h["blocks"].cuda()])
    ts = torch.cat([vol.tsdf, h["tsdf"].cuda()])
    W = torch.cat([vol.weight, h["weight"].cuda()])
    order = torch.argsort(sequence._packed_keys(b))
    return b[order], ts[order], W[order]


def walk(dev, budget, rows=None, profile=False):
    vol = sequence.SparseTsdfVolume(VS, (0.0011, -0.0007, 0.0003), color=False, max_device_blocks=budget)
    torch.cuda.reset_peak_memory_stats()
    moved_us, moved_blocks = 0.0, 0
    for s in range(0, N, CHUNK):
        sl = slice(s, s + CHUNK)
        fn = lambda: vol.integrate(dev["d"][sl], dev["K"], dev["R"][sl], dev["t"][sl])   # noqa: E731
        if profile:
            _, ev = device_events(fn)
            moved_us += sum(e.time_range.elapsed_us() for e in ev if "sparse_evict_kernel" in e.name or "sparse_restore_kernel" in e.name)
            moved_blocks += vol.last_blocks_in + vol.last_blocks_out
            continue
        ms, = call_times(fn, 1, warmup=0)
        rows.add({"bench": "stream_integrate", "budget": budget, "frames": [s, s + CHUNK], "voxel_size": VS, "ms": ms, "ms_per_frame": ms / CHUNK,
                  "device_blocks": int(vol.blocks.shape[0]), "host_blocks": int(vol.host["blocks"].shape[0]), "blocks_in": vol.last_blocks_in,
                  "blocks_out": vol.last_blocks_out, "peak_device_blocks": vol.peak_device_blocks, "device_bytes": vol.nbytes,
                  "host_bytes": vol.host_nbytes, "max_memory_allocated": torch.cuda.max_memory_allocated()})
    return vol, moved_us, moved_blocks


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_sparse_stream.jsonl"))
    args = ap.parse_args()
    rows = Rows(args.out)
    dev = frames()
    ref, _, _ = walk(dev, None, rows)
    total = int(ref.blocks.shape[0])
    ref_state = state(ref)
    mesh_ref = call_times(ref.mesh, 1, warmup=1)[0]
    tri_ref = int(ref.mesh()[2].shape[0])
    sl = slice(0, N, 4)
    far = torch.full((len(range(0, N, 4)),), 8.0, device="cuda")
    ray_ref = call_times(lambda: ref.raycast(dev["K"], dev["R"][sl], dev["t"][sl], far=far), 1, warmup=1)[0]
    rows.add({"bench": "stream_final", "budget": None, "blocks": total, "mesh_ms": mesh_ref, "triangles": tri_ref, "raycast_ms": ray_ref,
              "raycast_frames": far.numel()})
    img_ref = ref.raycast(dev["K"], dev["R"][sl], dev["t"][sl], far=far)["depth"]
    del ref
    torch.cuda.empty_cache()
    for budget in (total // 4, total // 16):
        vol, _, _ = walk(dev, budget, rows)
        fin = state(vol)
        equal = all(torch.equal(a, b) for a, b in zip(fin, ref_state))
        again, us, moved = walk(dev, budget, profile=True)
        same = all(torch.equal(a, b) for a, b in zip(state(again), fin))
        del again
        mesh_ms = call_times(vol.mesh, 1, warmup=1)[0]
        tri = int(vol.mesh()[2].shape[0])
        ray_ms = call_times(lambda: vol.raycast(dev["K"], dev["R"][sl], dev["t"][sl], far=far), 1, warmup=1)[0]
        img = vol.raycast(dev["K"], dev["R"][sl], dev["t"][sl], far=far)["depth"]
        rows.add({"bench": "stream_final", "budget": budget, "blocks": int(fin[0].shape[0]), "equal_to_unbudgeted": bool(equal),
                  "profiled_run_equal": bool(same), "transfer_kernel_ms": us / 1000.0, "blocks_moved": moved,
                  "transfer_GBps": moved * BLOCK_BYTES / (us * 1e3) if us else None, "mesh_ms": mesh_ms, "mesh_ms_unbudgeted": mesh_ref,
                  "triangles": tri, "triangles_unbudgeted": tri_ref, "raycast_ms": ray_ms, "raycast_ms_unbudgeted": ray_ref,
                  "raycast_equal": bool(torch.equal(img.nan_to_num(-1), img_ref.nan_to_num(-1)))})
        del vol
        torch.cuda.empty_cache()
    rows.save()


if __name__ == "__main__":
    main()
