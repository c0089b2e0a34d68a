"""Times the video reconstruction (README, DESIGN.md §3.9): TSDF integration of 64 and 256 frames of 192x256 depth into
256^3 voxels with and without colour, marching cubes of the result, chain_pairs at P = 255, reconstruct end to end from
640x480 uint8 frames with synthetic v1 weights at batch 64, and a single-core numpy run of the oracle's integrate and
marching cubes (tests/sequence_oracle.py) on the same input.  Device times are CUDA events around the call, after a warm-up
call, median of --reps.  The integrate lines give voxel-frame updates per second and the bytes the kernel must move (the
volume state read and written once, each frame's depth and image read once) over its time.  Appends JSON lines to --out.

    python tools/bench_sequence.py [--reps 10] [--out profiles/h100_sequence.jsonl]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from demon_b200 import sequence                                  # noqa: E402
from demon_b200 import weights as W1                             # noqa: E402
from demon_b200.networks_original import DemonPipeline, Session  # noqa: E402
import sequence_oracle as so                                     # noqa: E402

HBM_PEAK = 3.35e12   # H100 SXM data sheet, bytes/s


def device_info():
    """The card's name and power limit, read in the same call as the timings."""
    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        info["power_limit"], info["max_sm_clock"] = [s.strip() for s in q.split(",")]
    except Exception as e:
        info["power_limit"] = "unknown (%s)" % type(e).__name__
    return info


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms)), float(np.min(ms)), float(np.max(ms))


def orbit_frames(n, h=192, w=256):
    """n depth maps of a room with a sphere, from cameras on a circle around the volume [-1,1]^3 looking at its centre, and
    random images: float32 depth [n,h,w], K [3,3], R [n,3,3], t [n,3], uint8 [n,h,w,3]."""
    K = so.K_pixels(so.NETWORK_INTRINSICS, w, h)
    ang = np.linspace(0, 2 * np.pi, n, endpoint=False)
    Rs, ts, ds = [], [], []
    for a in ang:
        R, t = so.look_at((2.5 * np.cos(a), 2.5 * np.sin(a), 0.6), (0, 0, 0))
        Rs.append(R)
        ts.append(t)
        ds.append(so.render_depth(R, t, K, h, w, sphere=((0.1, 0, 0), 0.5), box=((-1, -1, -1), (1, 1, 1.2))))
    img = np.random.RandomState(0).randint(0, 256, (n, h, w, 3)).astype(np.uint8)
    return np.array(ds, np.float32), K.astype(np.float32), np.array(Rs, np.float32), np.array(ts, np.float32), img


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_sequence.jsonl"))
    args = ap.parse_args()
    info = device_info()
    rows = []

    def emit(row):
        row.update(info)
        rows.append(row)
        print(json.dumps(row), flush=True)

    dims, origin, vs = (256, 256, 256), (-1.25, -1.25, -1.25), 2.5 / 255
    nvox = int(np.prod(dims))
    d, K, R, t, img = orbit_frames(256)
    dev = {k: torch.from_numpy(v).cuda() for k, v in dict(d=d, R=R, t=t, img=img).items()}
    Kd = torch.from_numpy(K).cuda()
    vol = None
    for n in (64, 256):
        for color in (False, True):
            vol = sequence.TsdfVolume(dims, origin, vs, color=color)
            args_n = (dev["d"][:n], Kd, dev["R"][:n], dev["t"][:n], dev["img"][:n] if color else None)
            ms, lo, hi = timed(lambda: vol.integrate(*args_n), args.reps)
            state = nvox * (20 if color else 8)
            frames = n * 192 * 256 * (7 if color else 4)
            moved = 2 * state + frames
            emit({"bench": "integrate", "frames": n, "color": color, "dims": dims, "ms": ms, "ms_min": lo, "ms_max": hi,
                  "voxel_frame_updates_per_s": nvox * n / (ms * 1e-3), "bytes": moved, "bytes_per_s": moved / (ms * 1e-3),
                  "bytes_share_of_hbm_peak": moved / (ms * 1e-3) / HBM_PEAK})
    # the last volume holds 256 frames with colour, integrated 1 + reps times: mesh a fresh single integration
    vol = sequence.TsdfVolume(dims, origin, vs)
    vol.integrate(dev["d"], Kd, dev["R"], dev["t"], dev["img"])
    ms, lo, hi = timed(vol.mesh, args.reps)
    v, c, f = vol.mesh()
    emit({"bench": "mesh", "frames": 256, "dims": dims, "triangles": int(f.shape[0]), "ms": ms, "ms_min": lo, "ms_max": hi})

    sc = so.orbit_pairs(frames=256, seed=0)
    inv, rot, tr = (torch.from_numpy(sc[k]).cuda() for k in ("inverse_depth", "rotation", "translation"))
    ms, lo, hi = timed(lambda: sequence.chain_pairs(inv, rot, tr), args.reps)
    ch = sequence.chain_pairs(inv, rot, tr)
    emit({"bench": "chain_pairs", "pairs": 255, "ms": ms, "ms_min": lo, "ms_max": hi,
          "max_scale_rel_err": float(np.abs(ch["scales"] / sc["scales"] - 1).max())})

    s = Session(precision="3xtf32")
    s.load_weights(W1.synthetic_weights(0))
    pipe = DemonPipeline(s, batch_size=64, iterations=3)
    T = 129
    rng = np.random.RandomState(1)
    base = rng.randint(0, 256, (60, (640 + 16 * T) // 8, 3)).astype(np.uint8)
    big = np.kron(base, np.ones((8, 8, 1), np.uint8))
    frames = torch.from_numpy(np.stack([big[:, 16 * k:16 * k + 640] for k in range(T)])).cuda()
    Kc = np.array([[520.0, 0, 318.0], [0, 515.0, 243.0], [0, 0, 1]])
    try:
        ms, lo, hi = timed(lambda: sequence.reconstruct(pipe, frames, Kc, min_ratios=1), max(3, args.reps // 3))
        res = sequence.reconstruct(pipe, frames, Kc, min_ratios=1)
        emit({"bench": "reconstruct", "frames": T, "pairs": T - 1, "batch": 64, "iterations": 3, "weights": "synthetic v1",
              "ms": ms, "ms_min": lo, "ms_max": hi, "frames_per_s": T / (ms * 1e-3), "dims": res["volume"].dims,
              "triangles": int(res["faces"].shape[0])})
    except ValueError as e:
        emit({"bench": "reconstruct", "frames": T, "error": str(e)})

    # the oracle on one core: 8 frames into the same volume, then marching cubes of the GPU's 256-frame volume
    nz, ny, nx = dims[::-1]
    ts, W, col = np.zeros((nz, ny, nx), np.float32), np.zeros((nz, ny, nx), np.float32), np.zeros((nz, ny, nx, 3), np.float32)
    t0 = time.perf_counter()
    so.integrate(ts, W, col, vol.origin, vol.voxel_size, vol.trunc, d[:8], np.broadcast_to(K, (8, 3, 3)), R[:8], t[:8], img[:8])
    sec = time.perf_counter() - t0
    emit({"bench": "oracle_integrate_numpy", "frames": 8, "color": True, "dims": dims, "s": sec,
          "voxel_frame_updates_per_s": nvox * 8 / sec})
    tsdf, wt, cc = vol.tsdf.cpu().numpy(), vol.weight.cpu().numpy(), vol.color.cpu().numpy()
    t0 = time.perf_counter()
    vr, cr, fr = so.marching_cubes(tsdf, wt, cc, vol.origin, vol.voxel_size)
    sec = time.perf_counter() - t0
    emit({"bench": "oracle_mesh_numpy", "frames": 256, "dims": dims, "s": sec, "triangles": int(fr.shape[0]),
          "equals_gpu": bool(np.array_equal(vr, v.cpu().numpy()) and np.array_equal(cr, c.cpu().numpy()))})

    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "a") as fh:
        for r in rows:
            fh.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
