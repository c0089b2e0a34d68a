"""Cost of adapting one batch of image pairs to DeMoN's intrinsics (the image part of the reference's adjust_intrinsics,
dataset_tools/view_tools.py:97-172): on the device (images.adjust_intrinsics, the LANCZOS or BILINEAR resize and the crop
in one kernel) against single-threaded Pillow on the host doing the same resize and crop with fill (oracle/intrinsics.py).
Prints one JSON line per camera, with the card name and power limit read in the same call.

    python tools/bench_intrinsics.py [--pairs 64] [--reps 50] [--out FILE]
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
from demon_b200 import images
from oracle import intrinsics as oi

CAMERAS = {(640, 480): (525.0, 525.0, 319.5, 239.5), (1920, 1080): (1400.0, 1400.0, 959.5, 539.5)}


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in out.split(","))
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception:
        return {"gpu": torch.cuda.get_device_name(), "power_limit": None, "max_sm_clock": None}


def device_ms(frames, K, reps):
    """CUDA-event milliseconds of one batch's adjust_intrinsics, averaged over `reps` batches after a warm-up"""
    run = lambda: images.adjust_intrinsics(frames, K)
    for _ in range(3):
        run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        run()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def host_ms(frames_np, k):
    """wall-clock milliseconds of Pillow doing the same resize and crop for the batch, one thread"""
    knew = images.intrinsics4(images.demon_intrinsics(), (), "K_new")
    t0 = time.perf_counter()
    for im in frames_np:
        oi.adjust_image(im, k, knew, 256, 192)
    return (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=64)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_intrinsics needs a CUDA device"
    import PIL
    info = gpu_info()
    lines = []
    for (w, h), k in CAMERAS.items():
        frames_np = np.random.default_rng(0).integers(0, 256, (2 * a.pairs, h, w, 3), dtype=np.uint8)
        frames = torch.from_numpy(frames_np).cuda()
        K = torch.tensor([k] * (2 * a.pairs), dtype=torch.float64, device="cuda")
        rw, rh, _, _, bilinear = oi.window(k, images.intrinsics4(images.demon_intrinsics(), (), "K_new"), w, h)
        rec = {"source": "%dx%d" % (w, h), "K": list(k), "resized": "%dx%d" % (rw, rh), "filter": "bilinear" if bilinear else "lanczos",
               "pairs": a.pairs, "images": 2 * a.pairs, "device_ms_per_batch": round(device_ms(frames, K, a.reps), 4),
               "host_pillow_ms_per_batch": round(host_ms(frames_np, k), 1), "pillow": PIL.__version__, **info}
        rec["host_over_device"] = round(rec["host_pillow_ms_per_batch"] / rec["device_ms_per_batch"], 1)
        print(json.dumps(rec), flush=True)
        lines.append(rec)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            for r in lines:
                fh.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
