"""Cost of the input preparation of examples/example.py:15-42 for one batch of image pairs: on the device (resize_u8_kernel:
both images of every pair to 256x192, then the second to 64x48, as DemonPipeline.forward_images stages them) against
single-threaded Pillow on the host doing the same resizes.  Prints one JSON line per source size and filter, with the card
name and power limit.

    python tools/bench_prepare.py [--pairs 64] [--reps 50] [--out FILE]
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

SIZES = [(640, 480), (1920, 1080)]
FILTERS = ["nearest", "bilinear", "bicubic"]


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in out.split(","))
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception:
        return {"gpu": torch.cuda.get_device_name(), "power_limit": None, "max_sm_clock": None}


def device_ms(pairs, reps, f):
    """CUDA-event milliseconds of one batch's resizes, averaged over `reps` batches after a warm-up"""
    run = lambda: images.resize(images.resize(pairs.reshape(-1, *pairs.shape[2:]), (256, 192), f).view(pairs.shape[0], 2, 192, 256, 3)[:, 1],
                                (64, 48), f)
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


def host_ms(pairs_np, f):
    """wall-clock milliseconds of Pillow doing the same resizes for the batch, one thread"""
    from PIL import Image
    code = images.resample_code(f)
    pil = [[Image.fromarray(p[i]) for i in range(2)] for p in pairs_np]
    t0 = time.perf_counter()
    for a, b in pil:
        a.resize((256, 192), code)
        b.resize((256, 192), code).resize((64, 48), code)
    return (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=64)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_prepare needs a CUDA device"
    try:
        import PIL
        pil_version = PIL.__version__
    except ImportError:
        pil_version = None
    info = gpu_info()
    lines = []
    for (w, h) in SIZES:
        pairs_np = np.random.default_rng(0).integers(0, 256, (a.pairs, 2, h, w, 3), dtype=np.uint8)
        pairs = torch.from_numpy(pairs_np).cuda()
        for f in FILTERS:
            rec = {"source": "%dx%d" % (w, h), "filter": f, "pairs": a.pairs, "device_ms_per_batch": round(device_ms(pairs, a.reps, f), 4),
                   "host_pillow_ms_per_batch": round(host_ms(pairs_np, f), 1) if pil_version else None,
                   "pillow": pil_version, **info}
            if rec["host_pillow_ms_per_batch"] is not None:
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
