"""HBM-roofline check of the standalone geometry ops at the BASELINE.json configs[4] size ([8,3,768,1024]) and at the
hot-path size ([64,*,48,64]): CUDA-event time per launch, algorithmic bytes / time, fraction of the measured copy peak."""
import json
import os

import torch

from benchkit import ROOT, span_ms
from demon_b200 import lmbspecialops as ops


def main():
    peak = 6590.9
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.isfile(p):
        peak = json.load(open(p))["hbm_gbs"]
    rows = []
    for tag, (n, h, w) in (("1024x768 x8", (8, 768, 1024)), ("64x48 x64", (64, 48, 64)), ("256x192 x64", (64, 192, 256))):
        img = torch.rand(n, 3, h, w, device="cuda") - 0.5
        # a smooth displacement field (what flow networks produce): low-frequency waves of +-2.5 % of the image size;
        # `rough` is the adversarial case, an independent random displacement per pixel (every gather misses its neighbours)
        yy, xx = torch.meshgrid(torch.linspace(0, 6.28, h, device="cuda"), torch.linspace(0, 6.28, w, device="cuda"), indexing="ij")
        disp = (0.025 * torch.stack([torch.sin(xx + 0.5 * yy), torch.cos(yy - 0.3 * xx)])[None].repeat(n, 1, 1, 1)).contiguous()
        rough = (torch.rand(n, 2, h, w, device="cuda") - 0.5) * 0.05
        depth = torch.rand(n, 1, h, w, device="cuda") + 0.3
        K = torch.tensor([[0.89115971, 1.18821287, 0.5, 0.5]], device="cuda").repeat(n, 1)
        r = (torch.rand(n, 3, device="cuda") - 0.5) * 0.1
        t = torch.tensor([[0.9, 0.1, -0.05]], device="cuda").repeat(n, 1)
        px = n * h * w
        cases = [
            ("warp2d (value, normalized)", lambda: ops.warp2d(img, disp, normalized=True, border_mode="value"), (3 + 2 + 3) * 4 * px),
            ("warp2d (random displacement per pixel)", lambda: ops.warp2d(img, rough, normalized=True, border_mode="value"), (3 + 2 + 3) * 4 * px),
            ("depth_to_flow", lambda: ops.depth_to_flow(depth, K, r, t, inverse_depth=True, normalize_flow=True), (1 + 2) * 4 * px),
            ("flow_to_depth", lambda: ops.flow_to_depth(disp, K, r, t, normalized_flow=True, inverse_depth=True, nowarning=True), (2 + 1) * 4 * px),
            ("median3x3_downsample", lambda: ops.median3x3_downsample(img), (3 + 0.75) * 4 * px),
            ("scale_invariant_gradient (5 deltas)", lambda: ops.scale_invariant_gradient(depth, [1, 2, 4, 8, 16], [1, .5, .25, .125, .0625]), (1 + 2) * 4 * px),
            ("leaky_relu", lambda: ops.leaky_relu(img), 2 * 3 * 4 * px),
        ]
        for name, fn, nbytes in cases:
            ms = span_ms(fn, 20)
            gbs = nbytes / (ms / 1e3) / 1e9
            rows.append((tag, name, ms, nbytes / 1e6, gbs, gbs / peak))
    print("| size | op | ms / launch (incl. output allocation) | algorithmic MB | GB/s | fraction of measured copy peak (%.0f GB/s) |" % peak)
    print("|---|---|---|---|---|---|")
    for tag, name, ms, mb, gbs, fr in rows:
        print("| %s | %s | %.4f | %.1f | %.0f | %.2f |" % (tag, name, ms, mb, gbs, fr))


if __name__ == "__main__":
    main()
