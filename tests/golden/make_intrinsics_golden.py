"""Writes tests/golden/intrinsics_digests.json: shape, status and SHA-256 of what Pillow gives for the image part of the
reference's adjust_intrinsics (oracle/intrinsics.py), the fixture of demon_b200.images.adjust_intrinsics (csrc/images.cu).

The inputs are regenerated from seeds, so no image is stored.  `digests(adjust, put, get)` runs every case through any
implementation: Pillow here (python tests/golden/make_intrinsics_golden.py), the device in tests/test_gpu_intrinsics.py.
`adjust(x, K, K_new, width_new, height_new)` maps [N,h,w,3] images with K [N,4] (fx, fy, cx, cy in pixels) and K_new [4] to
([N,height_new,width_new,3], status [N]).  Cases (K_new is DeMoN's 256x192 unless a case says otherwise):
  camera   640x480 (fx = fy = 525), 1920x1080 (fx ~ 1400) and 4032x3024 (fx ~ 3000) photos, a 640x480 view cut out of a larger
           image (read in place), and four 640x480 images with a different K each, one of them leaving the resized image
  scan     full-image LANCZOS resizes, one digest over all targets: a 2500-pixel row to every width 1..2048, 30x3000 and
           7x700 images (no more than 100 times taller than wide) to every height 1..2048 with scale_x = 1 (the latter also
           upscales).  K_new puts the window on the whole resized image: cx_new = cx * scale_x = 0 and width_new = rw, with
           scale = (t + 0.5) / side, so that int(side * scale) = t
  axes     LANCZOS down in x and up in y; BILINEAR up in x and down in y; scale_x exactly 1 (LANCZOS, the x pass skipped);
           rw == w with scale_x > 1 (BILINEAR, the x pass skipped)
  leave    windows leaving the left, right, top and bottom of the resized image, and one entirely outside it
  round    crop offsets exactly k + 0.5 (round() is half to even), and w * scale_x just below an integer (int() truncates)
"""
import hashlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
PATH = os.path.join(HERE, "intrinsics_digests.json")
NET = (0.89115971 * 256, 1.18821287 * 192, 0.5 * 256, 0.5 * 192)   # demon_b200.images.demon_intrinsics() as (fx, fy, cx, cy)
CAMERAS = {(640, 480): (525.0, 525.0, 319.5, 239.5), (1920, 1080): (1400.0, 1400.0, 959.5, 539.5),
           (4032, 3024): (3000.0, 3000.0, 2015.5, 1511.5)}
SCAN_MAX = 2048
SCANS = [("width", 2500, 1), ("height", 3000, 30), ("height", 700, 7)]   # axis, its source size, the other side
CROP = (800, 600, 37, 53, 640, 480)   # source width, height; crop x0, y0, width, height
BATCH_K = [(525.0, 525.0, 319.5, 239.5), (500.0, 510.0, 330.0, 230.0), (600.0, 600.0, 300.0, 250.0), (400.0, 450.0, 100.0, 240.0)]


def image(seed, h, w, n=None):
    shape = (h, w, 3) if n is None else (n, h, w, 3)
    return np.random.default_rng(seed).integers(0, 256, shape, dtype=np.uint8)


def small_cases():
    """(name, K, K_new, width_new, height_new) on a 320x240 image"""
    below = lambda v: float(np.nextafter(v, 0.0))
    return [
        ("axes/lanczos_x_down_y_up", (300.0, 100.0, 160.0, 120.0), NET, 256, 192),
        ("axes/bilinear_x_up_y_down", (150.0, 400.0, 160.0, 120.0), NET, 256, 192),
        ("axes/scale_x_1", (NET[0], 150.0, 128.0, 120.0), NET, 256, 192),
        ("axes/rw_equals_w", (NET[0] / 1.001, 180.0, 160.0, 120.0), NET, 256, 192),
        ("leave/none", (260.0, 260.0, 160.0, 120.0), NET, 256, 192),
        ("leave/left", (260.0, 260.0, 130.0, 120.0), NET, 256, 192),
        ("leave/right", (260.0, 260.0, 190.0, 120.0), NET, 256, 192),
        ("leave/top", (260.0, 260.0, 160.0, 100.0), NET, 256, 192),
        ("leave/bottom", (260.0, 260.0, 160.0, 140.0), NET, 256, 192),
        ("leave/outside", (260.0, 260.0, 600.0, 120.0), NET, 256, 192),
        ("round/tie_2.5_-2.5", (200.0, 200.0, 105.0, 95.0), (100.0, 100.0, 50.0, 50.0), 64, 64),
        ("round/tie_3.5_-3.5", (200.0, 200.0, 107.0, 93.0), (100.0, 100.0, 50.0, 50.0), 64, 64),
        ("round/truncation", (1.0, 1.0, 0.0, 0.0), (below(0.9375), below(0.75), 0.0, 0.0), 299, 179),
    ]


def cases():
    """(name, source seed and shape [N,h,w], view (x0, y0, w, h) or None, calls [(K [N,4], K_new, width_new, height_new)])"""
    out = []
    for i, ((w, h), k) in enumerate(sorted(CAMERAS.items())):
        out.append(("camera/%dx%d" % (w, h), (100 + i, 1, h, w), None, [([k], NET, 256, 192)]))
    sw, sh, x0, y0, cw, ch = CROP
    out.append(("camera/crop/%dx%d+%d+%d" % (cw, ch, x0, y0), (110, 1, sh, sw), (x0, y0, cw, ch), [([CAMERAS[(640, 480)]], NET, 256, 192)]))
    out.append(("camera/batch/4x640x480", (111, 4, 480, 640), None, [(BATCH_K, NET, 256, 192)]))
    for i, (axis, n, m) in enumerate(SCANS):
        calls = []
        for t in range(1, SCAN_MAX + 1):
            s = (t + 0.5) / n
            calls.append(([(1.0, 1.0, 0.0, 0.0)], (s, 1.0, 0.0, 0.0) if axis == "width" else (1.0, s, 0.0, 0.0),
                          t if axis == "width" else m, t if axis == "height" else m))
        out.append(("scan/%s/%d" % (axis, n), (120 + i, 1, m, n) if axis == "width" else (120 + i, 1, n, m), None, calls))
    for i, (name, k, knew, ow, oh) in enumerate(small_cases()):
        out.append((name, (130 + i, 1, 240, 320), None, [([k], knew, ow, oh)]))
    return out


def _entry(arrays, status):
    h = hashlib.sha256()
    shapes = []
    for a in arrays:
        a = np.ascontiguousarray(a)
        shapes.append(list(a.shape))
        h.update(a.tobytes())
    return {"shape": shapes[0] if len(shapes) == 1 else [len(shapes)] + shapes[-1], "sha256": h.hexdigest(),
            "status": "".join(str(int(v)) for v in status)}


def digests(adjust, put=lambda a: a, get=np.asarray):
    out = {}
    for name, (seed, n, h, w), view, calls in cases():
        src = image(seed, h, w, n)
        x = put(src)
        if view is not None:
            vx, vy, vw, vh = view
            x = x[:, vy:vy + vh, vx:vx + vw]
        arrays, status = [], []
        for K, knew, ow, oh in calls:
            a, s = adjust(x, np.asarray(K, dtype=np.float64), np.asarray(knew, dtype=np.float64), ow, oh)
            arrays.append(get(a))
            status.extend(np.asarray(get(s)).reshape(-1).tolist())
        out[name] = _entry(arrays, status)
    return out


def lanczos_pairs():
    """Every (input size, output size) of an axis that the cases resize with LANCZOS (the axes the weight check covers)."""
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
    from oracle.intrinsics import window
    pairs = set()
    for _, (_, n, h, w), view, calls in cases():
        if view is not None:
            w, h = view[2], view[3]
        for K, knew, _, _ in calls:
            for k in K:
                rw, rh, _, _, bilinear = window(k, knew, w, h)
                if not bilinear:
                    pairs.update(p for p in ((w, rw), (h, rh)) if p[0] != p[1])
    return sorted(pairs)


def pillow_adjust(x, K, K_new, ow, oh):
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
    from oracle.intrinsics import adjust_image
    res = [adjust_image(im, k, K_new, ow, oh) for im, k in zip(x, K)]
    return np.stack([r[0] for r in res]), np.array([r[1] for r in res], dtype=np.uint8)


def pillow_digests():
    return digests(pillow_adjust)


def main():
    import PIL
    d = pillow_digests()
    d["_pillow"] = PIL.__version__
    with open(PATH, "w") as fh:
        json.dump(d, fh, indent=1, sort_keys=True)
        fh.write("\n")
    print("wrote %d digests to %s (Pillow %s)" % (len(d) - 1, PATH, PIL.__version__))


if __name__ == "__main__":
    main()
