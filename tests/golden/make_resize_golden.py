"""Writes tests/golden/resize_digests.json: the shape and SHA-256 of what Pillow's `Image.resize` returns for RGB uint8 images,
the fixture of demon_b200.images.resize (csrc/images.cu).

The inputs are regenerated from seeds with numpy.random.default_rng, so no image is stored.  `digests(resize, put, get)`
runs every case through any implementation of the resize: Pillow here (python tests/golden/make_resize_golden.py), the
device in tests/test_gpu_images.py.  Cases, each for NEAREST, BILINEAR and BICUBIC:
  2d      images of the sizes in SIZES_2D resized to 256x192, and that result resized to 64x48 (examples/example.py:15-22)
  scan    one-row images of every width 1..2048 resized to 256 and to 64 wide (one digest over all widths), and the same for
          one-column images and heights: this pins the index arithmetic, e.g. NEAREST's running sum
  crop    a 640x480 view cut out of a larger image (examples/example.py:53-59 tells users to crop), resized to 256x192
  batch   four different 333x251 images in one call
  extreme the largest downscale of one side allowed (8192 -> 2), where one output sample has thousands of taps
  tall    images just below and just above 100 times taller than wide: above, Pillow runs the vertical pass first when the
          height shrinks, and the horizontal pass first when it grows (TALL_TARGETS)
"""
import hashlib
import json
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
PATH = os.path.join(HERE, "resize_digests.json")
FILTERS = {"nearest": 0, "bilinear": 2, "bicubic": 3}
SIZES_2D = [(640, 480), (1920, 1080), (4096, 3072), (333, 251), (257, 193), (128, 96), (1, 1), (256, 192), (300, 192), (256, 100)]
SCAN_MAX = 2048
CROP = (800, 600, 37, 53, 640, 480)   # source width, height; crop x0, y0, width, height
SIZES_TALL = [(3, 300), (3, 301), (20, 2000), (20, 2001), (64, 6400), (64, 6401)]
TALL_TARGETS = [((3, 301), (6, 302)), ((3, 301), (6, 300)), ((20, 2001), (40, 2100)), ((20, 2001), (40, 2000)),
                ((10, 1001), (5, 1002)), ((10, 1001), (5, 1000)), ((10, 5000), (5, 5001)), ((10, 5000), (5, 4999))]


def image(seed, h, w, n=None):
    shape = (h, w, 3) if n is None else (n, h, w, 3)
    return np.random.default_rng(seed).integers(0, 256, shape, dtype=np.uint8)


def _entry(arrays):
    """shape of the first array (all of them for a list) and the SHA-256 of their bytes in order"""
    h = hashlib.sha256()
    shapes = []
    for a in arrays:
        a = np.ascontiguousarray(a)
        shapes.append(list(a.shape))
        h.update(a.tobytes())
    return {"shape": shapes[0] if len(shapes) == 1 else [len(shapes)] + shapes[-1], "sha256": h.hexdigest()}


def digests(resize, put=lambda a: a, get=np.asarray):
    """resize(x, (width, height), filter) maps [N,h,w,3] images of the backend to [N,height,width,3]; put() makes a backend
    array of a numpy array and get() a numpy array of a backend array.  Returns {case: {"shape", "sha256"}}."""
    out = {}
    for i, (w, h) in enumerate(SIZES_2D):
        x = put(image(1000 + i, h, w)[None])
        for name, f in FILTERS.items():
            a = resize(x, (256, 192), f)
            b = resize(a, (64, 48), f)
            out["2d/%dx%d/%s/256x192" % (w, h, name)] = _entry([get(a)[0]])
            out["2d/%dx%d/%s/64x48" % (w, h, name)] = _entry([get(b)[0]])
    base = put(image(7, 1, SCAN_MAX)[None])                        # [1,1,2048,3]
    col = put(np.ascontiguousarray(get(base).transpose(0, 2, 1, 3)))  # [1,2048,1,3]
    for name, f in FILTERS.items():
        for target in (256, 64):
            out["scan/width/%s/%d" % (name, target)] = _entry(
                [get(resize(base[:, :, :w], (target, 1), f)) for w in range(1, SCAN_MAX + 1)])
            out["scan/height/%s/%d" % (name, target)] = _entry(
                [get(resize(col[:, :hh], (1, target), f)) for hh in range(1, SCAN_MAX + 1)])
    sw, sh, x0, y0, cw, ch = CROP
    big = put(image(11, sh, sw)[None])
    batch = put(image(12, 251, 333, n=4))
    wide, tall = put(image(13, 64, 8192)[None]), put(image(14, 8192, 64)[None])
    for name, f in FILTERS.items():
        out["crop/%dx%d+%d+%d/%s/256x192" % (cw, ch, x0, y0, name)] = _entry([get(resize(big[:, y0:y0 + ch, x0:x0 + cw], (256, 192), f))[0]])
        out["batch/4x333x251/%s/256x192" % name] = _entry([get(resize(batch, (256, 192), f))])
        out["extreme/8192x64/%s/2x2" % name] = _entry([get(resize(wide, (2, 2), f))[0]])
        out["extreme/64x8192/%s/2x2" % name] = _entry([get(resize(tall, (2, 2), f))[0]])
    for i, (w, h) in enumerate(SIZES_TALL):
        x = put(image(2000 + i, h, w)[None])
        for name, f in FILTERS.items():
            out["tall/%dx%d/%s/5x7" % (w, h, name)] = _entry([get(resize(x, (5, 7), f))[0]])
    for i, ((w, h), (ow, oh)) in enumerate(TALL_TARGETS):
        x = put(image(3000 + i, h, w)[None])
        for name, f in FILTERS.items():
            out["tall/%dx%d/%s/%dx%d" % (w, h, name, ow, oh)] = _entry([get(resize(x, (ow, oh), f))[0]])
    return out


def pillow_resize(x, size, f):
    from PIL import Image
    return np.stack([np.asarray(Image.fromarray(np.ascontiguousarray(im)).resize(size, f)) for im in x])


def pillow_digests():
    return digests(pillow_resize)


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
