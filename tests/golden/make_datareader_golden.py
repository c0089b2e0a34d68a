"""Writes tests/golden/datareader_resize_digests.json: the shape and SHA-256 of what OpenCV's `cv::resize` returns for the
two calls of the multi-view reader's prepareScene (multivih5datareader.cpp:1439-1440 and :1481-1482), the fixture of
demon_b200.datareader.ViewPool.add (csrc/datareader.cu):
  area     cv::resize(image, (w, h), INTER_AREA) of a uint8 [sh, sw, 3] image, h <= sh and w <= sw;
  nearest  cv::resize(depth, (w, h), INTER_NEAREST) of a float32 [sh, sw] plane holding NaN of both signs (quiet and with a
           payload), +-inf and -0; the digest is over the bits.

The inputs are regenerated from seeds with numpy.random.default_rng, so no image is stored.  `digests(area, nearest)` runs
every case through any backend: OpenCV here (python tests/golden/make_datareader_golden.py, which records its version
under "_opencv"), the oracle in tests/test_datareader_opencv.py and the device in tests/test_gpu_datareader_resize.py.
`area(images, h, w)` and `nearest(planes, h, w)` map a list of sources of any sizes to the list of their h x w results.

INTER_AREA takes one of three paths (oracle/datareader.py, area_path), and the cases pick each of them at its edges:
  train    training.py's 640x480 -> 256x192 (general path, every weight k/25)
  2x2      the factor-2 vector path, on random data and on blocks whose sums sweep every value 0..1020 (every tie)
  fast     the other integer factors (kx x ky): 2x1, 1x2, 3x3, 4x4, 2x3, 16x16, and 14, 26, 28 and 30 along a row, where
           float(sum) * (1.f / area) is not the exact mean rounded; block sums sweep every value here too.  At an area
           above 2^24 that float cannot hold (2049 x 8191) 1.f / (float)area is not float(1.0 / area): the block sums are
           chosen where the two round differently.  OpenCV sums a block in int, which wraps above 2^31 (4096 x 4096 of
           values from 128 up)
  divisible  sides divisible by the output side whose scale is not integral (98 -> 2, 147 -> 3, ...): the general path;
           with block sums swept at 6272 -> 64 and 3920 -> 40 (factor 98) the integer path would round some differently
  near     general-path factors k +- 1/w around integers, 640x480 -> 213x160, 131x97 -> 61x83
  sliver   outputs wider or higher than 1000, where a cell's overlap can be a sliver of at most 1e-3 of a source cell that
           computeResizeAreaTab drops (1024 -> 1023: output 0 overlaps source cell 1 by 1/1023)
  edge     equal size, 1x1 outputs, sources one pixel wide or high
  scan     one-row images of every width w..2048 resized to w in {256, 83, 64, 61} (one digest over all widths), and
           one-column images of every height the same way (the vertical accumulation)
  f16      float16 depths (NaN of both signs, +-inf, -0, subnormals) of three sources that take the three paths to 256x192;
           the nearest digest is over OpenCV's resize of their exact float32 values
"""
import hashlib
import json
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
PATH = os.path.join(HERE, "datareader_resize_digests.json")
# (name, source height, source width, height, width, data): data 'random', 'sums' (block sums sweep 0..255*area) or
# 'split' (one block whose sums round differently with 1.f / (float)area and float(1.0 / area)) or 'bright' (128..255)
CASES = [
    ("train/640x480-256x192", 480, 640, 192, 256, "random"),
    ("2x2/512x384-256x192", 384, 512, 192, 256, "random"),
    ("2x2/512x384-256x192/sums", 384, 512, 192, 256, "sums"),
    ("2x2/128x96-64x48", 96, 128, 48, 64, "random"),
    ("2x2/128x96-64x48/sums", 96, 128, 48, 64, "sums"),
    ("fast/2x1/128x48-64x48", 48, 128, 48, 64, "sums"),
    ("fast/1x2/64x96-64x48", 96, 64, 48, 64, "sums"),
    ("fast/3x3/192x144-64x48", 144, 192, 48, 64, "sums"),
    ("fast/4x4/256x192-64x48", 192, 256, 48, 64, "sums"),
    ("fast/2x3/128x144-64x48", 144, 128, 48, 64, "sums"),
    ("fast/16x16/4096x3072-256x192", 3072, 4096, 192, 256, "random"),
    ("fast/14x1/896x1-64x1", 1, 896, 1, 64, "sums"),
    ("fast/26x1/1664x1-64x1", 1, 1664, 1, 64, "sums"),
    ("fast/28x1/1792x1-64x1", 1, 1792, 1, 64, "sums"),
    ("fast/30x1/1920x1-64x1", 1, 1920, 1, 64, "sums"),
    ("fast/1x14/8x56-8x4", 56, 8, 4, 8, "sums"),
    ("fast/2049x8191/2049x8191-1x1", 8191, 2049, 1, 1, "split"),
    ("fast/4096x4096/4096x4096-1x1/wrap", 4096, 4096, 1, 1, "bright"),
    ("divisible/98x1-2x1", 1, 98, 1, 2, "random"),
    ("divisible/147x1-3x1", 1, 147, 1, 3, "random"),
    ("divisible/49x1-1x1", 1, 49, 1, 1, "random"),
    ("divisible/1x98-1x2", 98, 1, 2, 1, "random"),
    ("divisible/98x147-2x3", 147, 98, 3, 2, "random"),
    ("divisible/1666x588-98x12", 588, 1666, 12, 98, "random"),
    ("divisible/8190x1-35x1", 1, 8190, 1, 35, "random"),
    ("divisible/1x8190-1x78", 8190, 1, 78, 1, "random"),
    ("divisible/198x196-2x4", 196, 198, 4, 2, "random"),
    ("divisible/6272x48-64x48/sums", 48, 6272, 48, 64, "sums"),
    ("divisible/48x6272-48x64/sums", 6272, 48, 64, 48, "sums"),
    ("divisible/3920x96-40x48/sums", 96, 3920, 48, 40, "sums"),
    ("near/129x97-64x48", 97, 129, 48, 64, "random"),
    ("near/127x95-64x48", 95, 127, 48, 64, "random"),
    ("near/641x481-320x240", 481, 641, 240, 320, "random"),
    ("near/639x479-320x240", 479, 639, 240, 320, "random"),
    ("near/769x577-256x192", 577, 769, 192, 256, "random"),
    ("near/767x575-256x192", 575, 767, 192, 256, "random"),
    ("near/513x383-256x192", 383, 513, 192, 256, "random"),
    ("near/640x480-213x160", 480, 640, 160, 213, "random"),
    ("near/131x97-61x83", 97, 131, 83, 61, "random"),
    ("sliver/1024x768-1023x767", 768, 1024, 767, 1023, "random"),
    ("sliver/2049x1-2048x1", 1, 2049, 1, 2048, "random"),
    ("sliver/1x2049-1x2048", 2049, 1, 2048, 1, "random"),
    ("sliver/8191x2-8000x1", 2, 8191, 1, 8000, "random"),
    ("edge/64x48-64x48", 48, 64, 48, 64, "random"),
    ("edge/41x37-1x1", 37, 41, 1, 1, "random"),
    ("edge/641x479-1x1", 479, 641, 1, 1, "random"),
    ("edge/300x1-7x1", 1, 300, 1, 7, "random"),
    ("edge/1x300-1x7", 300, 1, 7, 1, "random"),
    ("edge/640x1-256x1", 1, 640, 1, 256, "random"),
    ("edge/1x480-1x192", 480, 1, 192, 1, "random"),
    ("edge/1x1-1x1", 1, 1, 1, 1, "random"),
]
SCAN_TARGETS = (256, 83, 64, 61)
SCAN_MAX = 2048
# three sources that take the general, 2x2 and fast paths to 256x192, with float16 depths
F16 = [("f16/640x480", 480, 640), ("f16/512x384", 384, 512), ("f16/4096x3072", 3072, 4096)]
F16_SIZE = (192, 256)


def image(seed, sh, sw, h, w, data):
    rng = np.random.default_rng(seed)
    img = rng.integers(128 if data == "bright" else 0, 256, (sh, sw, 3), dtype=np.uint8)
    if data == "sums":   # every (ky x kx) block gets the sum (block index * 7 + channel) mod (255 * area + 1), spread evenly
        ky, kx = sh // h, sw // w
        area = ky * kx
        s = (np.arange(h * w * 3).reshape(h, w, 3) * 7 + np.arange(3)) % (255 * area + 1)
        q, r = s // area, s % area
        k = np.arange(area).reshape(ky, kx)
        blocks = q[:, None, :, None] + (k[None, :, None, :, None] < r[:, None, :, None])   # [h, ky, w, kx, 3]
        img = rng.permuted(blocks.reshape(h, ky, w, kx, 3), axis=3).astype(np.uint8).reshape(sh, sw, 3)
    if data == "split":
        area = sh * sw
        img = np.zeros((sh, sw, 3), np.uint8)
        mean = 40
        for c in range(3):   # block means below 2^31 / area: OpenCV's int block sum does not wrap
            while True:
                mean += 1
                cand = np.arange(int((mean + 0.5) * area) - 2 ** 20, int((mean + 0.5) * area) + 2 ** 20)
                f = cand.astype(np.float32)
                at = np.nonzero(np.rint(f * (np.float32(1) / np.float32(area))) != np.rint(f * np.float32(1.0 / area)))[0]
                if at.size:
                    break
            total = int(cand[at[0]])
            plane = img[:, :, c].reshape(-1)
            plane[:] = total // area
            plane[:total % area] += 1
    return img


SPECIAL_BITS = np.array([0x7fc00000, 0xffc00000, 0x7fc12345, 0xffd00001, 0x7f800000, 0xff800000, 0x80000000, 0x00000000],
                        np.uint32)


def depth(seed, sh, sw):
    """float32 [sh, sw] in [0.5, 10) with every eighth value one of SPECIAL_BITS, at random places"""
    rng = np.random.default_rng(seed)
    d = rng.uniform(0.5, 10.0, (sh, sw)).astype(np.float32)
    bits = d.reshape(-1).view(np.uint32)
    at = rng.random(bits.size) < 0.125
    bits[at] = rng.choice(SPECIAL_BITS, int(at.sum()))
    return d


SPECIAL_HALF = np.array([0x7e00, 0xfe00, 0x7c00, 0xfc00, 0x8000, 0x0000, 0x0001, 0x83ff], np.uint16)


def depth16(seed, sh, sw):
    """float16 [sh, sw] in [0.5, 10) with every eighth value quiet NaN of either sign, +-inf, +-0 or a subnormal"""
    rng = np.random.default_rng(seed)
    d = rng.uniform(0.5, 10.0, (sh, sw)).astype(np.float16)
    bits = d.reshape(-1).view(np.uint16)
    at = rng.random(bits.size) < 0.125
    bits[at] = rng.choice(SPECIAL_HALF, int(at.sum()))
    return d


def scan_row(target):
    """one-row uint8 images of every width target..SCAN_MAX, and float32 planes of the same widths"""
    base = image(7, 1, SCAN_MAX, 1, SCAN_MAX, "random")
    plane = depth(8, 1, SCAN_MAX)
    return [base[:, :w] for w in range(target, SCAN_MAX + 1)], [plane[:, :w] for w in range(target, SCAN_MAX + 1)]


def scan_col(target):
    imgs, planes = scan_row(target)
    return [np.ascontiguousarray(a.transpose(1, 0, 2)) for a in imgs], [np.ascontiguousarray(p.T) for p in planes]


def _entry(arrays):
    """shape of the first array (all of them for a list) and the SHA-256 of their bytes in order"""
    h = hashlib.sha256()
    shapes = []
    for a in arrays:
        a = np.ascontiguousarray(a)
        shapes.append(list(a.shape))
        h.update(a.tobytes())
    return {"shape": shapes[0] if len(shapes) == 1 else [len(shapes)] + shapes[-1], "sha256": h.hexdigest()}


def digests(area, nearest):
    """Every case through one backend: area(list of uint8 [sh,sw,3], h, w) and nearest(list of float32 [sh,sw], h, w)
    return the lists of [h,w,3] uint8 and [h,w] float32 results.  Returns {case: {"shape", "sha256"}}."""
    out = {}
    for i, (name, sh, sw, h, w, data) in enumerate(CASES):
        out["area/" + name] = _entry(area([image(100 + i, sh, sw, h, w, data)], h, w))
        out["nearest/" + name] = _entry(nearest([depth(300 + i, sh, sw)], h, w))
    for target in SCAN_TARGETS:
        for kind, make, size in (("width", scan_row, (1, target)), ("height", scan_col, (target, 1))):
            imgs, planes = make(target)
            out["area/scan/%s/%d" % (kind, target)] = _entry(area(imgs, *size))
            out["nearest/scan/%s/%d" % (kind, target)] = _entry(nearest(planes, *size))
    for i, (name, sh, sw) in enumerate(F16):
        out["nearest/" + name] = _entry(nearest([depth16(500 + i, sh, sw).astype(np.float32)], *F16_SIZE))
    return out


def opencv_area(images, h, w):
    import cv2
    return [cv2.resize(im, (w, h), interpolation=cv2.INTER_AREA).reshape(h, w, 3) for im in images]


def opencv_nearest(planes, h, w):
    import cv2
    return [cv2.resize(p, (w, h), interpolation=cv2.INTER_NEAREST).reshape(h, w) for p in planes]


def opencv_digests():
    return digests(opencv_area, opencv_nearest)


def main():
    import cv2
    d = opencv_digests()
    d["_opencv"] = cv2.__version__
    with open(PATH, "w") as fh:
        json.dump(d, fh, indent=1, sort_keys=True)
        fh.write("\n")
    print("wrote %d digests to %s (OpenCV %s)" % (len(d) - 1, PATH, cv2.__version__))


if __name__ == "__main__":
    main()
