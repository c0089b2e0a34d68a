"""ORACLE (test infrastructure) -- the reference's dataset tools (python/depthmotionnet/dataset_tools) in three forms:

* numpy restatements of its compute, which the CPU tests hold to the reference and the GPU tests hold the device to:
  `depth_ratios_numpy` (compute_depth_ratios of view_tools_cython.pyx, float32 operations in the .pyx's order) and
  `sharpness_numpy` (measure_sharpness: Pillow's grey, scipy's Laplacian, numpy's pairwise float32 variance);
* `reference_depth_ratios`, the reference's own Cython compute_depth_ratios from oracle/_ref/view_tools_cython.so (built by
  oracle/view_tools.py), or its stored digests (tests/golden/dataset_tools_digests.json, recorded with DEMON_REF_RECORD);
* the reference's helpers.py and sun3d_utils.py, loaded where they lie in the reference tree next to DEMON_REF_SRC
  (nothing is copied), and a deterministic synthetic SUN3D sequence to run them on.

The reference's modules import h5py and view_io's lz4 / webp wrappers, none of which this project needs: stub modules
stand in for them while the reference is loaded, `view_tools_cython` is the extension oracle/view_tools.py compiles from the
reference's own .pyx, and `FakeH5File` records what create_samples_from_sequence writes (require_group, attrs,
write_view) in dicts.  `reference_groups` turns that record into the groups demon_b200.dataset_tools.sun3d_view_groups
returns; tests/golden/sun3d_groups.json holds them (with the sequence's sharpness) for machines without the reference.

Only tests/, __graft_entry__ and tools/ may import this module.
"""
import hashlib
import importlib
import json
import os
import sys
import types

import numpy as np
from PIL import Image

from . import view_tools as vt
from .recorded import REF_SRC, Recorded, Store, entry, record

_HERE = os.path.dirname(os.path.abspath(__file__))
DATASET_TOOLS = (os.path.normpath(os.path.join(REF_SRC, "..", "..", "python", "depthmotionnet", "dataset_tools")) if REF_SRC
                 else "")
GOLDEN = os.path.join(os.path.dirname(_HERE), "tests", "golden", "sun3d_groups.json")
SEQ_NAME = "synthetic_lab/seq_1"
BASELINE_RANGE = (0.05, 0.6)
SHARPNESS_WINDOW = 5
MAX_VIEWS_NUM = 3
_PKG = "_demon_reference_dataset_tools"


def have_reference():
    return bool(DATASET_TOOLS) and os.path.isfile(os.path.join(DATASET_TOOLS, "sun3d_utils.py")) and vt.have_module()


# ---- compute_depth_ratios (view_tools_cython.pyx:107-191) -------------------------------------------------------------
_RATIOS = Store("dataset_tools_digests.json")
RecordedRatios = Recorded   # the digest of a stored ratio map: NaNs canonicalised like every other


def depth_ratios_numpy(depth1, depth2, K1, R1, t1, P2):
    """_compute_depth_ratios (view_tools_cython.pyx:107-159) over the whole image at once, float32 operations in the loop's
    order.  Returns (ratios, out_of_array): where the .pyx reads depth2 at flat index y2*w + x2 >= h*w (x2 = w on the last
    row, or y2 = h) its result is undefined; those pixels are NaN here and flagged in out_of_array."""
    f = np.float32
    depth1, depth2 = np.asarray(depth1, dtype=f), np.asarray(depth2, dtype=f)
    K1, R1, t1, P2 = (np.asarray(a, dtype=f) for a in (K1, R1, t1, P2))
    RT = R1.T
    h, w = depth1.shape
    h2, w2 = depth2.shape
    px = (np.arange(w) + 0.5).astype(f)[None, :]
    py = (np.arange(h) + 0.5).astype(f)[:, None]
    with np.errstate(all='ignore'):
        d = depth1
        valid = np.isfinite(d) & (d > f(0))
        p0 = d * (px - K1[0, 2]) / K1[0, 0]
        p1 = d * (py - K1[1, 2]) / K1[1, 1]
        p2 = d
        p0 = p0 - t1[0]
        p1 = p1 - t1[1]
        p2 = p2 - t1[2]
        q = [RT[r, 0] * p0 + RT[r, 1] * p1 + RT[r, 2] * p2 for r in range(3)]
        pr = [P2[r, 0] * q[0] + P2[r, 1] * q[1] + P2[r, 2] * q[2] + P2[r, 3] * f(1) for r in range(3)]
        front = pr[2] > f(0)
        u = pr[0] / pr[2]
        v = pr[1] / pr[2]
        inside = valid & front & (u > f(0)) & (v > f(0)) & (u < f(w2)) & (v < f(h2))
        # int(round(x)) of Python's round: half to even, which np.rint is
        x2 = np.clip(np.where(inside, np.rint(u), 0), 0, w2).astype(np.int64)
        y2 = np.clip(np.where(inside, np.rint(v), 0), 0, h2).astype(np.int64)
        flat = y2 * w2 + x2
        out_of_array = inside & (flat >= h2 * w2)
        look = inside & ~out_of_array
        d2 = np.full((h, w), np.nan, dtype=f)
        d2[look] = depth2.reshape(-1)[flat[look]]
        ok = look & (d2 > f(0)) & np.isfinite(d2)
        ratios = np.full((h, w), np.nan, dtype=f)
        ratios[ok] = pr[2][ok] / d2[ok]
    return ratios, out_of_array


def ratios_available():
    return vt.have_module() or bool(_RATIOS.entries())


def reference_depth_ratios(depth1, depth2, K1, R1, t1, K2, R2, t2):
    """compute_depth_ratios(view1, view2) of the reference's Cython for one ordered view pair (float32 camera-z depths of one
    size, float64 cameras).  The pixels the .pyx reads past depth2 for (depth_ratios_numpy's out_of_array) are set to NaN,
    so the result is defined.  Returns the float32 map, or its Recorded digest (tests/golden/dataset_tools_digests.json,
    recorded with DEMON_REF_RECORD=<json path>)."""
    depth1 = np.ascontiguousarray(depth1, dtype=np.float32)
    depth2 = np.ascontiguousarray(depth2, dtype=np.float32)
    arrays = [depth1, depth2] + [np.asarray(a) for a in (K1, R1, t1, K2, R2, t2)]
    h = hashlib.sha256(b"depth_ratios")
    for a in arrays:
        a = np.ascontiguousarray(a)
        h.update(("%s|%s" % (a.dtype.str, a.shape)).encode())
        h.update(a.tobytes())
    key = h.hexdigest()
    if not vt.have_module():
        return Recorded(_RATIOS.lookup(key, "result for this compute_depth_ratios call"))
    v1 = vt.View(R=np.asarray(R1), t=np.asarray(t1), K=np.asarray(K1), image=None, depth=depth1, depth_metric='camera_z')
    v2 = vt.View(R=np.asarray(R2), t=np.asarray(t2), K=np.asarray(K2), image=None, depth=depth2, depth_metric='camera_z')
    ratios = np.array(vt.module().compute_depth_ratios(v1, v2), dtype=np.float32)
    _, oob = depth_ratios_numpy(depth1, depth2, *vt.operands(K1, R1, t1, K2, R2, t2))
    ratios[oob] = np.nan
    record(key, entry(ratios))
    return ratios


def ratio_edge_cases():
    """View pairs (depth1, depth2, K1, R1, t1, K2, R2, t2) the tests hold the device, the numpy restatement and the
    reference's Cython to: NaN, +-inf, 0, negative and denormal depths in both views, points behind the second camera,
    projections exactly on .5 (half to even and half away from zero differ) and in [w-0.5, w) (the lookup at x2 = w reads
    the next row's first pixel, or past the array on the last row), realistic camera motion, and a 480x640 pair."""
    from demon_b200.evaluation import angleaxis_to_rotation_matrix, intrinsics_vector_to_K
    rng = np.random.RandomState(20172)
    cases = []

    def depth_map(h, w, lo=0.3, hi=8.0):
        d = rng.uniform(lo, hi, (h, w)).astype(np.float32)
        d[rng.rand(h, w) < 0.04] = np.nan
        d[rng.rand(h, w) < 0.03] = 0.0
        d[rng.rand(h, w) < 0.03] *= -1.0
        d[rng.rand(h, w) < 0.01] = np.inf
        d[rng.rand(h, w) < 0.01] = -np.inf
        d[rng.rand(h, w) < 0.01] = np.float32(1e-40)   # denormal: pr2 / d2 overflows to inf
        return d
    sun3d = np.array([0.891, 1.188, 0.5, 0.5])
    for h, w in ((7, 9), (48, 64), (31, 17)):
        K = intrinsics_vector_to_K(sun3d, w, h)
        R = angleaxis_to_rotation_matrix(rng.normal(0, 0.05, 3))
        t = rng.normal(0, 0.1, 3)
        cases.append((depth_map(h, w), depth_map(h, w), K, np.eye(3), np.zeros(3), K, R, t))
    for h, w in ((20, 30), (33, 41)):
        K1 = intrinsics_vector_to_K(np.array([0.8, 1.1, 0.45, 0.55]), w, h)
        K2 = intrinsics_vector_to_K(sun3d, w, h)
        cases.append((depth_map(h, w, 2.0, 8.0), depth_map(h, w, 2.0, 8.0), K1, angleaxis_to_rotation_matrix(rng.normal(0, 0.05, 3)),
                      rng.normal(0, 0.1, 3), K2, angleaxis_to_rotation_matrix(rng.normal(0, 0.05, 3)), rng.normal(0, 0.1, 3)))
    # points behind the second camera: it sits 5 units in front of view 1 looking back along z
    h, w = 16, 24
    K = intrinsics_vector_to_K(sun3d, w, h)
    cases.append((depth_map(h, w, 0.5, 10.0), depth_map(h, w, 0.5, 10.0), K, np.eye(3), np.zeros(3), K,
                  angleaxis_to_rotation_matrix(np.array([0.0, np.pi, 0.0])), np.array([0.0, 0.0, 5.0])))
    # depth 1, fx = fy = 2 and the principal point at the centre put pixel (x, y) at u = x + 0.5 + 2 tx, v = y + 0.5 + 2 ty,
    # exactly: with tx = 0 every u is a tie (rint sends x + 0.5 to the even neighbour) and the last column's u = w - 0.5
    # rounds to w for even w; ty = 0 does the same to v and the last row (y2 = h is past the array)
    for (h, w), (tx, ty) in (((12, 10), (0.0, 0.0)), ((12, 10), (0.0, -0.125)), ((9, 14), (-0.125, 0.0)), ((11, 7), (0.0, 0.0))):
        K = np.array([[2.0, 0.0, w / 2], [0.0, 2.0, h / 2], [0.0, 0.0, 1.0]])
        d2 = rng.uniform(0.85, 1.2, (h, w)).astype(np.float32)
        cases.append((np.ones((h, w), dtype=np.float32), d2, K, np.eye(3), np.zeros(3), K, np.eye(3), np.array([tx, ty, 0.0])))
    # a 480x640 pair of a smooth scene at the sun3d intrinsics
    h, w = 480, 640
    K = intrinsics_vector_to_K(sun3d, w, h)
    yy, xx = np.mgrid[0:h, 0:w]
    d = (2.0 + np.sin(xx / 50.0) + 0.5 * np.cos(yy / 30.0)).astype(np.float32)
    d[rng.rand(h, w) < 0.02] = np.nan
    d2 = (d * np.float32(1.02) + rng.normal(0, 0.02, (h, w))).astype(np.float32)
    cases.append((d, d2, K, np.eye(3), np.zeros(3), K, angleaxis_to_rotation_matrix(np.array([0.02, -0.1, 0.01])),
                  np.array([0.3, -0.05, 0.1])))
    return cases


# ---- measure_sharpness (helpers.py:23-31) ---------------------------------------------------------------------------
def grey_pillow(rgb):
    """Image.convert('L') of uint8 RGB [..., h, w, 3]: (R*19595 + G*38470 + B*7471 + 0x8000) >> 16, as int64."""
    c = np.asarray(rgb, dtype=np.int64)
    return (c[..., 0] * 19595 + c[..., 1] * 38470 + c[..., 2] * 7471 + 0x8000) >> 16


def laplace_reflect(grey):
    """scipy.ndimage.laplace(mode='reflect') of integer images [..., h, w]: [1,-2,1] along each axis, edge samples repeated."""
    g = np.asarray(grey, dtype=np.int64)
    ym = np.concatenate([g[..., :1, :], g[..., :-1, :]], axis=-2)
    yp = np.concatenate([g[..., 1:, :], g[..., -1:, :]], axis=-2)
    xm = np.concatenate([g[..., :1], g[..., :-1]], axis=-1)
    xp = np.concatenate([g[..., 1:], g[..., -1:]], axis=-1)
    return (ym + yp - 2 * g) + (xm + xp - 2 * g)


def pairwise_leaves(n):
    """The leaves (offset, length) of numpy's pairwise float32 sum of n elements, in order, and the tree as nested tuples."""
    def node(off, m):
        if m <= 128:
            return (off, m)
        n2 = m // 2
        n2 -= n2 % 8
        return (node(off, n2), node(off + n2, m - n2))
    return node(0, n)


def pairwise_sum_f32(a):
    """numpy's pairwise summation of float32 a [..., n] along the last axis, vectorised over the leading axes."""
    a = np.asarray(a, dtype=np.float32)
    f = np.float32

    def leaf(off, m):
        x = a[..., off:off + m]
        if m < 8:
            res = np.zeros(a.shape[:-1], dtype=f)
            for i in range(m):
                res = res + x[..., i]
            return res
        r = [x[..., j].copy() for j in range(8)]
        i = 8
        while i < m - m % 8:
            for j in range(8):
                r[j] = r[j] + x[..., i + j]
            i += 8
        res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
        for k in range(i, m):
            res = res + x[..., k]
        return res

    def walk(t):
        if isinstance(t[0], tuple):
            return walk(t[0]) + walk(t[1])
        return leaf(*t)
    return walk(pairwise_leaves(a.shape[-1]))


def sharpness_numpy(rgb):
    """measure_sharpness of uint8 RGB [..., h, w, 3] restated: np.var(laplace(grey)) as numpy computes it, float32
    mean = pairwise(lap) / n and var = pairwise((lap - mean)^2) / n.  Returns float32 [...]."""
    rgb = np.asarray(rgb)
    lap = laplace_reflect(grey_pillow(rgb)).astype(np.float32)
    lead = lap.shape[:-2]
    n = lap.shape[-2] * lap.shape[-1]
    x = lap.reshape(lead + (n,))
    mean = pairwise_sum_f32(x) / np.float32(n)
    dv = x - np.asarray(mean, dtype=np.float32)[..., None]
    return (pairwise_sum_f32(dv * dv) / np.float32(n)).astype(np.float32)


class FakeH5Group(dict):
    def __init__(self):
        super().__init__()
        self.attrs = {}
        self.views = []


class FakeH5File:
    """The parts of h5py.File create_samples_from_sequence uses: require_group(path), file[name]['frames/t0'].attrs."""

    def __init__(self):
        self.groups = {}

    def require_group(self, path):
        return self.groups.setdefault(path, FakeH5Group())

    def __getitem__(self, name):
        file = self

        class Sub:
            def __getitem__(self, sub):
                return file.require_group(name + '/' + sub)
        return Sub()


def _stub(name, **attrs):
    m = types.ModuleType(name)
    for k, v in attrs.items():
        setattr(m, k, v)
    return m


_ref = None


def reference():
    """The reference's (helpers, sun3d_utils, view_tools) modules, loaded once by path with the stubs in place."""
    global _ref
    if _ref is None:
        if not have_reference():
            raise RuntimeError("the reference's dataset_tools and oracle/_ref/view_tools_cython.so are needed")
        pkg = types.ModuleType(_PKG)
        pkg.__path__ = [DATASET_TOOLS]
        stubs = {
            _PKG: pkg,
            _PKG + ".lz4": _stub(_PKG + ".lz4", lz4_uncompress=None, lz4_compress_HC=None),
            _PKG + ".webp": _stub(_PKG + ".webp", webp_encode_array=None, webp_encode_image=None),
            _PKG + ".view_tools_cython": vt.module(),
        }
        temporary = {"h5py": _stub("h5py"), "pyximport": _stub("pyximport", install=lambda *a, **k: None)}
        saved = {k: sys.modules.get(k) for k in temporary}
        sys.modules.update(stubs)
        sys.modules.update(temporary)
        try:
            helpers = importlib.import_module(_PKG + ".helpers")
            sun3d = importlib.import_module(_PKG + ".sun3d_utils")
            view_tools = importlib.import_module(_PKG + ".view_tools")
        finally:
            for k, v in saved.items():
                if v is None:
                    sys.modules.pop(k, None)
                else:
                    sys.modules[k] = v

        def write_view(h5_group, view):   # replaces view_io.write_view (webp / lz4 encoding) in sun3d_utils' namespace
            h5_group.views.append(view)
        sun3d.write_view = write_view
        _ref = (helpers, sun3d, view_tools)
    return _ref


# ---- the synthetic sequence ---------------------------------------------------------------------------------------------
def write_sequence(root, seed=5, frames=40, h=48, w=64):
    """A SUN3D sequence under root/SEQ_NAME: image/<id>-<timestamp>.jpg holding PNG bytes (Pillow opens files by content,
    so no lossy codec is involved), depthTSDF/<id>-<timestamp>.png 16-bit depth with SUN3D's bit rotation, one
    extrinsics/*.txt with camera-to-world [R|c] rows per frame, and intrinsics.txt.  The camera walks along a wall with a
    slight yaw; the depth is the wall's camera z, with some frames broken (scaled: inconsistent; mostly zero: too little
    valid depth) and blurred images in between sharp ones.  Returns the sequence path."""
    from PIL import Image
    rng = np.random.RandomState(seed)
    seq = os.path.join(root, SEQ_NAME)
    for d in ('image', 'depthTSDF', 'extrinsics'):
        os.makedirs(os.path.join(seq, d), exist_ok=True)
    K = np.array([[58.0, 0.0, 31.5], [0.0, 58.0, 23.5], [0.0, 0.0, 1.0]])
    np.savetxt(os.path.join(seq, 'intrinsics.txt'), K, fmt='%.17g')
    texture = rng.randint(0, 256, (h * 3, w * 6, 3)).astype(np.float64)
    rows = []
    for f in range(frames):
        yaw = 0.02 * np.sin(f / 5.0)
        c = np.array([0.045 * f, 0.01 * np.cos(f / 3.0), 0.0])
        Rcw = np.array([[np.cos(yaw), 0, np.sin(yaw)], [0, 1, 0], [-np.sin(yaw), 0, np.cos(yaw)]])
        rows.append(np.concatenate([Rcw, c[:, None]], axis=1))
        # the wall z_world = 3 + 0.1 x_world: camera z along each pixel's ray
        yy, xx = np.mgrid[0:h, 0:w]
        ray = Rcw.dot(np.stack([(xx + 0.5 - K[0, 2]) / K[0, 0], (yy + 0.5 - K[1, 2]) / K[1, 1], np.ones((h, w))]).reshape(3, -1))
        s = (3.0 + 0.1 * c[0] - c[2]) / (ray[2] - 0.1 * ray[0])
        mm = np.clip(np.round(s * 1000), 0, 65535).reshape(h, w)
        if f % 7 == 3:
            mm = np.clip(mm * 1.4, 0, 65535)   # inconsistent with its neighbours
        if f % 11 == 5:
            mm[:, : int(w * 0.6)] = 0          # under half the pixels valid
        mm = mm.astype(np.uint32)
        raw = (((mm << 3) | (mm >> 13)) & 0xffff).astype(np.uint16)
        Image.fromarray(raw).save(os.path.join(seq, 'depthTSDF', '%07d-%012d.png' % (f, 1000 * f + 7)))
        x0 = int(3 * f) % (texture.shape[1] - w)
        img = texture[h:2 * h, x0:x0 + w]
        blur = (f % 4) * 0.25
        img = (1 - blur) * img + blur * np.roll(img, 1, axis=1)
        Image.fromarray(np.clip(img, 0, 255).astype(np.uint8)).save(os.path.join(seq, 'image', '%07d-%012d.jpg' % (f, 1000 * f)),
                                                                    format='PNG')
    np.savetxt(os.path.join(seq, 'extrinsics', '20000101000000.txt'), np.concatenate(rows, axis=0), fmt='%.17g')
    return seq


def reference_groups(root, sharpness=None):
    """create_samples_from_sequence of the reference on the sequence under root: (sharpness [F] float32 of the reference's
    compute_sharpness, groups as [{'name', 'frames', 'viewpoint_pairs'}] in write order)."""
    helpers, sun3d, _ = reference()
    if sharpness is None:
        sharpness = sun3d.compute_sharpness(root, SEQ_NAME)
    h5 = FakeH5File()
    n = sun3d.create_samples_from_sequence(h5, root, SEQ_NAME, BASELINE_RANGE, sharpness, sharpness_window=SHARPNESS_WINDOW,
                                           max_views_num=MAX_VIEWS_NUM)
    image_files = sorted(os.listdir(os.path.join(root, SEQ_NAME, 'image')))
    groups = {}
    for path, g in h5.groups.items():
        name, rest = path.split('/frames/t0')
        if rest:
            groups.setdefault(name, {})['v'] = groups.get(name, {}).get('v', []) + [(int(rest[2:]), g.views[0])]
        else:
            groups.setdefault(name, {})['pairs'] = g.attrs['viewpoint_pairs']
    out = []
    for name, g in groups.items():
        views = [v for _, v in sorted(g['v'], key=lambda x: x[0])]
        frames = [image_files.index(os.path.basename(v.image.filename)) for v in views]
        out.append({'name': name, 'frames': frames, 'viewpoint_pairs': np.asarray(g['pairs'], dtype=np.int32)})
    assert n == len(out)
    return np.asarray(sharpness, dtype=np.float32), out


def to_json(sharpness, groups):
    return {"seq_name": SEQ_NAME, "baseline_range": list(BASELINE_RANGE), "sharpness_window": SHARPNESS_WINDOW,
            "max_views_num": MAX_VIEWS_NUM, "sharpness_f32_bits": [int(v) for v in np.asarray(sharpness, np.float32).view(np.uint32)],
            "groups": [{"name": g['name'], "frames": [int(f) for f in g['frames']],
                        "viewpoint_pairs": [int(p) for p in g['viewpoint_pairs']]} for g in groups]}


def golden():
    """tests/golden/sun3d_groups.json: (sharpness float32 [F], groups) of the reference on write_sequence's directory."""
    d = json.load(open(GOLDEN))
    sharp = np.asarray(d["sharpness_f32_bits"], dtype=np.uint32).view(np.float32)
    groups = [{'name': g['name'], 'frames': g['frames'], 'viewpoint_pairs': np.asarray(g['viewpoint_pairs'], dtype=np.int32)}
              for g in d["groups"]]
    return sharp, groups


def _read_Rt(extrinsics, frame):
    """sun3d_utils.read_Rt (sun3d_utils.py:74-88)."""
    Rt = extrinsics[3 * frame:3 * frame + 3]
    R = Rt[0:3, 0:3].transpose()
    return R, -np.dot(R, Rt[0:3, 3])


def sequence_inputs(root):
    """What create_samples_from_sequence reads from the sequence under root, on the host: (R [F,3,3], t [F,3], K [3,3],
    depth [F,h,w] float32 of the depth file each frame maps to, image ids [F])."""
    seq = os.path.join(root, SEQ_NAME)
    image_files = sorted(f for f in os.listdir(os.path.join(seq, 'image')) if f.endswith('.jpg'))
    depth_files = sorted(f for f in os.listdir(os.path.join(seq, 'depthTSDF')) if f.endswith('.png'))
    K = np.loadtxt(os.path.join(seq, 'intrinsics.txt'))
    ext = np.loadtxt(os.path.join(seq, 'extrinsics', sorted(os.listdir(os.path.join(seq, 'extrinsics')))[-1]))
    ids = np.asarray([int(f.split('-')[0]) for f in image_files])
    its = np.asarray([int(f[:-4].split('-')[1]) for f in image_files])
    dts = np.asarray([int(f[:-4].split('-')[1]) for f in depth_files])
    F = len(image_files)
    R, t = np.empty((F, 3, 3)), np.empty((F, 3))
    depth = []
    for f in range(F):
        R[f], t[f] = _read_Rt(ext, f)
        raw = np.array(Image.open(os.path.join(seq, 'depthTSDF', depth_files[np.argmin(abs(dts - its[f]))]))).astype(np.uint16)
        depth.append(((raw >> 3) | (raw << 13)).astype(np.uint16) / 1000)
    depth = np.stack(depth).astype(np.float32)
    return R, t, K, depth, ids


if __name__ == "__main__":
    # python -m oracle.dataset_tools <scratch dir>: regenerate tests/golden/sun3d_groups.json from the reference
    root = sys.argv[1]
    write_sequence(root)
    s, g = reference_groups(root)
    with open(GOLDEN, "w") as f:
        json.dump(to_json(s, g), f, indent=1)
    print(len(g), "groups")
