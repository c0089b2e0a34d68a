"""The compute of the reference's multi-view training reader (`multi_vi_h5_data_reader`,
multivih5datareaderop/multivih5datareader.cpp) on the device: what training/v2/training.py gets every batch from.

    pool = ViewPool(256, 192)
    idx = pool.add(views)                                   # dataset_tools.View tuples -> prepared views on the device
    aug = draw_augmentation(reader_params, 32, np.random.default_rng(0))
    batch = build_batch(pool, [(idx[0], idx[1]), ...], reader_params, aug)
    batch['IMAGE_PAIR'], batch['MOTION'], batch.used         # float32 CUDA tensors; the entries of `pairs` used

`ViewPool.add` does prepareScene's work (:1384-1520) once per view in one launch (csrc/datareader.cu); `build_batch` does
the batch loop (:1585-1950): the per-item pose math here on the host in float64, every per-pixel output in one launch.
Reading HDF5 / webp / lz4, the scene pool's sampling and the builder threads are not part of this module: the caller
chooses which views the pool holds and which pairs make a batch.  There is no CPU fallback.
"""
import ctypes
import math
from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch

from . import _lib

OUTPUTS = ('IMAGE_PAIR', 'MOTION', 'FLOW', 'DEPTH', 'INTRINSICS', 'DEPTHMASKS')
MOTION_SIZES = {'ANGLEAXIS6': 6, 'ANGLEAXIS7': 7, 'QUATERNION': 7, 'FMATRIX': 8}
# multivih5datareader.h:113-133
DEFAULTS = {
    'batch_size': 1, 'test_phase': False, 'augment_rot180': 0.5, 'augment_mirror_x': 0.5, 'image_range_min': -0.5,
    'image_range_max': 0.5, 'motion_format': 'FMATRIX', 'depth_pair': False, 'norm_trans_scale_depth': True,
    'inverse_depth': False, 'min_depth': -1.0, 'max_depth': -1.0, 'depthmask_border1': 3, 'depthmask_border2': 5,
    'top_output': OUTPUTS,
}
# the colour augmentation's keys (a source's keys in the reader) and their values when absent (:656-668)
COLOUR_KEYS = ('aug_hsv_hue', 'aug_hsv_sat', 'aug_hsv_val', 'aug_contrast', 'aug_brightness', 'aug_gamma')
COLOUR_DEFAULTS = (0.0, 0.0, 0.0, 1.0, 0.0, 1.0)
# the reader's I/O keys: accepted and ignored.  scaled_width / scaled_height must match the pool when given.
IO_KEYS = ('source', 'scene_pool_size', 'builder_threads', 'scaled_width', 'scaled_height', 'convert_to_gray_values')
MAX_SIDE = 8192
MAX_HUE = 1e6   # the reader wraps the hue with `while` loops; a hue draw far beyond this would never finish

_VIEW_DTYPE = np.dtype({'names': ['image_offset', 'depth_offset', 'pool_index', 'width', 'height', 'depth_f16', 'ray_length', 'k', 'pad'],
                        'formats': ['<i8', '<i8', '<i8', '<i4', '<i4', '<i4', '<i4', ('<f4', 5), '<i4'],
                        'offsets': [0, 8, 16, 24, 28, 32, 36, 40, 60], 'itemsize': 64})
_ITEM_DTYPE = np.dtype({'names': ['view1', 'view2', 'flags', 'pad', 'depth_scale_factor', 'aug', 'cam'],
                        'formats': ['<i4', '<i4', '<i4', '<i4', '<f8', ('<f4', 6), ('<f4', (2, 17))],
                        'offsets': [0, 4, 8, 12, 16, 24, 48], 'itemsize': 184})


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _device():
    if not torch.cuda.is_available():
        raise RuntimeError("demon_b200.datareader needs a CUDA device (there is no CPU fallback)")
    return torch.device("cuda", torch.cuda.current_device())


def _host(a):
    if isinstance(a, torch.Tensor):
        return a.detach().cpu().numpy()
    return np.asarray(a)


def _align(n, a=16):
    return (n + a - 1) // a * a


class ViewPool:
    """Prepared views in device memory: `images` uint8 [n,h,w,3] and `depths` float32 [n,h,w] camera z at the scaled size,
    and per view its source size and its camera (the intrinsics normalised as prepareScene normalises them).  Views of
    different source sizes share one pool.  There is no eviction: the caller decides which views the pool holds."""

    def __init__(self, scaled_width=256, scaled_height=192):
        w, h = int(scaled_width), int(scaled_height)
        if not (1 <= w <= MAX_SIDE and 1 <= h <= MAX_SIDE):
            raise ValueError("scaled size %dx%d out of range (1..%d)" % (w, h, MAX_SIDE))
        self.width, self.height = w, h
        self._n = 0
        self._image = None
        self._depth = None
        self.source_sizes = np.zeros((0, 2), np.int64)   # (height, width) of each view's source
        self.cameras = np.zeros((0, 17), np.float64)      # fx/W, skew, cx/W, fy/H, cy/H, R row-major, t

    def __len__(self):
        return self._n

    @property
    def images(self):
        return self._image[:self._n]

    @property
    def depths(self):
        return self._depth[:self._n]

    def _reserve(self, n, dev):
        cap = 0 if self._image is None else self._image.shape[0]
        if n <= cap:
            return
        cap = max(n, 2 * cap, 16)
        img = torch.empty((cap, self.height, self.width, 3), dtype=torch.uint8, device=dev)
        dep = torch.empty((cap, self.height, self.width), dtype=torch.float32, device=dev)
        if self._n:
            img[:self._n].copy_(self._image[:self._n])
            dep[:self._n].copy_(self._depth[:self._n])
        self._image, self._depth = img, dep

    def add(self, views):
        """Prepares `views` (dataset_tools.View tuples: image uint8 [H,W,3] RGB as an array, a PIL image or a tensor;
        depth float32 or float16 [H,W]; K [3,3] in pixels, with skew; R [3,3]; t [3]; depth_metric 'camera_z' or
        'ray_length') in one launch and returns their pool indices.  The source must be at least the scaled size."""
        views = list(views)
        recs = np.zeros(len(views), _VIEW_DTYPE)
        cams = np.zeros((len(views), 17), np.float64)
        sizes = np.zeros((len(views), 2), np.int64)
        chunks, off = [], _align(len(views) * _VIEW_DTYPE.itemsize)
        for i, v in enumerate(views):
            img = np.ascontiguousarray(_host(v.image))
            if img.dtype != np.uint8 or img.ndim != 3 or img.shape[2] != 3:
                raise ValueError("view %d: image must be uint8 [H,W,3], got %s %s" % (i, img.dtype, img.shape))
            hs, ws = img.shape[:2]
            if not (1 <= hs <= MAX_SIDE and 1 <= ws <= MAX_SIDE):
                raise ValueError("view %d: source size %dx%d out of range (1..%d)" % (i, ws, hs, MAX_SIDE))
            if ws < self.width or hs < self.height:
                raise ValueError("view %d: %dx%d -> %dx%d would upscale; INTER_AREA's upscaling (bilinear) is not built"
                                 % (i, ws, hs, self.width, self.height))
            dep = np.ascontiguousarray(_host(v.depth))
            if dep.dtype not in (np.float32, np.float16) or dep.shape != (hs, ws):
                raise ValueError("view %d: depth must be float32 or float16 [%d,%d], got %s %s" % (i, hs, ws, dep.dtype, dep.shape))
            if v.depth_metric not in ('camera_z', 'ray_length'):
                raise ValueError("view %d: depth_metric must be 'camera_z' or 'ray_length', got %r" % (i, v.depth_metric))
            K = np.asarray(_host(v.K), np.float64)
            R = np.asarray(_host(v.R), np.float64)
            t = np.asarray(_host(v.t), np.float64).reshape(-1)
            if K.shape != (3, 3) or R.shape != (3, 3) or t.shape != (3,):
                raise ValueError("view %d: K and R must be [3,3] and t [3]" % i)
            if K[1, 0] != 0 or K[2, 0] != 0 or K[2, 1] != 0 or K[2, 2] != 1:
                raise ValueError("view %d: K must be [[fx, s, cx], [0, fy, cy], [0, 0, 1]]" % i)
            # prepareScene :1393-1396 in double; the skew K(0,1) stays in pixels
            cams[i, :5] = (K[0, 0] / ws, K[0, 1], K[0, 2] / ws, K[1, 1] / hs, K[1, 2] / hs)
            cams[i, 5:14] = R.reshape(-1)
            cams[i, 14:] = t
            sizes[i] = (hs, ws)
            r = recs[i]
            r['image_offset'] = off
            chunks.append((off, img.reshape(-1)))
            off = _align(off + img.nbytes)
            r['depth_offset'] = off
            chunks.append((off, dep.reshape(-1).view(np.uint8)))
            off = _align(off + dep.nbytes)
            r['pool_index'] = self._n + i
            r['width'], r['height'] = ws, hs
            r['depth_f16'] = int(dep.dtype == np.float16)
            r['ray_length'] = int(v.depth_metric == 'ray_length')
            r['k'] = cams[i, :5].astype(np.float32)
        if not views:
            return np.zeros(0, np.int64)
        dev = _device()
        staging = np.empty(off, np.uint8)
        staging[:recs.nbytes] = recs.view(np.uint8)
        for o, a in chunks:
            staging[o:o + a.nbytes] = a.view(np.uint8)
        buf = torch.from_numpy(staging).to(dev)
        self._reserve(self._n + len(views), dev)
        _lib.check(_lib.load().demon_datareader_prepare(buf.data_ptr(), buf.data_ptr(), len(views), self.height, self.width,
                                                        self._image.data_ptr(), self._depth.data_ptr(), _stream()))
        idx = np.arange(self._n, self._n + len(views), dtype=np.int64)
        self._n += len(views)
        self.source_sizes = np.concatenate([self.source_sizes, sizes])
        self.cameras = np.concatenate([self.cameras, cams])
        return idx


@dataclass
class Augmentation:
    """Each batch item's decisions: rot180 and mirror_x bool [B]; colour float32 [B,6] (hue, sat, val, contrast,
    brightness, gamma) or None, in which case the colour step does not run (:653)."""
    rot180: np.ndarray
    mirror_x: np.ndarray
    colour: Optional[np.ndarray] = None


def _random_param(spec, rng, key):
    if not isinstance(spec, dict):
        raise ValueError("%s must be a dict with 'normal' or 'uniform', got %r" % (key, spec))
    unknown = set(spec) - {'normal', 'uniform'}
    if unknown:
        raise ValueError("%s: unknown keys %s" % (key, sorted(unknown)))
    if 'normal' in spec:   # getRandomParam (:615-631); Normal() is mean 0, stddev 1 and Uniform() is a 0, b 1
        n = spec['normal']
        return rng.normal(float(n.get('mean', 0.0)), float(n.get('stddev', 1.0)))
    if 'uniform' in spec:
        u = spec['uniform']
        return rng.uniform(float(u.get('a', 0.0)), float(u.get('b', 1.0)))
    return 0.0


def draw_augmentation(params, batch_size, rng):
    """Draws every item's rot180, mirror_x and colour parameters from the numpy Generator `rng` with the reader's
    semantics: Bernoulli(augment_rot180 / augment_mirror_x) in training, `item < p*batch_size` with test_phase
    (:1587-1596); the colour draws only if one of the aug_* keys is present (:653), each absent key at its default."""
    b = int(batch_size)
    test = bool(params.get('test_phase', DEFAULTS['test_phase']))
    p_rot = float(params.get('augment_rot180', DEFAULTS['augment_rot180']))
    p_mir = float(params.get('augment_mirror_x', DEFAULTS['augment_mirror_x']))
    colour = None
    if any(k in params for k in COLOUR_KEYS):
        colour = np.empty((b, 6), np.float32)
    rot, mir = np.zeros(b, bool), np.zeros(b, bool)
    for i in range(b):
        if test:
            rot[i], mir[i] = i < p_rot * b, i < p_mir * b
        else:
            rot[i], mir[i] = rng.random() < p_rot, rng.random() < p_mir
        if colour is not None:
            for j, (k, d) in enumerate(zip(COLOUR_KEYS, COLOUR_DEFAULTS)):
                colour[i, j] = _random_param(params[k], rng, k) if k in params else d
    return Augmentation(rot, mir, colour)


def reader_params(params):
    """The reader's parameter dict with its defaults filled in; unknown keys and values are refused."""
    unknown = set(params) - set(DEFAULTS) - set(IO_KEYS) - set(COLOUR_KEYS)
    if unknown:
        raise ValueError("unknown reader parameters: %s" % sorted(unknown))
    p = dict(DEFAULTS)
    p.update({k: v for k, v in params.items() if k in DEFAULTS})
    if p['motion_format'] not in MOTION_SIZES:
        raise ValueError("motion_format must be one of %s, got %r" % (sorted(MOTION_SIZES), p['motion_format']))
    top = tuple(p['top_output'])
    if not top or any(t not in OUTPUTS for t in top) or len(set(top)) != len(top):
        raise ValueError("top_output must name distinct outputs of %s, got %r" % (OUTPUTS, top))
    p['top_output'] = top
    if int(p['batch_size']) < 1:
        raise ValueError("batch_size must be at least 1")
    if params.get('convert_to_gray_values'):
        raise ValueError("convert_to_gray_values is not built")
    return p


# ---- pose math, float64, per item (Eigen's fixed-size products sum left to right, as oracle/ref_stub/eigen_stub.h) ----
def _mm(A, B):
    return [[_dot_cols(A[i], B, j) for j in range(len(B[0]))] for i in range(len(A))]


def _dot_cols(row, B, j):
    s = row[0] * B[0][j]
    for k in range(1, len(row)):
        s = s + row[k] * B[k][j]
    return s


def _mv(A, v):
    return [(A[i][0] * v[0] + A[i][1] * v[1]) + A[i][2] * v[2] for i in range(3)]


def _tr(A):
    return [[A[j][i] for j in range(3)] for i in range(3)]


def _norm(v):
    return math.sqrt((v[0] * v[0] + v[1] * v[1]) + v[2] * v[2])


def _rot180(R, t):   # rotateCamera180DegAroundZ (:307-313)
    C = [-c for c in _mv(_tr(R), t)]
    R = [[-x for x in R[0]], [-x for x in R[1]], list(R[2])]
    return R, [-c for c in _mv(R, C)]


def _quaternion(m):   # Eigen 3.3 quaternion_assign_impl<.,3,3>: (w, x, y, z)
    t = (m[0][0] + m[1][1]) + m[2][2]
    q = [0.0, 0.0, 0.0]
    if t > 0:
        t = math.sqrt(t + 1.0)
        w = 0.5 * t
        t = 0.5 / t
        q = [(m[2][1] - m[1][2]) * t, (m[0][2] - m[2][0]) * t, (m[1][0] - m[0][1]) * t]
    else:
        i = 1 if m[1][1] > m[0][0] else 0
        if m[2][2] > m[i][i]:
            i = 2
        j, k = (i + 1) % 3, (i + 2) % 3
        t = math.sqrt(((m[i][i] - m[j][j]) - m[k][k]) + 1.0)
        q[i] = 0.5 * t
        t = 0.5 / t
        w = (m[k][j] - m[j][k]) * t
        q[j] = (m[j][i] + m[i][j]) * t
        q[k] = (m[k][i] + m[i][k]) * t
    return w, q


def _angle_axis(m):   # Eigen 3.3 AngleAxis(Matrix3d) through its quaternion; axis * angle
    w, v = _quaternion(m)
    n = _norm(v)
    if n < 2.220446049250313e-16:   # stableNorm
        s = max(abs(x) for x in v)
        n = 0.0 if s == 0 else s * _norm([x / s for x in v])
    if n == 0:
        return [0.0, 0.0, 0.0]
    angle = 2.0 * math.atan2(n, abs(w))
    if w < 0:
        n = -n
    return [(x / n) * angle for x in v]


def _det4(m):   # Eigen 3.3 determinant_impl<.,4>
    def h(j, k, a, b):
        return (m[j][0] * m[k][1] - m[k][0] * m[j][1]) * (m[a][2] * m[b][3] - m[b][2] * m[a][3])
    return ((((h(0, 1, 2, 3) - h(0, 2, 1, 3)) + h(0, 3, 1, 2)) + h(1, 2, 0, 3)) - h(1, 3, 0, 2)) + h(2, 3, 0, 1)


def _fundamental(P1, P2):   # computeFundamentalFromCameras (:264-304): F(i,j) = det [X_j ; Y_i]
    X = [[P1[1], P1[2]], [P1[2], P1[0]], [P1[0], P1[1]]]
    Y = [[P2[1], P2[2]], [P2[2], P2[0]], [P2[0], P2[1]]]
    return [[_det4(X[j] + Y[i]) for j in range(3)] for i in range(3)]


def _k_matrix(c):
    return [[c[0], c[1], c[2]], [0.0, c[3], c[4]], [0.0, 0.0, 1.0]]


def item_motion(cam1, cam2, rot180, mirror_x, params):
    """The motion block of the batch loop (:1650-1781) for one pair: (motion float64 [m], depth_scale_factor), or None
    where the reader skips the pair (|t12| < 1e-6, or |F(2,2)| < 1e-6 for FMATRIX)."""
    R1, t1 = [list(cam1[5 + 3 * i:8 + 3 * i]) for i in range(3)], list(cam1[14:17])
    R2, t2 = [list(cam2[5 + 3 * i:8 + 3 * i]) for i in range(3)], list(cam2[14:17])
    if rot180:
        R1, t1 = _rot180(R1, t1)
        R2, t2 = _rot180(R2, t2)
    R12 = _mm(R2, _tr(R1))
    Rt1 = _mv(R12, t1)
    t12 = [t2[i] - Rt1[i] for i in range(3)]
    if mirror_x:   # :1669-1676
        C2 = [-c for c in _mv(_tr(R12), t12)]
        C2[0] = -C2[0]
        for r in range(3):
            R12[r][0] = -R12[r][0]
        R12[0] = [-x for x in R12[0]]
        t12 = [-c for c in _mv(R12, C2)]
    n = _norm(t12)
    if n < 1e-6:
        return None
    dsf = 1.0
    if params['norm_trans_scale_depth']:
        dsf = 1 / n
        t12 = [x / n for x in t12]
    fmt = params['motion_format']
    if fmt == 'ANGLEAXIS6':
        return _angle_axis(R12) + t12, dsf
    if fmt == 'ANGLEAXIS7':
        aa = _angle_axis(R12)
        mag = _norm(aa)
        aa = [0.0, 0.0, 0.0] if mag < 1e-6 else [x / mag for x in aa]
        return [mag] + aa + t12, dsf
    if fmt == 'QUATERNION':
        w, q = _quaternion(R12)
        return [w] + q + t12, dsf
    P1 = _mm(_k_matrix(cam1), [R1[i] + [t1[i]] for i in range(3)])
    P2 = _mm(_k_matrix(cam2), [R2[i] + [t2[i]] for i in range(3)])
    F = _fundamental(P1, P2)
    if abs(F[2][2]) < 1e-6:
        return None
    normalizer = 1 / F[2][2]
    return [F[i][j] * normalizer for j in range(3) for i in range(3)][:8], dsf


def item_intrinsics(cam1, rot180, mirror_x):   # :1790-1813, in float
    fx, fy, cx, cy = (np.float32(c) for c in (cam1[0], cam1[3], cam1[2], cam1[4]))
    one = np.float32(1)
    if rot180:
        cx, cy = one - cx, one - cy
    if mirror_x:
        cx = one - cx
    return [fx, fy, cx, cy]


class Batch(dict):
    """The outputs keyed by the reader's names; `used` = the indices into `pairs` of the pairs that filled the items."""
    used: np.ndarray


def build_batch(pool, pairs, params, augmentation):
    """One batch of the reader from pool views: `pairs` [(view1, view2), ...] in order, a pair the reader skips
    (|t12| < 1e-6; |F(2,2)| < 1e-6 for FMATRIX) replaced by the next; `params` the reader's parameter dict;
    `augmentation` each item's decisions (draw_augmentation).  Returns float32 CUDA tensors for the keys of top_output:
    IMAGE_PAIR [B,6,h,w], MOTION [B,6|7|8], FLOW [B,2,h,w], DEPTH [B,1|2,h,w], INTRINSICS [B,4], DEPTHMASKS [B,1|2,h,w]."""
    p = reader_params(params)
    for k in ('scaled_width', 'scaled_height'):
        if k in params and int(params[k]) != (pool.width if k == 'scaled_width' else pool.height):
            raise ValueError("%s=%s does not match the pool's %dx%d" % (k, params[k], pool.width, pool.height))
    b = int(p['batch_size'])
    rot = np.asarray(augmentation.rot180, bool).reshape(-1)
    mir = np.asarray(augmentation.mirror_x, bool).reshape(-1)
    colour = augmentation.colour
    if rot.shape != (b,) or mir.shape != (b,):
        raise ValueError("augmentation: rot180 and mirror_x must have batch_size = %d entries" % b)
    if colour is not None:
        colour = np.asarray(colour, np.float32)
        if colour.shape != (b, 6) or not np.all(np.isfinite(colour)) or np.any(np.abs(colour[:, 0]) > MAX_HUE):
            raise ValueError("augmentation: colour must be finite float32 [%d,6] with |hue| <= %g" % (b, MAX_HUE))
    pairs = np.asarray(pairs, np.int64).reshape(-1, 2)
    if pairs.size and (pairs.min() < 0 or pairs.max() >= len(pool)):
        raise ValueError("pairs: view index out of range for a pool of %d views" % len(pool))

    m = MOTION_SIZES[p['motion_format']]
    items = np.zeros(b, _ITEM_DTYPE)
    motion = np.empty((b, m), np.float32)
    intr = np.empty((b, 4), np.float32)
    used = []
    cams = pool.cameras
    k = 0
    for s in range(b):
        res = None
        while res is None:
            if k >= len(pairs):
                raise ValueError("too few usable pairs: %d pairs filled %d of %d items" % (len(pairs), s, b))
            v1, v2 = int(pairs[k, 0]), int(pairs[k, 1])
            res = item_motion(cams[v1], cams[v2], rot[s], mir[s], p)
            k += 1
        used.append(k - 1)
        motion[s] = res[0]
        intr[s] = item_intrinsics(cams[v1], rot[s], mir[s])
        it = items[s]
        it['view1'], it['view2'] = v1, v2
        it['flags'] = int(rot[s]) | (int(mir[s]) << 1)
        it['depth_scale_factor'] = res[1]
        if colour is not None:
            it['aug'] = colour[s]
        it['cam'] = np.stack([cams[v1], cams[v2]]).astype(np.float32)

    # one upload: the item table, then MOTION and INTRINSICS
    off_m = _align(items.nbytes)
    off_i = _align(off_m + motion.nbytes)
    host = np.zeros(off_i + intr.nbytes, np.uint8)
    host[:items.nbytes] = items.view(np.uint8)
    host[off_m:off_m + motion.nbytes] = motion.reshape(-1).view(np.uint8)
    host[off_i:] = intr.reshape(-1).view(np.uint8)
    dev = _device()
    buf = torch.from_numpy(host).to(dev)
    top = p['top_output']
    h, w = pool.height, pool.width
    nd = 2 if p['depth_pair'] else 1
    out = Batch()
    for name, shape in (('IMAGE_PAIR', (b, 6, h, w)), ('FLOW', (b, 2, h, w)), ('DEPTH', (b, nd, h, w)), ('DEPTHMASKS', (b, nd, h, w))):
        if name in top:
            out[name] = torch.empty(shape, dtype=torch.float32, device=dev)
    if 'MOTION' in top:
        out['MOTION'] = buf[off_m:off_m + motion.nbytes].view(torch.float32).view(b, m)
    if 'INTRINSICS' in top:
        out['INTRINSICS'] = buf[off_i:].view(torch.float32).view(b, 4)

    def ptr(name):
        return out[name].data_ptr() if name in out else None
    _lib.check(_lib.load().demon_datareader_batch(
        pool.images.data_ptr(), pool.depths.data_ptr(), h, w, buf.data_ptr(), b, int(colour is not None),
        float(p['image_range_min']), float(p['image_range_max']), float(p['min_depth']), float(p['max_depth']),
        int(bool(p['inverse_depth'])), int(bool(p['depth_pair'])), int(p['depthmask_border1']), int(p['depthmask_border2']),
        ptr('IMAGE_PAIR'), ptr('FLOW'), ptr('DEPTH'), ptr('DEPTHMASKS'), _stream()))
    result = Batch((name, out[name]) for name in top)
    result.used = np.asarray(used, np.int64)
    return result
