"""Reconstruction of a video on the device: the two-view predictions of consecutive frames chained into one scaled
trajectory, and their depth maps fused into a TSDF volume and meshed (csrc/fusion.cu).

    res = reconstruct(pipeline, frames, K)                  # CUDA uint8 [T,H,W,3] frames, K in pixels
    export_sequence_to_ply('out/seq', res)                  # out/seq_mesh.ply, out/seq_cameras.ply
    ch = chain_pairs(out['predict_depth0'], out['predict_rotation'], out['predict_translation'])
    vol = TsdfVolume((256, 256, 256), origin, voxel_size)   # or SparseTsdfVolume(voxel_size): hashed 8^3 blocks, no box
    vol.integrate(ch['depth'], K, ch['R'][:-1], ch['t'][:-1], image)
    vertices, colors, faces = vol.mesh()

DeMoN normalises every pair to |t| = 1 and scales its depth to match, so each pair has its own unknown scale.  Pair k+1
is brought to pair k's scale by the lower median of the depth ratios (dataset_tools.depth_ratios) of frame k+1 as pair k
sees it against frame k+1 as pair k+1 sees it.  There is no loop closure and no bundle adjustment: the drift of the chain
is the drift of the pairs.  There is no CPU fallback.
"""
import ctypes
import math

import numpy as np
import torch

from . import _lib, images, vis
from .dataset_tools import depth_ratios
from .evaluation import intrinsics_vector_to_K, projection_matrix

DEPTH_SHAPE = (192, 256)   # the network's output size, (h, w)


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _device():
    if not torch.cuda.is_available():
        raise RuntimeError("demon_b200.sequence needs a CUDA device (there is no CPU fallback)")
    return torch.device("cuda", torch.cuda.current_device())


def _shape(x):
    return tuple(x.shape) if hasattr(x, "shape") else np.shape(x)


def _cuda(x, dtype):
    if isinstance(x, torch.Tensor):
        t = x if x.is_cuda else x.to(_device())
    else:
        t = torch.from_numpy(np.ascontiguousarray(np.asarray(x))).to(_device())
    return t.to(dtype).contiguous()


def _host64(x):
    return (x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)).astype(np.float64)


def _intrinsics(intrinsics):
    intr = np.asarray(images.NETWORK_INTRINSICS if intrinsics is None else _host64(intrinsics), dtype=np.float64).reshape(-1)
    if intr.shape != (4,) or not np.all(np.isfinite(intr)) or intr[0] <= 0 or intr[1] <= 0:
        raise ValueError("intrinsics: expected finite normalised (fx, fy, cx, cy) with fx, fy > 0, got %s" % (intr.tolist(),))
    return intr


def _check_pairs(inverse_depth, rotation, translation):
    """[P,1,192,256] (or [P,192,256]), [P,3], [P,3] -> P; ValueError before anything touches a device."""
    s = _shape(inverse_depth)
    if len(s) == 4 and s[1] == 1:
        s = (s[0],) + s[2:]
    if len(s) != 3 or s[1:] != DEPTH_SHAPE or s[0] < 1:
        raise ValueError("inverse_depth: expected [P,1,%d,%d] with P >= 1, got %s" % (DEPTH_SHAPE + (_shape(inverse_depth),)))
    p = s[0]
    for name, x in (("rotation", rotation), ("translation", translation)):
        if _shape(x) != (p, 3):
            raise ValueError("%s: expected [%d,3] for %d pairs, got %s" % (name, p, p, _shape(x)))
    return p


def rotation_matrices(rotation):
    """float64 [P,3,3]: vis.angleaxis_to_rotation_matrix (depthmotionnet/helpers.py's Rodrigues) of every float64 angle-axis row."""
    return np.stack([vis.angleaxis_to_rotation_matrix(a) for a in _host64(rotation).reshape(-1, 3)])


def ratio_operands(rotation, translation, intrinsics=None):
    """The depth_ratios operands of the P depth maps of a chain, as float32 CUDA tensors K [P,3,3], R [P,3,3], t [P,3] and P
    [P,3,4]: K = vis.prediction_K for every view, R = I and t = 0 (every depth map is in its own first camera's frame), and
    view k+1 projected by K [R_k | t_k] of pair k's motion (evaluation.projection_matrix; view 0's P is K [I | 0], unused)."""
    intr = _intrinsics(intrinsics)
    h, w = DEPTH_SHAPE
    rm, tr = rotation_matrices(rotation), _host64(translation).reshape(-1, 3)
    n = rm.shape[0]
    K64 = intrinsics_vector_to_K(intr, w, h)
    K = np.broadcast_to(K64.astype(np.float32), (n, 3, 3))
    R = np.broadcast_to(np.eye(3, dtype=np.float32), (n, 3, 3))
    t = np.zeros((n, 3), dtype=np.float32)
    P = np.stack([projection_matrix(K64, np.eye(3), np.zeros(3))] + [projection_matrix(K64, rm[k], tr[k]) for k in range(n - 1)])
    dev = _device()
    return tuple(torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (K, R, t, P))


def pair_ratios(inverse_depth, rotation, translation, intrinsics=None):
    """CUDA float32 [P-1,192,256]: map k holds the depth ratios (dataset_tools.depth_ratios, unchanged) of depth map k
    (1/inverse_depth_k) against depth map k+1 through pair k's motion, NaN where there is none.  Its finite values estimate
    the scale of pair k+1 relative to pair k."""
    p = _check_pairs(inverse_depth, rotation, translation)
    inv = _cuda(inverse_depth, torch.float32).reshape((p,) + DEPTH_SHAPE)
    K, R, t, P = ratio_operands(rotation, translation, intrinsics)
    pairs = np.stack([np.arange(p - 1), np.arange(1, p)], axis=1)
    return depth_ratios(1.0 / inv, K, R, t, P, pairs)


def chain_pairs(inverse_depth, rotation, translation, intrinsics=None, min_ratios=1000):
    """One trajectory from the P pairs (k, k+1), k = 0..P-1, of a video: inverse_depth [P,1,192,256] (predict_depth0),
    rotation and translation [P,3] (angle-axis and translation of frame k+1 relative to frame k, as the pipelines return
    them), intrinsics normalised (fx, fy, cx, cy) (default: images.NETWORK_INTRINSICS, the camera images.adjust_intrinsics
    adapts to).

    Returns a dict:
      scales [P-1] float64   s_k, the lower median of the finite ratios of pair_ratios map k (computed on the device)
      sigma  [P]   float64   the scale of pair k in frame 0's pair's units: sigma_0 = 1, sigma_{k+1} = sigma_k s_k
      R [P+1,3,3], t [P+1,3] float64 world-to-camera poses of frames 0..P with frame 0 as the world:
                             R_{k+1} = R(w_k) R_k, t_{k+1} = R(w_k) t_k + sigma_k t_pair_k
      depth  [P,192,256]     CUDA float32 camera z of frame k in world units, sigma_k / inverse_depth_k
    A pair with fewer than `min_ratios` finite ratios raises ValueError.  The motions come to the host once (they make the
    projections of the ratios), the medians and counts once."""
    p = _check_pairs(inverse_depth, rotation, translation)
    _intrinsics(intrinsics)
    if int(min_ratios) < 1:
        raise ValueError("min_ratios must be at least 1, got %r" % (min_ratios,))
    aa, tr = _host64(rotation), _host64(translation)
    rm = rotation_matrices(aa)
    scales = np.zeros((0,), dtype=np.float64)
    if p > 1:
        r = pair_ratios(inverse_depth, aa, tr, intrinsics).reshape(p - 1, -1)
        finite = torch.isfinite(r)
        med = torch.nanmedian(torch.where(finite, r, torch.full_like(r, float("nan"))), dim=1).values
        host = torch.stack([med.double(), finite.sum(dim=1).double()]).cpu().numpy()
        scales, counts = host[0], host[1].astype(np.int64)
        few = np.flatnonzero(counts < int(min_ratios))
        if few.size:
            k = int(few[0])
            raise ValueError("pairs %d and %d (frames %d..%d) share %d finite depth ratios, fewer than min_ratios = %d: their scales "
                             "cannot be chained" % (k, k + 1, k, k + 2, counts[k], int(min_ratios)))
    sigma = np.cumprod(np.concatenate([[1.0], scales]))
    R = np.empty((p + 1, 3, 3))
    t = np.empty((p + 1, 3))
    R[0], t[0] = np.eye(3), 0.0
    for k in range(p):
        R[k + 1] = rm[k].dot(R[k])
        t[k + 1] = rm[k].dot(t[k]) + sigma[k] * tr[k]
    inv = _cuda(inverse_depth, torch.float32).reshape((p,) + DEPTH_SHAPE)
    sig = torch.from_numpy(sigma.astype(np.float32)).to(inv.device).reshape(p, 1, 1)
    return {"scales": scales, "sigma": sigma, "R": R, "t": t, "depth": sig / inv}


def _grid(origin, voxel_size, trunc):
    """float32 origin [3], voxel_size and trunc (default 3 voxels) of a volume, checked."""
    org = np.asarray(origin, dtype=np.float32).reshape(-1)
    if org.shape != (3,) or not np.all(np.isfinite(org)):
        raise ValueError("origin must be 3 finite numbers, got %r" % (origin,))
    vs = np.float32(voxel_size)
    tr = np.float32(3 * vs if trunc is None else trunc)
    if not (np.isfinite(vs) and vs > 0 and np.isfinite(tr) and tr > 0):
        raise ValueError("voxel_size and trunc must be finite and > 0, got %r and %r" % (voxel_size, trunc))
    return org, vs, tr


def _frames(depth, K, R, t, image, color):
    """The frames of an integrate call as CUDA tensors: depth [n,h,w] float32, K, R [n,3,3], t [n,3] float32 and image
    [n,h,w,3] uint8 or None.  The shapes, and image against `color`, are checked before anything touches a device."""
    s = _shape(depth)
    if len(s) == 4 and s[1] == 1:
        s = (s[0],) + tuple(s[2:])
    if len(s) != 3:
        raise ValueError("depth must be [n,h,w] or [n,1,h,w], got %s" % (_shape(depth),))
    n, h, w = s
    if h * w >= 2 ** 24:
        raise ValueError("depth: %dx%d pixels is too many (h*w must be below 2^24)" % (h, w))
    for name, x, shape in (("K", K, (3, 3)), ("R", R, (3, 3)), ("t", t, (3,))):
        if _shape(x) not in (shape, (n,) + shape):
            raise ValueError("%s has shape %s; want %s or %s" % (name, _shape(x), shape, (n,) + shape))
    if (image is None) == color:
        raise ValueError("image is required with a colour volume and refused without one")
    if image is not None:
        if not vis._is_uint8(image):
            raise ValueError("image must be uint8, got %s" % (image.dtype,))
        if _shape(image) != (n, h, w, 3):
            raise ValueError("image: expected %s, got %s" % ((n, h, w, 3), _shape(image)))
    d = _cuda(depth, torch.float32).reshape(n, h, w)
    im = None if image is None else _cuda(image, torch.uint8)
    return d, vis._per_view(K, n, (3, 3), "K"), vis._per_view(R, n, (3, 3), "R"), vis._per_view(t, n, (3,), "t"), im


class TsdfVolume:
    """A truncated signed distance volume on the device (include/demon_b200.h: demon_tsdf_integrate_f32): dims (nx, ny, nz)
    voxels, voxel (i,j,k) at origin + voxel_size*(i,j,k), truncation `trunc` (default 3 voxels), and a colour average with
    `color`.  `tsdf` and `weight` are CUDA float32 [nz,ny,nx], `color` [nz,ny,nx,3] or None; they start at 0 and belong to
    the caller, so `integrate` can add a long video in chunks."""

    def __init__(self, dims, origin, voxel_size, trunc=None, color=True):
        try:
            nx, ny, nz = (int(d) for d in dims)
        except (TypeError, ValueError):
            raise ValueError("dims must be (nx, ny, nz), got %r" % (dims,))
        if min(nx, ny, nz) < 2 or nx * ny * nz >= 2 ** 31 or 15 * (nx - 1) * (ny - 1) * (nz - 1) >= 2 ** 31:
            raise ValueError("dims %s: at least 2 voxels per axis and a volume the mesh indices fit" % ((nx, ny, nz),))
        org, vs, tr = _grid(origin, voxel_size, trunc)
        self.dims, self.origin, self.voxel_size, self.trunc = (nx, ny, nz), org, vs, tr
        dev = _device()
        self.tsdf = torch.zeros((nz, ny, nx), dtype=torch.float32, device=dev)
        self.weight = torch.zeros((nz, ny, nx), dtype=torch.float32, device=dev)
        self.color = torch.zeros((nz, ny, nx, 3), dtype=torch.float32, device=dev) if color else None

    def _origin(self):
        return (ctypes.c_float * 3)(*(float(v) for v in self.origin))

    def integrate(self, depth, K, R, t, image=None):
        """Adds n frames in order: depth [n,h,w] (or [n,1,h,w]) float32 camera z, K [n,3,3] pixels (or one [3,3]), R [n,3,3]
        and t [n,3] world-to-camera, image [n,h,w,3] uint8 RGB (required with a colour volume, refused without).  Asynchronous
        on the current stream."""
        d, Kd, Rd, td, im = _frames(depth, K, R, t, image, self.color is not None)
        n, h, w = d.shape
        nx, ny, nz = self.dims
        with torch.cuda.device(self.tsdf.device):
            _lib.check(_lib.load().demon_tsdf_integrate_f32(
                self.tsdf.data_ptr(), self.weight.data_ptr(), None if self.color is None else self.color.data_ptr(), nx, ny, nz,
                ctypes.cast(self._origin(), ctypes.c_void_p), float(self.voxel_size), float(self.trunc), d.data_ptr(), Kd.data_ptr(),
                Rd.data_ptr(), td.data_ptr(), None if im is None else im.data_ptr(), n, h, w, _stream()))
        return self

    def mesh(self):
        """The zero surface as a triangle soup (include/demon_b200.h: demon_marching_cubes_f32): CUDA vertices [m,3] float32,
        colors [m,3] uint8 (None without colour) and faces [m/3,3] int32 = 0, 1, 2, ...  Cubes with a corner of weight 0
        are skipped; the order is the cube's linear index, then the table's.  Reads the triangle count back, so it
        synchronises."""
        lib = _lib.load()
        nx, ny, nz = self.dims
        dev = self.tsdf.device
        with torch.cuda.device(dev):
            scratch = torch.empty((lib.demon_marching_cubes_scratch_bytes(nx, ny, nz),), dtype=torch.uint8, device=dev)
            total = torch.empty((1,), dtype=torch.int64, device=dev)
            _lib.check(lib.demon_marching_cubes_count_f32(self.tsdf.data_ptr(), self.weight.data_ptr(), nx, ny, nz, scratch.data_ptr(),
                                                          total.data_ptr(), _stream()))
            tri = int(total.item())
            vertices = torch.empty((3 * tri, 3), dtype=torch.float32, device=dev)
            colors = None if self.color is None else torch.empty((3 * tri, 3), dtype=torch.uint8, device=dev)
            faces = torch.empty((tri, 3), dtype=torch.int32, device=dev)
            if tri:
                _lib.check(lib.demon_marching_cubes_f32(
                    self.tsdf.data_ptr(), self.weight.data_ptr(), None if self.color is None else self.color.data_ptr(), nx, ny, nz,
                    ctypes.cast(self._origin(), ctypes.c_void_p), float(self.voxel_size), scratch.data_ptr(), vertices.data_ptr(),
                    None if colors is None else colors.data_ptr(), faces.data_ptr(), _stream()))
        return vertices, colors, faces


class SparseTsdfVolume:
    """A TSDF volume of 8x8x8 voxel blocks kept in a hash table on the device, allocated where depth is seen
    (include/demon_b200.h: demon_sparse_tsdf_*), so memory and integration work follow the observed surface rather than a
    bounding box.  Voxel g = 8 b + l (block b, |b| < 2^20 per axis) is the point origin + voxel_size * g, with
    TsdfVolume's arithmetic; `trunc` defaults to 3 voxels.

    State, CUDA tensors in allocation order, views of a pool that doubles as it fills (m = the number of blocks):
      blocks [m,3] int32 (bx, by, bz), tsdf and weight [m,8,8,8] float32 (z, y, x; x fastest), color [m,8,8,8,3] float32
      or None.
    `integrate` first allocates, one thread per pixel, every block within 2 voxels of the pixel's band cell (its pixel square
    between camera z d - trunc and d + trunc); a pixel whose cell would span more than DEMON_SPARSE_TSDF_MAX_SPAN (4) blocks
    along an axis, or leaves the key range, allocates nothing and is counted in `last_skipped_pixels`.  The call's new
    blocks are sorted by key and appended, then every block integrates the call's frames exactly as TsdfVolume does.  So a
    block holds the dense integration of every frame from the call that allocated it onward: blocks of the first call equal
    a dense volume's voxels bit for bit, and a block first seen in a later call has missed the free-space updates of the
    earlier calls, as in every voxel-hashing fusion."""

    MAX_SPAN = 4   # DEMON_SPARSE_TSDF_MAX_SPAN
    _POOL_BLOCKS = 64
    _TABLE_SLOTS = 1024

    def __init__(self, voxel_size, origin=(0, 0, 0), trunc=None, color=True):
        self.origin, self.voxel_size, self.trunc = _grid(origin, voxel_size, trunc)
        self._color = bool(color)
        self.last_skipped_pixels = 0
        self._m = 0
        self._pool = None    # blocks, tsdf, weight, color: the device state, made by the first call that needs it
        self._table = None   # keys, values, counters

    def _state(self):
        if self._pool is None:
            dev = _device()
            with torch.cuda.device(dev):
                self._pool = self._new_pool(self._POOL_BLOCKS, dev)
                self._table = self._rehash(self._TABLE_SLOTS, dev)
        return self._pool

    def _new_pool(self, capacity, dev):
        pool = {"blocks": torch.zeros((capacity, 3), dtype=torch.int32, device=dev),
                "tsdf": torch.zeros((capacity, 8, 8, 8), dtype=torch.float32, device=dev),
                "weight": torch.zeros((capacity, 8, 8, 8), dtype=torch.float32, device=dev),
                "color": torch.zeros((capacity, 8, 8, 8, 3), dtype=torch.float32, device=dev) if self._color else None}
        if self._pool is not None:
            for k, v in pool.items():
                if v is not None:
                    v[:self._m] = self._pool[k][:self._m]
        return pool

    def _rehash(self, slots, dev):
        """A table of `slots` slots holding the current table's entries."""
        old = self._table
        keys = torch.empty((slots,), dtype=torch.int64, device=dev)
        values = torch.empty((slots,), dtype=torch.int32, device=dev)
        counters = old[2] if old is not None else torch.empty((4,), dtype=torch.int64, device=dev)
        _lib.check(_lib.load().demon_sparse_tsdf_rehash(
            None if old is None else old[0].data_ptr(), None if old is None else old[1].data_ptr(), 0 if old is None else old[0].numel(),
            keys.data_ptr(), values.data_ptr(), slots, counters.data_ptr(), _stream()))
        return keys, values, counters

    def _view(self, name):
        t = self._state()[name]
        return None if t is None else t[:self._m]

    @property
    def blocks(self):
        return self._view("blocks")

    @property
    def tsdf(self):
        return self._view("tsdf")

    @property
    def weight(self):
        return self._view("weight")

    @property
    def color(self):
        return self._view("color") if self._color else None

    @property
    def capacity(self):
        """Blocks the pool holds before it doubles again."""
        return self._state()["blocks"].shape[0]

    @property
    def table_slots(self):
        self._state()
        return self._table[0].numel()

    @property
    def nbytes(self):
        """Device bytes of the pool and the hash table."""
        tensors = list(self._state().values()) + list(self._table)
        return sum(t.numel() * t.element_size() for t in tensors if t is not None)

    def _origin(self):
        return ctypes.cast((ctypes.c_float * 3)(*(float(v) for v in self.origin)), ctypes.c_void_p)

    def integrate(self, depth, K, R, t, image=None):
        """Adds n frames in order, with TsdfVolume.integrate's arguments: allocates their blocks, then integrates them into
        every block.  Synchronises once, to read the number of new blocks and grow the pool (and once more each time the
        hash table has to double)."""
        d, Kd, Rd, td, im = _frames(depth, K, R, t, image, self._color)
        n, h, w = d.shape
        pool = self._state()
        lib = _lib.load()
        dev = pool["tsdf"].device
        args = (self._origin(), float(self.voxel_size), float(self.trunc), d.data_ptr(), Kd.data_ptr(), Rd.data_ptr(), td.data_ptr())
        with torch.cuda.device(dev):
            while True:
                keys, values, counters = self._table
                _lib.check(lib.demon_sparse_tsdf_allocate_f32(keys.data_ptr(), values.data_ptr(), keys.numel(), counters.data_ptr(),
                                                              *args, n, h, w, _stream()))
                occupied, overflow, skipped = counters[:3].tolist()
                if not overflow:
                    break
                self._table = self._rehash(2 * keys.numel(), dev)
            new = occupied - self._m
            if new:
                fresh = torch.empty((new,), dtype=torch.int64, device=dev)
                _lib.check(lib.demon_sparse_tsdf_gather_new(keys.data_ptr(), values.data_ptr(), keys.numel(), counters.data_ptr(),
                                                            fresh.data_ptr(), _stream()))
                fresh = torch.sort(fresh).values
                cap = pool["blocks"].shape[0]
                if self._m + new > cap:
                    while cap < self._m + new:
                        cap *= 2
                    pool = self._pool = self._new_pool(cap, dev)
                _lib.check(lib.demon_sparse_tsdf_commit(keys.data_ptr(), values.data_ptr(), keys.numel(), fresh.data_ptr(), new, self._m,
                                                        pool["blocks"].data_ptr(), _stream()))
                self._m += new
            self.last_skipped_pixels = skipped
            _lib.check(lib.demon_sparse_tsdf_integrate_f32(
                pool["tsdf"].data_ptr(), pool["weight"].data_ptr(), None if pool["color"] is None else pool["color"].data_ptr(),
                pool["blocks"].data_ptr(), self._m, *args, None if im is None else im.data_ptr(), n, h, w, _stream()))
        return self

    def mesh(self):
        """TsdfVolume.mesh on the blocks: a cube is skipped when a corner lies in a block that is not allocated or has weight
        0; the order is the block's pool index, the cube's local linear index (x fastest), then the table's.  Faces are
        int32, so a mesh of 2^31 vertices or more raises ValueError.  Reads the triangle count back, so it synchronises."""
        pool = self._state()
        lib = _lib.load()
        dev, m = pool["tsdf"].device, self._m
        with torch.cuda.device(dev):
            tri = 0
            if m:
                keys, values, _ = self._table
                scratch = torch.empty((lib.demon_sparse_tsdf_mesh_scratch_bytes(m),), dtype=torch.uint8, device=dev)
                total = torch.empty((1,), dtype=torch.int64, device=dev)
                _lib.check(lib.demon_sparse_tsdf_mesh_count_f32(pool["tsdf"].data_ptr(), pool["weight"].data_ptr(), pool["blocks"].data_ptr(),
                                                                m, keys.data_ptr(), values.data_ptr(), keys.numel(), scratch.data_ptr(),
                                                                total.data_ptr(), _stream()))
                tri = int(total.item())
                if 3 * tri >= 2 ** 31:
                    raise ValueError("the mesh has %d triangles: its int32 faces cannot index 3x that many vertices" % tri)
            vertices = torch.empty((3 * tri, 3), dtype=torch.float32, device=dev)
            colors = None if pool["color"] is None else torch.empty((3 * tri, 3), dtype=torch.uint8, device=dev)
            faces = torch.empty((tri, 3), dtype=torch.int32, device=dev)
            if tri:
                _lib.check(lib.demon_sparse_tsdf_mesh_f32(
                    pool["tsdf"].data_ptr(), pool["weight"].data_ptr(), None if colors is None else pool["color"].data_ptr(),
                    pool["blocks"].data_ptr(), m, self._origin(), float(self.voxel_size), scratch.data_ptr(), vertices.data_ptr(),
                    None if colors is None else colors.data_ptr(), faces.data_ptr(), _stream()))
        return vertices, colors, faces


def volume_from_points(points, dims=(256, 256, 256), low=5.0, high=95.0, color=True):
    """A TsdfVolume of at most `dims` voxels with cubic voxels around the `low`..`high` percentile box of points [m,3]
    (CUDA float32), each axis's percentiles taken on its own (torch.kthvalue, so any m works)."""
    m = points.shape[0]
    if m < 1:
        raise ValueError("no points to bound the volume with")

    def pct(q):
        return torch.kthvalue(points, 1 + int(round(q / 100.0 * (m - 1))), dim=0).values
    box = torch.stack([pct(low), pct(high)]).double().cpu().numpy()
    lo, ext = box[0], np.maximum(box[1] - box[0], 1e-6)
    vs = float(np.max(ext / (np.asarray(dims, dtype=np.float64) - 1)))
    n = [max(2, min(int(d), int(math.ceil(e / vs)) + 1)) for d, e in zip(dims, ext)]
    return TsdfVolume(n, lo, vs, color=color)


def reconstruct(pipeline, frames, intrinsics, volume=None, resample="bicubic", min_ratios=1000):
    """A video end to end: frames CUDA uint8 [T,H,W,3] (T >= 2, HWC RGB) with their intrinsics in pixels ([3,3], [T,3,3] or
    [T,4], as images.adjust_intrinsics takes them).  Every frame is adapted once to DeMoN's camera at 256x192
    (images.adjust_intrinsics), and its 64x48 image2_2 resized from the adapted frame with `resample`, as forward_views makes
    it.  The pairs (k, k+1) run through pipeline.forward_u8 (DemonPipeline or DemonPipelineV2) batch_size at a time; a
    partial last batch repeats its last pair, whose outputs are dropped.  The pairs are chained (chain_pairs) and the P
    depth maps integrated, coloured by adapted frame k, into `volume` (a TsdfVolume or a SparseTsdfVolume, which is added to)
    or, by default, a new 256^3 TsdfVolume around the 5th..95th percentiles of the chained points.

    Returns a dict: chain_pairs' scales, sigma, R, t and depth, inverse_depth / rotation / translation [P,...] of the pairs,
    the adapted frames [T,192,256,3] and their status (images.adjust_intrinsics), K [3,3] of the adapted frames in pixels,
    volume, and the mesh: vertices, colors, faces."""
    if not (isinstance(frames, torch.Tensor) and frames.dim() == 4 and frames.shape[0] >= 2):
        raise ValueError("frames: expected a CUDA uint8 tensor [T,H,W,3] with T >= 2, got %s" % (_shape(frames),))
    if volume is not None and not isinstance(volume, (TsdfVolume, SparseTsdfVolume)):
        raise ValueError("volume must be a TsdfVolume, a SparseTsdfVolume or None")
    adapted, K_new, status = images.adjust_intrinsics(frames, intrinsics)
    small = images.resize(adapted, (64, 48), resample)
    T, b = frames.shape[0], pipeline.batch_size
    p = T - 1
    h, w = DEPTH_SHAPE
    dev = adapted.device
    inv = torch.empty((p, 1, h, w), dtype=torch.float32, device=dev)
    rot = torch.empty((p, 3), dtype=torch.float32, device=dev)
    trans = torch.empty((p, 3), dtype=torch.float32, device=dev)
    for s in range(0, p, b):
        m = min(b, p - s)
        idx = torch.arange(s, s + b, device=dev).clamp_(max=s + m - 1)
        out = pipeline.forward_u8(torch.stack((adapted[idx], adapted[idx + 1]), dim=1), small[idx + 1])
        inv[s:s + m] = out["predict_depth0"][:m]
        rot[s:s + m] = out["predict_rotation"][:m]
        trans[s:s + m] = out["predict_translation"][:m]
    ch = chain_pairs(inv, rot, trans, None, min_ratios)   # adjust_intrinsics adapts to the default intrinsics
    K = torch.from_numpy(vis.prediction_K(images.NETWORK_INTRINSICS, 1, h, w)[0]).to(dev)
    R32 = torch.from_numpy(ch["R"][:p].astype(np.float32)).to(dev)
    t32 = torch.from_numpy(ch["t"][:p].astype(np.float32)).to(dev)
    if volume is None:
        pc = vis.point_clouds(ch["depth"], K, R32, t32)
        valid = torch.arange(h * w, device=dev)[None, :] < pc["counts"][:, None].long()
        volume = volume_from_points(pc["points"][valid])
    volume.integrate(ch["depth"], K, R32, t32, adapted[:p] if volume.color is not None else None)
    vertices, colors, faces = volume.mesh()
    return dict(ch, inverse_depth=inv, rotation=rot, translation=trans, adapted=adapted, status=status, K=K_new, volume=volume,
                vertices=vertices, colors=colors, faces=faces)


def export_sequence_to_ply(prefix, result):
    """Writes prefix + '_mesh.ply' (the coloured mesh of `result`) and prefix + '_cameras.ply' (vis.camera_mesh of every
    pose of result['R'] / result['t'], one mesh), in vis.write_ply's format."""
    col = result.get("colors")
    vis.write_ply(prefix + "_mesh.ply", result["vertices"].cpu().numpy(), None if col is None else col.cpu().numpy(),
                  result["faces"].cpu().numpy())
    verts, faces = [], []
    for k, (R, t) in enumerate(zip(result["R"], result["t"])):
        v, f = vis.camera_mesh(R, t)
        verts.append(v)
        faces.append(f + k * v.shape[0])
    vis.write_ply(prefix + "_cameras.ply", np.concatenate(verts), faces=np.concatenate(faces))
