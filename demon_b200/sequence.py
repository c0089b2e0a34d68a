"""Reconstruction of a video on the device: the two-view predictions of consecutive frames chained into one scaled
trajectory, and their depth maps fused into a TSDF volume and meshed (csrc/fusion.cu).

    res = reconstruct(pipeline, frames, K)                  # CUDA uint8 [T,H,W,3] frames, K in pixels
    export_sequence_to_ply('out/seq', res)                  # out/seq_mesh.ply, out/seq_cameras.ply
    ch = chain_pairs(out['predict_depth0'], out['predict_rotation'], out['predict_translation'])
    vol = TsdfVolume((256, 256, 256), origin, voxel_size)   # or SparseTsdfVolume(voxel_size): hashed 8^3 blocks, no box
    vol.integrate(ch['depth'], K, ch['R'][:-1], ch['t'][:-1], image)
    vertices, colors, faces = vol.mesh()

The fused volume renders back to images (ray casting, csrc/fusion.cu): fused depth, normals and colour for every input
frame at its own chained pose, or from any other camera.

    K = vis.prediction_K(images.NETWORK_INTRINSICS, 1, 192, 256)[0]
    img = res['volume'].raycast(K, res['R'][:-1], res['t'][:-1])   # img['depth'] [P,192,256]: fused depth of frames 0..P-1

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


def _per_frame(x, n, name):
    """float32 [n] from one number or n of them, all finite."""
    v = np.asarray(_host64(x), dtype=np.float32).reshape(-1)
    if v.size == 1:
        v = np.repeat(v, n)
    if v.shape != (n,) or not np.all(np.isfinite(v)):
        raise ValueError("%s: expected one finite number or %d of them, got %r" % (name, n, x))
    return v


class _Render:
    """The checked arguments of a raycast call: the frame count n from R (or t, or K), the image size, step, and near and
    far [n] float32 (far None for the volume's default).  Everything is checked before anything touches a device."""

    def __init__(self, K, R, t, height, width, near, far, step):
        try:
            self.h, self.w = int(height), int(width)
        except (TypeError, ValueError):
            raise ValueError("height and width must be integers, got %r and %r" % (height, width))
        if self.h < 1 or self.w < 1 or self.h * self.w >= 2 ** 24:
            raise ValueError("image size %dx%d: at least 1x1 and fewer than 2^24 pixels" % (self.h, self.w))
        self.step = np.float32(step)
        if not (np.isfinite(self.step) and 0 < self.step <= 1):
            raise ValueError("step must be finite and in (0, 1] voxels, got %r" % (step,))
        sK, sR, st = _shape(K), _shape(R), _shape(t)
        self.n = sR[0] if len(sR) == 3 else st[0] if len(st) == 2 else sK[0] if len(sK) == 3 else 1
        for name, x, shape in (("K", K, (3, 3)), ("R", R, (3, 3)), ("t", t, (3,))):
            if _shape(x) not in (shape, (self.n,) + shape):
                raise ValueError("%s has shape %s; want %s or %s" % (name, _shape(x), shape, (self.n,) + shape))
        self.near = _per_frame(near, self.n, "near")
        if (self.near < 0).any():
            raise ValueError("near must be >= 0, got %r" % (near,))
        self.far = None if far is None else _per_frame(far, self.n, "far")
        self.K, self.R, self.t = K, R, t

    def cameras(self):
        """CUDA float32 K, R [n,3,3] and t [n,3]."""
        n = self.n
        return vis._per_view(self.K, n, (3, 3), "K"), vis._per_view(self.R, n, (3, 3), "R"), vis._per_view(self.t, n, (3,), "t")

    def outputs(self, color, dev):
        """The all-miss result: depth and normals NaN, colours 0."""
        n, h, w = self.n, self.h, self.w
        return {"depth": torch.full((n, h, w), float("nan"), dtype=torch.float32, device=dev),
                "normals": torch.full((n, 3, h, w), float("nan"), dtype=torch.float32, device=dev),
                "colors": torch.zeros((n, h, w, 3), dtype=torch.uint8, device=dev) if color else None}

    def limits(self, dev, far):
        """near and far as CUDA float32 [n]; far(R, t) gives the default."""
        nr = torch.from_numpy(self.near).to(dev)
        return nr, far if self.far is None else torch.from_numpy(self.far).to(dev)


def _far_of_corners(X, Rd, td):
    """CUDA float32 [n]: the largest camera z ((R_20 X_0 + R_21 X_1) + R_22 X_2) + t_2 of the float32 points X [c,3]."""
    X = torch.from_numpy(np.ascontiguousarray(X, dtype=np.float32)).to(Rd.device)
    z = ((Rd[:, 2, 0:1] * X[None, :, 0] + Rd[:, 2, 1:2] * X[None, :, 1]) + Rd[:, 2, 2:3] * X[None, :, 2]) + td[:, 2:3]
    return z.amax(dim=1)


def _check_normals(normals):
    if not isinstance(normals, (bool, np.bool_)):
        raise ValueError("normals must be True or False, got %r" % (normals,))


def _ptr(t):
    return None if t is None else t.data_ptr()


def _indexed_outputs(nv, tri, normals, color, dev):
    """The empty CUDA outputs of an indexed mesh of nv vertices and tri triangles; ValueError past int32 indices."""
    if nv >= 2 ** 31:
        raise ValueError("the mesh has %d vertices: its int32 faces cannot index them" % nv)
    return {"vertices": torch.empty((nv, 3), dtype=torch.float32, device=dev),
            "normals": torch.empty((nv, 3), dtype=torch.float32, device=dev) if normals else None,
            "colors": torch.empty((nv, 3), dtype=torch.uint8, device=dev) if color else None,
            "faces": torch.empty((tri, 3), dtype=torch.int32, device=dev)}


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

    def indexed_mesh(self, normals=True):
        """The zero surface as an indexed mesh (include/demon_b200.h: demon_tsdf_indexed_mesh_f32): one vertex per edge
        that a meshed cube's triangles use, in ascending 3 (linear voxel index) + axis, at the soup's position and colour
        bit for bit; faces are mesh()'s triangles in its order, each corner the index of its edge's vertex, so
        vertices[faces] is mesh()'s vertices.  Returns a dict of CUDA tensors: vertices [V,3] float32, normals [V,3] float32
        (unit, towards free space; NaN where a voxel the central differences read is not stored; None with
        normals=False), colors [V,3] uint8 (None without colour), faces [T,3] int32.  Reads the counts back, so it
        synchronises."""
        _check_normals(normals)
        lib = _lib.load()
        nx, ny, nz = self.dims
        dev = self.tsdf.device
        with torch.cuda.device(dev):
            scratch = torch.empty((lib.demon_tsdf_indexed_mesh_scratch_bytes(nx, ny, nz),), dtype=torch.uint8, device=dev)
            counts = torch.empty((2,), dtype=torch.int64, device=dev)
            _lib.check(lib.demon_tsdf_indexed_mesh_count_f32(self.tsdf.data_ptr(), self.weight.data_ptr(), nx, ny, nz, scratch.data_ptr(),
                                                             counts.data_ptr(), _stream()))
            nv, tri = counts.tolist()
            out = _indexed_outputs(nv, tri, normals, self.color is not None, dev)
            if nv:
                _lib.check(lib.demon_tsdf_indexed_mesh_f32(
                    self.tsdf.data_ptr(), self.weight.data_ptr(), None if self.color is None else self.color.data_ptr(), nx, ny, nz,
                    ctypes.cast(self._origin(), ctypes.c_void_p), float(self.voxel_size), scratch.data_ptr(), out["vertices"].data_ptr(),
                    _ptr(out["normals"]), _ptr(out["colors"]), out["faces"].data_ptr(), _stream()))
        return out

    def default_far(self, R, t):
        """CUDA float32 [n]: raycast's default far, the largest camera z of the box's 8 corners for each world-to-camera
        R [n,3,3] (CUDA float32) and t [n,3]."""
        corners = [self.origin[a] + self.voxel_size * np.float32(self.dims[a] - 1) for a in range(3)]
        X = [[self.origin[a] if (q >> a) & 1 == 0 else corners[a] for a in range(3)] for q in range(8)]
        return _far_of_corners(np.array(X, dtype=np.float32), R, t)

    def raycast(self, K, R, t, height=192, width=256, near=0.0, far=None, step=0.5):
        """Renders the volume's surface from n cameras (include/demon_b200.h: demon_tsdf_raycast_f32, which states the rule):
        K [n,3,3] pixels (or one [3,3]), R [n,3,3] and t [n,3] world-to-camera, as integrate takes them; an image of
        height x width.  Each pixel's ray is sampled every `step` voxels (0 < step <= 1) in camera z from `near` (default 0,
        >= 0) to `far` (default: the largest camera z of the box's corners), one number or one per frame; the first crossing
        of the trilinear tsdf from >= 0 to < 0 between valid samples is the hit.

        Returns a dict of CUDA tensors: depth [n,h,w] float32 camera z (NaN: no hit), normals [n,3,h,w] float32 unit
        normals in the camera frame, towards the camera on a visible surface (NaN where not all 6 neighbours are valid),
        colors [n,h,w,3] uint8 (None without colour; 0 where not valid).  Asynchronous on the current stream."""
        rq = _Render(K, R, t, height, width, near, far, step)
        dev = self.tsdf.device
        with torch.cuda.device(dev):
            out = rq.outputs(self.color is not None, dev)
            if rq.n == 0:
                return out
            Kd, Rd, td = rq.cameras()
            nr, fr = rq.limits(dev, None if rq.far is not None else self.default_far(Rd, td))
            nx, ny, nz = self.dims
            _lib.check(_lib.load().demon_tsdf_raycast_f32(
                self.tsdf.data_ptr(), self.weight.data_ptr(), None if self.color is None else self.color.data_ptr(), nx, ny, nz,
                ctypes.cast(self._origin(), ctypes.c_void_p), float(self.voxel_size), Kd.data_ptr(), Rd.data_ptr(), td.data_ptr(),
                nr.data_ptr(), fr.data_ptr(), float(rq.step), rq.n, rq.h, rq.w, out["depth"].data_ptr(), out["normals"].data_ptr(),
                None if out["colors"] is None else out["colors"].data_ptr(), _stream()))
        return out


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
    earlier calls, as in every voxel-hashing fusion.

    With `max_device_blocks` (an integer >= 1; default None: every block stays on the device), the blocks beyond that many
    stream to pinned host memory after each integrate and raycast call, least recently reached first (ties by ascending
    packed key, z then y then x), and every host block a call's cameras reach (include/demon_b200.h:
    demon_sparse_tsdf_reach_f32) comes back before the call does any work, appended in key order.  A call that reaches
    more blocks than the budget keeps them all until it ends (`peak_device_blocks`).  The table still indexes every block
    and the host blocks' coordinates stay on the device, so the union of device and host blocks equals an unbudgeted
    volume fed the same calls, voxel for voxel, and raycast and mesh return what it returns.  `blocks`, `tsdf`, `weight`,
    `color`, `capacity` and `nbytes` describe the device; `host`, `host_nbytes`, `last_blocks_in` and `last_blocks_out`
    the rest.  A long video is fused in bounded device memory by calling integrate once per chunk of frames."""

    MAX_SPAN = 4   # DEMON_SPARSE_TSDF_MAX_SPAN
    _POOL_BLOCKS = 64
    _TABLE_SLOTS = 1024

    def __init__(self, voxel_size, origin=(0, 0, 0), trunc=None, color=True, max_device_blocks=None):
        self.origin, self.voxel_size, self.trunc = _grid(origin, voxel_size, trunc)
        if max_device_blocks is not None and (isinstance(max_device_blocks, bool) or not isinstance(max_device_blocks, (int, np.integer))
                                              or max_device_blocks < 1):
            raise ValueError("max_device_blocks must be an integer >= 1 or None, got %r" % (max_device_blocks,))
        self.max_device_blocks = None if max_device_blocks is None else int(max_device_blocks)
        self._color = bool(color)
        self.last_skipped_pixels = 0
        self._m = 0
        self._pool = None    # blocks, tsdf, weight, color (and stamp with a budget): the device state, made by the first call
        self._table = None   # keys, values, counters
        # with a budget: the host store (pinned tsdf, weight, color; device blocks, stamp, live), its slots in use
        # [0, _hend) and the free ones among them (ascending), and the index of the last integrate or raycast call
        self._host, self._hend, self._free, self._calls = None, 0, [], 0
        self.last_blocks_in = self.last_blocks_out = self.peak_device_blocks = 0

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
        if self.max_device_blocks is not None:
            pool["stamp"] = torch.zeros((capacity,), dtype=torch.int32, device=dev)   # the last call that reached the block
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

    @property
    def host(self):
        """The blocks on the host in slot order, as CPU tensors: blocks [h,3] int32, tsdf and weight [h,8,8,8], color
        [h,8,8,8,3] or None.  Synchronises (the transfers are asynchronous)."""
        if self._host is None:
            return {"blocks": torch.zeros((0, 3), dtype=torch.int32), "tsdf": torch.zeros((0, 8, 8, 8)), "weight": torch.zeros((0, 8, 8, 8)),
                    "color": torch.zeros((0, 8, 8, 8, 3)) if self._color else None}
        hs = self._host
        torch.cuda.current_stream(hs["blocks"].device).synchronize()
        live = torch.nonzero(hs["live"][:self._hend]).reshape(-1)
        idx = live.cpu()
        return {"blocks": hs["blocks"][live].cpu(), "tsdf": hs["tsdf"][idx], "weight": hs["weight"][idx],
                "color": None if hs["color"] is None else hs["color"][idx]}

    @property
    def host_nbytes(self):
        """Bytes of the pinned host store (it doubles as it fills; slots freed by returning blocks are reused)."""
        if self._host is None:
            return 0
        return sum(self._host[k].numel() * self._host[k].element_size() for k in ("tsdf", "weight", "color") if self._host[k] is not None)

    def _host_blocks(self):
        return self._hend - len(self._free)

    def _grow_host(self, slots, dev):
        """Makes the host store hold `slots` slots: the smallest doubling of its capacity that does."""
        old = self._host
        cap = 0 if old is None else old["tsdf"].shape[0]
        if slots <= cap:
            return
        new = max(cap, 1)
        while new < slots:
            new *= 2
        store = {"tsdf": torch.empty((new, 8, 8, 8), dtype=torch.float32, pin_memory=True),
                 "weight": torch.empty((new, 8, 8, 8), dtype=torch.float32, pin_memory=True),
                 "color": torch.empty((new, 8, 8, 8, 3), dtype=torch.float32, pin_memory=True) if self._color else None,
                 "blocks": torch.zeros((new, 3), dtype=torch.int32, device=dev), "stamp": torch.zeros((new,), dtype=torch.int32, device=dev),
                 "live": torch.zeros((new,), dtype=torch.bool, device=dev)}
        if old is not None:
            torch.cuda.current_stream(dev).synchronize()   # the device has written the old store
            for k, v in store.items():
                if v is not None:
                    v[:cap] = old[k]
        self._host = store

    def _reach(self, blocks, m, trunc, tiles, cams, n, h, w, out, mark):
        Kd, Rd, td = cams
        _lib.check(_lib.load().demon_sparse_tsdf_reach_f32(blocks.data_ptr(), m, self._origin(), float(self.voxel_size), float(trunc),
                                                            tiles.data_ptr(), Kd.data_ptr(), Rd.data_ptr(), td.data_ptr(), n, h, w,
                                                            out.data_ptr(), mark, _stream()))

    def _bring_back(self, tiles, trunc, cams, n, h, w):
        """A new call: stamps the device blocks its cameras reach and brings back the host blocks they reach, in key order."""
        self._calls += 1
        pool, dev = self._pool, self._pool["tsdf"].device
        self._reach(pool["blocks"], self._m, trunc, tiles, cams, n, h, w, pool["stamp"], self._calls)
        r = 0
        if self._host_blocks():
            hs = self._host
            flags = torch.zeros((self._hend,), dtype=torch.int32, device=dev)
            self._reach(hs["blocks"], self._hend, trunc, tiles, cams, n, h, w, flags, 1)
            slots = torch.nonzero((flags > 0) & hs["live"][:self._hend]).reshape(-1)
            r = slots.numel()
            if r:
                slots = slots[torch.argsort(_packed_keys(hs["blocks"][slots]))]
                src = slots.to(torch.int32)   # named: a pointer's tensor must outlive the call
                cap = pool["blocks"].shape[0]
                if self._m + r > cap:
                    while cap < self._m + r:
                        cap *= 2
                    pool = self._pool = self._new_pool(cap, dev)
                keys, values, _ = self._table
                dst = torch.arange(self._m, self._m + r, dtype=torch.int32, device=dev)
                _lib.check(_lib.load().demon_sparse_tsdf_restore(
                    hs["tsdf"].data_ptr(), hs["weight"].data_ptr(), None if hs["color"] is None else hs["color"].data_ptr(),
                    hs["blocks"].data_ptr(), src.data_ptr(), dst.data_ptr(), r, pool["tsdf"].data_ptr(),
                    pool["weight"].data_ptr(), None if pool["color"] is None else pool["color"].data_ptr(), pool["blocks"].data_ptr(),
                    pool["stamp"].data_ptr(), self._calls, keys.data_ptr(), values.data_ptr(), keys.numel(), _stream()))
                hs["live"][slots] = False
                self._free = sorted(self._free + slots.tolist())
                while self._free and self._free[-1] == self._hend - 1:
                    self._free.pop()
                    self._hend -= 1
                self._m += r
        self.last_blocks_in = r

    def _stream_out(self):
        """The end of a call: moves the device blocks beyond the budget to the host, least recently reached first (ties
        by key), and compacts the pool in order."""
        pool, m, dev = self._pool, self._m, self._pool["tsdf"].device
        self.peak_device_blocks = max(self.peak_device_blocks, m)
        e = m - self.max_device_blocks
        self.last_blocks_out = max(e, 0)
        if e <= 0:
            return
        order = torch.argsort(_packed_keys(pool["blocks"][:m]))
        order = order[torch.sort(pool["stamp"][:m][order], stable=True).indices]
        out = order[:e]
        src = out.to(torch.int32)
        reuse = min(e, len(self._free))
        slots = self._free[:reuse] + list(range(self._hend, self._hend + e - reuse))
        self._free = self._free[reuse:]
        self._hend += e - reuse
        self._grow_host(self._hend, dev)
        hs = self._host
        slots = torch.tensor(slots, dtype=torch.int32, device=dev)
        keys, values, _ = self._table
        _lib.check(_lib.load().demon_sparse_tsdf_evict(
            pool["tsdf"].data_ptr(), pool["weight"].data_ptr(), None if pool["color"] is None else pool["color"].data_ptr(),
            pool["blocks"].data_ptr(), pool["stamp"].data_ptr(), keys.data_ptr(), values.data_ptr(), keys.numel(),
            src.data_ptr(), slots.data_ptr(), e, hs["tsdf"].data_ptr(), hs["weight"].data_ptr(),
            None if hs["color"] is None else hs["color"].data_ptr(), hs["blocks"].data_ptr(), hs["stamp"].data_ptr(), _stream()))
        hs["live"][slots.long()] = True
        keep = torch.ones((m,), dtype=torch.bool, device=dev)
        keep[out] = False
        first = int(out.min())   # blocks before it keep their index
        tail = torch.nonzero(keep[first:]).reshape(-1) + first
        for v in pool.values():
            if v is not None:
                v[first:m - e] = v[tail]
                v[m - e:m] = 0   # new blocks are committed onto zeroed slots
        self._m = m - e
        _lib.check(_lib.load().demon_sparse_tsdf_index(keys.data_ptr(), values.data_ptr(), keys.numel(), pool["blocks"].data_ptr(), first,
                                                       self._m - first, _stream()))

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
            if self.max_device_blocks is not None:
                tiles = torch.empty((n, -(-h // 8), -(-w // 8)), dtype=torch.float32, device=dev)
                _lib.check(lib.demon_sparse_tsdf_depth_tiles_f32(d.data_ptr(), n, h, w, tiles.data_ptr(), _stream()))
                self._bring_back(tiles, self.trunc, (Kd, Rd, td), n, h, w)
                pool = self._pool
            while True:
                keys, values, counters = self._table
                _lib.check(lib.demon_sparse_tsdf_allocate_f32(keys.data_ptr(), values.data_ptr(), keys.numel(), counters.data_ptr(),
                                                              *args, n, h, w, _stream()))
                occupied, overflow, skipped = counters[:3].tolist()
                if not overflow:
                    break
                self._table = self._rehash(2 * keys.numel(), dev)
            new = occupied - self._m - self._host_blocks()   # the table also holds the blocks on the host
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
                if self.max_device_blocks is not None:
                    pool["stamp"][self._m:self._m + new] = self._calls
                self._m += new
            self.last_skipped_pixels = skipped
            _lib.check(lib.demon_sparse_tsdf_integrate_f32(
                pool["tsdf"].data_ptr(), pool["weight"].data_ptr(), None if pool["color"] is None else pool["color"].data_ptr(),
                pool["blocks"].data_ptr(), self._m, *args, None if im is None else im.data_ptr(), n, h, w, _stream()))
            if self.max_device_blocks is not None:
                self._stream_out()
        return self

    def mesh(self):
        """TsdfVolume.mesh on the blocks: a cube is skipped when a corner lies in a block that is not allocated or has weight
        0; the order is the block's pool index, the cube's local linear index (x fastest), then the table's.  Faces are
        int32, so a mesh of 2^31 vertices or more raises ValueError.  Reads the triangle count back, so it synchronises.

        With blocks on the host, every block is meshed: all blocks in ascending key order, max_device_blocks at a time, each
        chunk copied with the neighbours its cubes need into a scratch pool on the device; the result is the chunk meshes
        concatenated, faces offset.  The volume's state does not change."""
        if self._host_blocks():
            return self._mesh_chunks()
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

    def _blocks_by_key(self):
        """Every block, on the device or the host, in ascending key order: packed keys [B] int64, coordinates [B,3] and
        where each is (its pool index, or -2 - host slot, as the table has it)."""
        pool, hs, m = self._pool, self._host, self._m
        dev = pool["tsdf"].device
        slots = torch.nonzero(hs["live"][:self._hend]).reshape(-1)
        coords = torch.cat([pool["blocks"][:m], hs["blocks"][slots]])
        where = torch.cat([torch.arange(m, device=dev), -2 - slots])
        keys = _packed_keys(coords)
        order = torch.argsort(keys)
        return keys[order], coords[order], where[order]

    @staticmethod
    def _chunk_selection(keys, coords, c0, c1, steps):
        """The key ranks of blocks c0 .. c1-1 of the key-ordered blocks, then those of their neighbours at `steps` that
        exist outside the chunk, ascending."""
        dev, total = keys.device, keys.numel()
        nk = []
        for step in steps:
            st = torch.tensor(step, dtype=torch.int32, device=dev)
            ok = ((coords[c0:c1] + st) <= _MAX_COORD).all(dim=1) & ((coords[c0:c1] + st) >= -_MAX_COORD).all(dim=1)
            nk.append(keys[c0:c1][ok] + (step[0] + (step[1] << 21) + (step[2] << 42)))
        nk = torch.unique(torch.cat(nk))
        pos = torch.searchsorted(keys, nk).clamp_(max=total - 1)
        pos = pos[(keys[pos] == nk) & ((pos < c0) | (pos >= c1))]
        return torch.cat([torch.arange(c0, c1, device=dev), pos])

    def _mesh_chunks(self):
        dev = self._pool["tsdf"].device
        out = ([], [], [])
        with torch.cuda.device(dev):
            keys, coords, where = self._blocks_by_key()
            total, vertices = keys.numel(), 0
            for c0 in range(0, total, self.max_device_blocks):
                c1 = min(total, c0 + self.max_device_blocks)
                sel = self._chunk_selection(keys, coords, c0, c1, _PLUS_STEPS)   # the neighbours the chunk's cubes read
                chunk = self._chunk_pool(coords[sel].contiguous(), where[sel])
                v, c, f = self._mesh_range(chunk, c1 - c0)
                if vertices + v.shape[0] >= 2 ** 31:
                    raise ValueError("the mesh has %d or more vertices: its int32 faces cannot index them" % (vertices + v.shape[0]))
                out[0].append(v)
                out[1].append(c)
                out[2].append(f + vertices)
                vertices += v.shape[0]
        return torch.cat(out[0]), torch.cat(out[1]) if self._color else None, torch.cat(out[2])

    def _chunk_pool(self, blocks, where):
        """A scratch pool of the blocks [t,3] (where: their pool index or -2 - host slot) with its own table."""
        pool, hs, lib = self._pool, self._host, _lib.load()
        dev, t = blocks.device, blocks.shape[0]
        chunk = {"blocks": blocks, "tsdf": torch.empty((t, 8, 8, 8), dtype=torch.float32, device=dev),
                 "weight": torch.empty((t, 8, 8, 8), dtype=torch.float32, device=dev),
                 "color": torch.empty((t, 8, 8, 8, 3), dtype=torch.float32, device=dev) if self._color else None}
        on = torch.nonzero(where >= 0).reshape(-1)
        for k in ("tsdf", "weight", "color"):
            if chunk[k] is not None:
                chunk[k][on] = pool[k][where[on]]
        off = torch.nonzero(where < 0).reshape(-1)
        if off.numel():
            src, dst = (-2 - where[off]).to(torch.int32), off.to(torch.int32)
            _lib.check(lib.demon_sparse_tsdf_restore(
                hs["tsdf"].data_ptr(), hs["weight"].data_ptr(), None if hs["color"] is None else hs["color"].data_ptr(), hs["blocks"].data_ptr(),
                src.data_ptr(), dst.data_ptr(), off.numel(), chunk["tsdf"].data_ptr(),
                chunk["weight"].data_ptr(), None if chunk["color"] is None else chunk["color"].data_ptr(), blocks.data_ptr(), None, 0, None,
                None, 0, _stream()))
        slots = 1024
        while slots < 2 * t:
            slots *= 2
        keys = torch.empty((slots,), dtype=torch.int64, device=dev)
        values = torch.empty((slots,), dtype=torch.int32, device=dev)
        counters = torch.empty((4,), dtype=torch.int64, device=dev)
        _lib.check(lib.demon_sparse_tsdf_rehash(None, None, 0, keys.data_ptr(), values.data_ptr(), slots, counters.data_ptr(), _stream()))
        _lib.check(lib.demon_sparse_tsdf_index(keys.data_ptr(), values.data_ptr(), slots, blocks.data_ptr(), 0, t, _stream()))
        chunk["table"] = (keys, values)
        return chunk

    def _mesh_range(self, chunk, count):
        """The mesh of the chunk pool's first `count` blocks (demon_sparse_tsdf_mesh_range_*)."""
        lib, t = _lib.load(), chunk["blocks"].shape[0]
        dev = chunk["tsdf"].device
        keys, values = chunk["table"]
        scratch = torch.empty((lib.demon_sparse_tsdf_mesh_scratch_bytes(count),), dtype=torch.uint8, device=dev)
        total = torch.empty((1,), dtype=torch.int64, device=dev)
        _lib.check(lib.demon_sparse_tsdf_mesh_range_count_f32(chunk["tsdf"].data_ptr(), chunk["weight"].data_ptr(), chunk["blocks"].data_ptr(), t,
                                                              0, count, keys.data_ptr(), values.data_ptr(), keys.numel(), scratch.data_ptr(),
                                                              total.data_ptr(), _stream()))
        tri = int(total.item())
        vertices = torch.empty((3 * tri, 3), dtype=torch.float32, device=dev)
        colors = None if chunk["color"] is None else torch.empty((3 * tri, 3), dtype=torch.uint8, device=dev)
        faces = torch.empty((tri, 3), dtype=torch.int32, device=dev)
        if tri:
            _lib.check(lib.demon_sparse_tsdf_mesh_range_f32(
                chunk["tsdf"].data_ptr(), chunk["weight"].data_ptr(), None if colors is None else chunk["color"].data_ptr(),
                chunk["blocks"].data_ptr(), t, 0, count, self._origin(), float(self.voxel_size), scratch.data_ptr(), vertices.data_ptr(),
                None if colors is None else colors.data_ptr(), faces.data_ptr(), _stream()))
        return vertices, colors, faces

    def indexed_mesh(self, normals=True):
        """TsdfVolume.indexed_mesh on the blocks (include/demon_b200.h: demon_sparse_tsdf_indexed_mesh_range_f32): one
        vertex per edge a meshed cube's triangles use, in ascending (packed key of the block holding the edge's first
        voxel, its local linear index, axis); faces are mesh()'s triangles moved into ascending block key, then the cube's
        local index and the table's order.  The result depends on the stored voxels alone, not on the pool's layout or
        max_device_blocks.  Returns TsdfVolume.indexed_mesh's dict; synchronises.

        With blocks on the host it runs twice over mesh()'s key-ordered chunks of max_device_blocks blocks, each copied
        with its 26 neighbours into a scratch pool: the first pass marks the edges, a scan over all blocks gives every
        block its first vertex, and the second writes the chunk's vertices and faces.  The edge masks cover every block
        (384 bytes per block on the device).  The volume's state does not change."""
        _check_normals(normals)
        if self._pool is None or self._m + self._host_blocks() == 0:
            return _indexed_outputs(0, 0, normals, self._color, self._pool["tsdf"].device if self._pool is not None else _device())
        dev = self._pool["tsdf"].device
        with torch.cuda.device(dev):
            if self._host_blocks():
                keys, coords, where = self._blocks_by_key()
                total = keys.numel()

                def chunks():
                    for c0 in range(0, total, self.max_device_blocks):
                        c1 = min(total, c0 + self.max_device_blocks)
                        sel = self._chunk_selection(keys, coords, c0, c1, _ALL_STEPS)
                        yield self._chunk_pool(coords[sel].contiguous(), where[sel]), c1 - c0, sel.to(torch.int32), None
                return self._indexed(normals, chunks, total)
            pool, m = self._pool, self._m
            order = torch.argsort(_packed_keys(pool["blocks"][:m]))
            rank = torch.empty_like(order)
            rank[order] = torch.arange(m, device=dev)
            whole = dict(pool, table=self._table[:2])
            return self._indexed(normals, lambda: [(whole, m, rank.to(torch.int32), order.to(torch.int32))], m)

    def _indexed(self, normals, chunks, total):
        """The indexed mesh of `total` blocks from two passes over chunks(), which yields (pool, count, rank, order): a pool
        with its table whose first count blocks are the chunk, the key rank of every pool block, and the key order of the
        chunk's blocks (None: already in key order)."""
        lib, dev = _lib.load(), self._pool["tsdf"].device
        masks = torch.zeros((total, 48), dtype=torch.int32, device=dev)
        for pool, count, rank, _ in chunks():
            keys, values = pool["table"]
            scratch = torch.empty((lib.demon_sparse_tsdf_mesh_scratch_bytes(count),), dtype=torch.uint8, device=dev)
            _lib.check(lib.demon_sparse_tsdf_edge_mark_f32(pool["tsdf"].data_ptr(), pool["weight"].data_ptr(), pool["blocks"].data_ptr(),
                                                           pool["blocks"].shape[0], 0, count, keys.data_ptr(), values.data_ptr(),
                                                           keys.numel(), rank.data_ptr(), scratch.data_ptr(), masks.data_ptr(), _stream()))
        base = torch.empty((total, 48), dtype=torch.int32, device=dev)
        scan = torch.empty((lib.demon_sparse_tsdf_edge_scan_bytes(total),), dtype=torch.uint8, device=dev)
        nv = torch.empty((1,), dtype=torch.int64, device=dev)
        _lib.check(lib.demon_sparse_tsdf_edge_scan(masks.data_ptr(), total, scan.data_ptr(), base.data_ptr(), nv.data_ptr(), _stream()))
        out = _indexed_outputs(int(nv.item()), 0, normals, self._color, dev)
        if out["vertices"].shape[0] == 0:   # no vertex, no triangle
            return out
        faces = []
        for pool, count, rank, order in chunks():
            keys, values = pool["table"]
            t = pool["blocks"].shape[0]
            scratch = torch.empty((lib.demon_sparse_tsdf_mesh_scratch_bytes(count),), dtype=torch.uint8, device=dev)
            tri = torch.empty((1,), dtype=torch.int64, device=dev)
            _lib.check(lib.demon_sparse_tsdf_indexed_mesh_range_count_f32(
                pool["tsdf"].data_ptr(), pool["weight"].data_ptr(), pool["blocks"].data_ptr(), t, 0, count, _ptr(order), keys.data_ptr(),
                values.data_ptr(), keys.numel(), scratch.data_ptr(), tri.data_ptr(), _stream()))
            f = torch.empty((int(tri.item()), 3), dtype=torch.int32, device=dev)
            _lib.check(lib.demon_sparse_tsdf_indexed_mesh_range_f32(
                pool["tsdf"].data_ptr(), pool["weight"].data_ptr(), None if out["colors"] is None else pool["color"].data_ptr(),
                pool["blocks"].data_ptr(), t, 0, count, _ptr(order), keys.data_ptr(), values.data_ptr(), keys.numel(), rank.data_ptr(),
                masks.data_ptr(), base.data_ptr(), self._origin(), float(self.voxel_size), scratch.data_ptr(), out["vertices"].data_ptr(),
                _ptr(out["normals"]), _ptr(out["colors"]), f.data_ptr() if f.shape[0] else None, _stream()))
            faces.append(f)
        out["faces"] = torch.cat(faces)
        return out

    def default_far(self, R, t):
        """CUDA float32 [n]: raycast's default far, the largest camera z of the 8 corners origin + voxel_size*(8b + (0 or 8))
        of every allocated block b, on the device or the host (include/demon_b200.h: demon_sparse_tsdf_far_f32), for each
        world-to-camera R [n,3,3] (CUDA float32) and t [n,3].  The volume must hold a block."""
        pool = self._state()
        n = R.shape[0]
        blocks, m = pool["blocks"], self._m
        if self._host_blocks():
            blocks = torch.cat([blocks[:m], self._host["blocks"][:self._hend][self._host["live"][:self._hend]]])
            m = blocks.shape[0]
        far = torch.empty((n,), dtype=torch.float32, device=R.device)
        _lib.check(_lib.load().demon_sparse_tsdf_far_f32(blocks.data_ptr(), m, self._origin(), float(self.voxel_size),
                                                        R.data_ptr(), t.data_ptr(), n, far.data_ptr(), _stream()))
        return far

    def raycast(self, K, R, t, height=192, width=256, near=0.0, far=None, step=0.5):
        """TsdfVolume.raycast on the blocks (include/demon_b200.h: demon_sparse_tsdf_raycast_f32): a sample is valid when
        its cube's 8 corners lie in allocated blocks with weight > 0, and far defaults to the largest camera z of the
        corners of every allocated block, reduced on the device.  The march jumps over blocks that are not allocated, with
        the result of evaluating every sample.  An empty volume renders no hit without a launch.  Asynchronous on the
        current stream, except with max_device_blocks: the host blocks its cameras reach (every tile at far, trunc 0) come
        back first, and the blocks beyond the budget stream out after it, which synchronises."""
        rq = _Render(K, R, t, height, width, near, far, step)
        dev = self._pool["tsdf"].device if self._pool is not None else _device()
        with torch.cuda.device(dev):
            out = rq.outputs(self._color, dev)
            if rq.n == 0 or self._m + self._host_blocks() == 0:
                return out
            Kd, Rd, td = rq.cameras()
            nr, fr = rq.limits(dev, None if rq.far is not None else self.default_far(Rd, td))
            if self.max_device_blocks is not None:
                tiles = fr[:, None, None].expand(rq.n, -(-rq.h // 8), -(-rq.w // 8)).contiguous()
                self._bring_back(tiles, 0.0, (Kd, Rd, td), rq.n, rq.h, rq.w)
                if self._m:
                    self._launch_raycast(rq, Kd, Rd, td, nr, fr, out)
                self._stream_out()
            else:
                self._launch_raycast(rq, Kd, Rd, td, nr, fr, out)
        return out

    def _launch_raycast(self, rq, Kd, Rd, td, nr, fr, out):
        pool, lib, m, dev = self._pool, _lib.load(), self._m, self._pool["tsdf"].device
        keys, values, _ = self._table
        scratch = torch.empty((lib.demon_sparse_tsdf_raycast_scratch_bytes(m),), dtype=torch.uint8, device=dev)
        _lib.check(lib.demon_sparse_tsdf_raycast_f32(
            pool["tsdf"].data_ptr(), pool["weight"].data_ptr(), None if pool["color"] is None else pool["color"].data_ptr(),
            pool["blocks"].data_ptr(), m, keys.data_ptr(), values.data_ptr(), keys.numel(), scratch.data_ptr(), self._origin(),
            float(self.voxel_size), Kd.data_ptr(), Rd.data_ptr(), td.data_ptr(), nr.data_ptr(), fr.data_ptr(), float(rq.step), rq.n,
            rq.h, rq.w, out["depth"].data_ptr(), out["normals"].data_ptr(),
            None if out["colors"] is None else out["colors"].data_ptr(), _stream()))


_MAX_COORD = (1 << 20) - 1   # DEMON_SPARSE_TSDF_MAX_COORD
_PLUS_STEPS = [[(q >> a) & 1 for a in range(3)] for q in range(1, 8)]   # the +x, +y, +z neighbours of a block
_ALL_STEPS = [[dx, dy, dz] for dz in (-1, 0, 1) for dy in (-1, 0, 1) for dx in (-1, 0, 1) if dx or dy or dz]


def _packed_keys(blocks):
    """int64 [m]: the table's packed key of each block [m,3] int32, 21 bits per axis offset by 2^20, z highest (fusion.cu's
    block_key), so ascending keys are ascending (z, y, x)."""
    b = blocks.long() + (1 << 20)
    return (b[:, 2] << 42) | (b[:, 1] << 21) | b[:, 0]


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


def reconstruct(pipeline, frames, intrinsics, volume=None, resample="bicubic", min_ratios=1000, indexed_mesh=False):
    """A video end to end: frames CUDA uint8 [T,H,W,3] (T >= 2, HWC RGB) with their intrinsics in pixels ([3,3], [T,3,3] or
    [T,4], as images.adjust_intrinsics takes them).  Every frame is adapted once to DeMoN's camera at 256x192
    (images.adjust_intrinsics), and its 64x48 image2_2 resized from the adapted frame with `resample`, as forward_views makes
    it.  The pairs (k, k+1) run through pipeline.forward_u8 (DemonPipeline or DemonPipelineV2) batch_size at a time; a
    partial last batch repeats its last pair, whose outputs are dropped.  The pairs are chained (chain_pairs) and the P
    depth maps integrated, coloured by adapted frame k, into `volume` (a TsdfVolume or a SparseTsdfVolume, which is added to)
    or, by default, a new 256^3 TsdfVolume around the 5th..95th percentiles of the chained points.

    Returns a dict: chain_pairs' scales, sigma, R, t and depth, inverse_depth / rotation / translation [P,...] of the pairs,
    the adapted frames [T,192,256,3] and their status (images.adjust_intrinsics), K [3,3] of the adapted frames in pixels,
    volume, and the mesh: vertices, colors, faces.  With indexed_mesh=True the mesh is volume.indexed_mesh()'s (shared
    vertices, and a `normals` key) instead of the soup."""
    if not isinstance(indexed_mesh, (bool, np.bool_)):
        raise ValueError("indexed_mesh must be True or False, got %r" % (indexed_mesh,))
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
    res = dict(ch, inverse_depth=inv, rotation=rot, translation=trans, adapted=adapted, status=status, K=K_new, volume=volume)
    if indexed_mesh:
        res.update(volume.indexed_mesh())
    else:
        res["vertices"], res["colors"], res["faces"] = volume.mesh()
    return res


def export_sequence_to_ply(prefix, result):
    """Writes prefix + '_mesh.ply' (the coloured mesh of `result`, with its normals when it has them) and prefix + '_cameras.ply' (vis.camera_mesh of every
    pose of result['R'] / result['t'], one mesh), in vis.write_ply's format."""
    col = result.get("colors")
    nrm = result.get("normals")
    vis.write_ply(prefix + "_mesh.ply", result["vertices"].cpu().numpy(), None if col is None else col.cpu().numpy(),
                  result["faces"].cpu().numpy(), None if nrm is None else nrm.cpu().numpy())
    verts, faces = [], []
    for k, (R, t) in enumerate(zip(result["R"], result["t"])):
        v, f = vis.camera_mesh(R, t)
        verts.append(v)
        faces.append(f + k * v.shape[0])
    vis.write_ply(prefix + "_cameras.ply", np.concatenate(verts), faces=np.concatenate(faces))
