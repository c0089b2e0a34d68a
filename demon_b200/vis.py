"""Mirror of `depthmotionnet.vis` (python/depthmotionnet/vis.py) without VTK: the point cloud of a depth map on the device
(csrc/vis.cu), bit for bit what the reference's `compute_point_cloud_from_depthmap` Cython (vis_cython.pyx) returns, and
`export_prediction_to_ply` writing the same three files as data.  There is no window and no renderer.

    pc = compute_point_cloud_from_depthmap(depth, K, R, t, normals, colors)   # vis_cython.pyx:142-173, one view
    pcs = point_clouds(depth, K, R, t, image=image, inverse_depth=True)       # a batch, padded, on the device
    pcs = prediction_point_clouds(out['predict_depth0'], intrinsics, image_pair[:, 0:3])   # visualize_prediction's operands
    export_prediction_to_ply('out/', inverse_depth, image=image)               # points.ply, cam1.ply, cam2.ply

A view's valid pixels are those with a finite depth > 0; they keep their row-major order.  There is no CPU fallback.
"""
import ctypes

import numpy as np
import torch

from . import _lib
from .evaluation import intrinsics_vector_to_K

SUN3D_INTRINSICS = (0.89115971, 1.18821287, 0.5, 0.5)   # vis.py:252, the network's sun3d constant

# create_camera_polydata (vis.py:50-142) with only_polys=True: the 11 corners of the camera glyph in camera coordinates
# before the 0.25 scale, and its 6 triangles in the order vis.py adds them (left, right, top, bottom, x-axis indicator,
# up vector)
CAMERA_POINTS = np.array([[0, 0, 0], [-1, -1, 1.5], [1, -1, 1.5], [1, 1, 1.5], [-1, 1, 1.5], [-0.5, 1, 1.5], [0.5, 1, 1.5],
                          [0, 1.2, 1.5], [1, -0.5, 1.5], [1, 0.5, 1.5], [1.2, 0, 1.5]], dtype=np.float64)
CAMERA_TRIANGLES = np.array([[0, 1, 4], [0, 3, 2], [0, 4, 3], [0, 2, 1], [8, 10, 9], [5, 6, 7]], dtype=np.int32)


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _device():
    if not torch.cuda.is_available():
        raise RuntimeError("demon_b200.vis needs a CUDA device (there is no CPU fallback)")
    return torch.device("cuda", torch.cuda.current_device())


def _cuda(x, dtype):
    """x (torch tensor or anything numpy converts) -> contiguous CUDA tensor of dtype."""
    if isinstance(x, torch.Tensor):
        t = x if x.is_cuda else x.to(_device())
    else:
        t = torch.from_numpy(np.ascontiguousarray(np.asarray(x))).to(_device())
    return t.to(dtype).contiguous()


def _host(x):
    return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def _shape(x):
    return tuple(x.shape)


def _is_uint8(x):
    return x.dtype == torch.uint8 if isinstance(x, torch.Tensor) else np.asarray(x).dtype == np.uint8


def _per_view(x, n, shape, name):
    """float32 CUDA [n, *shape] from [n, *shape] or one [*shape] shared by every view."""
    t = _cuda(x, torch.float32)
    if _shape(t) == shape:
        t = t.expand((n,) + shape).contiguous()
    if _shape(t) != (n,) + shape:
        raise ValueError("%s has shape %s; want %s or %s" % (name, _shape(t), shape, (n,) + shape))
    return t


def point_clouds(depth, K, R, t, normals=None, colors=None, image=None, inverse_depth=False):
    """The point clouds of n views on the device (include/demon_b200.h: demon_point_cloud_f32).

    depth [n,h,w] or [n,1,h,w] float32 camera z (inverse depth with `inverse_depth`: d = 1/inverse_depth in float32
    first); K [n,3,3], R [n,3,3], t [n,3] (or one [3,3] / [3] for all views); normals [n,3,h,w] float32; colors [n,3,h,w]
    uint8, or image [n,3,h,w] float32 taken as ((image+0.5)*255).astype(np.uint8) (vis.py:276, numpy's x86 cast for every
    value).  Returns {'points': [n,h*w,3] float32, 'normals'?: [n,h*w,3] float32, 'colors'?: [n,h*w,3] uint8, 'counts': [n]
    int32}, CUDA tensors: view i's cloud is rows 0..counts[i]-1, and rows past them are left unwritten.  Nothing
    synchronises, so with CUDA-tensor arguments the call can be captured in torch.cuda.graph and replayed with new
    contents.  A zero focal length is not checked here (compute_point_cloud_from_depthmap raises for it)."""
    d = _cuda(depth, torch.float32)
    if d.dim() == 4 and d.shape[1] == 1:
        d = d[:, 0]
    if d.dim() != 3:
        raise ValueError("depth must be [n,h,w] or [n,1,h,w], got %s" % (_shape(d),))
    n, h, w = d.shape
    if colors is not None and image is not None:
        raise ValueError("pass colors (uint8) or image (float), not both")
    Kd, Rd, td = _per_view(K, n, (3, 3), "K"), _per_view(R, n, (3, 3), "R"), _per_view(t, n, (3,), "t")
    nd = cd = im = None
    if normals is not None:
        nd = _cuda(normals, torch.float32)
        if _shape(nd) != (n, 3, h, w):
            raise ValueError("shape mismatch: normals %s, depth %s" % (_shape(nd), _shape(d)))
    if colors is not None:
        if not _is_uint8(colors):
            raise ValueError("colors must be uint8, got %s" % (colors.dtype,))
        cd = _cuda(colors, torch.uint8)
        if _shape(cd) != (n, 3, h, w):
            raise ValueError("shape mismatch: colors %s, depth %s" % (_shape(cd), _shape(d)))
    if image is not None:
        im = _cuda(image, torch.float32)
        if _shape(im) != (n, 3, h, w):
            raise ValueError("shape mismatch: image %s, depth %s" % (_shape(im), _shape(d)))
    lib = _lib.load()
    dev = d.device
    out = {'points': torch.empty((n, h * w, 3), dtype=torch.float32, device=dev)}
    if nd is not None:
        out['normals'] = torch.empty((n, h * w, 3), dtype=torch.float32, device=dev)
    if cd is not None or im is not None:
        out['colors'] = torch.empty((n, h * w, 3), dtype=torch.uint8, device=dev)
    out['counts'] = torch.empty((n,), dtype=torch.int32, device=dev)
    scratch = torch.empty((max(1, lib.demon_point_cloud_scratch_bytes(n, h, w)),), dtype=torch.uint8, device=dev)

    def ptr(x):
        return None if x is None else x.data_ptr()
    fn = lib.demon_point_cloud_inverse_f32 if inverse_depth else lib.demon_point_cloud_f32
    _lib.check(fn(d.data_ptr(), Kd.data_ptr(), Rd.data_ptr(), td.data_ptr(), ptr(nd), ptr(cd), ptr(im), n, h, w, scratch.data_ptr(),
                  out['points'].data_ptr(), ptr(out.get('normals')), ptr(out.get('colors')), out['counts'].data_ptr(), _stream()))
    return out


def compute_point_cloud_from_depthmap(depth, K, R, t, normals=None, colors=None):
    """vis_cython.pyx:142-173 for one view, on the device: depth [h,w] (squeezed if it has more dimensions), K [3,3], R
    [3,3], t [3], normals [3,h,w], colors [3,h,w] uint8.  Returns {'points' [m,3] float32, 'normals' [m,3] float32 if
    normals were given, 'colors' [m,3] uint8 if colors were given} for the m valid pixels, bit for bit the reference's.
    numpy in gives numpy out; a CUDA tensor depth gives CUDA tensors.  Errors as the reference's: AssertionError for
    colours that are not uint8, ValueError for a depth with more than 2 non-unit dimensions or normals / colours of
    another size, ZeroDivisionError for K[0,0] or K[1,1] == 0.  Reads the point count back, so it synchronises."""
    assert _is_uint8(colors) if colors is not None else True
    was_np = not isinstance(depth, torch.Tensor)
    shape = _shape(depth) if hasattr(depth, "shape") else np.shape(depth)
    if len(shape) > 2:
        shape = tuple(s for s in shape if s != 1)
    if len(shape) > 2:
        raise ValueError("wrong number of dimensions for depth")
    if len(shape) != 2:
        raise ValueError("Buffer has wrong number of dimensions (expected 2, got %d)" % len(shape))
    # the reference checks the shape after the channel; a channel count other than 3 would read past its buffer
    if normals is not None and (_shape(normals)[1:] != shape or _shape(normals)[0] != 3):
        raise ValueError("shape mismatch: normals {0}, depth {1}".format(_shape(normals), _shape(depth)))
    if colors is not None and (_shape(colors)[1:] != shape or _shape(colors)[0] != 3):
        raise ValueError("shape mismatch: colors {0}, depth {1}".format(_shape(colors), _shape(depth)))
    K32, R32, t32 = (_host(a).astype(np.float32) for a in (K, R, t))
    if K32[0, 0] == 0 or K32[1, 1] == 0:   # the .pyx's 1/K[0,0], 1/K[1,1] are checked divisions
        raise ZeroDivisionError("float division")
    d = _cuda(depth, torch.float32).reshape(shape)
    pc = point_clouds(d[None], K32[None], R32[None], t32.reshape(1, 3), None if normals is None else normals[None],
                      None if colors is None else colors[None])
    m = int(pc['counts'][0])
    res = {k: v[0, :m] for k, v in pc.items() if k != 'counts'}
    return {k: v.cpu().numpy() for k, v in res.items()} if was_np else res


def prediction_K(intrinsics, n, h, w):
    """float32 [n,3,3]: K of visualize_prediction (vis.py:251-258) for intrinsics None (sun3d), [4] or [n,4] normalised
    (fx, fy, cx, cy), as evaluation.intrinsics_vector_to_K builds it (the same float32 values as vis.py's construction)."""
    intr = np.array(SUN3D_INTRINSICS) if intrinsics is None else _host(intrinsics)
    intr = np.broadcast_to(intr.reshape(-1, 4), (n, 4)) if intr.size == 4 else intr.reshape(n, 4)
    return np.stack([intrinsics_vector_to_K(intr[i], w, h).astype(np.float32) for i in range(n)])


def prediction_point_clouds(inverse_depth, intrinsics=None, image=None, normals=None):
    """The point clouds visualize_prediction / export_prediction_to_ply compute (vis.py:246-278), for a batch on the
    device: inverse_depth [B,1,h,w] (the network's predict_depth0; depth = 1/inverse_depth), intrinsics None (sun3d),
    [4] or [B,4], image [B,3,h,w] float32 in [-0.5,0.5] (colours ((image+0.5)*255).astype(uint8)), normals [B,3,h,w];
    the first camera at the origin (R = I, t = 0).  Returns point_clouds' padded dict.  K is built on the host and
    copied over; to capture a graph, call point_clouds with device K instead."""
    d = _cuda(inverse_depth, torch.float32)
    if d.dim() == 3:
        d = d[:, None]
    if d.dim() != 4 or d.shape[1] != 1:
        raise ValueError("inverse_depth must be [B,1,h,w], got %s" % (_shape(d),))
    n, _, h, w = d.shape
    K = torch.from_numpy(prediction_K(intrinsics, n, h, w)).to(d.device)
    R = torch.eye(3, dtype=torch.float32, device=d.device)
    t = torch.zeros(3, dtype=torch.float32, device=d.device)
    return point_clouds(d, K, R, t, normals=normals, image=image, inverse_depth=True)


def angleaxis_to_rotation_matrix(aa):
    """depthmotionnet/helpers.py:37-57 (Rodrigues' formula, not the quaternion form of evaluation.angleaxis_to_rotation_matrix):
    float64 [3,3] R = c I + (1-c) u u^T + s [u]x for angle = |aa| > 1e-6, else I, computed in aa's own precision."""
    aa = np.asarray(aa)
    angle = np.sqrt(aa.dot(aa))
    if not angle > 1e-6:
        return np.eye(3)
    c, s = np.cos(angle), np.sin(angle)
    u = np.array([aa[0] / angle, aa[1] / angle, aa[2] / angle])
    cross = np.array([[0, -u[2], u[1]], [u[2], 0, -u[0]], [-u[1], u[0], 0]], dtype=u.dtype)
    R = np.empty((3, 3))
    R[...] = np.outer(u, u) * (1 - c) + c * np.eye(3, dtype=u.dtype) + cross * s
    return R


def camera_mesh(R, t):
    """create_camera_polydata(R, t, only_polys=True) (vis.py:50-142) as arrays: float64 vertices [11,3]
    (0.25*CAMERA_POINTS - t).dot(R) and int32 triangles [6,3] (CAMERA_TRIANGLES)."""
    return (0.25 * CAMERA_POINTS - np.asarray(t)).dot(np.asarray(R)), CAMERA_TRIANGLES.copy()


def write_ply(path, vertices, colors=None, faces=None, normals=None):
    """A binary little-endian PLY file: vertices [m,3] as float x y z, normals [m,3] as float nx ny nz, colors [m,3] uint8
    as uchar red green blue, faces [k,3] as list uchar int vertex_indices.  The header is

        ply
        format binary_little_endian 1.0
        element vertex <m>
        property float x
        property float y
        property float z
        property float nx           (with normals)
        property float ny
        property float nz
        property uchar red          (with colours)
        property uchar green
        property uchar blue
        element face <k>            (with faces)
        property list uchar int vertex_indices
        end_header

    followed by the m packed vertex records and the k face records (a count byte 3 and three int32 indices)."""
    v = np.asarray(vertices).reshape(-1, 3)
    fields = [('x', '<f4'), ('y', '<f4'), ('z', '<f4')]
    if normals is not None:
        fields += [('nx', '<f4'), ('ny', '<f4'), ('nz', '<f4')]
    if colors is not None:
        fields += [('red', 'u1'), ('green', 'u1'), ('blue', 'u1')]
    rec = np.empty(v.shape[0], dtype=np.dtype(fields))
    rec['x'], rec['y'], rec['z'] = v[:, 0], v[:, 1], v[:, 2]
    if normals is not None:
        nv = np.asarray(normals, dtype=np.float32).reshape(-1, 3)
        if nv.shape[0] != v.shape[0]:
            raise ValueError("%d normals for %d vertices" % (nv.shape[0], v.shape[0]))
        rec['nx'], rec['ny'], rec['nz'] = nv[:, 0], nv[:, 1], nv[:, 2]
    if colors is not None:
        c = np.asarray(colors, dtype=np.uint8).reshape(-1, 3)
        if c.shape[0] != v.shape[0]:
            raise ValueError("%d colours for %d vertices" % (c.shape[0], v.shape[0]))
        rec['red'], rec['green'], rec['blue'] = c[:, 0], c[:, 1], c[:, 2]
    head = ["ply", "format binary_little_endian 1.0", "element vertex %d" % v.shape[0],
            "property float x", "property float y", "property float z"]
    if normals is not None:
        head += ["property float nx", "property float ny", "property float nz"]
    if colors is not None:
        head += ["property uchar red", "property uchar green", "property uchar blue"]
    frec = None
    if faces is not None:
        fc = np.asarray(faces).reshape(-1, 3)
        frec = np.empty(fc.shape[0], dtype=np.dtype([('n', 'u1'), ('i', '<i4', (3,))]))
        frec['n'], frec['i'] = 3, fc
        head += ["element face %d" % fc.shape[0], "property list uchar int vertex_indices"]
    head.append("end_header")
    with open(path, "wb") as f:
        f.write(("\n".join(head) + "\n").encode("ascii"))
        f.write(rec.tobytes())
        if frec is not None:
            f.write(frec.tobytes())


def export_prediction_to_ply(output_prefix, inverse_depth, intrinsics=None, normals=None, rotation=None, translation=None,
                             image=None):
    """vis.py:322-401 without VTK: writes output_prefix + 'points.ply' (the valid pixels' points, coloured when `image` is
    given), 'cam1.ply' (the camera mesh at the origin) and 'cam2.ply' (the mesh at R2 = Rodrigues(rotation), t2 =
    translation if both are given, else at the origin too), in write_ply's format.  inverse_depth [h,w] (any unit
    dimensions are squeezed), intrinsics [4] or None (sun3d), normals [3,h,w] (checked, not written: the reference does
    not write them either), rotation / translation [3], image [3,h,w] float32 in [-0.5,0.5].  numpy arrays or tensors."""
    inv = _cuda(inverse_depth, torch.float32).squeeze()
    if inv.dim() != 2:
        raise ValueError("inverse_depth must hold one [h,w] map, got %s" % (_shape(inverse_depth),))
    h, w = inv.shape
    if normals is not None and tuple(s for s in _shape(normals) if s != 1) != (3, h, w):
        raise ValueError("shape mismatch: normals {0}, depth {1}".format(_shape(normals), (h, w)))
    img = None if image is None else _cuda(image, torch.float32).reshape(1, 3, h, w)
    pc = prediction_point_clouds(inv[None, None], None if intrinsics is None else _host(intrinsics).reshape(4), img)
    m = int(pc['counts'][0])
    points = pc['points'][0, :m].cpu().numpy()
    colors = pc['colors'][0, :m].cpu().numpy() if 'colors' in pc else None
    if rotation is not None and translation is not None:
        R2, t2 = angleaxis_to_rotation_matrix(_host(rotation).squeeze()), _host(translation).squeeze()
    else:
        R2, t2 = np.eye(3), np.zeros((3,))
    write_ply(output_prefix + 'points.ply', points, colors)
    for name, (R, t) in (('cam1.ply', (np.eye(3), np.zeros((3,)))), ('cam2.ply', (R2, t2))):
        v, f = camera_mesh(R, t)
        write_ply(output_prefix + name, v, faces=f)
