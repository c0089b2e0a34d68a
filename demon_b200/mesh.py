"""Connected components of an indexed mesh on the device, and the removal of its small pieces (csrc/mesh.cu).

    comps = components(faces, num_vertices)            # labels [V], triangles [C], vertices [C]
    clean = remove_small_components(res, min_triangles=200)
    export_sequence_to_ply(prefix, dict(res, **clean))

Two vertices are connected when a face contains both; a component is a class of that relation, by index, not by
position, and a vertex no face uses is a component of its own.  Components are numbered in ascending order of their
smallest vertex.  The rule is in include/demon_b200.h (demon_mesh_*).  There is no CPU fallback.
"""
import ctypes
import numbers

import numpy as np
import torch

from . import _lib

_INT_DTYPES = (torch.int32, torch.int64)


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _device():
    if not torch.cuda.is_available():
        raise RuntimeError("demon_b200.mesh needs a CUDA device (there is no CPU fallback)")
    return torch.device("cuda", torch.cuda.current_device())


def _ptr(t):
    return None if t is None else t.data_ptr()


def _is_int(x):
    return isinstance(x, numbers.Integral) and not isinstance(x, (bool, np.bool_))


def _array(x, name):
    """A torch tensor as it is, anything else through numpy; ValueError for what numpy cannot take."""
    if isinstance(x, torch.Tensor):
        return x
    try:
        return np.asarray(x)
    except Exception as e:
        raise ValueError("%s: cannot be read as an array (%s)" % (name, e))


def _check_faces(faces, num_vertices):
    """faces [F,3] int32 / int64 (tensor or array) with every index in [0, num_vertices), and 0 <= num_vertices < 2^31:
    ValueError otherwise.  A host array is checked on the host; a CUDA tensor by its minimum and maximum before any of
    this module's kernels sees it.  Returns the faces as they came."""
    if not _is_int(num_vertices) or not 0 <= num_vertices < 2 ** 31:
        raise ValueError("num_vertices must be an integer in [0, 2^31), got %r" % (num_vertices,))
    f = _array(faces, "faces")
    if isinstance(f, torch.Tensor):
        ok = f.dtype in _INT_DTYPES
    else:
        ok = f.dtype in (np.int32, np.int64)
    if not ok:
        raise ValueError("faces must be int32 or int64, got %s" % (f.dtype,))
    if len(f.shape) != 2 or f.shape[1] != 3:
        raise ValueError("faces must be [F,3], got %s" % (tuple(f.shape),))
    if f.shape[0]:
        if isinstance(f, torch.Tensor):
            lo, hi = (int(v) for v in torch.aminmax(f))
        else:
            lo, hi = int(f.min()), int(f.max())
        if lo < 0 or hi >= num_vertices:
            raise ValueError("faces index vertices %d .. %d; want every index in [0, %d)" % (lo, hi, num_vertices))
    return f


def _device_faces(f, dev):
    t = f if isinstance(f, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(f))
    return t.to(device=dev, dtype=torch.int32).contiguous()


def _components(f, nv, dev):
    """components() on checked int32 CUDA faces, with the scratch it used."""
    lib = _lib.load()
    nf = f.shape[0]
    scratch = torch.empty((max(1, lib.demon_mesh_components_scratch_bytes(nv, nf)),), dtype=torch.uint8, device=dev)
    labels = torch.empty((nv,), dtype=torch.int32, device=dev)
    count = torch.empty((1,), dtype=torch.int64, device=dev)
    _lib.check(lib.demon_mesh_components_count(_ptr(f), nf, nv, scratch.data_ptr(), labels.data_ptr(), count.data_ptr(), _stream()))
    c = int(count.item())
    tri = torch.empty((c,), dtype=torch.int64, device=dev)
    ver = torch.empty((c,), dtype=torch.int64, device=dev)
    _lib.check(lib.demon_mesh_component_sizes(_ptr(f), nf, labels.data_ptr(), nv, c, tri.data_ptr(), ver.data_ptr(), _stream()))
    return {"labels": labels, "triangles": tri, "vertices": ver}, scratch


def components(faces, num_vertices):
    """The connected components of a mesh of num_vertices vertices (include/demon_b200.h: demon_mesh_components_count):
    faces [F,3] int32 or int64, a tensor or anything numpy converts, with every index in [0, num_vertices) (checked before
    any kernel runs: ValueError).  Returns CUDA tensors {"labels": [V] int32, each vertex's component, numbered 0 .. C-1 in
    ascending order of the component's smallest vertex; "triangles": [C] int64 and "vertices": [C] int64, each
    component's faces and vertices}.  A face's component is labels[faces[f,0]].  Reads C back, so it synchronises."""
    f = _check_faces(faces, num_vertices)
    dev = _device()
    with torch.cuda.device(dev):
        return _components(_device_faces(f, dev), num_vertices, dev)[0]


def _float3(x, name, nv, dtype):
    t = _array(x, name)
    t = t if isinstance(t, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(t))
    if t.dtype != dtype or tuple(t.shape) != (nv, 3):
        raise ValueError("%s must be %s [%d,3], got %s %s" % (name, dtype, nv, t.dtype, tuple(t.shape)))
    return t


def remove_small_components(mesh, min_triangles=1, keep_largest=None):
    """The mesh without its small components (include/demon_b200.h: demon_mesh_filter): a component is kept when it has
    at least min_triangles triangles, and with keep_largest=k only the k kept components with the most triangles remain
    (ties go to the smaller label).  mesh is a dict with "vertices" [V,3] float32, "faces" [F,3] int32 / int64 and optional
    "normals" [V,3] float32 and "colors" [V,3] uint8 (a missing key or None: none), such as indexed_mesh()'s dict or a
    reconstruct(..., indexed_mesh=True) result; tensors or arrays.  Returns a new dict of CUDA tensors with those four keys:
    the kept vertices in ascending original index, their normals and colours copied bit for bit (None where the input
    had none), and the kept faces in their original order, renumbered.  Every argument is checked before any device
    work (ValueError).  Reads two counts back, so it synchronises."""
    if not isinstance(mesh, dict) or "vertices" not in mesh or "faces" not in mesh:
        raise ValueError("mesh must be a dict with 'vertices' and 'faces'")
    if not _is_int(min_triangles) or min_triangles < 0:
        raise ValueError("min_triangles must be an integer >= 0, got %r" % (min_triangles,))
    if keep_largest is not None and (not _is_int(keep_largest) or keep_largest < 1):
        raise ValueError("keep_largest must be None or an integer >= 1, got %r" % (keep_largest,))
    v = _array(mesh["vertices"], "vertices")
    if len(v.shape) != 2 or v.shape[1] != 3:
        raise ValueError("vertices must be [V,3], got %s" % (tuple(v.shape),))
    nv = int(v.shape[0])
    f = _check_faces(mesh["faces"], nv)
    v = _float3(v, "vertices", nv, torch.float32)
    n = None if mesh.get("normals") is None else _float3(mesh["normals"], "normals", nv, torch.float32)
    c = None if mesh.get("colors") is None else _float3(mesh["colors"], "colors", nv, torch.uint8)
    dev = _device()
    with torch.cuda.device(dev):
        fd = _device_faces(f, dev)
        v, n, c = (None if x is None else x.to(dev).contiguous() for x in (v, n, c))
        comps, scratch = _components(fd, nv, dev)
        tri = comps["triangles"]
        select = None
        if keep_largest is not None and keep_largest < tri.shape[0]:
            # the k largest of the kept components; a stable descending sort leaves ties in label order
            key = torch.where(tri >= min_triangles, tri, torch.full_like(tri, -1))
            top = torch.sort(key, descending=True, stable=True).indices[:keep_largest]
            select = torch.zeros(tri.shape, dtype=torch.uint8, device=dev)
            select[top] = 1
        lib = _lib.load()
        nf = fd.shape[0]
        counts = torch.empty((2,), dtype=torch.int64, device=dev)
        args = (_ptr(fd), nf, comps["labels"].data_ptr(), nv, tri.data_ptr(), int(min_triangles), _ptr(select), scratch.data_ptr())
        _lib.check(lib.demon_mesh_filter_count(*args, counts.data_ptr(), _stream()))
        kv, kf = counts.tolist()
        out = {"vertices": torch.empty((kv, 3), dtype=torch.float32, device=dev),
               "normals": None if n is None else torch.empty((kv, 3), dtype=torch.float32, device=dev),
               "colors": None if c is None else torch.empty((kv, 3), dtype=torch.uint8, device=dev),
               "faces": torch.empty((kf, 3), dtype=torch.int32, device=dev)}
        if kv:
            _lib.check(lib.demon_mesh_filter(*args, v.data_ptr(), _ptr(n), _ptr(c), out["vertices"].data_ptr(), _ptr(out["normals"]),
                                             _ptr(out["colors"]), _ptr(out["faces"]) if kf else None, _stream()))
    return out
