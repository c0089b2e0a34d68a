"""ORACLE (test infrastructure) -- compute_point_cloud_from_depthmap of the reference's python/depthmotionnet/vis_cython.pyx,
in two forms:

* the reference's own Cython, cythonized unmodified from the reference tree next to DEMON_REF_SRC and compiled with
  -O2 -ffp-contract=off into oracle/_ref/vis_cython.so (vis.mk; a build product, git-ignored).  Where neither the extension
  nor the reference tree exists, `reference_point_cloud` returns the stored digests of the same call
  (tests/golden/vis_digests.json, recorded with DEMON_REF_RECORD=<json path> like oracle/ref.py's);
* `point_cloud_numpy`, a numpy restatement of the .pyx loop (float32 element-wise operations in the .pyx's order), which
  the CPU tests hold to the Cython bit for bit and the GPU tests hold the device to.

Digests hash the arrays with every NaN canonicalised (oracle/recorded.py:digest): a rotated NaN normal or an overflowing point
carries an x86 NaN payload the GPU does not reproduce.  Only tests/, __graft_entry__ and tools/ may import this module.
"""
import hashlib
import importlib.util
import os
import sys

import numpy as np

from .recorded import REF_SRC, Recorded, Store, build_artefact, digest, entry, record  # noqa: F401  (digest: re-exported)

_HERE = os.path.dirname(os.path.abspath(__file__))
_EXT_PATH = os.path.join(_HERE, "_ref", "vis_cython.so")
PYX = (os.path.normpath(os.path.join(REF_SRC, "..", "..", "python", "depthmotionnet", "vis_cython.pyx")) if REF_SRC else "")
_STORE = Store("vis_digests.json")

# vis.py:252
SUN3D_INTRINSICS = (0.89115971, 1.18821287, 0.5, 0.5)


def build(force=False):
    """Compile _ref/vis_cython.so if the reference tree is present; returns the path or None."""
    return build_artefact(_EXT_PATH, [PYX], ["vis.mk"], ["-f", "vis.mk", "vis", "PYTHON=" + sys.executable], force)


_mod = None


def have_module():
    return build() is not None


def module():
    global _mod
    if _mod is None:
        path = build()
        if path is None:
            raise RuntimeError("oracle/_ref/vis_cython.so is not built and DEMON_REF_SRC names no reference tree")
        spec = importlib.util.spec_from_file_location("vis_cython", path)
        _mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(_mod)
    return _mod


def available():
    return have_module() or bool(_STORE.entries())


def _key(arrays):
    h = hashlib.sha256(b"compute_point_cloud_from_depthmap")
    for a in arrays:
        if a is None:
            h.update(b"None")
            continue
        a = np.ascontiguousarray(a)
        h.update(("%s|%s" % (a.dtype.str, a.shape)).encode())
        h.update(a.tobytes())
    return h.hexdigest()


def reference_point_cloud(depth, K, R, t, normals=None, colors=None):
    """The reference's compute_point_cloud_from_depthmap for one view: depth [h,w] float32, K [3,3], R [3,3], t [3],
    normals [3,h,w] float32 or None, colors [3,h,w] uint8 or None.  Returns its dict of arrays, or a dict of their
    Recorded digests."""
    depth = np.ascontiguousarray(depth, dtype=np.float32)
    K, R, t = (np.asarray(a) for a in (K, R, t))
    key = _key([depth, K, R, t, normals, colors])
    if not have_module():
        stored = _STORE.lookup(key, "result for this compute_point_cloud_from_depthmap call")
        return {name: Recorded(v) for name, v in stored.items()}
    out = module().compute_point_cloud_from_depthmap(depth, K, R, t, normals, colors)
    out = {name: np.asarray(v) for name, v in out.items()}
    record(key, {name: entry(v) for name, v in out.items()})
    return out


def image_to_colors(image):
    """vis.py:276: ((image+0.5)*255).astype(np.uint8) of a float32 [3,h,w] image (numpy's own cast)."""
    with np.errstate(all='ignore'):
        return ((np.asarray(image, dtype=np.float32) + 0.5) * 255).astype(np.uint8)


def point_cloud_numpy(depth, K, R, t, normals=None, colors=None):
    """_compute_point_cloud_from_depthmap (vis_cython.pyx:24-135) over the whole image at once: float32 operations in the
    loop's order (every numpy operation here is float32 op float32 -> float32, rounded like C's; 1/K[0,0] is the .pyx's
    double division rounded to float32, which equals the float32 division)."""
    f = np.float32
    depth = np.asarray(depth, dtype=f)
    K, R, t = (np.asarray(a, dtype=f) for a in (K, R, t))
    h, w = depth.shape
    inv_fx, inv_fy = f(1.0 / np.float64(K[0, 0])), f(1.0 / np.float64(K[1, 1]))
    cx, cy = K[0, 2], K[1, 2]
    px = (np.arange(w, dtype=f) + f(0.5))[None, :]
    py = (np.arange(h, dtype=f) + f(0.5))[:, None]
    with np.errstate(all='ignore'):
        valid = np.isfinite(depth) & (depth > f(0))
        d = depth
        tmp = [d * (px - cx) * inv_fx - t[0], d * (py - cy) * inv_fy - t[1], d - t[2]]
        X = [R[0, c] * tmp[0] + R[1, c] * tmp[1] + R[2, c] * tmp[2] for c in range(3)]
        out = {'points': np.stack([x[valid] for x in X], axis=1).astype(f).reshape(-1, 3)}
        if normals is not None:
            nrm = np.asarray(normals, dtype=f)
            N = [R[0, c] * nrm[0] + R[1, c] * nrm[1] + R[2, c] * nrm[2] for c in range(3)]
            out['normals'] = np.stack([x[valid] for x in N], axis=1).astype(f).reshape(-1, 3)
    if colors is not None:
        col = np.asarray(colors)
        out['colors'] = np.stack([col[c][valid] for c in range(3)], axis=1).astype(np.uint8).reshape(-1, 3)
    return out


def edge_cases():
    """Views the tests hold the device kernel, the numpy restatement and the reference's Cython to: dicts with `depth`
    ([h,w] float32 camera z, or None) or `inverse_depth` (the same, inverse), K [3,3], R [3,3], t [3] float64, `normals`
    ([3,h,w] float32 or None), `colors` ([3,h,w] uint8 or None) or `image` ([3,h,w] float32 in about [-0.5,0.5], or None)."""
    from demon_b200.evaluation import angleaxis_to_rotation_matrix, intrinsics_vector_to_K
    rng = np.random.RandomState(20172)
    f = np.float32
    cases = []

    def depth_map(h, w, lo=0.3, hi=8.0):
        d = rng.uniform(lo, hi, (h, w)).astype(f)
        special = np.array([np.nan, np.inf, -np.inf, 0.0, -0.0, -1.5, 1e-45, 1e-40, np.finfo(f).max, -np.finfo(f).max], dtype=f)
        m = rng.rand(h, w) < 0.15
        d[m] = special[rng.randint(0, len(special), m.sum())]
        return d

    def normal_map(h, w):
        nrm = rng.normal(0, 1, (3, h, w)).astype(f)
        nrm[:, rng.rand(h, w) < 0.1] = np.nan
        return nrm

    def image(h, w, lo=-0.5, hi=0.5):
        return rng.uniform(lo, hi, (3, h, w)).astype(f)

    sun3d = np.array(SUN3D_INTRINSICS)
    other = np.array([0.8, 1.1, 0.45, 0.55])
    I3, z3 = np.eye(3), np.zeros(3)
    # every size, the sun3d camera at the origin, camera-z depth with every special value, normals and colours
    for h, w in ((1, 1), (7, 9), (31, 17), (48, 64), (192, 256), (768, 1024)):
        K = intrinsics_vector_to_K(sun3d, w, h)
        cases.append(dict(depth=depth_map(h, w), K=K, R=I3, t=z3, normals=normal_map(h, w),
                          colors=rng.randint(0, 256, (3, h, w)).astype(np.uint8)))
    # non-identity R with a translation and other intrinsics; with and without normals and colours
    for h, w in ((7, 9), (31, 17), (48, 64)):
        K = intrinsics_vector_to_K(other, w, h)
        R = angleaxis_to_rotation_matrix(rng.normal(0, 0.4, 3))
        t = rng.normal(0, 0.5, 3)
        cases.append(dict(depth=depth_map(h, w), K=K, R=R, t=t, normals=normal_map(h, w), colors=None))
        cases.append(dict(depth=depth_map(h, w), K=K, R=R, t=t, normals=None,
                          colors=rng.randint(0, 256, (3, h, w)).astype(np.uint8)))
        cases.append(dict(depth=depth_map(h, w), K=K, R=R, t=t))
    # all invalid (count 0) and all valid
    h, w = 31, 17
    K = intrinsics_vector_to_K(sun3d, w, h)
    bad = np.array([np.nan, np.inf, -np.inf, 0.0, -0.0, -2.0], dtype=f)[rng.randint(0, 6, (h, w))]
    cases.append(dict(depth=bad, K=K, R=I3, t=z3, normals=normal_map(h, w), colors=rng.randint(0, 256, (3, h, w)).astype(np.uint8)))
    cases.append(dict(depth=rng.uniform(0.5, 3.0, (h, w)).astype(f), K=K, R=angleaxis_to_rotation_matrix(np.array([0.1, 0.2, -0.3])),
                      t=np.array([0.2, -0.1, 0.4]), normals=normal_map(h, w), colors=rng.randint(0, 256, (3, h, w)).astype(np.uint8)))
    # inverse depth (visualize_prediction): 0, -0, subnormal (1/x is inf), negative, NaN, and images out of range
    for h, w in ((7, 9), (48, 64), (192, 256), (768, 1024)):
        inv = rng.uniform(0.05, 2.0, (h, w)).astype(f)
        special = np.array([0.0, -0.0, 1e-45, 1e-39, 3e-39, -0.5, np.nan, np.inf, 1e30], dtype=f)
        m = rng.rand(h, w) < 0.15
        inv[m] = special[rng.randint(0, len(special), m.sum())]
        img = image(h, w)
        sel = rng.rand(3, h, w)
        img[sel < 0.05] = rng.uniform(-3.0, -0.5, (sel < 0.05).sum())             # below -0.5
        img[(sel >= 0.05) & (sel < 0.1)] = rng.uniform(0.5 + 1 / 255, 5.0, ((sel >= 0.05) & (sel < 0.1)).sum())
        img[(sel >= 0.1) & (sel < 0.12)] = np.nan
        img[(sel >= 0.12) & (sel < 0.13)] = np.array([np.inf, -np.inf, 1e10, -1e10, 255.0, -300.0], dtype=f)[
            rng.randint(0, 6, ((sel >= 0.12) & (sel < 0.13)).sum())]
        cases.append(dict(inverse_depth=inv, K=intrinsics_vector_to_K(sun3d, w, h), R=I3, t=z3,
                          normals=normal_map(h, w) if h <= 48 else None, image=img))
    # inverse depth with another camera pose and intrinsics, uint8 colours
    h, w = 31, 17
    inv = rng.uniform(0.1, 1.0, (h, w)).astype(f)
    inv[rng.rand(h, w) < 0.2] = 0.0
    cases.append(dict(inverse_depth=inv, K=intrinsics_vector_to_K(other, w, h), R=angleaxis_to_rotation_matrix(np.array([0.3, -0.2, 0.1])),
                      t=np.array([0.5, 0.25, -1.0]), normals=None, colors=rng.randint(0, 256, (3, h, w)).astype(np.uint8)))
    return cases


def case_operands(case):
    """The operands the reference's Cython sees for a case: (depth float32 camera z, K, R, t, normals, colors uint8) -- 1/inverse
    depth and ((image+0.5)*255).astype(uint8) taken in numpy as vis.py:246, 276 do."""
    if case.get('inverse_depth') is not None:
        with np.errstate(all='ignore'):
            depth = 1 / case['inverse_depth']
    else:
        depth = case['depth']
    colors = case.get('colors')
    if case.get('image') is not None:
        colors = image_to_colors(case['image'])
    return depth, case['K'], case['R'], case['t'], case.get('normals'), colors
