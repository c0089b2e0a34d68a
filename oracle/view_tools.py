"""ORACLE (test infrastructure) -- compute_visible_points_mask of the reference's
python/depthmotionnet/dataset_tools/view_tools_cython.pyx, in two forms:

* the reference's own Cython, cythonized unmodified from the reference tree next to DEMON_REF_SRC and compiled with
  -O2 -ffp-contract=off into oracle/_ref/view_tools_cython.so (view_tools.mk; a build product, git-ignored).  Where neither
  the extension nor the reference tree exists, `reference_mask` returns the stored digest of the same call
  (tests/golden/view_tools_digests.json, recorded with DEMON_REF_RECORD=<json path> like oracle/ref.py's);
* `visible_points_mask_numpy`, a numpy restatement of the .pyx loop (float32 element-wise operations in the .pyx's
  order), which the CPU tests hold to the Cython bit for bit and which composes the GPU tests' oracle tables.

Only tests/, __graft_entry__ and tools/ may import this module.
"""
import hashlib
import importlib.util
import os
import sys
from collections import namedtuple

import numpy as np

from .recorded import REF_SRC, Recorded, Store, build_artefact, digest, entry, record  # noqa: F401  (digest: re-exported)

_HERE = os.path.dirname(os.path.abspath(__file__))
_EXT_PATH = os.path.join(_HERE, "_ref", "view_tools_cython.so")
PYX = (os.path.normpath(os.path.join(REF_SRC, "..", "..", "python", "depthmotionnet", "dataset_tools", "view_tools_cython.pyx"))
       if REF_SRC else "")
_STORE = Store("view_tools_digests.json")

# dataset_tools/view.py:25
View = namedtuple('View', ['R', 't', 'K', 'image', 'depth', 'depth_metric'])


def build(force=False):
    """Compile _ref/view_tools_cython.so if the reference tree is present; returns the path or None."""
    return build_artefact(_EXT_PATH, [PYX], ["view_tools.mk"],
                          ["-f", "view_tools.mk", "view_tools", "PYTHON=" + sys.executable], force)


_mod = None


def have_module():
    return build() is not None


def module():
    global _mod
    if _mod is None:
        path = build()
        if path is None:
            raise RuntimeError("oracle/_ref/view_tools_cython.so is not built and DEMON_REF_SRC names no reference tree")
        spec = importlib.util.spec_from_file_location("view_tools_cython", path)
        _mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(_mod)
    return _mod


def available():
    return have_module() or bool(_STORE.entries())


def _key(arrays, ints):
    h = hashlib.sha256(("visible_points_mask|%s" % (ints,)).encode())
    for a in arrays:
        a = np.ascontiguousarray(a)
        h.update(("%s|%s" % (a.dtype.str, a.shape)).encode())
        h.update(a.tobytes())
    return h.hexdigest()


def reference_mask(depth, K1, R1, t1, K2, R2, t2, borderx=0, bordery=0):
    """compute_visible_points_mask(view1, view2, borderx, bordery) of the reference's Cython for one view pair: depth [h,w]
    float32 camera z of view 1 (view 2 has the same size).  Returns the uint8 mask, or its Recorded digest."""
    depth = np.ascontiguousarray(depth, dtype=np.float32)
    arrays = [depth] + [np.asarray(a) for a in (K1, R1, t1, K2, R2, t2)]
    key = _key(arrays, (int(borderx), int(bordery)))
    if not have_module():
        return Recorded(_STORE.lookup(key, "result for this compute_visible_points_mask call"))
    v1 = View(R=np.asarray(R1), t=np.asarray(t1), K=np.asarray(K1), image=None, depth=depth, depth_metric='camera_z')
    v2 = View(R=np.asarray(R2), t=np.asarray(t2), K=np.asarray(K2), image=None, depth=depth, depth_metric='camera_z')
    mask = np.asarray(module().compute_visible_points_mask(v1, v2, borderx, bordery))
    record(key, entry(mask))
    return mask


def operands(K1, R1, t1, K2, R2, t2):
    """The float32 operands the .pyx wrapper passes to its loop (view_tools_cython.pyx:81-102)."""
    P2 = np.empty((3, 4), dtype=np.float32)
    P2[:, 0:3] = R2
    P2[:, 3:4] = np.asarray(t2).reshape((3, 1))
    P2 = np.asarray(K2).dot(P2)
    return (np.asarray(K1).astype(np.float32), np.asarray(R1).astype(np.float32), np.asarray(t1).astype(np.float32),
            P2.astype(np.float32))


def visible_points_mask_numpy(depth, K1, R1, t1, P2, width2, height2, borderx=0, bordery=0):
    """_compute_visible_points_mask (view_tools_cython.pyx:9-58) over the whole image at once: float32 operations in the
    loop's order (every numpy operation here is float32 op float32 -> float32, rounded like C's)."""
    f = np.float32
    depth = np.asarray(depth, dtype=f)
    K1, R1, t1, P2 = (np.asarray(a, dtype=f) for a in (K1, R1, t1, P2))
    RT = R1.T
    h, w = depth.shape
    px = (np.arange(w) + 0.5).astype(f)[None, :]
    py = (np.arange(h) + 0.5).astype(f)[:, None]
    with np.errstate(all='ignore'):
        d = depth
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
        inside = (u > f(borderx)) & (v > f(bordery)) & (u < f(width2 - borderx)) & (v < f(height2 - bordery))
    return (valid & front & inside).astype(np.uint8)


def edge_cases():
    """View pairs the tests hold the device kernel, the numpy restatement and the reference's Cython to: (depth, K1, R1,
    t1, K2, R2, t2, borderx, bordery) with float64 cameras, camera-z float32 depth."""
    from demon_b200.evaluation import angleaxis_to_rotation_matrix, intrinsics_vector_to_K
    rng = np.random.RandomState(20171)
    cases = []

    def depth_map(h, w, lo=0.3, hi=8.0):
        d = rng.uniform(lo, hi, (h, w)).astype(np.float32)
        d[rng.rand(h, w) < 0.04] = np.nan
        d[rng.rand(h, w) < 0.03] = 0.0
        d[rng.rand(h, w) < 0.03] *= -1.0
        d[rng.rand(h, w) < 0.01] = np.inf
        return d
    sun3d = np.array([0.891, 1.188, 0.5, 0.5])
    # identity view 1, moving view 2 (the evaluation's use), with and without borders
    for h, w in ((7, 9), (48, 64), (31, 17)):
        K = intrinsics_vector_to_K(sun3d, w, h)
        R = angleaxis_to_rotation_matrix(rng.normal(0, 0.2, 3))
        t = rng.normal(0, 0.5, 3)
        for b in ((0, 0), (2, 3)):
            cases.append((depth_map(h, w), K, np.eye(3), np.zeros(3), K, R, t) + b)
    # non-identity R1 / t1 and different K2
    for h, w in ((20, 30), (33, 41)):
        K1 = intrinsics_vector_to_K(np.array([0.8, 1.1, 0.45, 0.55]), w, h)
        K2 = intrinsics_vector_to_K(sun3d, w, h)
        cases.append((depth_map(h, w, 2.0, 8.0), K1, angleaxis_to_rotation_matrix(rng.normal(0, 0.05, 3)), rng.normal(0, 0.1, 3), K2,
                      angleaxis_to_rotation_matrix(rng.normal(0, 0.05, 3)), rng.normal(0, 0.1, 3), 1, 1))
    # points behind the second camera: it sits 5 units in front of view 1 looking back along z
    h, w = 16, 24
    K = intrinsics_vector_to_K(sun3d, w, h)
    cases.append((depth_map(h, w, 0.5, 10.0), K, np.eye(3), np.zeros(3), K, angleaxis_to_rotation_matrix(np.array([0.0, np.pi, 0.0])),
                  np.array([0.0, 0.0, 5.0]), 0, 0))
    # projections exactly on the border: depth 1, fx = fy = 2 and a -1/4 translation put every point at u = x, v = y
    # (exact in float32), so the strict tests drop column / row `border` and keep the next one
    h, w = 12, 10
    K = np.array([[2.0, 0.0, w / 2], [0.0, 2.0, h / 2], [0.0, 0.0, 1.0]])
    ones = np.ones((h, w), dtype=np.float32)
    for b in ((0, 0), (2, 3)):
        cases.append((ones, K, np.eye(3), np.zeros(3), K, np.eye(3), np.array([-0.25, -0.25, 0.0])) + b)
    # a 480x640 ground truth at the sun3d intrinsics
    h, w = 480, 640
    K = intrinsics_vector_to_K(sun3d, w, h)
    yy, xx = np.mgrid[0:h, 0:w]
    d = (2.0 + np.sin(xx / 50.0) + 0.5 * np.cos(yy / 30.0)).astype(np.float32)
    d[rng.rand(h, w) < 0.02] = np.nan
    cases.append((d, K, np.eye(3), np.zeros(3), K, angleaxis_to_rotation_matrix(np.array([0.02, -0.1, 0.01])),
                  np.array([0.3, -0.05, 0.1]), 0, 0))
    return cases
