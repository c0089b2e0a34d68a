"""GPU: the fusion kernels (csrc/fusion.cu) past their internal boundaries, bit for bit against the numpy restatements
(sequence_oracle, sparse_tsdf_oracle, raycast_oracle) and, on the grid-aligned plane, against exact arithmetic
(tests/fusion_boundary_scenes.py).

* More than 64 frames per call: the cameras are staged in shared memory 64 frames at a time, so calls of 63, 64, 65, 129
  frames (each frame with its own intrinsics) run one, two and three chunks; split calls give one call's bytes.
* The plane: voxels on u = 0 and u = w, sdf = -trunc, f = +-1, band cells ending on block faces, tsdf corners at exactly
  0, and ray samples on voxel planes and block faces.
* Meshes of more than 1024 tiles of 2048 cubes, where the one-CTA offset scan sums several tiles per thread."""
import numpy as np
import pytest
import torch

import fusion_boundary_scenes as fb
import raycast_oracle as ro
import sequence_oracle as so
import sparse_tsdf_oracle as sp
from demon_b200 import _lib, sequence

pytestmark = pytest.mark.gpu
f32 = np.float32


def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(x):
    return None if x is None else x.cpu().numpy()


def bits(a):
    return np.ascontiguousarray(host(a) if isinstance(a, torch.Tensor) else a, dtype=f32).view(np.uint32).reshape(-1)


def same(a, b):
    """Equal bytes, NaN matching NaN whatever its payload."""
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype.kind != "f":
        return a.shape == b.shape and np.array_equal(a, b)
    na, nb = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))


def frames(d, K, R, t, img, sl=slice(None), color=True):
    return cuda(d[sl]), cuda(K[sl]), cuda(R[sl]), cuda(t[sl]), cuda(img[sl]) if color else None


def sorted_by_key(b):
    return np.array_equal(np.lexsort((b[:, 0], b[:, 1], b[:, 2])), np.arange(b.shape[0]))


def triangles(v, c, f):
    """The mesh as a sorted multiset of triangles: rows of 9 vertex floats' bits and 9 colour bytes."""
    v, f = np.asarray(v), np.asarray(f)
    rows = v[f].reshape(-1, 9).view(np.uint32)
    if c is not None:
        rows = np.concatenate([rows, np.asarray(c)[f].reshape(-1, 9).astype(np.uint32)], axis=1)
    return rows[np.lexsort(rows.T[::-1])]


def dense_at(dense, g, name):
    """The dense volume's field `name` at grid coordinates g [N,3], as numpy."""
    x = getattr(dense, name)
    idx = tuple(torch.from_numpy(g[:, a]).cuda() for a in (2, 1, 0))
    return host(x[idx])


# ---- A: more than 64 frames per call ----------------------------------------------------------------------------------
ORIGIN_A, VOXEL_A, DIMS_A = (-1.2, -1.2, -1.2), 0.043, (49, 50, 51)
TRUNC_A = f32(3 * f32(VOXEL_A))
COUNTS = (63, 64, 65, 129)


@pytest.fixture(scope="module")
def spheres():
    """129 sphere views of 48x64 and the oracle's state (colour) after the first n of them, for every n of COUNTS."""
    d, K, R, t, img = fb.varied_sphere_views(129)
    nx, ny, nz = DIMS_A
    ts, W, col = np.zeros((nz, ny, nx), f32), np.zeros((nz, ny, nx), f32), np.zeros((nz, ny, nx, 3), f32)
    state, done = {}, 0
    for n in COUNTS:
        sl = slice(done, n)
        so.integrate(ts, W, col, ORIGIN_A, VOXEL_A, TRUNC_A, d[sl], K[sl], R[sl], t[sl], img[sl])
        state[n], done = (ts.copy(), W.copy(), col.copy()), n
    return (d, K, R, t, img), state


@pytest.mark.parametrize("color", [True, False])
@pytest.mark.parametrize("n", COUNTS)
def test_dense_call_of_n_frames_equals_the_oracle(spheres, n, color):
    views, state = spheres
    vol = sequence.TsdfVolume(DIMS_A, ORIGIN_A, VOXEL_A, color=color)
    vol.integrate(*frames(*views, slice(0, n), color))
    ts, W, col = state[n]
    assert np.array_equal(bits(vol.tsdf), bits(ts)) and np.array_equal(bits(vol.weight), bits(W))
    if color:
        assert np.array_equal(bits(vol.color), bits(col))
    if n > 64:   # the frames of the second and third chunk change voxels
        assert (W != state[64][1]).sum() > 1000
    _lib.check_errors()


@pytest.mark.parametrize("split", [(64, 65), (1, 128), (63, 66)])
def test_dense_split_calls_give_the_bytes_of_one_call(spheres, split):
    views, state = spheres
    one = sequence.TsdfVolume(DIMS_A, ORIGIN_A, VOXEL_A)
    one.integrate(*frames(*views))
    two = sequence.TsdfVolume(DIMS_A, ORIGIN_A, VOXEL_A)
    two.integrate(*frames(*views, slice(0, split[0])))
    two.integrate(*frames(*views, slice(split[0], None)))
    for name, ref in zip(("tsdf", "weight", "color"), state[129]):
        assert np.array_equal(bits(getattr(two, name)), bits(getattr(one, name))), name
        assert np.array_equal(bits(getattr(one, name)), bits(ref)), name
    _lib.check_errors()


def check_sparse_against_oracle_and_dense(views, color, oracle):
    """One SparseTsdfVolume call: the block set and skipped pixels of sparse_tsdf_oracle, blocks in key order, and every
    stored voxel equal to a dense volume of the same call on the same grid and to the oracle's dense state `oracle`
    (tsdf, weight, color on DIMS_A)."""
    d, K, R, t, _ = views
    vol = sequence.SparseTsdfVolume(VOXEL_A, ORIGIN_A, color=color)
    vol.integrate(*frames(*views, color=color))
    ref, skipped = sp.allocate(d, K, R, t, ORIGIN_A, VOXEL_A, vol.trunc)
    b = host(vol.blocks)
    assert set(map(tuple, b.tolist())) == ref and len(ref) == b.shape[0] and sorted_by_key(b)
    assert vol.last_skipped_pixels == skipped
    dense = sequence.TsdfVolume(DIMS_A, ORIGIN_A, VOXEL_A, trunc=vol.trunc, color=color)
    dense.integrate(*frames(*views, color=color))
    g = fb.block_grid(b)
    assert g.min() >= 0 and (g.max(axis=0) < np.array(DIMS_A)).all()   # the dense box holds every block
    for name, ref in zip(("tsdf", "weight", "color"), oracle):
        if name != "color" or color:
            got = bits(getattr(vol, name))
            assert np.array_equal(got, bits(dense_at(dense, g, name))), name
            assert np.array_equal(got, bits(ref[g[:, 2], g[:, 1], g[:, 0]])), name
    assert (host(vol.weight) > 0).mean() > 0.2
    return dense


@pytest.mark.parametrize("color", [True, False])
@pytest.mark.parametrize("n", COUNTS)
def test_sparse_call_of_n_frames_equals_the_oracle_and_the_dense_volume(spheres, n, color):
    (d, K, R, t, img), state = spheres
    sl = slice(0, n)
    check_sparse_against_oracle_and_dense((d[sl], K[sl], R[sl], t[sl], img[sl]), color, state[n])
    _lib.check_errors()


def test_70_frames_of_192x256_in_one_call():
    views = fb.varied_sphere_views(70, 192, 256, seed=2)
    nx, ny, nz = DIMS_A
    ts, W, col = np.zeros((nz, ny, nx), f32), np.zeros((nz, ny, nx), f32), np.zeros((nz, ny, nx, 3), f32)
    so.integrate(ts, W, col, ORIGIN_A, VOXEL_A, TRUNC_A, *views)
    dense = check_sparse_against_oracle_and_dense(views, True, (ts, W, col))
    for name, ref in zip(("tsdf", "weight", "color"), (ts, W, col)):
        assert np.array_equal(bits(getattr(dense, name)), bits(ref)), name
    _lib.check_errors()


# ---- B: the grid-aligned plane, exact ---------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def plane():
    """The plane's 129 frames, the oracle's dense state (colour) and the closed form's tsdf and weight."""
    d, K, R, t, img = fb.plane_frames()
    nx, ny, nz = fb.DIMS
    ts, W, col = np.zeros((nz, ny, nx), f32), np.zeros((nz, ny, nx), f32), np.zeros((nz, ny, nx, 3), f32)
    so.integrate(ts, W, col, fb.ORIGIN, fb.VOXEL, fb.TRUNC, d, K, R, t, img)
    closed_t, closed_w, _ = fb.plane_state(fb.box_grid())
    return (d, K, R, t, img), (ts, W, col), (closed_t, closed_w)


@pytest.mark.parametrize("color", [True, False])
def test_plane_dense_equals_the_closed_form_and_the_oracle(plane, color):
    views, (ts, W, col), (closed_t, closed_w) = plane
    vol = sequence.TsdfVolume(fb.DIMS, fb.ORIGIN, fb.VOXEL, trunc=fb.TRUNC, color=color)
    vol.integrate(*frames(*views, color=color))
    assert np.array_equal(bits(vol.tsdf), bits(closed_t)) and np.array_equal(bits(vol.weight), bits(closed_w))
    assert np.array_equal(bits(vol.tsdf), bits(ts)) and np.array_equal(bits(vol.weight), bits(W))
    if color:
        assert np.array_equal(bits(vol.color), bits(col))
    # marching cubes on corners at exactly 0: the oracle's mesh, and the closed form's plane
    v, c, f = (host(x) for x in vol.mesh())
    vr, cr, fr = so.marching_cubes(ts, W, col if color else None, fb.ORIGIN, fb.VOXEL)
    assert np.array_equal(bits(v), bits(vr)) and np.array_equal(f, fr)
    if color:
        assert np.array_equal(c, cr)
    assert f.shape[0] == 2 * fb.plane_mesh_cubes(W).sum() > 1000 and (v[:, 2] == fb.PLANE_Z).all()
    _lib.check_errors()


def test_plane_sparse_equals_the_closed_form_and_the_oracle(plane):
    views = plane[0]
    d, K, R, t, img = views
    vol = sequence.SparseTsdfVolume(fb.VOXEL, fb.ORIGIN, trunc=fb.TRUNC)
    vol.integrate(*frames(*views))
    b = host(vol.blocks)
    ref, faces = fb.plane_blocks()
    assert set(map(tuple, b.tolist())) == ref == sp.allocate(d, K, R, t, fb.ORIGIN, fb.VOXEL, fb.TRUNC)[0] and len(ref) == b.shape[0]
    assert faces["lo"] > 0 and faces["hi"] > 0 and vol.last_skipped_pixels == 0
    g = fb.block_grid(b)
    closed_t, closed_w, _ = fb.plane_state(g)
    assert np.array_equal(bits(vol.tsdf), bits(closed_t)) and np.array_equal(bits(vol.weight), bits(closed_w))
    m = b.shape[0]
    ts, W, col = np.zeros((m, 8, 8, 8), f32), np.zeros((m, 8, 8, 8), f32), np.zeros((m, 8, 8, 8, 3), f32)
    sp.integrate_blocks(ts, W, col, b, fb.ORIGIN, fb.VOXEL, fb.TRUNC, d, K, R, t, img)
    assert np.array_equal(bits(vol.color), bits(col))
    # the mesh: the oracle's on a box around the blocks holding their state, weight 0 elsewhere (a cube with a corner
    # outside the blocks is skipped either way); every coordinate is dyadic, so the shifted origin is exact
    lo = b.min(axis=0)
    nx, ny, nz = 8 * (b.max(axis=0) - lo + 1)
    bt, bw, bc = np.zeros((nz, ny, nx), f32), np.zeros((nz, ny, nx), f32), np.zeros((nz, ny, nx, 3), f32)
    gl = g - 8 * lo
    bt[gl[:, 2], gl[:, 1], gl[:, 0]], bw[gl[:, 2], gl[:, 1], gl[:, 0]] = ts.reshape(-1), W.reshape(-1)
    bc[gl[:, 2], gl[:, 1], gl[:, 0]] = col.reshape(-1, 3)
    origin = tuple(o + 8 * fb.VOXEL * float(x) for o, x in zip(fb.ORIGIN, lo))
    v, c, f = (host(x) for x in vol.mesh())
    vr, cr, fr = so.marching_cubes(bt, bw, bc, origin, fb.VOXEL)
    assert f.shape[0] == fr.shape[0] > 1000 and (v[:, 2] == fb.PLANE_Z).all()
    assert np.array_equal(triangles(v, c, f), triangles(vr, cr, fr))
    _lib.check_errors()


@pytest.mark.parametrize("storage", ["dense", "sparse"])
def test_plane_raycast_at_step_1_equals_the_oracle(plane, storage):
    """near = 0.5 is a voxel plane, so the on-axis ray samples every voxel plane (trilinear weights 0) and, in the sparse
    volume, marches through the unallocated block 0 in front of the plane to its face z = 1.25."""
    views = plane[0]
    if storage == "dense":
        vol = sequence.TsdfVolume(fb.DIMS, fb.ORIGIN, fb.VOXEL, trunc=fb.TRUNC)
    else:
        vol = sequence.SparseTsdfVolume(fb.VOXEL, fb.ORIGIN, trunc=fb.TRUNC)
    vol.integrate(*frames(*views))
    K, R, t = fb.plane_render_cameras()
    got = vol.raycast(cuda(K), cuda(R), cuda(t), height=fb.H, width=fb.W, near=0.5, step=1.0)
    far = host(vol.default_far(cuda(R), cuda(t)))
    if storage == "dense":
        state = ro.Dense(host(vol.tsdf), host(vol.weight), host(vol.color))
    else:
        state = ro.Sparse(host(vol.blocks), host(vol.tsdf), host(vol.weight), host(vol.color))
        assert host(vol.blocks)[:, 2].min() == 1
    ref = ro.raycast(state, fb.ORIGIN, fb.VOXEL, K, R, t, 0.5, far, 1.0, fb.H, fb.W)
    for k in ("depth", "normals", "colors"):
        assert same(host(got[k]), ref[k]), k
    dep = host(got["depth"])
    assert (dep[:, 11, 15] == fb.PLANE_Z).all() and np.isfinite(dep).mean() > 0.5 and np.isfinite(ref["normals"]).any()
    _lib.check_errors()


# ---- C: meshes of more than 1024 tiles --------------------------------------------------------------------------------
ORIGIN_C, VOXEL_C, DIMS_C = (0.1, -0.2, 0.3), 0.01, (131, 137, 130)   # 2 280 720 cubes: 1114 tiles, the last one ragged


@pytest.fixture(scope="module")
def field():
    s, w, c = fb.two_spheres(DIMS_C)
    return (s, w, c), so.marching_cubes(s, w, c, ORIGIN_C, VOXEL_C)


@pytest.mark.parametrize("color", [True, False])
def test_dense_mesh_past_1024_tiles_equals_the_oracle(field, color):
    (s, w, c), (vr, cr, fr) = field
    nx, ny, nz = DIMS_C
    cubes = (nx - 1) * (ny - 1) * (nz - 1)
    assert -(-cubes // 2048) > 1024 and cubes % 2048
    assert (np.signbit(s) & (s == 0) & (w > 0)).any() and (~np.signbit(s) & (s == 0) & (w > 0)).any()
    vol = sequence.TsdfVolume(DIMS_C, ORIGIN_C, VOXEL_C, color=color)
    vol.tsdf.copy_(cuda(s))
    vol.weight.copy_(cuda(w))
    if color:
        vol.color.copy_(cuda(c))
    v, cg, f = (host(x) for x in vol.mesh())
    assert np.array_equal(bits(v), bits(vr)) and np.array_equal(f, fr)
    if color:
        assert np.array_equal(cg, cr)
    # triangles in the tiles past 1024 (cube layers z >= 119) and in the last tile (layer 128, rows y >= 127)
    g = (vr.astype(np.float64) - np.array(ORIGIN_C)) / VOXEL_C
    assert (g[:, 2] > 119.5).sum() > 100 and ((g[:, 1] > 127.05) & (g[:, 2] > 128.05)).sum() > 10
    _lib.check_errors()


def test_sparse_mesh_past_1024_tiles_equals_the_dense_mesh():
    """A sphere at 5 mm voxels from 24 views of 192x256: about 9 000 blocks, over 2 000 tiles; the dense box around the
    blocks meshes over 10 000 tiles."""
    views = fb.varied_sphere_views(24, 192, 256)
    origin, vs = (-0.75, -0.75, -0.75), 0.005
    vol = sequence.SparseTsdfVolume(vs, origin)
    vol.integrate(*frames(*views))
    b = host(vol.blocks)
    assert b.shape[0] > 4 * 1024 and b.min() >= 0 and vol.last_skipped_pixels == 0
    dense = sequence.TsdfVolume(tuple(int(8 * (x + 1)) for x in b.max(axis=0)), origin, vs, trunc=vol.trunc)
    dense.integrate(*frames(*views))
    ms, md = [[host(x) for x in m] for m in (vol.mesh(), dense.mesh())]
    assert ms[2].shape[0] > 100000 and ms[2].shape == md[2].shape
    assert np.array_equal(ms[2].reshape(-1), np.arange(3 * ms[2].shape[0]))
    assert np.array_equal(triangles(*ms), triangles(*md))
    _lib.check_errors()
