"""CPU: the indexed-mesh oracle (tests/indexed_mesh_oracle.py) against marching cubes' soup (sequence_oracle), the
topology and normals of fused scenes, and the argument checks of the indexed-mesh calls."""
import numpy as np
import pytest
import torch

import fusion_boundary_scenes as fb
import indexed_mesh_oracle as imo
import sequence_oracle as so
from demon_b200 import sequence, vis

f32 = np.float32
DIMS, ORIGIN, VOXEL = (48, 48, 48), (-1.0, -1.0, -1.0), 2.0 / 47


@pytest.fixture(scope="module")
def sphere():
    """so.sphere_views (a sphere of radius 0.6) fused into a 48^3 box, with colour."""
    d, K, R, t, img = so.sphere_views()
    nx, ny, nz = DIMS
    s, w, c = np.zeros((nz, ny, nx), f32), np.zeros((nz, ny, nx), f32), np.zeros((nz, ny, nx, 3), f32)
    so.integrate(s, w, c, ORIGIN, VOXEL, f32(3 * f32(VOXEL)), d, K, R, t, img)
    return s, w, c


def test_oracle_vertices_of_faces_are_the_soup(sphere):
    s, w, c = sphere
    v, col, f = so.marching_cubes(s, w, c, ORIGIN, VOXEL)
    m = imo.dense(s, w, c, ORIGIN, VOXEL)
    assert np.array_equal(m["vertices"][m["faces"]].reshape(-1, 3).view(np.uint32), v.view(np.uint32))
    assert np.array_equal(m["colors"][m["faces"]].reshape(-1, 3), col)
    # every soup corner of one edge is the same bits: the edge is the vertex
    assert np.array_equal(np.unique(m["soup_keys"]).size, m["vertices"].shape[0])
    assert np.all(np.diff(np.unique(m["soup_keys"])) > 0)


def test_fused_sphere_is_closed_by_index(sphere):
    s, w, c = sphere
    m = imo.dense(s, w, c, ORIGIN, VOXEL)
    f = m["faces"].astype(np.int64)
    nv, nf = m["vertices"].shape[0], f.shape[0]
    e = np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), axis=1)
    _, counts = np.unique(e, axis=0, return_counts=True)
    assert (counts == 2).all()
    assert nv - counts.size + nf == 2 and 2 * nv == nf + 4   # V = F/2 + 2: a sixth of the soup's 3F vertices
    assert np.array_equal(np.unique(f), np.arange(nv))


def test_sphere_normals_are_radial(sphere):
    """The normal of a vertex on a fused sphere is within 25 degrees of its radial direction.  The bound: the fused tsdf
    of a sphere of radius r = 14 voxels is, near the surface, a truncated distance along each camera's rays, whose
    gradient leans from the radial direction by at most the angle between a ray and the normal where the surface
    is seen (under 20 degrees here: the cameras stand 5 radii away and a voxel's update comes from views within
    about 60 degrees of its normal, each with weight 1), and the central differences over 2 voxels on a sphere of
    14 voxels add at most atan(1/14), about 4 degrees."""
    s, w, c = sphere
    m = imo.dense(s, w, c, ORIGIN, VOXEL)
    n, v = m["normals"], m["vertices"].astype(np.float64)
    ok = ~np.isnan(n).any(axis=1)
    assert ok.mean() > 0.95
    assert np.allclose(np.linalg.norm(n[ok], axis=1), 1, atol=1e-6)
    radial = v[ok] / np.linalg.norm(v[ok], axis=1, keepdims=True)
    angle = np.degrees(np.arccos(np.clip((n[ok] * radial).sum(axis=1), -1, 1)))
    assert angle.max() < 25.0 and np.median(angle) < 5.0


def test_plane_normals_are_exactly_minus_z():
    """The grid-aligned plane's closed-form state: a vertex per column at mu = 0 on the plane's voxels, and every normal
    that is not NaN exactly -e_z (towards the cameras, which stand at z = 0 and look along +z)."""
    g = fb.box_grid()
    tsdf, weight, _ = fb.plane_state(g)
    nx, ny, nz = fb.DIMS
    s, w = tsdf.reshape(nz, ny, nx), weight.reshape(nz, ny, nx)
    m = imo.dense(s, w, None, fb.ORIGIN, fb.VOXEL)
    n = m["normals"]
    ok = ~np.isnan(n).any(axis=1)
    assert ok.sum() > 100
    assert np.array_equal(n[ok], np.tile(np.array([0, 0, -1], f32), (ok.sum(), 1)))
    z = (m["vertices"][:, 2] - f32(fb.ORIGIN[2])) / f32(fb.VOXEL)
    assert np.all(z == (fb.PLANE_Z - fb.ORIGIN[2]) / fb.VOXEL)   # mu = 0: on the plane's voxels
    v, _, f = so.marching_cubes(s, w, None, fb.ORIGIN, fb.VOXEL)
    assert np.array_equal(m["vertices"][m["faces"]].reshape(-1, 3), v)


def test_coincident_vertices_stay_separate():
    """A voxel at exactly 0 whose +x and +z neighbours are inside: both edges give mu = 0, so two vertices at the same
    point, which welding by coordinates would merge."""
    s = np.ones((3, 3, 3), f32)
    s[1, 1, 1] = 0.0
    s[1, 1, 2] = s[2, 1, 1] = -1.0
    w = np.ones_like(s)
    m = imo.dense(s, w, None, (0, 0, 0), 1.0)
    v = m["vertices"]
    _, first, counts = np.unique(v, axis=0, return_index=True, return_counts=True)
    assert (counts > 1).any() and v.shape[0] > first.size
    assert np.array_equal(m["vertices"][m["faces"]].reshape(-1, 3), so.marching_cubes(s, w, None, (0, 0, 0), 1.0)[0])
    n = m["normals"]
    assert np.isnan(n).all()   # every vertex reads a voxel outside the 3^3 box


def test_sparse_oracle_orders_by_key():
    """Blocks laid into a box and back: the vertices ascend in (block key, local index, axis)."""
    s = np.full((2, 8, 8, 8), 0.5, f32)
    s[0, :, :, 5:] = -0.5   # a wall inside block 0, x = 5..7, continued into block 1 at x = 8 ...
    s[1] = -0.5
    s[1, :, :, 2:] = 0.5    # ... and ending at x = 10
    w = np.ones_like(s)
    blocks = np.array([[-1, 0, 0], [-2, 0, 0]])   # pool order is not key order
    m = imo.sparse(blocks, s[::-1].copy(), w, None, (0, 0, 0), 1.0)
    d = imo.dense(np.concatenate([s[0], s[1]], axis=2), np.ones((8, 8, 16), f32), None, (-16, 0, 0), 1.0)
    assert m["faces"].shape == d["faces"].shape and m["vertices"].shape == d["vertices"].shape

    def rows(x):
        x = x.reshape(x.shape[0], -1)
        return x[np.lexsort(x.T[::-1])]
    assert np.array_equal(rows(m["vertices"][m["faces"]]), rows(d["vertices"][d["faces"]]))   # the same triangles
    key = imo.packed_keys(np.floor(m["vertices"] / 8).astype(np.int64))
    assert np.all(np.diff(key) >= 0) and key[0] != key[-1]


def test_arguments_are_checked_before_any_device():
    vol = sequence.SparseTsdfVolume(0.1)
    for bad in ("yes", 1, None):
        with pytest.raises(ValueError, match="normals"):
            vol.indexed_mesh(normals=bad)
    assert vol._pool is None
    with pytest.raises(ValueError, match="indexed_mesh"):
        sequence.reconstruct(None, torch.zeros((2, 4, 4, 3), dtype=torch.uint8), np.eye(3), indexed_mesh="yes")
    with pytest.raises(ValueError, match="normals"):
        vis.write_ply("/nonexistent/x.ply", np.zeros((3, 3), f32), normals=np.zeros((2, 3), f32))
