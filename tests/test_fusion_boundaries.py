"""CPU: the grid-aligned plane scene of tests/fusion_boundary_scenes.py, whose fused state is known in exact arithmetic,
against the numpy restatements of integration, allocation, marching cubes and ray casting (sequence_oracle,
sparse_tsdf_oracle, raycast_oracle).  The scene reaches the rules' boundaries exactly: voxels on u = 0 and u = w,
sdf = -trunc, f = +-1, band cells that end on block faces, and tsdf corners at exactly 0.  So the GPU tests of the same
scene compare the kernels with exact arithmetic, not only with a restatement of the kernels' own order."""
import numpy as np
import pytest

import fusion_boundary_scenes as fb
import raycast_oracle as ro
import sequence_oracle as so
import sparse_tsdf_oracle as sp

f32 = np.float32


def bits(a):
    return np.ascontiguousarray(a, dtype=f32).view(np.uint32)


@pytest.fixture(scope="module")
def plane():
    d, K, R, t, img = fb.plane_frames()
    nx, ny, nz = fb.DIMS
    ts, W = np.zeros((nz, ny, nx), f32), np.zeros((nz, ny, nx), f32)
    so.integrate(ts, W, None, fb.ORIGIN, fb.VOXEL, fb.TRUNC, d, K, R, t)
    return (d, K, R, t, img), ts, W


def test_plane_closed_form_equals_the_integration_oracle(plane):
    _, ts, W = plane
    ref_t, ref_w, edges = fb.plane_state(fb.box_grid())
    assert np.array_equal(bits(ts).reshape(-1), bits(ref_t)) and np.array_equal(bits(W).reshape(-1), bits(ref_w))
    # the scene reaches every boundary of the rule, many times
    assert min(edges.values()) >= 20, edges
    seen = ref_w > 0
    assert (ref_t[seen] == -1).any() and (ref_t[seen] == 1).any() and (ref_t[seen] == 0).any()
    assert len(np.unique(ref_w)) > 30 and ref_w.max() == 129 and (~seen).any()


def test_plane_closed_form_blocks_equal_the_allocation_oracle():
    d, K, R, t, _ = fb.plane_frames()
    ref, faces = fb.plane_blocks()
    blocks, skipped = sp.allocate(d, K, R, t, fb.ORIGIN, fb.VOXEL, fb.TRUNC)
    assert skipped == 0 and blocks == ref
    assert faces["lo"] > 1000 and faces["hi"] > 1000, faces
    # the band's near end, z = 1.5 - 2 voxels, is the face z = 1.25 of block 1: the blocks in front stay unallocated
    assert {b[2] for b in blocks} == {1, 2}


def test_plane_closed_form_on_blocks_equals_the_block_oracle():
    d, K, R, t, _ = fb.plane_frames()
    blocks = np.array(sorted(fb.plane_blocks()[0]))
    m = len(blocks)
    ts, W = np.zeros((m, 8, 8, 8), f32), np.zeros((m, 8, 8, 8), f32)
    sp.integrate_blocks(ts, W, None, blocks, fb.ORIGIN, fb.VOXEL, fb.TRUNC, d, K, R, t)
    ref_t, ref_w, _ = fb.plane_state(fb.block_grid(blocks))
    assert np.array_equal(bits(ts).reshape(-1), bits(ref_t)) and np.array_equal(bits(W).reshape(-1), bits(ref_w))
    assert (ref_w > 0).mean() > 0.2


def test_plane_oracle_mesh_is_the_plane(plane):
    """Marching cubes on corners at exactly 0 (outside) over corners at -1/4: two triangles per cube of the slice z = 2
    whose corners were all seen, every vertex at mu = 0 on a voxel of the plane."""
    _, ts, W = plane
    v, c, f = so.marching_cubes(ts, W, None, fb.ORIGIN, fb.VOXEL)
    cubes = fb.plane_mesh_cubes(W)
    assert cubes.sum() > 500 and f.shape[0] == 2 * cubes.sum()
    assert (v[:, 2] == fb.PLANE_Z).all()
    g = (v[:, :2].astype(np.float64) - np.array(fb.ORIGIN[:2])) / fb.VOXEL
    assert np.array_equal(g, np.round(g))


@pytest.mark.parametrize("storage", ["dense", "sparse"])
def test_plane_oracle_raycast_hits_the_plane_on_axis(plane, storage):
    """Step 1 from near = 0.5, a voxel plane: the on-axis ray samples the voxels themselves, reads tsdf 0 at z = 2 and
    -1/4 one voxel further, and its crossing is z = 2 exactly."""
    _, ts, W = plane
    if storage == "dense":
        vol = ro.Dense(ts, W)
        far = ro.dense_far(fb.DIMS, fb.ORIGIN, fb.VOXEL, *fb.plane_render_cameras()[1:])
    else:
        blocks = np.array(sorted(fb.plane_blocks()[0]))
        bt, bw, _ = fb.plane_state(fb.block_grid(blocks))
        vol = ro.Sparse(blocks, bt, bw)
        far = ro.sparse_far(blocks, fb.ORIGIN, fb.VOXEL, *fb.plane_render_cameras()[1:])
    K, R, t = fb.plane_render_cameras()
    out = ro.raycast(vol, fb.ORIGIN, fb.VOXEL, K, R, t, 0.5, far, 1.0, fb.H, fb.W)
    assert (out["depth"][:, 11, 15] == fb.PLANE_Z).all()
    assert np.isfinite(out["depth"]).mean() > 0.5
