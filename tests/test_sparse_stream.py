"""CPU: the reach rule that streams a sparse TSDF volume's blocks (tests/sparse_stream_oracle.py, the numpy restatement of
include/demon_b200.h: demon_sparse_tsdf_reach_f32) is conservative and tight.  Every block holding a voxel that
sequence_oracle.integrate changes, every block sparse_tsdf_oracle.allocate inserts and every block holding a corner of a
sample raycast_oracle.raycast evaluates is reached; in a ring corridor, most blocks are not reached from the far side."""
from unittest import mock

import numpy as np
import pytest

import fusion_boundary_scenes as fb
import raycast_oracle as ro
import sequence_oracle as so
import sparse_stream_oracle as ss
import sparse_tsdf_oracle as sp
from demon_b200 import sequence

f32 = np.float32


def sphere_views_with_bad_pixels(n, seed):
    d, K, R, t, img = so.sphere_views(n=n, seed=seed)
    rng = np.random.RandomState(seed)
    for bad in (np.nan, 0.0, -1.0, np.inf):
        m = rng.rand(*d.shape) < 0.03
        d[m & np.isfinite(d)] = bad
    return d, K, R, t, img


def box_around(blocks, pad=1):
    """A dense box (dims, grid offset in voxels) covering the blocks with `pad` blocks around them."""
    lo, hi = blocks.min(axis=0) - pad, blocks.max(axis=0) + pad + 1
    return tuple(int(x) for x in 8 * (hi - lo)), 8 * lo


def check_integration_reach(d, K, R, t, origin, vs, trunc):
    """Per frame, over every block of a box around the allocated ones: the blocks of the voxels integration changes and
    the blocks allocation inserts are all reached."""
    n, h, w = d.shape
    alloc, _ = sp.allocate(d, K, R, t, origin, vs, trunc)
    blocks = np.array(sorted(alloc), np.int64)
    dims, g0 = box_around(blocks)
    lo = g0 // 8
    grid = np.stack(np.meshgrid(*(np.arange(dims[a] // 8) + lo[a] for a in range(3)), indexing="ij"), axis=-1).reshape(-1, 3)
    tiles = ss.depth_tiles(d)
    changed_total = 0
    for f in range(n):
        sl = slice(f, f + 1)
        reached = ss.reach(grid, origin, vs, trunc, tiles[sl], K[sl], R[sl], t[sl], h, w)[0]
        got = set(map(tuple, grid[reached].tolist()))
        ts, W = np.zeros(dims[::-1], f32), np.zeros(dims[::-1], f32)
        g = [np.asarray(p) for p in np.meshgrid(*(np.arange(dims[a]) + g0[a] for a in (2, 1, 0)), indexing="ij")]
        exact = [np.asarray(origin, f32)[a] + f32(vs) * g[2 - a].reshape(-1).astype(f32) for a in range(3)]
        with mock.patch.object(so, "voxel_points", lambda dims_, o_, vs_: exact):
            so.integrate(ts, W, None, origin, vs, trunc, d[sl], K[sl], R[sl], t[sl])
        kz, ky, kx = np.nonzero(W > 0)
        vox = np.stack([kx + g0[0], ky + g0[1], kz + g0[2]], axis=1)
        changed = set(map(tuple, sp.block_of(vox).tolist()))
        changed_total += len(changed)
        assert changed <= got, (f, sorted(changed - got)[:5])
        new, _ = sp.allocate(d[sl], K[sl], R[sl], t[sl], origin, vs, trunc)
        assert new <= got, (f, sorted(new - got)[:5])
    assert changed_total > 0
    return blocks


def check_raycast_reach(blocks, tsdf, weight, origin, vs, K, R, t, h, w, step=0.5):
    """Every block holding a corner of a sample the ray cast evaluates, of a normal's sample or of the colour lookup is
    reached with every tile at far and trunc 0."""
    vol = ro.Sparse(blocks, tsdf, weight)
    far = ro.sparse_far(blocks, origin, vs, R, t)
    seen = []
    real_cube = ro.cube

    def cube(v, X, o, s):
        out = real_cube(v, X, o, s)
        seen.append(out[3][(out[3] != ro.NO_CUBE).all(axis=1)])
        return out
    n = R.shape[0]
    for f in range(n):
        seen.clear()
        sl = slice(f, f + 1)
        with mock.patch.object(ro, "cube", cube):
            ro.raycast(vol, origin, vs, K[sl], R[sl], t[sl], 0.0, far[sl], step, h, w)
        c = np.concatenate(seen)
        corners = (c[:, None, :] + so.CORNERS[None]).reshape(-1, 3)
        need = set(map(tuple, np.unique(sp.block_of(corners), axis=0).tolist())) & set(map(tuple, blocks.tolist()))
        reached = ss.reach(blocks, origin, vs, 0.0, ss.raycast_tiles(far[sl], h, w), K[sl], R[sl], t[sl], h, w)[0]
        got = set(map(tuple, blocks[reached].tolist()))
        assert need and need <= got, (f, sorted(need - got)[:5])


def fused(blocks, origin, vs, trunc, d, K, R, t):
    m = blocks.shape[0]
    ts, W = np.zeros((m, 8, 8, 8), f32), np.zeros((m, 8, 8, 8), f32)
    sp.integrate_blocks(ts, W, None, blocks, origin, vs, trunc, d, K, R, t)
    return ts, W


def test_depth_tiles():
    d = np.full((2, 10, 17), np.nan, f32)
    d[0, 3, 4], d[0, 5, 6], d[0, 9, 16], d[1, 0, 0] = 2.0, 3.0, 1.5, np.inf
    d[1, 8, 9], d[1, 8, 10] = -1.0, 0.0
    tl = ss.depth_tiles(d)
    assert tl.shape == (2, 2, 3) and tl.dtype == f32
    assert tl[0, 0, 0] == 3.0 and tl[0, 1, 2] == 1.5 and np.isneginf(tl[1]).all()
    assert np.isneginf(tl[0, 0, 1:]).all() and np.isneginf(tl[0, 1, :2]).all()


def test_sphere_views_with_invalid_pixels():
    d, K, R, t, _ = sphere_views_with_bad_pixels(6, 2)
    origin, vs = (0.013, -0.021, 0.007), 0.043
    blocks = check_integration_reach(d, K, R, t, origin, vs, f32(3 * vs))
    ts, W = fused(blocks, origin, vs, f32(3 * vs), d, K, R, t)
    check_raycast_reach(blocks, ts, W, origin, vs, K[:3], R[:3], t[:3], 24, 32)


def test_varied_sphere_views():
    d, K, R, t, _ = fb.varied_sphere_views(5, seed=3)
    origin, vs = (-0.31, 0.12, 0.05), 0.05
    check_integration_reach(d, K, R, t, origin, vs, f32(3 * vs))


def test_grid_aligned_plane():
    """Voxels at sdf = -trunc and on u = w are reached."""
    d, K, R, t, _ = fb.plane_frames(6)
    check_integration_reach(d, K, R, t, fb.ORIGIN, fb.VOXEL, fb.TRUNC)


def test_orbit():
    p = so.orbit_pairs(frames=4, h=48, w=64, intrinsics=so.NETWORK_INTRINSICS)
    d = np.asarray(p["depth"], f32)
    n = d.shape[0]
    K = np.broadcast_to(so.K_pixels(so.NETWORK_INTRINSICS, 64, 48).astype(f32), (n, 3, 3))
    Rw = np.asarray(p["R"], f32)
    tw = np.asarray(p["t"] * p["baselines"][0], f32)
    check_integration_reach(d, K, Rw, tw, (0.01, -0.02, 0.03), 0.2, f32(0.6))


def test_ring_corridor_is_reached_and_tight():
    d, K, R, t, _ = ss.ring_walk(24)
    origin, vs, trunc = (0.003, -0.002, 0.001), 0.05, f32(0.15)
    n, h, w = d.shape
    blocks = check_integration_reach(d[:12], K[:12], R[:12], t[:12], origin, vs, trunc)
    ts, W = fused(blocks, origin, vs, trunc, d[:12], K[:12], R[:12], t[:12])
    check_raycast_reach(blocks, ts, W, origin, vs, K[:2], R[:2], t[:2], h, w)
    # tightness: a longer loop's blocks against one frame on its far side
    d, K, R, t, _ = ss.ring_walk(24, L=4.0)
    alloc, _ = sp.allocate(d, K, R, t, origin, vs, trunc)
    allb = np.array(sorted(alloc), np.int64)
    f = 9   # half a loop from frame 0
    reached = ss.reach(allb, origin, vs, trunc, ss.depth_tiles(d[f:f + 1]), K[f:f + 1], R[f:f + 1], t[f:f + 1], h, w)[0]
    frac = 1.0 - reached.mean()
    print("ring corridor: %d blocks, %.1f %% not reached from frame %d" % (allb.shape[0], 100 * frac, f))
    assert frac > 0.6


@pytest.mark.parametrize("bad", [0, -3, 2.5, "4", True, np.nan])
def test_max_device_blocks_is_checked_before_any_device(bad):
    with mock.patch.object(sequence, "_device", side_effect=AssertionError("device touched")):
        with pytest.raises(ValueError, match="max_device_blocks"):
            sequence.SparseTsdfVolume(0.1, max_device_blocks=bad)
        vol = sequence.SparseTsdfVolume(0.1, max_device_blocks=np.int64(7))
    assert vol.max_device_blocks == 7 and sequence.SparseTsdfVolume(0.1).max_device_blocks is None
