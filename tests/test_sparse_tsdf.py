"""CPU: the allocation rule of the sparse TSDF volume (tests/sparse_tsdf_oracle.py) against the dense numpy integration
(tests/sequence_oracle.py) on small scenes: every voxel an update with f < 1 reached, and every corner of a cube with a
corner below zero, lies in an allocated block.  And the argument checks of SparseTsdfVolume that come before any device."""
import numpy as np
import pytest

import sequence_oracle as so
import sparse_tsdf_oracle as sp
from demon_b200 import sequence


def spoil(d, seed):
    """NaN, 0, negative and inf pixels in 3% of the finite depths each."""
    d = d.copy()
    rng = np.random.RandomState(seed)
    for bad in (np.nan, 0.0, -1.0, np.inf):
        m = rng.rand(*d.shape) < 0.03
        d[m & np.isfinite(d)] = bad
    return d


def orbit_views(n=6, h=36, w=48):
    """Depth maps of a box with a sphere in it from cameras on a circle around it, looking at its centre (as
    tools/bench_sequence.py's orbit_frames), at a small size: depth [n,h,w], K [n,3,3], R [n,3,3], t [n,3] float32."""
    K = so.K_pixels(so.NETWORK_INTRINSICS, w, h)
    Rs, ts, ds = [], [], []
    for a in np.linspace(0, 2 * np.pi, n, endpoint=False):
        R, t = so.look_at((2.5 * np.cos(a), 2.5 * np.sin(a), 0.6), (0, 0, 0))
        Rs.append(R)
        ts.append(t)
        ds.append(so.render_depth(R, t, K, h, w, sphere=((0.1, 0, 0), 0.5), box=((-1, -1, -1), (1, 1, 1.2))))
    return (np.array(ds, np.float32), np.broadcast_to(K.astype(np.float32), (n, 3, 3)).copy(), np.array(Rs, np.float32),
            np.array(ts, np.float32))


def scenes():
    d, K, R, t, _ = so.sphere_views(n=6, h=24, w=32)
    yield "sphere", spoil(d, 1), K, R, t, (-1.0, -1.0, -1.0), 0.05, (40, 40, 40)
    d, K, R, t = orbit_views()
    yield "orbit", spoil(d, 2), K, R, t, (-3.0, -3.0, -1.5), 0.1, (60, 60, 32)


@pytest.mark.parametrize("scene", list(scenes()), ids=lambda s: s[0])
def test_allocation_covers_every_updated_voxel_and_every_surface_cube(scene):
    _, d, K, R, t, origin, vs, dims = scene
    trunc = np.float32(3 * np.float32(vs))
    blocks, skipped = sp.allocate(d, K, R, t, origin, vs, trunc)
    assert skipped == 0 and len(blocks) > 0
    nx, ny, nz = dims
    ts, W = np.zeros((nz, ny, nx), np.float32), np.zeros((nz, ny, nx), np.float32)
    so.integrate(ts, W, None, origin, vs, trunc, d, K, R, t)
    assert (W > 0).any() and (ts < 0).any()

    def allocated(g):   # g [..., 3] voxel coordinates (x, y, z) -> bool
        b = sp.block_of(g)
        return np.array([tuple(x) in blocks for x in b.reshape(-1, 3).tolist()]).reshape(b.shape[:-1])

    k, j, i = np.nonzero((W > 0) & (ts < 1))
    assert allocated(np.stack([i, j, k], axis=1)).all()
    # every cube (of the dense box) with a corner below zero: all 8 corners allocated
    neg = ts < 0
    low = np.zeros((nz - 1, ny - 1, nx - 1), bool)
    for dx, dy, dz in so.CORNERS:
        low |= neg[dz:dz + nz - 1, dy:dy + ny - 1, dx:dx + nx - 1]
    k, j, i = np.nonzero(low)
    g = np.stack([i, j, k], axis=1)
    for c in so.CORNERS:
        assert allocated(g + c).all()
    # the dense box holds every voxel an update with f < 1 reached, so nothing was missed at its border
    band = (W > 0) & (ts < 1)
    assert not any(band[s].any() for s in (np.s_[0], np.s_[-1], np.s_[:, 0], np.s_[:, -1], np.s_[:, :, 0], np.s_[:, :, -1]))


def test_allocation_skips_far_and_out_of_range_pixels():
    """A pixel whose cell spans more than MAX_SPAN blocks, or whose blocks leave the key range, allocates nothing."""
    d, K, R, t, _ = so.sphere_views(n=2, h=8, w=8)
    d[:] = 1.0
    d[0, 0, 0] = 1e3       # a wide cell
    d[0, 0, 1] = 1e30      # past the key range
    d[1, 0, 0] = np.nan    # invalid: neither allocated nor counted
    blocks, skipped = sp.allocate(d, K, R, t, (0, 0, 0), 0.05, 0.15)
    assert skipped == 2
    near, _ = sp.allocate(np.where(d > 10, np.nan, d), K, R, t, (0, 0, 0), 0.05, 0.15)
    assert blocks == near


@pytest.mark.parametrize("kwargs, match", [
    (dict(voxel_size=0.0), "voxel_size"),
    (dict(voxel_size=np.nan), "voxel_size"),
    (dict(voxel_size=0.1, trunc=-1.0), "trunc"),
    (dict(voxel_size=0.1, trunc=np.inf), "trunc"),
    (dict(voxel_size=0.1, origin=(0, 0)), "origin"),
    (dict(voxel_size=0.1, origin=(0, np.inf, 0)), "origin"),
])
def test_sparse_volume_refuses_bad_arguments(kwargs, match):
    with pytest.raises(ValueError, match=match):
        sequence.SparseTsdfVolume(**kwargs)


@pytest.mark.parametrize("color, change, match", [
    (False, dict(depth=np.ones((8, 8), np.float32)), "depth"),
    (False, dict(depth=np.ones((2, 2, 8, 8), np.float32)), "depth"),
    (False, dict(depth=np.ones((1, 4096, 4096), np.float32)), "too many"),
    (False, dict(K=np.eye(3, dtype=np.float32)[None].repeat(3, 0)), "K"),
    (False, dict(R=np.eye(4, dtype=np.float32)), "R"),
    (False, dict(t=np.zeros((2, 4), np.float32)), "t"),
    (False, dict(image=np.zeros((2, 8, 8, 3), np.uint8)), "image"),
    (True, dict(), "image"),
    (True, dict(image=np.zeros((2, 8, 8, 3), np.float32)), "uint8"),
    (True, dict(image=np.zeros((2, 8, 7, 3), np.uint8)), "image"),
])
def test_sparse_integrate_refuses_bad_arguments_before_the_device(color, change, match):
    args = dict(depth=np.ones((2, 8, 8), np.float32), K=np.eye(3, dtype=np.float32), R=np.eye(3, dtype=np.float32)[None].repeat(2, 0),
                t=np.zeros((2, 3), np.float32), image=None)
    args.update(change)
    vol = sequence.SparseTsdfVolume(0.1, color=color)
    with pytest.raises(ValueError, match=match):
        vol.integrate(**args)


def test_reconstruct_takes_a_sparse_volume_only_as_a_volume():
    import torch
    with pytest.raises(ValueError, match="SparseTsdfVolume"):
        sequence.reconstruct(None, torch.zeros((2, 48, 64, 3), dtype=torch.uint8), np.eye(3), volume="sparse")
