"""CPU: the numpy restatements of the video reconstruction (tests/sequence_oracle.py) on synthetic scenes with analytic
depth, and the argument checks of demon_b200.sequence that come before any device is needed."""
import numpy as np
import pytest
import torch

import sequence_oracle as so
from demon_b200 import sequence


@pytest.mark.parametrize("seed", [0, 3])
def test_oracle_chain_recovers_scales_and_poses(seed):
    """Pairs normalised to |t| = 1 with their depth scaled to match, with random baselines: the chain gives back the
    baseline ratios and the poses in pair 0's units."""
    sc = so.orbit_pairs(frames=6, seed=seed)
    ch = so.chain(sc["inverse_depth"], sc["rotation"], sc["translation"])
    assert np.all(ch["counts"] > 10000)
    np.testing.assert_allclose(ch["scales"], sc["scales"], rtol=1e-5)
    np.testing.assert_allclose(ch["R"], sc["R"], rtol=0, atol=1e-5)
    np.testing.assert_allclose(ch["t"], sc["t"], rtol=0, atol=1e-5 * np.abs(sc["t"]).max())
    # the chained depth of every frame is its true depth in pair 0's units
    finite = np.isfinite(sc["depth"][:-1])
    np.testing.assert_allclose(ch["depth"][finite] * sc["baselines"][0], sc["depth"][:-1][finite], rtol=1e-5)


def test_oracle_marching_cubes_sphere_is_closed():
    """An analytic sphere SDF: every welded edge is shared by exactly two faces, every vertex lies within half a voxel of
    the sphere."""
    n, r = 33, 0.63
    vs, org = np.float32(2.0 / (n - 1)), np.float32([-1, -1, -1])
    X = so.voxel_points((n, n, n), org, vs)
    sdf = (np.sqrt(sum(x.astype(np.float64) ** 2 for x in X)) - r).astype(np.float32).reshape(n, n, n)
    v, c, f = so.marching_cubes(sdf, np.ones_like(sdf), None, org, vs)
    assert c is None and f.shape[0] > 1000
    assert np.array_equal(f.reshape(-1), np.arange(v.shape[0]))
    assert set(so.welded_edges(v, f)) == {2}
    assert np.abs(np.linalg.norm(v.astype(np.float64), axis=1) - r).max() <= vs / 2


def test_oracle_fused_sphere_is_closed():
    """Depth maps of a sphere from cameras all around it, integrated and meshed: closed, coloured, near the sphere."""
    d, K, R, t, img = so.sphere_views()
    n = 40
    vs, org = np.float32(2.0 / (n - 1)), np.float32([-1, -1, -1])
    tsdf, W = np.zeros((n, n, n), np.float32), np.zeros((n, n, n), np.float32)
    col = np.zeros((n, n, n, 3), np.float32)
    so.integrate(tsdf, W, col, org, vs, 3 * vs, d, K, R, t, img)
    v, c, f = so.marching_cubes(tsdf, W, col, org, vs)
    assert f.shape[0] > 1000 and c.dtype == np.uint8 and c.shape == v.shape
    assert set(so.welded_edges(v, f)) == {2}
    assert np.abs(np.linalg.norm(v.astype(np.float64), axis=1) - 0.6).max() <= vs / 2


def test_triangle_table_separates_every_case():
    """Each case's triangles use exactly the edges whose corners differ in sign."""
    for case, row in enumerate(so.TRIANGLES):
        inside = [(case >> q) & 1 for q in range(8)]
        crossing = {e for e, (a, b) in enumerate(so.EDGES) if inside[a] != inside[b]}
        assert len(row) % 3 == 0 and set(row) == crossing, case


def test_chain_pairs_refuses_bad_arguments():
    inv = np.ones((3, 1, 192, 256), np.float32)
    m = np.zeros((3, 3), np.float32)
    with pytest.raises(ValueError, match="inverse_depth"):
        sequence.chain_pairs(np.ones((3, 1, 96, 128), np.float32), m, m)
    with pytest.raises(ValueError, match="inverse_depth"):
        sequence.chain_pairs(np.ones((0, 1, 192, 256), np.float32), m[:0], m[:0])
    with pytest.raises(ValueError, match="rotation"):
        sequence.chain_pairs(inv, m[:2], m)
    with pytest.raises(ValueError, match="translation"):
        sequence.chain_pairs(inv, m, np.zeros((3, 4), np.float32))
    with pytest.raises(ValueError, match="intrinsics"):
        sequence.chain_pairs(inv, m, m, intrinsics=(0.0, 1.0, 0.5, 0.5))
    with pytest.raises(ValueError, match="intrinsics"):
        sequence.chain_pairs(inv, m, m, intrinsics=(1.0, 1.0, 0.5))
    with pytest.raises(ValueError, match="min_ratios"):
        sequence.chain_pairs(inv, m, m, min_ratios=0)


@pytest.mark.parametrize("kwargs, match", [
    (dict(dims=(1, 8, 8)), "dims"),
    (dict(dims=(8, 8)), "dims"),
    (dict(dims=(2048, 2048, 1024)), "dims"),
    (dict(origin=(0, 0)), "origin"),
    (dict(origin=(0, np.nan, 0)), "origin"),
    (dict(voxel_size=0.0), "voxel_size"),
    (dict(voxel_size=np.inf), "voxel_size"),
    (dict(trunc=-1.0), "trunc"),
])
def test_tsdf_volume_refuses_bad_arguments(kwargs, match):
    args = dict(dims=(8, 8, 8), origin=(0, 0, 0), voxel_size=0.1)
    args.update(kwargs)
    with pytest.raises(ValueError, match=match):
        sequence.TsdfVolume(**args)


def test_reconstruct_refuses_bad_arguments():
    with pytest.raises(ValueError, match="T >= 2"):
        sequence.reconstruct(None, torch.zeros((1, 48, 64, 3), dtype=torch.uint8), np.eye(3))
    with pytest.raises(ValueError, match="T >= 2"):
        sequence.reconstruct(None, np.zeros((4, 48, 64, 3), np.uint8), np.eye(3))
    with pytest.raises(ValueError, match="volume"):
        sequence.reconstruct(None, torch.zeros((2, 48, 64, 3), dtype=torch.uint8), np.eye(3), volume=object())
