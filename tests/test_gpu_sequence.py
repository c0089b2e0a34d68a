"""GPU: demon_b200.sequence against its numpy restatement (tests/sequence_oracle.py): the chain's scales and float64 poses,
the TSDF integration and marching cubes bit for bit (odd volume sizes, colour or not, chunked calls, invalid depth, voxels
behind a camera and outside every frustum), and reconstruct end to end against forward_views, chain_pairs and integrate."""
import numpy as np
import pytest
import torch

import sequence_oracle as so
from demon_b200 import _lib, images, sequence

pytestmark = pytest.mark.gpu


def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def test_chain_pairs_equals_lower_median_and_oracle_poses():
    sc = so.orbit_pairs(frames=7, seed=2)
    inv, rot, tr = cuda(sc["inverse_depth"]), cuda(sc["rotation"]), cuda(sc["translation"])
    ch = sequence.chain_pairs(inv, rot, tr)
    ratios = sequence.pair_ratios(inv, rot, tr).cpu().numpy()
    ref = so.pair_ratios(sc["inverse_depth"], sc["rotation"], sc["translation"])
    assert np.array_equal(ratios, ref, equal_nan=True)
    med = np.array([so.lower_median(r)[0] for r in ratios], dtype=np.float64)
    assert np.array_equal(ch["scales"], med)
    sigma, R, t = so.chain_poses(sc["rotation"], sc["translation"], med)
    assert np.array_equal(ch["sigma"], sigma) and np.array_equal(ch["R"], R) and np.array_equal(ch["t"], t)
    assert np.array_equal(ch["depth"].cpu().numpy(), sigma.astype(np.float32)[:, None, None] / sc["inverse_depth"][:, 0])
    np.testing.assert_allclose(ch["scales"], sc["scales"], rtol=1e-5)
    # one pair: no ratios, the pair's own motion
    one = sequence.chain_pairs(inv[:1], rot[:1], tr[:1])
    assert one["scales"].shape == (0,) and np.array_equal(one["t"][1], sc["translation"][0].astype(np.float64))


def test_chain_pairs_names_the_pair_without_ratios():
    sc = so.orbit_pairs(frames=5, seed=1)
    inv = sc["inverse_depth"].copy()
    inv[2] = np.nan
    with pytest.raises(ValueError, match="pairs 1 and 2"):
        sequence.chain_pairs(cuda(inv), cuda(sc["rotation"]), cuda(sc["translation"]))


def views(n, seed):
    """Sphere views with NaN, 0, negative and inf pixels."""
    d, K, R, t, img = so.sphere_views(n=n, seed=seed)
    rng = np.random.RandomState(seed)
    for bad in (np.nan, 0.0, -1.0, np.inf):
        m = rng.rand(*d.shape) < 0.03
        d[m & np.isfinite(d)] = bad
    return d, K, R, t, img


@pytest.mark.parametrize("dims, origin, voxel", [
    ((37, 29, 23), (-3.6, -3.6, -3.6), 0.2),        # around the sphere and past the cameras: behind and outside frustums
    ((41, 39, 45), (-0.9, -0.85, -0.95), 0.043),   # the sphere at a fine voxel
])
@pytest.mark.parametrize("color", [True, False])
def test_integrate_and_mesh_match_the_oracle(dims, origin, voxel, color):
    d, K, R, t, img = views(8, 4)
    vol = sequence.TsdfVolume(dims, origin, voxel, color=color)
    im = img if color else None
    vol.integrate(cuda(d[:3]), cuda(K[:3]), cuda(R[:3]), cuda(t[:3]), None if im is None else cuda(im[:3]))
    vol.integrate(cuda(d[3:]), cuda(K[3:]), cuda(R[3:]), cuda(t[3:]), None if im is None else cuda(im[3:]))
    one = sequence.TsdfVolume(dims, origin, voxel, color=color)
    one.integrate(cuda(d), cuda(K), cuda(R), cuda(t), None if im is None else cuda(im))
    nx, ny, nz = dims
    ts, W = np.zeros((nz, ny, nx), np.float32), np.zeros((nz, ny, nx), np.float32)
    col = np.zeros((nz, ny, nx, 3), np.float32) if color else None
    so.integrate(ts, W, col, vol.origin, vol.voxel_size, vol.trunc, d, K, R, t, im)
    for v in (vol, one):
        assert np.array_equal(v.tsdf.cpu().numpy(), ts) and np.array_equal(v.weight.cpu().numpy(), W)
        if color:
            assert np.array_equal(v.color.cpu().numpy(), col)
    assert 0 < (W > 0).mean() < 1   # some voxels are never updated
    vg, cg, fg = vol.mesh()
    vr, cr, fr = so.marching_cubes(ts, W, col, vol.origin, vol.voxel_size)
    assert fr.shape[0] > 0
    assert np.array_equal(vg.cpu().numpy(), vr) and np.array_equal(fg.cpu().numpy(), fr)
    assert (cg is None) == (not color)
    if color:
        assert np.array_equal(cg.cpu().numpy(), cr)
    _lib.check_errors()


def test_fused_sphere_mesh_is_closed():
    d, K, R, t, img = so.sphere_views(n=24)
    n = 48
    vs = 2.0 / (n - 1)
    vol = sequence.TsdfVolume((n, n, n), (-1, -1, -1), vs)
    vol.integrate(cuda(d), cuda(K), cuda(R), cuda(t), cuda(img))
    v, c, f = (x.cpu().numpy() for x in vol.mesh())
    vr, cr, fr = so.marching_cubes(vol.tsdf.cpu().numpy(), vol.weight.cpu().numpy(), vol.color.cpu().numpy(), vol.origin, vol.voxel_size)
    assert np.array_equal(v, vr) and np.array_equal(c, cr) and np.array_equal(f, fr)
    assert set(so.welded_edges(v, f)) == {2}
    assert np.abs(np.linalg.norm(v.astype(np.float64), axis=1) - 0.6).max() <= vs / 2


def test_mesh_of_an_empty_volume():
    vol = sequence.TsdfVolume((5, 6, 7), (0, 0, 0), 0.1)
    v, c, f = vol.mesh()
    assert v.shape == (0, 3) and c.shape == (0, 3) and f.shape == (0, 3)


def video(T, seed, h=480, w=640):
    """A smooth synthetic video: a textured plane panning sideways, so that consecutive frames overlap."""
    rng = np.random.RandomState(seed)
    base = rng.randint(0, 256, (h // 8, (w + 16 * T) // 8, 3)).astype(np.uint8)
    big = np.kron(base, np.ones((8, 8, 1), np.uint8))
    return cuda(np.stack([big[:, 16 * k:16 * k + w] for k in range(T)]))


@pytest.fixture(scope="module")
def sessions(synthetic_weights):
    from demon_b200.networks_original import Session
    from demon_b200.v2 import weights as W2
    from demon_b200.v2.networks import Session as SessionV2
    s1 = Session(precision="3xtf32")
    s1.load_weights(synthetic_weights)
    s2 = SessionV2(precision="3xtf32")
    s2.load_weights(W2.synthetic_weights(0))
    return {"v1": s1, "v2": s2}


@pytest.mark.parametrize("net", ["v1", "v2"])
@pytest.mark.parametrize("T, batch", [(2, 1), (7, 4)])
def test_reconstruct_equals_forward_views_chain_and_integrate(sessions, net, T, batch):
    from demon_b200.networks_original import DemonPipeline
    from demon_b200.v2.networks import DemonPipelineV2
    cls = DemonPipeline if net == "v1" else DemonPipelineV2
    pipe = cls(sessions[net], batch_size=batch, iterations=1)
    frames = video(T, 3)
    K = np.array([[520.0, 0, 318.0], [0, 515.0, 243.0], [0, 0, 1]])
    res = sequence.reconstruct(pipe, frames, K, min_ratios=1)

    # the composition: forward_views on the raw pairs (the last batch padded the same way), then chain_pairs and integrate
    p = T - 1
    inv, rot, tr = [], [], []
    for s in range(0, p, batch):
        m = min(batch, p - s)
        idx = np.minimum(np.arange(s, s + batch), s + m - 1)
        pairs = torch.stack((frames[idx], frames[idx + 1]), dim=1)
        out = pipe.forward_views(pairs, np.broadcast_to(K, (batch, 2, 3, 3)))
        assert torch.all(out["status"] < 2)
        inv.append(out["predict_depth0"][:m].clone())
        rot.append(out["predict_rotation"][:m].clone())
        tr.append(out["predict_translation"][:m].clone())
    inv, rot, tr = torch.cat(inv), torch.cat(rot), torch.cat(tr)
    assert torch.equal(res["inverse_depth"], inv) and torch.equal(res["rotation"], rot) and torch.equal(res["translation"], tr)
    ch = sequence.chain_pairs(inv, rot, tr, min_ratios=1)
    for k in ("scales", "sigma", "R", "t"):
        assert np.array_equal(res[k], ch[k]), k
    assert torch.equal(res["depth"], ch["depth"])
    adapted, _, _ = images.adjust_intrinsics(frames, K)
    assert torch.equal(res["adapted"], adapted)
    v0 = res["volume"]
    vol = sequence.TsdfVolume(v0.dims, v0.origin, v0.voxel_size, v0.trunc)
    Kp = torch.from_numpy(so.K_pixels(so.NETWORK_INTRINSICS, 256, 192).astype(np.float32)).cuda()
    vol.integrate(ch["depth"], Kp, cuda(ch["R"][:p].astype(np.float32)), cuda(ch["t"][:p].astype(np.float32)), adapted[:p])
    assert torch.equal(vol.tsdf, v0.tsdf) and torch.equal(vol.weight, v0.weight) and torch.equal(vol.color, v0.color)
    v, c, f = vol.mesh()
    assert torch.equal(v, res["vertices"]) and torch.equal(c, res["colors"]) and torch.equal(f, res["faces"])
    assert v0.dims[0] <= 256 and v0.dims[1] <= 256 and v0.dims[2] <= 256 and max(v0.dims) == 256
    _lib.check_errors()


def test_export_sequence_to_ply(tmp_path):
    d, K, R, t, img = so.sphere_views(n=12)
    vol = sequence.TsdfVolume((32, 32, 32), (-1, -1, -1), 2.0 / 31)
    vol.integrate(cuda(d), cuda(K), cuda(R), cuda(t), cuda(img))
    v, c, f = vol.mesh()
    Rs, ts = np.concatenate([np.eye(3)[None], R.astype(np.float64)]), np.concatenate([np.zeros((1, 3)), t.astype(np.float64)])
    prefix = str(tmp_path / "seq")
    sequence.export_sequence_to_ply(prefix, {"vertices": v, "colors": c, "faces": f, "R": Rs, "t": ts})
    mesh = open(prefix + "_mesh.ply", "rb").read()
    cams = open(prefix + "_cameras.ply", "rb").read()
    m = v.shape[0]
    assert (b"element vertex %d\n" % m) in mesh and b"property uchar red" in mesh and (b"element face %d\n" % (m // 3)) in mesh
    assert (b"element vertex %d\n" % (11 * 13)) in cams and (b"element face %d\n" % (6 * 13)) in cams
    body = mesh[mesh.index(b"end_header\n") + 11:]
    assert len(body) == m * 15 + (m // 3) * 13
