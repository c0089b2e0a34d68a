"""GPU: demon_b200.sequence.SparseTsdfVolume against its numpy restatement (tests/sparse_tsdf_oracle.py) and the dense
TsdfVolume: the allocated block set and skipped pixels, every stored voxel and the mesh bit for bit against a dense volume
on the same origin, negative block coordinates, chunked calls that grow the pool and the hash table, determinism, mesh
edge cases, and reconstruct with a sparse volume against its parts composed by hand."""
import numpy as np
import pytest
import torch

import sequence_oracle as so
import sparse_tsdf_oracle as sp
from demon_b200 import _lib, images, sequence

pytestmark = pytest.mark.gpu


def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def views(n, seed):
    """Sphere views with NaN, 0, negative and inf pixels."""
    d, K, R, t, img = so.sphere_views(n=n, seed=seed)
    rng = np.random.RandomState(seed)
    for bad in (np.nan, 0.0, -1.0, np.inf):
        m = rng.rand(*d.shape) < 0.03
        d[m & np.isfinite(d)] = bad
    return d, K, R, t, img


def frames(d, K, R, t, img, sl=slice(None), color=True):
    return cuda(d[sl]), cuda(K[sl]), cuda(R[sl]), cuda(t[sl]), cuda(img[sl]) if color else None


def sorted_by_key(b):
    """Rows of blocks [m,3] in ascending packed key order: z, then y, then x."""
    return np.array_equal(np.lexsort((b[:, 0], b[:, 1], b[:, 2])), np.arange(b.shape[0]))


def triangles(v, c, f):
    """The mesh as a sorted multiset of triangles: rows of 9 vertex floats' bits and 9 colour bytes."""
    v, f = v.cpu().numpy(), f.cpu().numpy()
    rows = v[f].reshape(-1, 9).view(np.uint32)
    if c is not None:
        rows = np.concatenate([rows, c.cpu().numpy()[f].reshape(-1, 9).astype(np.uint32)], axis=1)
    return rows[np.lexsort(rows.T[::-1])]


def test_allocation_equals_the_oracle():
    """Odd intrinsics, invalid depths, a camera facing away from the scene, and pixels past the span cap and the key range."""
    d, K, R, t, _ = views(6, 3)
    K = K.copy()
    K[:, 0, 0], K[:, 1, 1], K[:, 0, 2], K[:, 1, 2] = 61.3, 57.9, 31.7, 22.1
    R = R.copy()
    R[5] = -R[5]
    R[5, 1] = -R[5, 1]           # a proper rotation facing the other way
    d[1, :4, :4] = 400.0         # wide cells: skipped
    d[2, 5, :7] = 1e30           # past the key range: skipped
    d[3, :, :] = np.where(np.isfinite(d[3]), d[3], 2.5)
    vol = sequence.SparseTsdfVolume(0.031, origin=(0.013, -0.021, 0.007), color=False)
    vol.integrate(cuda(d), cuda(K), cuda(R), cuda(t))
    ref, skipped = sp.allocate(d, K, R, t, vol.origin, vol.voxel_size, vol.trunc)
    assert skipped >= 16 + 7 and vol.last_skipped_pixels == skipped
    b = vol.blocks.cpu().numpy()
    assert set(map(tuple, b.tolist())) == ref and len(ref) == b.shape[0]
    assert sorted_by_key(b) and (b < 0).any()
    _lib.check_errors()


@pytest.mark.parametrize("color", [True, False])
def test_one_call_equals_the_dense_volume(color):
    d, K, R, t, img = views(8, 4)
    origin, vs = (-1.2, -1.2, -1.2), 0.043
    vol = sequence.SparseTsdfVolume(vs, origin, color=color)
    vol.integrate(*frames(d, K, R, t, img, color=color))
    assert vol.last_skipped_pixels == 0
    b = vol.blocks.cpu().numpy()
    assert b.min() >= 0
    bx, by, bz = (int(x) + 1 for x in b.max(axis=0))
    dense = sequence.TsdfVolume((8 * bx, 8 * by, 8 * bz), origin, vs, trunc=vol.trunc, color=color)
    dense.integrate(*frames(d, K, R, t, img, color=color))

    def by_block(x):   # dense [nz,ny,nx,...] -> [bz,by,bx,8,8,8,...]
        x = x.reshape((bz, 8, by, 8, bx, 8) + tuple(x.shape[3:]))
        return x.permute((0, 2, 4, 1, 3, 5) + tuple(range(6, x.dim())))

    idx = tuple(torch.from_numpy(b[:, a]).long().cuda() for a in (2, 1, 0))
    assert torch.equal(by_block(dense.tsdf)[idx], vol.tsdf) and torch.equal(by_block(dense.weight)[idx], vol.weight)
    if color:
        assert torch.equal(by_block(dense.color)[idx], vol.color)
    else:
        assert vol.color is None
    stored = torch.zeros((bz, by, bx), dtype=torch.bool, device="cuda")
    stored[idx] = True
    outside = ~stored[:, :, :, None, None, None].expand(-1, -1, -1, 8, 8, 8)
    Wd, Td = by_block(dense.weight), by_block(dense.tsdf)
    assert bool(((Wd == 0) | (Td == 1))[outside].all())
    assert bool((Wd[outside] > 0).any())   # free space outside the blocks was seen
    ms, md = vol.mesh(), dense.mesh()
    assert ms[2].shape[0] > 0 and ms[2].shape == md[2].shape
    assert np.array_equal(ms[2].cpu().numpy().reshape(-1), np.arange(3 * ms[2].shape[0]))
    assert np.array_equal(triangles(*ms), triangles(*md))
    _lib.check_errors()


def test_negative_block_coordinates_equal_the_oracle():
    d, K, R, t, img = views(6, 5)
    vol = sequence.SparseTsdfVolume(0.05, origin=(0.01, -0.02, 0.0))
    vol.integrate(*frames(d, K, R, t, img))
    b = vol.blocks.cpu().numpy()
    assert (b < 0).any() and (b >= 0).any()
    m = b.shape[0]
    ts, W, col = np.zeros((m, 8, 8, 8), np.float32), np.zeros((m, 8, 8, 8), np.float32), np.zeros((m, 8, 8, 8, 3), np.float32)
    sp.integrate_blocks(ts, W, col, b, vol.origin, vol.voxel_size, vol.trunc, d, K, R, t, img)
    assert np.array_equal(vol.tsdf.cpu().numpy(), ts) and np.array_equal(vol.weight.cpu().numpy(), W)
    assert np.array_equal(vol.color.cpu().numpy(), col)
    assert (W > 0).any() and (ts < 0).any()
    _lib.check_errors()


def test_chunked_calls_grow_the_pool_and_table():
    """Three calls: each call's new blocks are appended in key order and hold the frames from that call onward."""
    d, K, R, t, img = so.sphere_views(n=9)
    vol = sequence.SparseTsdfVolume(0.02, origin=(0.01, -0.02, 0.0))
    firsts, caps, known = [0], [], set()
    for c in range(3):
        sl = slice(3 * c, 3 * c + 3)
        vol.integrate(*frames(d, K, R, t, img, sl))
        ref, skipped = sp.allocate(d[sl], K[sl], R[sl], t[sl], vol.origin, vol.voxel_size, vol.trunc)
        b = vol.blocks.cpu().numpy()
        new = b[firsts[-1]:]
        assert set(map(tuple, new.tolist())) == ref - known and sorted_by_key(new) and vol.last_skipped_pixels == skipped
        known |= ref
        firsts.append(b.shape[0])
        caps.append(vol.capacity)
    assert caps[0] >= 4 * sequence.SparseTsdfVolume._POOL_BLOCKS and caps[1] > caps[0]
    assert vol.table_slots > sequence.SparseTsdfVolume._TABLE_SLOTS
    b = vol.blocks.cpu().numpy()
    for c in range(3):
        blk = b[firsts[c]:firsts[c + 1]]
        m = blk.shape[0]
        ts, W, col = np.zeros((m, 8, 8, 8), np.float32), np.zeros((m, 8, 8, 8), np.float32), np.zeros((m, 8, 8, 8, 3), np.float32)
        sl = slice(3 * c, None)
        sp.integrate_blocks(ts, W, col, blk, vol.origin, vol.voxel_size, vol.trunc, d[sl], K[sl], R[sl], t[sl], img[sl])
        assert np.array_equal(vol.tsdf[firsts[c]:firsts[c + 1]].cpu().numpy(), ts), c
        assert np.array_equal(vol.weight[firsts[c]:firsts[c + 1]].cpu().numpy(), W), c
        assert np.array_equal(vol.color[firsts[c]:firsts[c + 1]].cpu().numpy(), col), c
    _lib.check_errors()


def test_same_calls_give_the_same_bytes():
    d, K, R, t, img = views(10, 6)
    out = []
    for _ in range(2):
        vol = sequence.SparseTsdfVolume(0.025, origin=(-0.3, 0.2, 0.1))
        vol.integrate(*frames(d, K, R, t, img, slice(0, 4)))
        vol.integrate(*frames(d, K, R, t, img, slice(4, None)))
        out.append([vol.blocks, vol.tsdf, vol.weight, vol.color] + list(vol.mesh()))
    assert out[0][6].shape[0] > 0
    for a, b in zip(*out):
        assert a.dtype == b.dtype and torch.equal(a, b)


def test_fused_sphere_mesh_is_closed():
    d, K, R, t, img = so.sphere_views(n=24)
    vs = 2.0 / 47
    vol = sequence.SparseTsdfVolume(vs, origin=(-1, -1, -1))
    vol.integrate(*frames(d, K, R, t, img))
    v, c, f = (x.cpu().numpy() for x in vol.mesh())
    assert f.shape[0] > 1000 and c.shape == v.shape
    assert set(so.welded_edges(v, f)) == {2}
    assert np.abs(np.linalg.norm(v.astype(np.float64), axis=1) - 0.6).max() <= vs / 2


def test_frames_without_valid_pixels():
    vol = sequence.SparseTsdfVolume(0.1)
    v, c, f = vol.mesh()
    assert v.shape == (0, 3) and c.shape == (0, 3) and f.shape == (0, 3)
    d = np.full((3, 6, 7), np.nan, np.float32)
    d[1] = 0.0
    d[2] = -1.0
    K = np.array([[5.0, 0, 3], [0, 5, 3], [0, 0, 1]], np.float32)
    vol.integrate(cuda(d), cuda(K), cuda(np.eye(3, dtype=np.float32)), cuda(np.zeros(3, np.float32)), cuda(np.zeros((3, 6, 7, 3), np.uint8)))
    assert vol.blocks.shape == (0, 3) and vol.tsdf.shape == (0, 8, 8, 8) and vol.last_skipped_pixels == 0
    v, c, f = vol.mesh()
    assert v.shape == (0, 3) and f.shape == (0, 3)
    _lib.check_errors()


def video(T, seed, h=480, w=640):
    """A smooth synthetic video: a textured plane panning sideways, so that consecutive frames overlap."""
    rng = np.random.RandomState(seed)
    base = rng.randint(0, 256, (h // 8, (w + 16 * T) // 8, 3)).astype(np.uint8)
    big = np.kron(base, np.ones((8, 8, 1), np.uint8))
    return cuda(np.stack([big[:, 16 * k:16 * k + w] for k in range(T)]))


@pytest.fixture(scope="module")
def session(synthetic_weights):
    from demon_b200.networks_original import Session
    s = Session(precision="3xtf32")
    s.load_weights(synthetic_weights)
    return s


@pytest.mark.parametrize("T, batch", [(2, 1), (7, 4)])
def test_reconstruct_into_a_sparse_volume(session, T, batch):
    from demon_b200.networks_original import DemonPipeline
    pipe = DemonPipeline(session, batch_size=batch, iterations=1)
    frames_u8 = video(T, 3)
    K = np.array([[520.0, 0, 318.0], [0, 515.0, 243.0], [0, 0, 1]])
    # the voxel size: 4 blocks across the default volume's box, whatever scale the synthetic weights give the depth
    box = sequence.reconstruct(pipe, frames_u8, K, min_ratios=1)["volume"]
    vs = float(box.voxel_size) * max(box.dims) / 32
    res = sequence.reconstruct(pipe, frames_u8, K, volume=sequence.SparseTsdfVolume(vs, box.origin), min_ratios=1)

    p = T - 1
    inv, rot, tr = [], [], []
    for s in range(0, p, batch):
        m = min(batch, p - s)
        idx = np.minimum(np.arange(s, s + batch), s + m - 1)
        out = pipe.forward_views(torch.stack((frames_u8[idx], frames_u8[idx + 1]), dim=1), np.broadcast_to(K, (batch, 2, 3, 3)))
        inv.append(out["predict_depth0"][:m].clone())
        rot.append(out["predict_rotation"][:m].clone())
        tr.append(out["predict_translation"][:m].clone())
    inv, rot, tr = torch.cat(inv), torch.cat(rot), torch.cat(tr)
    assert torch.equal(res["inverse_depth"], inv) and torch.equal(res["rotation"], rot) and torch.equal(res["translation"], tr)
    ch = sequence.chain_pairs(inv, rot, tr, min_ratios=1)
    adapted, _, _ = images.adjust_intrinsics(frames_u8, K)
    vol = sequence.SparseTsdfVolume(vs, box.origin)
    Kp = torch.from_numpy(so.K_pixels(so.NETWORK_INTRINSICS, 256, 192).astype(np.float32)).cuda()
    vol.integrate(ch["depth"], Kp, cuda(ch["R"][:p].astype(np.float32)), cuda(ch["t"][:p].astype(np.float32)), adapted[:p])
    v0 = res["volume"]
    assert isinstance(v0, sequence.SparseTsdfVolume) and v0.blocks.shape[0] > 0
    for k in ("blocks", "tsdf", "weight", "color"):
        assert torch.equal(getattr(vol, k), getattr(v0, k)), k
    assert vol.last_skipped_pixels == v0.last_skipped_pixels
    v, c, f = vol.mesh()
    assert torch.equal(v, res["vertices"]) and torch.equal(c, res["colors"]) and torch.equal(f, res["faces"])
    _lib.check_errors()
