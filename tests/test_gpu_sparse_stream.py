"""GPU: streaming a SparseTsdfVolume's blocks to pinned host memory (max_device_blocks).  The depth tiles and the reach
kernel equal their numpy restatement (tests/sparse_stream_oracle.py) bit for bit; a budgeted volume walked 1.3 times
round a ring corridor equals an unbudgeted one after every call, block for block, and so do its ray casts and meshes;
identical calls give identical bytes; reconstruct takes a budgeted volume."""
import numpy as np
import pytest
import torch

import sparse_stream_oracle as ss
from demon_b200 import _lib, images, sequence
from test_gpu_sparse_tsdf import cuda, session, triangles, video   # noqa: F401  (session is a fixture)

pytestmark = pytest.mark.gpu

VS, ORIGIN, CHUNK = 0.05, (0.003, -0.002, 0.001), 8


@pytest.fixture(scope="module")
def walk():
    return ss.ring_walk(40)


def calls(walk, color):
    d, K, R, t, img = walk
    for c0 in range(0, d.shape[0], CHUNK):
        sl = slice(c0, c0 + CHUNK)
        yield cuda(d[sl]), cuda(K[sl]), cuda(R[sl]), cuda(t[sl]), cuda(img[sl]) if color else None


def by_block(vol):
    """{block coordinates: (tsdf, weight, color) bytes} over the device and the host."""
    out = {}
    h = vol.host
    parts = [(vol.blocks.cpu(), vol.tsdf.cpu(), vol.weight.cpu(), None if vol.color is None else vol.color.cpu()),
             (h["blocks"], h["tsdf"], h["weight"], h["color"])]
    for b, ts, W, c in parts:
        for i, key in enumerate(map(tuple, b.numpy().tolist())):
            assert key not in out
            out[key] = (ts[i].numpy().tobytes(), W[i].numpy().tobytes(), None if c is None else c[i].numpy().tobytes())
    return out


def test_reach_kernel_equals_the_oracle(walk):
    d, K, R, t, _ = walk
    d = d[:6].copy()
    d[0, :3, :5], d[1, 7:9, :] = np.nan, np.inf
    d[2, 10:12, 3:40] = 0.0
    n, h, w = d.shape
    lib = _lib.load()
    tiles = torch.empty((n, 6, 8), dtype=torch.float32, device="cuda")
    dd = cuda(d)
    _lib.check(lib.demon_sparse_tsdf_depth_tiles_f32(dd.data_ptr(), n, h, w, tiles.data_ptr(), None))
    ref = ss.depth_tiles(d)
    assert np.array_equal(tiles.cpu().numpy().view(np.uint32), ref.view(np.uint32))
    g = np.arange(-8, 8)
    blocks = np.stack(np.meshgrid(g, g, np.arange(-2, 4), indexing="ij"), axis=-1).reshape(-1, 3).astype(np.int32)
    m = blocks.shape[0]
    o = sequence.ctypes.cast((sequence.ctypes.c_float * 3)(*ORIGIN), sequence.ctypes.c_void_p)
    far = np.array([0.5, 3.0, 7.5, 1.0, 2.0, 12.0], np.float32)
    for tl, trunc in ((ref, np.float32(3 * VS)), (ss.raycast_tiles(far, h, w), 0.0)):
        got = []
        for f in range(n):
            out = torch.zeros((m,), dtype=torch.int32, device="cuda")
            x = [cuda(a) for a in (blocks, tl[f:f + 1], K[f:f + 1], R[f:f + 1], t[f:f + 1])]   # alive through the call
            _lib.check(lib.demon_sparse_tsdf_reach_f32(x[0].data_ptr(), m, o, VS, float(trunc), x[1].data_ptr(), x[2].data_ptr(),
                                                       x[3].data_ptr(), x[4].data_ptr(), 1, h, w, out.data_ptr(), 5, None))
            got.append(out.cpu().numpy())
        want = ss.reach(blocks, ORIGIN, VS, trunc, tl, K[:n], R[:n], t[:n], h, w)
        got = np.stack(got)
        bad = np.argwhere(got != np.where(want, 5, 0))
        assert bad.size == 0, (trunc, bad[:5].tolist(), blocks[bad[:5, 1]].tolist(), got[tuple(bad[:5].T)].tolist())
        assert 0 < want.mean() < 0.9
    _lib.check_errors()


@pytest.mark.parametrize("color", [True, False])
@pytest.mark.parametrize("kind", ["below_one_call", "quarter", "tenth"])
def test_budgeted_walk_equals_the_unbudgeted_volume(walk, color, kind):
    ref = sequence.SparseTsdfVolume(VS, ORIGIN, color=color)
    states = []
    for args in calls(walk, color):
        ref.integrate(*args)
        states.append(by_block(ref))
    total = len(states[-1])
    budget = {"below_one_call": len(states[0]) - 1, "quarter": total // 4, "tenth": total // 10}[kind]
    vol = sequence.SparseTsdfVolume(VS, ORIGIN, color=color, max_device_blocks=budget)
    ins, outs = [], []
    for c, args in enumerate(calls(walk, color)):
        vol.integrate(*args)
        assert by_block(vol) == states[c], c
        assert vol.blocks.shape[0] <= budget
        ins.append(vol.last_blocks_in)
        outs.append(vol.last_blocks_out)
    assert sum(outs) > 0 and vol.host["blocks"].shape[0] > 0
    assert max(ins[-2:]) > 0   # the revisit brings blocks back
    assert vol.peak_device_blocks >= budget and vol.host_nbytes > 0
    _lib.check_errors()


@pytest.mark.parametrize("color", [True, False])
def test_raycast_and_mesh_equal_the_unbudgeted_volume(walk, color):
    ref = sequence.SparseTsdfVolume(VS, ORIGIN, color=color)
    for args in calls(walk, color):
        ref.integrate(*args)
    total = ref.blocks.shape[0]
    vol = sequence.SparseTsdfVolume(VS, ORIGIN, color=color, max_device_blocks=total // 5)
    for args in calls(walk, color):
        vol.integrate(*args)
    assert vol.host["blocks"].shape[0] > 0
    mr, mv = ref.mesh(), vol.mesh()
    assert mv[2].shape[0] > 0 and np.array_equal(mv[2].cpu().numpy().reshape(-1), np.arange(3 * mv[2].shape[0]))
    assert np.array_equal(triangles(*mv), triangles(*mr))
    d, K, R, t, _ = walk
    for sl, far in ((slice(0, 40, 5), None), (slice(3, 40, 7), 2.5)):
        a = ref.raycast(cuda(K[sl]), cuda(R[sl]), cuda(t[sl]), 48, 64, far=far)
        b = vol.raycast(cuda(K[sl]), cuda(R[sl]), cuda(t[sl]), 48, 64, far=far)
        for k in ("depth", "normals", "colors"):
            if a[k] is None:
                assert b[k] is None
            else:
                assert np.array_equal(a[k].cpu().numpy().view(np.uint8), b[k].cpu().numpy().view(np.uint8)), k
        assert torch.isfinite(a["depth"]).any()
        assert by_block(vol) == by_block(ref)   # a ray cast moves blocks but changes none
    _lib.check_errors()


def test_mesh_without_host_blocks_is_the_same_mesh(walk):
    ref = sequence.SparseTsdfVolume(VS, ORIGIN)
    vol = sequence.SparseTsdfVolume(VS, ORIGIN, max_device_blocks=10 ** 6)
    for args in calls(walk, True):
        ref.integrate(*args)
        vol.integrate(*args)
    assert vol.host["blocks"].shape[0] == 0 and vol.last_blocks_out == 0
    for a, b in zip(ref.mesh(), vol.mesh()):
        assert torch.equal(a, b)
    for k in ("blocks", "tsdf", "weight", "color"):
        assert torch.equal(getattr(ref, k), getattr(vol, k)), k


def test_same_calls_give_the_same_bytes(walk):
    out = []
    for _ in range(2):
        vol = sequence.SparseTsdfVolume(VS, ORIGIN, max_device_blocks=300)
        for args in calls(walk, True):
            vol.integrate(*args)
        h = vol.host
        out.append([vol.blocks, vol.tsdf, vol.weight, vol.color, h["blocks"], h["tsdf"], h["weight"], h["color"]])
    assert out[0][4].shape[0] > 0
    for a, b in zip(*out):
        assert torch.equal(a.cpu(), b.cpu())


def test_reconstruct_into_a_budgeted_volume(session):   # noqa: F811
    from demon_b200.networks_original import DemonPipeline
    pipe = DemonPipeline(session, batch_size=4, iterations=1)
    frames_u8 = video(7, 3)
    K = np.array([[520.0, 0, 318.0], [0, 515.0, 243.0], [0, 0, 1]])
    box = sequence.reconstruct(pipe, frames_u8, K, min_ratios=1)["volume"]
    vs = float(box.voxel_size) * max(box.dims) / 32
    full = sequence.reconstruct(pipe, frames_u8, K, volume=sequence.SparseTsdfVolume(vs, box.origin), min_ratios=1)
    budget = max(1, full["volume"].blocks.shape[0] // 4)
    res = sequence.reconstruct(pipe, frames_u8, K, volume=sequence.SparseTsdfVolume(vs, box.origin, max_device_blocks=budget), min_ratios=1)
    p = 6
    ch = sequence.chain_pairs(res["inverse_depth"], res["rotation"], res["translation"], min_ratios=1)
    adapted, _, _ = images.adjust_intrinsics(frames_u8, K)
    vol = sequence.SparseTsdfVolume(vs, box.origin, max_device_blocks=budget)
    Kp = torch.from_numpy(sequence.vis.prediction_K(images.NETWORK_INTRINSICS, 1, 192, 256)[0]).cuda()
    vol.integrate(ch["depth"], Kp, cuda(ch["R"][:p].astype(np.float32)), cuda(ch["t"][:p].astype(np.float32)), adapted[:p])
    v0 = res["volume"]
    assert v0.host["blocks"].shape[0] > 0
    assert by_block(vol) == by_block(v0) == by_block(full["volume"])
    v, c, f = vol.mesh()
    assert torch.equal(v, res["vertices"]) and torch.equal(c, res["colors"]) and torch.equal(f, res["faces"])
    assert np.array_equal(triangles(v, c, f), triangles(full["vertices"], full["colors"], full["faces"]))
    _lib.check_errors()
