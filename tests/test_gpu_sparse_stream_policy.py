"""GPU: which blocks a budgeted SparseTsdfVolume keeps on the device, call by call, against the numpy model of its policy
(tests/sparse_stream_model.py): the device blocks in pool order, the host blocks in slot order, the traffic counters and
the sizes of the pool, the host store and the hash table, over two ring walks, interleaved integrate and ray cast calls
and meshes at budgets 1 and 2, while every block, ray cast and mesh equals an unbudgeted volume's.  The depth tiles and
the reach kernel equal tests/sparse_stream_oracle.py bit for bit at frame sizes that are not whole 8x8 tiles."""
import functools

import numpy as np
import pytest
import torch

import sparse_stream_model as sm
import sparse_stream_oracle as ss
from demon_b200 import _lib, sequence
from test_gpu_sparse_stream import by_block
from test_gpu_sparse_tsdf import cuda, triangles

pytestmark = pytest.mark.gpu

f32 = np.float32
BAD = (np.nan, np.inf, 0.0, -1.0, -np.inf)


def ragged_depth(n, h, w):
    """Ring walk frames of h x w whose clipped last row and column of tiles hold NaN, inf, 0 and negative pixels with
    each tile's largest depth in its last pixel; in the last frame those tiles hold no valid pixel at all."""
    d, K, R, t, _ = ss.ring_walk(n, h=h, w=w, f=40.0 * w / 64)
    th, tw = -(-h // 8), -(-w // 8)
    ragged = [(ty, tx) for ty in range(th) for tx in range(tw) if (h % 8 and ty == th - 1) or (w % 8 and tx == tw - 1)]
    for f in range(n):
        for k, (ty, tx) in enumerate(ragged):
            tile = d[f, 8 * ty:8 * ty + 8, 8 * tx:8 * tx + 8]   # a view, clipped to the image
            if f == n - 1:
                tile[...] = np.resize(np.array(BAD, f32), tile.shape)
                continue
            flat = tile.reshape(-1).copy()
            top = f32(flat.max() + 1.0)
            for i in range(k % 3, flat.size - 1, 3):
                flat[i] = BAD[(i // 3) % len(BAD)]
            flat[-1] = top
            tile[...] = flat.reshape(tile.shape)
    return d, K, R, t, ragged


def device_tiles(d):
    n, h, w = d.shape
    tiles = torch.full((n, -(-h // 8), -(-w // 8)), 7.0, dtype=torch.float32, device="cuda")
    dd = cuda(d)
    _lib.check(_lib.load().demon_sparse_tsdf_depth_tiles_f32(dd.data_ptr(), n, h, w, tiles.data_ptr(), None))
    return tiles.cpu().numpy()


def device_reach(blocks, tiles, trunc, K, R, t, h, w):
    """bool [n, m], one launch per frame; one more launch of every frame must give their union."""
    lib, m = _lib.load(), blocks.shape[0]
    o = sequence.ctypes.cast((sequence.ctypes.c_float * 3)(*sm.ORIGIN), sequence.ctypes.c_void_p)
    got = []
    for f in range(tiles.shape[0]):
        out = torch.zeros((m,), dtype=torch.int32, device="cuda")
        x = [cuda(a) for a in (blocks, tiles[f:f + 1], K[f:f + 1], R[f:f + 1], t[f:f + 1])]   # alive through the call
        _lib.check(lib.demon_sparse_tsdf_reach_f32(x[0].data_ptr(), m, o, sm.VS, float(trunc), x[1].data_ptr(), x[2].data_ptr(),
                                                   x[3].data_ptr(), x[4].data_ptr(), 1, h, w, out.data_ptr(), 3, None))
        got.append(out.cpu().numpy())
    out = torch.zeros((m,), dtype=torch.int32, device="cuda")   # all frames in one launch, as a call runs them
    x = [cuda(a) for a in (blocks, tiles, K, R, t)]
    _lib.check(lib.demon_sparse_tsdf_reach_f32(x[0].data_ptr(), m, o, sm.VS, float(trunc), x[1].data_ptr(), x[2].data_ptr(),
                                               x[3].data_ptr(), x[4].data_ptr(), tiles.shape[0], h, w, out.data_ptr(), 3, None))
    got = np.stack(got)
    assert np.isin(got, (0, 3)).all() and np.isin(out.cpu().numpy(), (0, 3)).all()
    assert np.array_equal(out.cpu().numpy() == 3, (got == 3).any(axis=0))
    return got == 3


@pytest.mark.parametrize("h,w", [(1, 1), (5, 3), (7, 9), (45, 61), (47, 64), (48, 63)])
def test_ragged_tiles_and_reach_equal_the_oracle(h, w):
    d, K, R, t, ragged = ragged_depth(4, h, w)
    tiles = device_tiles(d)
    ref = ss.depth_tiles(d)
    assert np.array_equal(tiles.view(np.uint32), ref.view(np.uint32))
    last = [ref[:-1, ty, tx] for ty, tx in ragged]
    assert np.isfinite(last).all() and np.isneginf([ref[-1, ty, tx] for ty, tx in ragged]).all()
    g = np.arange(-8, 8)
    blocks = np.stack(np.meshgrid(g, g, np.arange(-2, 4), indexing="ij"), axis=-1).reshape(-1, 3).astype(np.int32)
    far = np.array([0.7, 2.0, 4.5, 9.0], f32)
    decided = 0
    for tl, trunc in ((ref, sm.TRUNC), (ss.raycast_tiles(far, h, w), f32(0))):
        got = device_reach(blocks, tl, trunc, K, R, t, h, w)
        want = ss.reach(blocks, sm.ORIGIN, sm.VS, trunc, tl, K, R, t, h, w)
        bad = np.argwhere(got != want)
        assert bad.size == 0, (trunc, bad[:5].tolist(), blocks[bad[:5, 1]].tolist())
        assert 0 < want.mean() < 1
        cut = tl.copy()
        for ty, tx in ragged:
            cut[:, ty, tx] = -np.inf
        decided += int((want != ss.reach(blocks, sm.ORIGIN, sm.VS, trunc, cut, K, R, t, h, w)).sum())
    assert decided > 0   # the clipped tiles alone reach some block
    _lib.check_errors()


@functools.lru_cache(maxsize=None)
def scene(name):
    frames, per_call = sm.scene(name)
    return frames, per_call, sm.budgets(frames, per_call)


def volume(color, budget=None):
    return sequence.SparseTsdfVolume(sm.VS, sm.ORIGIN, color=color, max_device_blocks=budget)


def args(call, color):
    d, K, R, t, img = call
    return cuda(d), cuda(K), cuda(R), cuda(t), cuda(img) if color else None


def check_state(vol, st, where):
    """The volume's public state equals the model's prediction; returns (predicted table size, table size)."""
    assert np.array_equal(vol.blocks.cpu().numpy(), st["blocks"]), where
    assert np.array_equal(vol.host["blocks"].numpy(), st["host"]), where
    got = (vol.last_blocks_in, vol.last_blocks_out, vol.peak_device_blocks, vol.host_nbytes, vol.capacity)
    assert got == tuple(st[k] for k in ("last_blocks_in", "last_blocks_out", "peak_device_blocks", "host_nbytes", "capacity")), where
    return st["table"], vol.table_slots


def check_tables(tables):
    """The table doubles only as its keys need: after every call it has the model's size, the smallest doubling of 1024
    slots that holds every block at most half full (so within the bound p <= slots <= 2p, and exactly p)."""
    assert all(p == slots for p, slots in tables), tables


@pytest.mark.parametrize("name,kind,color", [("A", "one", True), ("A", "below_peak", False), ("A", "tenth", True), ("A", "third", False),
                                             ("B", "one", False), ("B", "below_peak", True), ("B", "tenth", False), ("B", "third", True)])
def test_walk_follows_the_model(name, kind, color):
    frames, per_call, budgets = scene(name)
    states, model = sm.walk(frames, per_call, budgets[kind], color)
    ref, vol = volume(color), volume(color, budgets[kind])
    tables, grew_with_host = [], False
    for c, call in enumerate(sm.chunks(frames, per_call)):
        a = args(call, color)
        ref.integrate(*a)
        slots, host = vol.table_slots, vol.host["blocks"].shape[0]
        vol.integrate(*a)
        grew_with_host |= host > 0 and vol.table_slots > slots
        tables.append(check_state(vol, states[c], c))
        assert by_block(vol) == by_block(ref), c
    check_tables(tables)
    assert grew_with_host == any(r["table_grew"] and r["host_at_start"] for r in model.log)
    _lib.check_errors()


def raycast_both(ref, vol, K, R, t, h, w, far):
    a = ref.raycast(cuda(K), cuda(R), cuda(t), h, w, far=far)
    b = vol.raycast(cuda(K), cuda(R), cuda(t), h, w, far=far)
    for k in ("depth", "normals", "colors"):
        if a[k] is None:
            assert b[k] is None
        else:
            assert np.array_equal(a[k].cpu().numpy().view(np.uint8), b[k].cpu().numpy().view(np.uint8)), k
    return a


@pytest.mark.parametrize("kind,color", [("tenth", True), ("one", False)])
def test_interleaved_calls_follow_the_model(kind, color):
    frames, per_call, budgets = scene("A")
    states, _ = sm.run_interleaved(frames, per_call, budgets[kind], color)
    ref, vol = volume(color), volume(color, budgets[kind])
    tables, hits = [], 0
    for c, (op, x) in enumerate(sm.interleaved_calls(frames, per_call)):
        if op == "integrate":
            a = args(x, color)
            ref.integrate(*a)
            vol.integrate(*a)
        else:
            K, R, t, h, w, far = x
            hits += int(torch.isfinite(raycast_both(ref, vol, K, R, t, h, w, far)["depth"]).sum())
        tables.append(check_state(vol, states[c], (c, op)))
        assert by_block(vol) == by_block(ref), (c, op)
    assert hits > 0
    check_tables(tables)
    _lib.check_errors()


@pytest.mark.parametrize("budget", [1, 2])
@pytest.mark.parametrize("color", [True, False])
def test_mesh_in_one_and_two_block_chunks(budget, color):
    frames, per_call, _ = scene("A")
    states, _ = sm.walk(frames, per_call, budget, color)
    ref, vol = volume(color), volume(color, budget)
    for call in sm.chunks(frames, per_call):
        a = args(call, color)
        ref.integrate(*a)
        vol.integrate(*a)
    check_state(vol, states[-1], "walk")
    before = by_block(vol)
    mr, mv = ref.mesh(), vol.mesh()
    assert mv[2].shape[0] > 0 and np.array_equal(mv[2].cpu().numpy().reshape(-1), np.arange(3 * mv[2].shape[0]))
    assert (mv[1] is None) == (not color)
    assert np.array_equal(triangles(*mv), triangles(*mr))
    check_state(vol, states[-1], "mesh")
    assert by_block(vol) == before
    _lib.check_errors()
