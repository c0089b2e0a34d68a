"""CPU: the numpy model of the sparse TSDF's hash table (tests/sparse_table_model.py), the blocks and frames the GPU tests
place in it, and the allocation rule at the ends of the key range, |b| <= MAX = 2^20 - 1 per axis: the guarantee of
tests/test_sparse_tsdf.py (every updated voxel and every corner of a surface cube allocated) with the grid coordinates
near +-2^23, where float32 resolves half a voxel, and pixels whose block range ends on or just past either end."""
import itertools

import numpy as np
import pytest
import torch

import indexed_mesh_oracle as imo
import sequence_oracle as so
import sparse_table_model as tm
import sparse_tsdf_oracle as sp
from demon_b200 import sequence

f32 = np.float32
M = tm.MAX_COORD


def random_keys(n, seed):
    b = np.unique(np.random.RandomState(seed).randint(-30, 30, size=(3 * n, 3)), axis=0)[:n]
    return tm.packed_key(b)


@pytest.mark.parametrize("extra", [0, 200, 450])
def test_occupied_slots_do_not_depend_on_insertion_order(extra):
    chain = tm.packed_key(tm.colliding_blocks(40, (1023,), 20))
    keys = np.concatenate([chain, random_keys(extra, extra)])
    want = tm.occupied_slots(keys, 1024)
    assert 1023 in want and 0 in want and len(want) == keys.size
    rng = np.random.RandomState(extra)
    tables = [tm.insert_in_order(keys[rng.permutation(keys.size)], 1024) for _ in range(5)]
    tables.append(tm.insert_in_order(np.sort(keys), 1024))
    for table in tables:
        assert set(np.flatnonzero(table != tm.EMPTY).tolist()) == want
        assert set(table[table != tm.EMPTY].tolist()) == set(keys.tolist())
    # the in-cluster order differs between orders, the set of slots does not
    assert len({tuple(t.tolist()) for t in tables}) > 1


def test_check_table_accepts_every_order_and_refuses_a_broken_probe():
    blocks = np.concatenate([tm.colliding_blocks(40, (1023,), 20), np.unique(np.random.RandomState(2).randint(-9, 9, (80, 3)), axis=0)])
    blocks = np.unique(blocks, axis=0)
    keys = tm.insert_in_order(tm.packed_key(blocks)[::-1], 1024)
    index = {k: i for i, k in enumerate(tm.packed_key(blocks).tolist())}
    values = np.array([index.get(k, -1) for k in keys.tolist()], np.int64)
    p = tm.check_table(keys, values, blocks, {}, set(map(tuple, blocks.tolist())))
    assert p.max() >= 39
    bad = keys.copy()   # a key one slot past an empty slot: its probe would stop before it
    s = int(np.flatnonzero(bad == tm.EMPTY)[0])
    bad[s], bad[s - 1] = bad[s - 1], tm.EMPTY
    if bad[s] != tm.EMPTY:
        with pytest.raises(AssertionError):
            tm.check_table(bad, values, blocks, {})
    host = {0: tuple(blocks[-1].tolist())}   # the last block on the host, slot 0
    hv = values.copy()
    hv[keys == tm.packed_key(blocks[-1:])[0]] = -2
    tm.check_table(keys, hv, blocks[:-1], host)
    with pytest.raises(AssertionError):
        tm.check_table(keys, values, blocks[:-1], host)


def test_colliding_blocks_collide_and_their_cluster_wraps():
    b = tm.colliding_blocks(40, (1023, 2047), 28, seed=5)
    k = tm.packed_key(b)
    assert np.unique(b, axis=0).shape[0] == 40 and np.abs(b).max() <= 28
    assert (tm.home_slot(k, 1023) == 1023).all() and (tm.home_slot(k, 2047) == 2047).all()
    assert np.array_equal(tm.decode(k), b)
    for cap in (1024, 2048):
        table = tm.insert_in_order(k, cap)
        assert tm.runs(set(np.flatnonzero(table != tm.EMPTY).tolist()), cap) == [(cap - 1, 40)]
        assert tm.probes(table, cap).max() == 39


ENDS = [((M, M, M), -8 * M), ((-M, -M, -M), 8 * M), ((-M + 1, 3, 3), 0), ((M, 2, -3), None), ((5, -M, 7), None),
        ((-17, 4, 2), 0)]


@pytest.mark.parametrize("block, shift", ENDS)
@pytest.mark.parametrize("k", [1, 4])
def test_one_block_frames_allocate_exactly_their_block(block, shift, k):
    vs = 0.05
    if shift is None:   # the origin puts the block's voxels near grid 0 along the axes at the range's end
        shift = 0
        origin = tuple(-8 * b * vs if abs(b) == M else 0.0 for b in block)
    else:
        origin = (shift * vs,) * 3
    d, K, R, t = tm.one_block_frames([block], origin, vs, k)
    blocks, skipped = sp.allocate(d, K, R, t, origin, vs, f32(f32(vs) / 2))
    assert blocks == {tuple(block)} and skipped == 0


def test_one_block_frames_of_many_blocks():
    b = np.concatenate([tm.colliding_blocks(30, (1023,), 20), [[3, -4, 5]]])
    d, K, R, t = tm.one_block_frames(b, (0.01, -0.02, 0.03), 0.05, 3)
    blocks, skipped = sp.allocate(d, K, R, t, (0.01, -0.02, 0.03), 0.05, f32(0.025))
    assert blocks == set(map(tuple, b.tolist())) and skipped == 0


@pytest.mark.parametrize("block, origin, allocated", [
    ((M, 0, 0), (-8 * M * 0.05, 0, 0), True),             # the range ends exactly at +MAX
    ((-M, 0, 0), (8 * M * 0.05, 0, 0), True),             # ... starts exactly at -MAX
    ((M + 1, 0, 0), (-8 * M * 0.05, 0, 0), False),        # one block past +MAX
    ((-M - 1, 0, 0), (8 * M * 0.05, 0, 0), False),        # one block past -MAX
    ((0, M + 1, 0), (0, -8 * M * 0.05, 0), False),
    ((0, 0, -M - 1), (0, 0, 8 * M * 0.05), False),
])
def test_pixels_at_and_past_the_ends_of_the_key_range(block, origin, allocated):
    d, K, R, t = tm.one_block_frames([block], origin, 0.05, 2)
    blocks, skipped = sp.allocate(d, K, R, t, origin, 0.05, f32(0.025))
    assert (blocks, skipped) == (({tuple(block)}, 0) if allocated else (set(), 4))


def test_a_range_across_the_end_is_skipped():
    """A pixel at local x 1 of block MAX reaches block MAX - 1 too, and one at local 7 reaches block MAX + 1: skipped."""
    vs, origin = 0.05, (-8 * M * 0.05, 0, 0)
    d, K, R, t = tm.one_block_frames([(M, 0, 0)] * 2, origin, vs, 1)
    t[0, 0] += f32(3 * vs)     # the camera moves +3 voxels in x: the voxel column is at local 1
    t[1, 0] -= f32(3 * vs)     # ... at local 7
    blocks, skipped = sp.allocate(d, K, R, t, origin, vs, f32(0.025))
    assert blocks == {(M - 1, 0, 0), (M, 0, 0)} and skipped == 1


def test_packed_keys_agree_at_the_ends_of_the_key_range():
    b = np.array([[M, M, M], [-M, -M, -M], [M, -M, 0], [-M, M, -M], [0, 0, M], [0, 0, -M], [M, 0, 0], [-M, 0, 0], [1, -1, 0],
                  [-M + 1, M - 1, 3]], np.int64)
    k = tm.packed_key(b)
    assert np.array_equal(k, imo.packed_keys(b))
    assert np.array_equal(k, sequence._packed_keys(torch.from_numpy(b.astype(np.int32))).numpy())
    assert np.array_equal(tm.decode(k), b) and (k > 0).all()
    order = np.argsort(k)
    assert np.array_equal(order, np.lexsort((b[:, 0], b[:, 1], b[:, 2])))


# ---- the allocation guarantee near g = +-2^23 ---------------------------------------------------------------------------
def shifted_scenes():
    """Sphere views with the origin moved so that the sphere's centre (world 0) sits at grid coordinate s (8 MAX - 30)
    on one, two or three axes (s = +1 or -1) and near 0 on the others, at voxel sizes where o + vs g rounds by about
    half a voxel."""
    d, K, R, t, _ = so.sphere_views(n=6, h=24, w=32, seed=7)
    g = 8 * M - 30
    for vs in (0.0599, 0.047, 0.05, 0.0625):
        for axes in ((0,), (1, 2), (0, 1, 2)):
            for s in (1, -1):
                centre = [s * g if a in axes else 3 for a in range(3)]
                origin = tuple(float(-f32(vs) * f32(c)) for c in centre)
                yield "%g-%s-%+d" % (vs, "".join("xyz"[a] for a in axes), s), d, K, R, t, origin, vs


@pytest.mark.parametrize("scene", list(shifted_scenes()), ids=lambda s: s[0])
def test_allocation_covers_every_updated_voxel_and_every_surface_cube_near_the_ends(scene):
    _, d, K, R, t, origin, vs = scene
    trunc = f32(3 * f32(vs))
    blocks, skipped = sp.allocate(d, K, R, t, origin, vs, trunc)
    assert skipped == 0 and len(blocks) > 0
    b = np.array(sorted(blocks))
    lo, hi = b.min(axis=0) - 1, b.max(axis=0) + 1     # the allocated blocks' box and a shell of one block
    assert (np.abs(lo) > 8 ** 6).any() and np.abs(hi).max() <= M
    box = np.stack(np.meshgrid(*[np.arange(lo[a], hi[a] + 1) for a in range(3)], indexing="ij"), axis=-1).reshape(-1, 3)
    m = box.shape[0]
    ts, W = np.zeros((m, 8, 8, 8), f32), np.zeros((m, 8, 8, 8), f32)
    sp.integrate_blocks(ts, W, None, box, origin, vs, trunc, d, K, R, t)
    assert (W > 0).any() and (ts < 0).any()
    l = np.arange(512)
    g = (8 * box[:, None, :] + np.stack([l & 7, (l >> 3) & 7, l >> 6], axis=1)[None]).reshape(-1, 3)
    keys = set(tm.packed_key(b).tolist())

    def allocated(x):
        return np.isin(tm.packed_key(sp.block_of(x)), list(keys))

    ts, W = ts.reshape(-1), W.reshape(-1)
    assert allocated(g[(W > 0) & (ts < 1)]).all()
    # every cube with a corner below zero has all 8 corners allocated: every voxel within one step of a negative voxel
    neg = g[(W > 0) & (ts < 0)]
    for dd in itertools.product((-1, 0, 1), repeat=3):
        assert allocated(neg + np.array(dd)).all(), dd
    # the band stays inside the box: no voxel of the outer shell was reached with f < 1
    shell = ~np.isin(tm.packed_key(box), list(keys))
    band = ((W > 0) & (ts < 1)).reshape(m, 512)
    assert not band[shell].any()
