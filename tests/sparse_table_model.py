"""numpy model of SparseTsdfVolume's hash table (csrc/fusion.cu: block_key, key_slot, insert_key) for the tests: the
packed key and home slot of a block, the slots linear probing fills, a check of a device table against both, blocks
whose keys all hash to the table's last slot (so their probe chain wraps to slot 0), and frames that allocate exactly
one chosen block each, so a test can place keys in the table on purpose."""
import numpy as np

import sparse_stream_model as sm

f32 = np.float32
MAX_COORD = 2 ** 20 - 1   # DEMON_SPARSE_TSDF_MAX_COORD
EMPTY = -1                # the empty key (~0 as int64)
_M1, _M2 = np.uint64(0xbf58476d1ce4e5b9), np.uint64(0x94d049bb133111eb)


def packed_key(b):
    """int64 [N]: block_key of blocks b [N,3], 21 bits per axis offset by 2^20, z highest."""
    b = np.asarray(b, dtype=np.int64).reshape(-1, 3) + (1 << 20)
    return (b[:, 2] << 42) | (b[:, 1] << 21) | b[:, 0]


def decode(key):
    """Blocks [N,3] of packed keys [N] (key_coord)."""
    k = np.asarray(key, dtype=np.int64).reshape(-1)
    return np.stack([((k >> (21 * a)) & ((1 << 21) - 1)) - (1 << 20) for a in range(3)], axis=1)


def home_slot(key, mask):
    """int64 [N]: key_slot, the splitmix64 finaliser of the keys in uint64 arithmetic, masked."""
    k = np.asarray(key, dtype=np.int64).reshape(-1).view(np.uint64).copy()
    k ^= k >> np.uint64(30)
    k *= _M1
    k ^= k >> np.uint64(27)
    k *= _M2
    k ^= k >> np.uint64(31)
    return (k & np.uint64(mask)).astype(np.int64)


def occupied_slots(keys, capacity):
    """The set of slots linear probing fills with the distinct keys (fewer than capacity), without placing them one by
    one: slot s is full when a key homed at s or a key carried past an earlier full slot reaches it.  Two sweeps round
    the table settle the carry that wraps past the last slot.  With no deletions this set is the same for every
    insertion order."""
    keys = np.unique(np.asarray(keys, dtype=np.int64))
    assert keys.size < capacity
    count = np.bincount(home_slot(keys, capacity - 1), minlength=capacity)
    full, carry = np.zeros(capacity, bool), 0
    for s in list(range(capacity)) * 2:
        carry += count[s]
        full[s] = carry > 0
        carry = max(carry - 1, 0)
    return set(np.flatnonzero(full).tolist())


def insert_in_order(keys, capacity):
    """keys [capacity] int64 of a table after inserting `keys` one by one in the given order (EMPTY where empty)."""
    table = np.full(capacity, EMPTY, np.int64)
    for k in np.asarray(keys, dtype=np.int64).reshape(-1).tolist():
        s = int(home_slot([k], capacity - 1)[0])
        while table[s] != EMPTY and table[s] != k:
            s = (s + 1) % capacity
        table[s] = k
    return table


def runs(full, capacity):
    """The maximal runs of full slots as (first slot, length), a run that passes the last slot wrapping to slot 0."""
    full = np.zeros(capacity, bool) if not full else np.isin(np.arange(capacity), sorted(full))
    if full.all():
        return [(0, capacity)]
    start = int(np.flatnonzero(~full)[0]) + 1   # sweep from just after an empty slot
    out, first, length = [], None, 0
    for i in range(capacity):
        s = (start + i) % capacity
        if full[s]:
            first = s if length == 0 else first
            length += 1
        elif length:
            out.append((first, length))
            length = 0
    if length:
        out.append((first, length))
    return out


def probes(keys, capacity):
    """int64 [capacity]: for each full slot of a table `keys`, how many slots past its key's home slot it sits (-1 where
    empty): the length of the probe that finds that key, less one."""
    keys = np.asarray(keys, dtype=np.int64)
    out = np.full(capacity, -1, np.int64)
    s = np.flatnonzero(keys != EMPTY)
    out[s] = (s - home_slot(keys[s], capacity - 1)) % capacity
    return out


def check_table(keys, values, blocks, host_blocks, expected=None):
    """A device table (keys int64 [capacity], values int32 [capacity]) against the model, for a pool of `blocks` [m,3]
    and host slots {slot: block}:
    - its keys are the packed keys of the pool and host blocks (and of `expected`, a set of blocks, when given), each once;
    - its full slots are occupied_slots of those keys;
    - every key sits in the run of full slots that starts at its home slot (no empty slot between, wrapping past the end);
    - every value is its block's pool index, or -2 - s for host slot s;
    - the capacity is the smallest doubling of 1024 slots that holds the keys at most half full.
    Returns probes() of the table."""
    keys, values = np.asarray(keys, np.int64), np.asarray(values, np.int64)
    blocks = np.asarray(blocks, np.int64).reshape(-1, 3)
    capacity = keys.size
    hs = sorted(host_blocks.items())
    stored = {int(k): v for k, v in zip(packed_key(blocks).tolist(), range(blocks.shape[0]))}
    for s, b in hs:
        k = int(packed_key([b])[0])
        assert k not in stored, ("a block both on the device and on the host", b)
        stored[k] = -2 - s
    assert len(stored) == blocks.shape[0] + len(hs), "a block twice in the pool"
    if expected is not None:
        assert set(stored) == set(packed_key(sorted(expected)).tolist()), "the stored blocks are not the expected ones"
    full = np.flatnonzero(keys != EMPTY)
    assert np.unique(keys[full]).size == full.size, "a key in two slots"
    assert set(keys[full].tolist()) == set(stored), "the table's keys are not the stored blocks"
    assert set(full.tolist()) == occupied_slots(list(stored), capacity), "full slots differ from linear probing's"
    p = probes(keys, capacity)
    for s in full.tolist():   # every slot from the key's home to its slot is full
        span = (s - np.arange(p[s] + 1)) % capacity
        assert (keys[span] != EMPTY).all(), ("an empty slot on the probe of", s)
    assert [int(values[s]) for s in full] == [stored[int(keys[s])] for s in full], "a value is not its block's place"
    assert capacity == sm.doubling(sm.TABLE_SLOTS, 2 * len(stored)), (capacity, len(stored))
    return p


def device_table(vol):
    """check_table's arguments of a SparseTsdfVolume: keys, values, pool blocks and host slots."""
    keys, values, _ = vol._table
    hosted = {}
    if vol._host is not None:
        hend = vol._hend
        live = vol._host["live"][:hend].cpu().numpy()
        hb = vol._host["blocks"][:hend].cpu().numpy()
        hosted = {s: tuple(hb[s].tolist()) for s in np.flatnonzero(live).tolist()}
    return keys.cpu().numpy(), values.cpu().numpy(), vol.blocks.cpu().numpy(), hosted


def colliding_blocks(n, masks, region, seed=0):
    """n distinct blocks [n,3] int64 in the cube [-region, region)^3 whose home slot is the last slot under every mask
    of `masks` (e.g. 1023 and 2047: their chain starts at the table's last slot and wraps, and still does after a
    doubling), found by a vectorised search over random blocks.  Raises when the region holds too few."""
    rng = np.random.RandomState(seed)
    found = np.zeros((0, 3), np.int64)
    for _ in range(64):
        b = rng.randint(-region, region, size=(1 << 20, 3)).astype(np.int64)
        key = packed_key(b)
        ok = np.ones(b.shape[0], bool)
        for m in masks:
            ok &= home_slot(key, m) == m
        found = np.unique(np.concatenate([found, b[ok]]), axis=0)
        if found.shape[0] >= n:
            return found[rng.permutation(found.shape[0])[:n]]
    raise ValueError("only %d blocks of [-%d, %d)^3 collide" % (found.shape[0], region, region))


def homed_blocks(n, mask, slots, region, exclude=(), seed=1):
    """n distinct blocks [n,3] of [-region, region)^3, none in `exclude`, whose home slot under `mask` is in `slots`."""
    rng = np.random.RandomState(seed)
    b = np.unique(rng.randint(-region, region, size=(1 << 20, 3)).astype(np.int64), axis=0)
    ok = np.isin(home_slot(packed_key(b), mask), list(slots)) & ~np.isin(packed_key(b), packed_key(np.reshape(exclude, (-1, 3))))
    b = b[ok]
    assert b.shape[0] >= n
    return b[rng.permutation(b.shape[0])[:n]]


def one_block_frames(blocks, origin, voxel_size, k=1):
    """Frames that allocate exactly the given blocks [N,3], one each: depth [N,k,k] = 1, K [N,3,3], R = I [N,3,3], t [N,3]
    float32.  Frame i looks down +z from 1 unit in front of block i's centre voxel (local 4, 4, 4), with fx = fy = 1000
    and cx = cy = k/2, so its k x k pixels all see that voxel's column within k/2000 units (threads racing on one key);
    with trunc = voxel_size / 2 the band cell widened by 2 voxels stays within local 1.5 .. 6.5 along every axis."""
    blocks = np.asarray(blocks, dtype=np.int64).reshape(-1, 3)
    n = blocks.shape[0]
    o, vs = np.asarray(origin, dtype=f32), f32(voxel_size)
    centre = np.stack([o[a] + vs * (8 * blocks[:, a] + 4).astype(f32) for a in range(3)], axis=1)
    t = -centre.astype(f32)
    t[:, 2] = (-(centre[:, 2].astype(np.float64) - 1.0)).astype(f32)
    K = np.array([[1000.0, 0, k / 2], [0, 1000.0, k / 2], [0, 0, 1]], f32)
    return (np.ones((n, k, k), f32), np.broadcast_to(K, (n, 3, 3)).copy(), np.broadcast_to(np.eye(3, dtype=f32), (n, 3, 3)).copy(), t)
