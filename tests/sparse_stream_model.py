"""numpy model of SparseTsdfVolume's block streaming policy (max_device_blocks), restated from DESIGN.md §3.9 "Policy"
and the class's docstrings, for the tests: which blocks stay on the device and in which order, which host slot each
evicted block takes, the traffic counters and the sizes of the pool, the host store and the hash table.  The reach rule
is tests/sparse_stream_oracle.py's and the allocation tests/sparse_tsdf_oracle.py's, so the model predicts a volume's
public state after every call exactly.  It also runs the scenes the GPU tests stream and records the policy's events,
so the CPU tests can pin what those scenes exercise."""
import numpy as np

import raycast_oracle as ro
import sparse_stream_oracle as ss
import sparse_tsdf_oracle as sp

f32 = np.float32
POOL_BLOCKS = 64      # the pool's first capacity; it doubles
TABLE_SLOTS = 1024    # the hash table's first size; it doubles and is never more than half full


def key_order(b):
    """Sort key of a block (bx, by, bz) in ascending packed key: z, then y, then x."""
    return (b[2], b[1], b[0])


def doubling(start, need):
    """The smallest start * 2^k (k >= 0) that is >= need."""
    c = start
    while c < need:
        c *= 2
    return c


def as_blocks(blocks):
    return np.array(blocks, dtype=np.int32).reshape(-1, 3)


class StreamModel:
    """The public state of SparseTsdfVolume(voxel_size, origin, trunc, color, max_device_blocks) after each call.

    `device` is the device blocks in pool order, `stamp` the index of the last call that reached each of them, `slots`
    the host store's slots in use (a block, or None for a free slot).  `log` holds one record per call that ran."""

    def __init__(self, max_device_blocks, origin, voxel_size, trunc, color=True):
        self.budget = int(max_device_blocks)
        self.origin, self.voxel_size, self.trunc, self.color = origin, f32(voxel_size), f32(trunc), color
        self.device, self.stamp, self.slots = [], {}, []
        self.calls = 0
        self.last_blocks_in = self.last_blocks_out = self.peak_device_blocks = 0
        self.capacity = POOL_BLOCKS
        self.host_capacity = 0
        self.table = TABLE_SLOTS
        self.log = []

    # ---- the public state -------------------------------------------------------------------------------------------
    @property
    def host_blocks(self):
        return [b for b in self.slots if b is not None]

    def known(self):
        return set(self.device) | set(self.host_blocks)

    @property
    def host_nbytes(self):
        """tsdf and weight (4 KB), and colour (6 KB more), per slot of capacity."""
        return self.host_capacity * (10240 if self.color else 4096)

    def state(self):
        return {"blocks": as_blocks(self.device), "host": as_blocks(self.host_blocks), "last_blocks_in": self.last_blocks_in,
                "last_blocks_out": self.last_blocks_out, "peak_device_blocks": self.peak_device_blocks,
                "host_nbytes": self.host_nbytes, "capacity": self.capacity, "table": self.table}

    # ---- the calls --------------------------------------------------------------------------------------------------
    def integrate(self, depth, K, R, t):
        depth = np.asarray(depth, f32)
        n, h, w = depth.shape
        rec = self._begin("integrate")
        self._bring_back(rec, ss.depth_tiles(depth), self.trunc, K, R, t, h, w)
        alloc, _ = sp.allocate(depth, K, R, t, self.origin, self.voxel_size, self.trunc)
        new = sorted(alloc - self.known(), key=key_order)
        self._grow_pool(len(self.device) + len(new))
        for b in new:
            self.device.append(b)
            self.stamp[b] = self.calls
        table = doubling(TABLE_SLOTS, 2 * len(self.known()))
        rec["table_grew"] = table > self.table
        self.table = table
        rec["new"] = len(new)
        self._stream_out(rec)

    def raycast(self, K, R, t, h, w, far=None):
        """Returns the far used per frame, or None when the call does nothing (no cameras or an empty volume)."""
        R = np.asarray(R, f32)
        n = R.shape[0]
        everything = self.device + self.host_blocks
        if n == 0 or not everything:
            return None
        if far is None:
            far = ro.sparse_far(as_blocks(everything), self.origin, self.voxel_size, R, t)
        far = np.broadcast_to(np.asarray(far, f32).reshape(-1), (n,)).copy()
        rec = self._begin("raycast")
        rec["table_grew"], rec["new"] = False, 0
        self._bring_back(rec, ss.raycast_tiles(far, h, w), f32(0), K, R, t, h, w)
        self._stream_out(rec)
        return far

    # ---- the policy -------------------------------------------------------------------------------------------------
    def _begin(self, kind):
        self.calls += 1
        rec = {"call": self.calls, "kind": kind, "host_at_start": len(self.host_blocks), "freed": set()}
        self.log.append(rec)
        return rec

    def _grow_pool(self, m):
        self.capacity = doubling(self.capacity, m)

    def _reached(self, blocks, tiles, trunc, K, R, t, h, w):
        if not blocks:
            return np.zeros(0, bool)
        return ss.reach(as_blocks(blocks), self.origin, self.voxel_size, trunc, tiles, K, R, t, h, w).any(axis=0)

    def _bring_back(self, rec, tiles, trunc, K, R, t, h, w):
        """Stamps the device blocks the call reaches; brings back the host blocks it reaches, appended in key order."""
        for b, hit in zip(self.device, self._reached(self.device, tiles, trunc, K, R, t, h, w)):
            if hit:
                self.stamp[b] = self.calls
        live = [s for s, b in enumerate(self.slots) if b is not None]
        hit = self._reached([self.slots[s] for s in live], tiles, trunc, K, R, t, h, w)
        back = [s for s, x in zip(live, hit) if x]
        blocks = sorted((self.slots[s] for s in back), key=key_order)
        rec["slot_order_differs"] = blocks != [self.slots[s] for s in back]
        self._grow_pool(len(self.device) + len(blocks))
        for b in blocks:
            self.device.append(b)
            self.stamp[b] = self.calls
        for s in back:
            self.slots[s] = None
        while self.slots and self.slots[-1] is None:
            self.slots.pop()
        rec["freed"] = {s for s in back if s < len(self.slots)}
        self.last_blocks_in = len(blocks)

    def _stream_out(self, rec):
        """Moves the device blocks beyond the budget to the host, least recently reached first, ties by ascending key;
        the others keep their order.  Evicted blocks take the free slots lowest first, then new slots at the end."""
        m = len(self.device)
        self.peak_device_blocks = max(self.peak_device_blocks, m)
        e = m - self.budget
        self.last_blocks_out = max(e, 0)
        rec.update(evicted=[], stamps=set(), reused_freed=False)
        if e <= 0:
            return
        order = sorted(self.device, key=lambda b: (self.stamp[b],) + key_order(b))
        out, kept = order[:e], order[e:]
        rec["evicted"] = out
        rec["stamps"] = {self.stamp[b] for b in self.device}
        rec["evicted_unreached_kept_reached"] = (any(self.stamp[b] < self.calls for b in out)
                                                 and any(self.stamp[b] == self.calls for b in kept))
        free = [s for s, b in enumerate(self.slots) if b is None]
        slots = free[:e] + list(range(len(self.slots), len(self.slots) + e - len(free[:e])))
        rec["reused_freed"] = bool(rec["freed"] & set(slots))
        self.slots.extend([None] * (slots[-1] + 1 - len(self.slots)))
        for b, s in zip(out, slots):
            self.slots[s] = b
        if len(self.slots) > self.host_capacity:
            self.host_capacity = doubling(max(self.host_capacity, 1), len(self.slots))
        gone = set(out)
        self.device = [b for b in self.device if b not in gone]
        for b in gone:
            del self.stamp[b]
        rec["host_capacity"] = self.host_capacity


# ---- the scenes the GPU tests stream ----------------------------------------------------------------------------------
VS, ORIGIN = 0.05, (0.003, -0.002, 0.001)
TRUNC = f32(3 * f32(VS))   # SparseTsdfVolume's default


def scene(name):
    """(frames, frames per call) of a scene: A is the ring walk at a ragged 45x61, B a ring twice as wide."""
    if name == "A":
        return ss.ring_walk(40, h=45, w=61), 8
    if name == "B":
        return ss.ring_walk(40, L=4.0), 4
    raise ValueError(name)


def chunks(frames, per_call):
    d = frames[0]
    return [tuple(a[c0:c0 + per_call] for a in frames) for c0 in range(0, d.shape[0], per_call)]


def walk(frames, per_call, budget, color=True):
    """The model after each integrate call of a walk: a list of states, and the model."""
    model = StreamModel(budget, ORIGIN, VS, TRUNC, color)
    states = []
    for d, K, R, t, _ in chunks(frames, per_call):
        model.integrate(d, K, R, t)
        states.append(model.state())
    return states, model


def budgets(frames, per_call):
    """{kind: budget}: 1, one below the largest number of blocks one call keeps on the device, about a tenth and about a
    third of the walk's blocks."""
    _, m1 = walk(frames, per_call, 1)
    total = len(m1.known())
    return {"one": 1, "below_peak": m1.peak_device_blocks - 1, "tenth": total // 10, "third": total // 3}


# The interleaved calls on scene A: integrate chunk i ("integrate", i); ray casts from the poses of chunk i with the
# default far, from its first pose with a far that reaches a few blocks, from a camera that sees nothing, at a ragged
# size, and with no cameras (before the first integrate too: an empty volume); and an integrate of depth with no valid
# pixel.
INTERLEAVED = [("empty", None), ("integrate", 0), ("integrate", 1), ("raycast_near", 0), ("integrate", 2), ("raycast", 0), ("blind", None),
               ("integrate", 3), ("invalid", None), ("raycast_ragged", 1), ("empty", None), ("integrate", 4), ("raycast", 2),
               ("integrate", 0)]
NEAR_FAR = 0.1
RAGGED = (13, 21)


def blind_camera():
    """K, R, t [1,...] of a camera 100 m below the scene looking down: every block is behind it."""
    K = np.array([[[40.0, 0, 32.0], [0, 40.0, 24.0], [0, 0, 1]]], f32)
    R = np.array([[[1, 0, 0], [0, -1, 0], [0, 0, -1]]], f32)
    t = np.array([[0, 0, -100.0]], f32)
    return K, R, t


def invalid_depth(h, w):
    """One frame with no valid pixel: NaN, +-inf, 0 and negative depths."""
    d = np.full((1, h, w), np.nan, f32)
    d[0, 1::4], d[0, 2::4], d[0, 3::4] = np.inf, 0.0, -1.0
    d[0, :, ::5] = -np.inf
    return d


def interleaved_calls(frames, per_call):
    """The INTERLEAVED script as (kind, args): ("integrate", (d, K, R, t, img)) or ("raycast", (K, R, t, h, w, far))."""
    ch = chunks(frames, per_call)
    h, w = frames[0].shape[1:]
    out = []
    for kind, i in INTERLEAVED:
        if kind == "integrate":
            out.append(("integrate", ch[i]))
        elif kind == "invalid":
            d0, K, R, t, img = ch[0]
            out.append(("integrate", (invalid_depth(h, w), K[:1], R[:1], t[:1], img[:1])))
        elif kind == "blind":
            out.append(("raycast", blind_camera() + (h, w, None)))
        elif kind == "empty":
            _, K, R, t, _ = ch[0]
            out.append(("raycast", (K[:0], R[:0], t[:0], h, w, None)))
        else:
            _, K, R, t, _ = ch[i]
            if kind == "raycast_near":
                K, R, t = K[:1], R[:1], t[:1]
            size = RAGGED if kind == "raycast_ragged" else (h, w)
            out.append(("raycast", (K, R, t) + size + (NEAR_FAR if kind == "raycast_near" else None,)))
    return out


def run_interleaved(frames, per_call, budget, color=True):
    """The model after each call of the interleaved script: a list of states, and the model."""
    model = StreamModel(budget, ORIGIN, VS, TRUNC, color)
    states = []
    for kind, args in interleaved_calls(frames, per_call):
        if kind == "integrate":
            model.integrate(*args[:4])
        else:
            model.raycast(*args)
        states.append(model.state())
    return states, model
