"""GPU: SparseTsdfVolume's hash table where linear probing and the key range are hardest, against the numpy model of the
table (tests/sparse_table_model.py) and the oracles, bit for bit:
- a chain of 48 keys homed on the table's last slot, wrapping to slot 0 with ordinary keys inside it, fed in one call,
  in three calls and in reverse;
- exactly 512 and 513 keys in a 1024-slot table, with the chain among them and every key raced by 9 threads;
- budgeted volumes whose evictions, restores and chunk pools go through the wrapped chain;
- blocks at the corners (+MAX, +MAX, +MAX) and (-MAX, -MAX, -MAX) and on the +x face of the key range, MAX = 2^20 - 1.
After every call the device table must be the model's: its keys, its full slots, each key in the run from its home
slot, each value its block's place, and its size."""
import numpy as np
import pytest
import torch

import indexed_mesh_oracle as imo
import raycast_oracle as ro
import sequence_oracle as so
import sparse_stream_model as sm
import sparse_table_model as tm
import sparse_tsdf_oracle as sp
from demon_b200 import _lib, sequence
from test_gpu_raycast import same
from test_gpu_sparse_stream import by_block
from test_gpu_sparse_tsdf import cuda, triangles

pytestmark = pytest.mark.gpu

f32 = np.float32
M = tm.MAX_COORD
VS, ORIGIN = 0.05, (0.003, -0.002, 0.001)
CHAIN_TRUNC = f32(f32(1.9) * f32(VS))   # under 2 voxels: a one-block frame stays in its block


def host(x):
    return None if x is None else x.cpu().numpy()


def check_table(vol, expected=None):
    return tm.check_table(*tm.device_table(vol), expected=expected)


# ---- the wrapped chain ------------------------------------------------------------------------------------------------
def patch_frame(block, origin, vs, size=12, f=24.0):
    """A size x size frame looking down +z at a plane at depth 1 through local z = 3.2 of `block`, centred on its voxel
    column (4, 4): it covers about 11 x 11 voxels, so its band allocates the 3 x 3 x 2 blocks around and below."""
    o, vs = np.asarray(origin, f32), f32(vs)
    c = [o[a] + vs * f32(8 * block[a] + 4) for a in range(2)] + [o[2] + vs * f32(8 * block[2] + 3.2)]
    t = np.array([-c[0], -c[1], -(np.float64(c[2]) - 1.0)], f32)
    K = np.array([[f, 0, size / 2], [0, f, size / 2], [0, 0, 1]], f32)
    return np.ones((size, size), f32), K, np.eye(3, dtype=f32), t


@pytest.fixture(scope="module")
def chain_scene():
    """Frames (depth [n,12,12], K, R, t, images) of 48 blocks homed on slot 1023 of 1024, 24 ordinary blocks homed in
    the slots the chain covers, and 3 plane patches centred on chain blocks at z layers 3 apart, so the meshes of the
    patches do not interleave in key order."""
    chain = tm.colliding_blocks(48, (1023,), 20, seed=3)
    zs = np.unique(chain[:, 2])
    centres = []
    for z in zs:
        if not centres or z >= centres[-1][2] + 3:
            centres.append(chain[chain[:, 2] == z][0])
    centres = centres[:3]
    fill = tm.homed_blocks(24, 1023, list(range(1000, 1023)) + list(range(0, 40)), 20, exclude=chain)
    one = tm.one_block_frames(np.concatenate([chain, fill]), ORIGIN, VS, k=12)
    pat = [patch_frame(c, ORIGIN, VS) for c in centres]
    d = np.concatenate([one[0], np.stack([p[0] for p in pat])])
    K = np.concatenate([one[1], np.stack([p[1] for p in pat])])
    R = np.concatenate([one[2], np.stack([p[2] for p in pat])])
    t = np.concatenate([one[3], np.stack([p[3] for p in pat])])
    img = np.random.RandomState(0).randint(0, 256, d.shape + (3,)).astype(np.uint8)
    perm = np.random.RandomState(1).permutation(d.shape[0])   # patches among the one-block frames
    return (d[perm], K[perm], R[perm], t[perm], img[perm]), chain, np.array(centres)


def split(frames, parts, reverse=False):
    idx = np.arange(frames[0].shape[0])[::-1] if reverse else np.arange(frames[0].shape[0])
    return [tuple(a[s] for a in frames) for s in np.array_split(idx, parts)]


def feed(vol, calls, color, check=True):
    """Integrates the calls, checking the table and the allocation after each; returns the model."""
    model = sm.StreamModel(10 ** 9, vol.origin, vol.voxel_size, vol.trunc, color)
    for d, K, R, t, img in calls:
        vol.integrate(cuda(d), cuda(K), cuda(R), cuda(t), cuda(img) if color else None)
        model.integrate(d, K, R, t)
        _, skipped = sp.allocate(d, K, R, t, vol.origin, vol.voxel_size, vol.trunc)
        assert vol.last_skipped_pixels == skipped
        assert np.array_equal(host(vol.blocks), sm.as_blocks(model.device))
        assert vol.table_slots == model.table
        if check:
            check_table(vol, set(model.device))
    return model


def expected_voxels(vol, calls, color):
    """The oracle's tsdf, weight and colour of the pool: a block integrates every frame from the call that made it on."""
    b = host(vol.blocks)
    m = b.shape[0]
    ts, W = np.zeros((m, 8, 8, 8), f32), np.zeros((m, 8, 8, 8), f32)
    col = np.zeros((m, 8, 8, 8, 3), f32) if color else None
    first = 0
    for c, call in enumerate(calls):
        new, _ = sp.allocate(*call[:4], vol.origin, vol.voxel_size, vol.trunc)
        known = set(map(tuple, b[:first].tolist()))
        end = first + len(new - known)
        rest = [np.concatenate([x[i] for x in calls[c:]]) for i in range(5 if color else 4)]
        sl = slice(first, end)
        sp.integrate_blocks(ts[sl], W[sl], None if col is None else col[sl], b[sl], vol.origin, vol.voxel_size, vol.trunc,
                            *rest[:4], rest[4] if color else None)
        first = end
    assert first == m
    return ts, W, col


def check_voxels(vol, calls, color):
    ts, W, col = expected_voxels(vol, calls, color)
    assert np.array_equal(host(vol.tsdf), ts) and np.array_equal(host(vol.weight), W)
    assert (W > 0).any() and (ts < 0).any()
    if color:
        assert np.array_equal(host(vol.color), col)


def layered_mesh_oracle(vol, centres):
    """imo.sparse of each patch's 4 x 4 x 3 blocks around its centre (every meshed cube and every voxel its normals
    read lies there), concatenated in key order: the groups' z layers do not overlap, so their keys do not interleave."""
    b, s, w, c = host(vol.blocks), host(vol.tsdf), host(vol.weight), host(vol.color)
    parts, nv = [], 0
    for centre in sorted(centres.tolist(), key=lambda x: x[2]):
        near = np.flatnonzero((np.abs(b[:, :2] - centre[:2]) <= 2).all(axis=1) & (b[:, 2] - centre[2] >= -2) & (b[:, 2] - centre[2] <= 1))
        out = imo.sparse(b[near], s[near], w[near], None if c is None else c[near], vol.origin, vol.voxel_size)
        assert out["faces"].shape[0] > 50
        out["faces"] = out["faces"] + nv
        nv += out["vertices"].shape[0]
        parts.append(out)
    return {k: None if parts[0][k] is None else np.concatenate([p[k] for p in parts]) for k in imo_keys()}


def imo_keys():
    return ("vertices", "normals", "colors", "faces")


def check_mesh(vol, want):
    got = {k: host(v) for k, v in vol.indexed_mesh().items()}
    for k in imo_keys():
        assert same(got[k], want[k]), k
    assert np.isfinite(got["normals"]).all(axis=1).any() and np.isnan(got["normals"]).any()
    v, c, f = vol.mesh()
    tri = {"vertices": torch.from_numpy(want["vertices"]), "faces": torch.from_numpy(want["faces"])}
    wc = None if want["colors"] is None else torch.from_numpy(want["colors"])
    assert np.array_equal(triangles(v, c, f), triangles(tri["vertices"], wc, tri["faces"]))


def chain_raycast(vol, frames, centres):
    """Ray casts from the patch cameras at the default far, against the oracle."""
    d, K, R, t, _ = frames
    sel = [i for i in range(d.shape[0]) if K[i, 0, 0] == 24.0]
    K, R, t = K[sel], R[sel], t[sel]
    far = vol.default_far(cuda(R), cuda(t))
    assert same(host(far), ro.sparse_far(host(vol.blocks), vol.origin, vol.voxel_size, R, t))
    got = vol.raycast(cuda(K), cuda(R), cuda(t), height=16, width=16)
    ref = ro.raycast(ro.Sparse(host(vol.blocks), host(vol.tsdf), host(vol.weight), host(vol.color)), vol.origin, vol.voxel_size,
                     K, R, t, 0.0, host(far), 0.5, 16, 16)
    for k in ("depth", "normals", "colors"):
        assert (got[k] is None) == (ref[k] is None) and (ref[k] is None or same(host(got[k]), ref[k])), k
    assert np.isfinite(ref["depth"]).sum() > 200
    return got


@pytest.mark.parametrize("order", ["one_call", "three_calls", "reversed"])
def test_wrapped_chain_equals_the_model_and_the_oracles(chain_scene, order):
    frames, chain, centres = chain_scene
    color = order == "one_call"
    calls = split(frames, 1) if order == "one_call" else split(frames, 3, reverse=order == "reversed")
    vol = sequence.SparseTsdfVolume(VS, ORIGIN, trunc=CHAIN_TRUNC, color=color)
    model = feed(vol, calls, color)
    probes = check_table(vol, set(model.device))
    keys = host(vol._table[0])
    # the chain wraps: its run holds slot 1023 and slot 0, its longest probe is past 32 slots, ordinary keys sit in it
    run = [r for r in tm.runs(set(np.flatnonzero(keys != tm.EMPTY).tolist()), 1024) if (r[0] + r[1] - 1) % 1024 < r[0]]
    assert len(run) == 1 and run[0][1] >= 48 and probes.max() >= 47
    in_run = (run[0][0] + np.arange(run[0][1])) % 1024
    homes = tm.home_slot(keys[in_run], 1023)
    assert (homes != 1023).sum() >= 10
    check_voxels(vol, calls, color)
    check_mesh(vol, layered_mesh_oracle(vol, centres))
    chain_raycast(vol, frames, centres)
    _lib.check_errors()


# ---- 512 and 513 keys ---------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def half_full_blocks():
    """513 blocks: 40 homed on slot 2047 of 2048 (so on 1023 of 1024 too), then ordinary ones."""
    chain = tm.colliding_blocks(40, (1023, 2047), 28, seed=5)
    rng = np.random.RandomState(6)
    other = np.unique(rng.randint(-28, 28, size=(2000, 3)), axis=0)
    other = other[~np.isin(tm.packed_key(other), tm.packed_key(chain))]
    other = other[rng.permutation(other.shape[0])[:473]]
    return np.concatenate([chain, other])


@pytest.mark.parametrize("n, parts", [(512, 1), (513, 1), (513, 2)])
def test_half_full_boundary(half_full_blocks, n, parts):
    """512 keys keep 1024 slots, 513 double them once, in one call (the launch overflows and reruns) or as 500 keys and
    then 13 (the rehash moves the full wrapped cluster)."""
    blocks = half_full_blocks[:n]
    d, K, R, t = tm.one_block_frames(blocks, ORIGIN, VS, k=3)   # 9 threads race on each key
    trunc = f32(f32(VS) / f32(2))
    vol = sequence.SparseTsdfVolume(VS, ORIGIN, trunc=trunc, color=False)
    cut = [0, n] if parts == 1 else [0, 500, n]
    calls = [(d[a:b], K[a:b], R[a:b], t[a:b], None) for a, b in zip(cut[:-1], cut[1:])]
    slots = []
    for c, (dd, KK, RR, tt, _) in enumerate(calls):
        vol.integrate(cuda(dd), cuda(KK), cuda(RR), cuda(tt))
        assert vol.last_skipped_pixels == 0
        slots.append(vol.table_slots)
        check_table(vol, set(map(tuple, blocks[:cut[c + 1]].tolist())))
    assert slots[-1] == (1024 if n == 512 else 2048) and (parts == 1 or slots[0] == 1024)
    keys = host(vol._table[0])
    cap = keys.size
    assert keys[cap - 1] != tm.EMPTY and keys[0] != tm.EMPTY   # the 40 keys homed on the last slot wrap
    assert tm.probes(keys, cap).max() >= 39
    # the pool: each call's new blocks in key order
    b = host(vol.blocks)
    for a, z in zip(cut[:-1], cut[1:]):
        part = blocks[a:z]
        assert np.array_equal(b[a:z], part[np.argsort(tm.packed_key(part))])
    ts, W = expected_voxels(vol, calls, False)[:2]
    assert np.array_equal(host(vol.tsdf), ts) and np.array_equal(host(vol.weight), W)
    _lib.check_errors()


# ---- streaming over the chain -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("budget", [1, 14])
def test_streaming_over_the_wrapped_chain(chain_scene, budget):
    frames, chain, centres = chain_scene
    calls = split(frames, 4)
    ref = sequence.SparseTsdfVolume(VS, ORIGIN, trunc=CHAIN_TRUNC, color=True)
    vol = sequence.SparseTsdfVolume(VS, ORIGIN, trunc=CHAIN_TRUNC, color=True, max_device_blocks=budget)
    model = sm.StreamModel(budget, ORIGIN, VS, CHAIN_TRUNC, True)
    for d, K, R, t, img in calls:
        a = (cuda(d), cuda(K), cuda(R), cuda(t), cuda(img))
        ref.integrate(*a)
        vol.integrate(*a)
        model.integrate(d, K, R, t)
        st = model.state()
        assert np.array_equal(host(vol.blocks), st["blocks"]) and np.array_equal(vol.host["blocks"].numpy(), st["host"])
        check_table(vol, model.known())
        assert by_block(vol) == by_block(ref)
    assert vol.host["blocks"].shape[0] > 100 and vol.last_blocks_in + sum(r["host_at_start"] > 0 for r in model.log) > 0
    # the chunk pools' tables: every chunk's blocks, values their chunk index, sized by the doubling
    seen = []
    chunk_pool = vol._chunk_pool

    def recorded(blocks, where):
        chunk = chunk_pool(blocks, where)
        keys, values = chunk["table"]
        tm.check_table(host(keys), host(values), host(blocks), {})
        seen.append(blocks.shape[0])
        return chunk
    vol._chunk_pool = recorded
    assert np.array_equal(triangles(*ref.mesh()), triangles(*vol.mesh()))   # the same soup, in key-ordered chunks
    ia, ib = ref.indexed_mesh(), vol.indexed_mesh()
    for k in imo_keys():
        assert same(host(ia[k]), host(ib[k])), k
    assert len(seen) > 0 and ib["faces"].shape[0] > 100
    d, K, R, t, _ = frames
    sel = [i for i in range(d.shape[0]) if K[i, 0, 0] == 24.0]
    ra = ref.raycast(cuda(K[sel]), cuda(R[sel]), cuda(t[sel]), height=16, width=16)
    rb = vol.raycast(cuda(K[sel]), cuda(R[sel]), cuda(t[sel]), height=16, width=16)
    for k in ("depth", "normals", "colors"):
        assert np.array_equal(host(ra[k]).view(np.uint8), host(rb[k]).view(np.uint8)), k
    model.raycast(K[sel], R[sel], t[sel], 16, 16)
    check_table(vol, model.known())
    assert np.array_equal(host(vol.blocks), model.state()["blocks"])
    _lib.check_errors()


# ---- the ends of the key range -----------------------------------------------------------------------------------------
END_SCENES = {
    # name: (voxel size, the grid coordinate of the sphere's centre (world 0), colour)
    "plus_corner": (0.05, (8 * M + 4,) * 3, True),
    "minus_corner": (0.047, (-8 * M + 4,) * 3, False),
    "plus_x_face": (0.0599, (8 * M + 3, 5, -6), False),
}


def end_scene(name):
    """A sphere of radius 0.6 at world 0 whose centre lies at the scene's grid coordinate: the origin is -vs * g."""
    vs, g, color = END_SCENES[name]
    origin = tuple(float(-f32(vs) * f32(x)) for x in g)
    d, K, R, t, img = so.sphere_views(n=6, h=24, w=32, seed=4)
    return vs, origin, color, (d, K, R, t, img)


def end_cameras(K, R, t):
    """Four integrated cameras, then two at the sphere's centre looking out along +x and -x: their rays leave the key range."""
    Ri, ti = so.look_at((0, 0, 0), (1, 0.2, 0.1))
    Rj, tj = so.look_at((0, 0, 0), (-1, 0.1, -0.2))
    return (np.concatenate([K[:4], K[:1], K[:1]]).astype(f32), np.concatenate([R[:4], [Ri, Rj]]).astype(f32),
            np.concatenate([t[:4], [ti, tj]]).astype(f32))


@pytest.mark.parametrize("name", list(END_SCENES))
def test_blocks_at_the_ends_of_the_key_range(name):
    vs, origin, color, (d, K, R, t, img) = end_scene(name)
    vol = sequence.SparseTsdfVolume(vs, origin, color=color)
    vol.integrate(cuda(d), cuda(K), cuda(R), cuda(t), cuda(img) if color else None)
    want, skipped = sp.allocate(d, K, R, t, vol.origin, vol.voxel_size, vol.trunc)
    b = host(vol.blocks)
    assert set(map(tuple, b.tolist())) == want and vol.last_skipped_pixels == skipped
    assert skipped > 0   # the band crosses the range's face
    edge = M if name.startswith("plus") else -M
    assert (b[:, 0] == edge).any() and np.abs(b).max() <= M
    check_table(vol, want)
    check_voxels(vol, [(d, K, R, t, img)], color)
    # the mesh: a cube whose corners need block 2^20 is skipped, a normal that needs block -2^20 is NaN
    want_mesh = imo.sparse(b, host(vol.tsdf), host(vol.weight), host(vol.color), vol.origin, vol.voxel_size)
    got = {k: host(v) for k, v in vol.indexed_mesh().items()}
    for k in imo_keys():
        assert same(got[k], want_mesh[k]), k
    assert got["faces"].shape[0] > 100
    v, c, f = vol.mesh()
    wc = None if want_mesh["colors"] is None else torch.from_numpy(want_mesh["colors"])
    assert np.array_equal(triangles(v, c, f), triangles(torch.from_numpy(want_mesh["vertices"]), wc, torch.from_numpy(want_mesh["faces"])))
    # ray casts, at the default far, from outside and from inside the range
    Kc, Rc, tc = end_cameras(K, R, t)
    far = vol.default_far(cuda(Rc), cuda(tc))
    assert same(host(far), ro.sparse_far(b, vol.origin, vol.voxel_size, Rc, tc))
    rc = vol.raycast(cuda(Kc), cuda(Rc), cuda(tc), height=24, width=32)
    ref = ro.raycast(ro.Sparse(b, host(vol.tsdf), host(vol.weight), host(vol.color)), vol.origin, vol.voxel_size, Kc, Rc, tc,
                     0.0, host(far), 0.5, 24, 32)
    for k in ("depth", "normals", "colors"):
        assert (rc[k] is None) == (ref[k] is None) and (ref[k] is None or same(host(rc[k]), ref[k])), k
    assert np.isfinite(ref["depth"][:4]).sum() > 200
    _lib.check_errors()


@pytest.mark.parametrize("name", ["plus_corner", "minus_corner"])
def test_budgeted_volume_at_the_ends_of_the_key_range(name):
    vs, origin, color, (d, K, R, t, img) = end_scene(name)
    trunc = f32(3 * f32(vs))
    ref = sequence.SparseTsdfVolume(vs, origin, color=color)
    for c in range(3):
        sl = slice(2 * c, 2 * c + 2)
        ref.integrate(cuda(d[sl]), cuda(K[sl]), cuda(R[sl]), cuda(t[sl]), cuda(img[sl]) if color else None)
    budget = max(1, ref.blocks.shape[0] // 6)
    vol = sequence.SparseTsdfVolume(vs, origin, color=color, max_device_blocks=budget)
    model = sm.StreamModel(budget, vol.origin, vs, trunc, color)
    for c in range(3):
        sl = slice(2 * c, 2 * c + 2)
        vol.integrate(cuda(d[sl]), cuda(K[sl]), cuda(R[sl]), cuda(t[sl]), cuda(img[sl]) if color else None)
        model.integrate(d[sl], K[sl], R[sl], t[sl])
        st = model.state()
        assert np.array_equal(host(vol.blocks), st["blocks"]) and np.array_equal(vol.host["blocks"].numpy(), st["host"]), c
        assert vol.last_blocks_in == st["last_blocks_in"] and vol.last_blocks_out == st["last_blocks_out"], c
        check_table(vol, model.known())
    assert by_block(vol) == by_block(ref) and vol.host["blocks"].shape[0] > 0
    assert sum(r["host_at_start"] > 0 and len(r["evicted"]) > 0 for r in model.log) > 0
    assert np.array_equal(triangles(*ref.mesh()), triangles(*vol.mesh()))   # the same soup, in key-ordered chunks
    ia, ib = ref.indexed_mesh(), vol.indexed_mesh()
    for k in imo_keys():
        assert same(host(ia[k]), host(ib[k])), k
    Kc, Rc, tc = end_cameras(K, R, t)
    ra = ref.raycast(cuda(Kc), cuda(Rc), cuda(tc), height=24, width=32)
    rb = vol.raycast(cuda(Kc), cuda(Rc), cuda(tc), height=24, width=32)
    for k in ("depth", "normals", "colors"):
        assert (ra[k] is None and rb[k] is None) or np.array_equal(host(ra[k]).view(np.uint8), host(rb[k]).view(np.uint8)), k
    model.raycast(Kc, Rc, tc, 24, 32)
    assert np.array_equal(host(vol.blocks), model.state()["blocks"])
    check_table(vol, model.known())
    _lib.check_errors()
