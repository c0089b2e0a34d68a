"""GPU: the indexed mesh (TsdfVolume.indexed_mesh, SparseTsdfVolume.indexed_mesh; csrc/fusion.cu's edge kernels) bit for
bit against tests/indexed_mesh_oracle.py and against mesh()'s soup, on dense boxes of odd size and past 1024 scan tiles,
sparse volumes with negative blocks and a pool out of key order, the ~9 000-block sphere, and budgeted ring walks whose
blocks stream to the host."""
import numpy as np
import pytest
import torch

import fusion_boundary_scenes as fb
import indexed_mesh_oracle as imo
import sequence_oracle as so
import sparse_stream_model as sm
from demon_b200 import _lib, sequence, vis

pytestmark = pytest.mark.gpu
f32 = np.float32
KEYS = ("vertices", "normals", "colors", "faces")


def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(x):
    return None if x is None else x.cpu().numpy()


def same(a, b):
    """Equal bytes (None matching None), NaN matching NaN whatever its payload."""
    if a is None or b is None:
        return a is None and b is None
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype.kind != "f":
        return a.shape == b.shape and np.array_equal(a, b)
    na, nb = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))


def check(got, want, normals=True):
    got = {k: host(v) for k, v in got.items()}
    for k in KEYS:
        w = want[k] if (k != "normals" or normals) else None
        assert same(got[k], w), k
    return got


def state(vol):
    """A sparse volume's whole state, device and host, as numpy."""
    hs = vol.host
    out = {k: host(getattr(vol, k)) for k in ("blocks", "tsdf", "weight", "color")}
    out.update({"host_" + k: None if v is None else v.numpy() for k, v in hs.items()})
    out["keys"], out["values"] = host(vol._table[0]), host(vol._table[1])
    return out


def frames(d, K, R, t, img, color=True):
    return cuda(d), cuda(K), cuda(R), cuda(t), cuda(img) if color else None


@pytest.fixture(scope="module")
def sphere_box():
    """24 sphere views fused into an odd 37x41x43 box, with and without colour, and the oracle's meshes."""
    d, K, R, t, img = so.sphere_views()
    dims, origin, vs = (37, 41, 43), (-0.81, -0.9, -0.94), 0.043
    vols = {}
    for color in (True, False):
        vol = sequence.TsdfVolume(dims, origin, vs, color=color)
        vol.integrate(*frames(d, K, R, t, img, color))
        s, w, c = host(vol.tsdf), host(vol.weight), host(vol.color)
        vols[color] = vol, imo.dense(s, w, c, origin, vs)
    return vols


@pytest.mark.parametrize("normals", [True, False])
@pytest.mark.parametrize("color", [True, False])
def test_dense_odd_box_equals_the_oracle_and_the_soup(sphere_box, color, normals):
    vol, want = sphere_box[color]
    got = check(vol.indexed_mesh(normals=normals), want, normals)
    assert got["faces"].shape[0] > 1000
    if normals:
        assert (~np.isnan(got["normals"]).any(axis=1)).mean() > 0.9
    sv, sc, sf = (host(x) for x in vol.mesh())
    assert same(got["vertices"][got["faces"]].reshape(-1, 3), sv)
    if color:
        assert same(got["colors"][got["faces"]].reshape(-1, 3), sc)
    assert 5 * got["vertices"].shape[0] < sv.shape[0]
    _lib.check_errors()


def test_dense_past_1024_tiles_equals_the_oracle():
    origin, vs, dims = (0.1, -0.2, 0.3), 0.01, (131, 137, 130)
    s, w, c = fb.two_spheres(dims)
    vol = sequence.TsdfVolume(dims, origin, vs)
    vol.tsdf.copy_(cuda(s))
    vol.weight.copy_(cuda(w))
    vol.color.copy_(cuda(c))
    want = imo.dense(s, w, c, origin, vs)
    got = check(vol.indexed_mesh(), want)
    assert np.isnan(got["normals"]).any() and (~np.isnan(got["normals"])).any()
    assert same(got["vertices"][got["faces"]].reshape(-1, 3), host(vol.mesh()[0]))
    _lib.check_errors()


def sparse_want(vol, normals=True):
    return imo.sparse(host(vol.blocks), host(vol.tsdf), host(vol.weight), host(vol.color), vol.origin, vol.voxel_size, normals)


@pytest.mark.parametrize("color", [True, False])
def test_sparse_negative_blocks_two_calls_equal_the_oracle_and_the_soup(color):
    d, K, R, t, img = so.sphere_views()
    vol = sequence.SparseTsdfVolume(0.043, (0.01, -0.02, 0.005), color=color)
    vol.integrate(*frames(d[:12], K[:12], R[:12], t[:12], img[:12], color))
    vol.integrate(*frames(d[12:], K[12:], R[12:], t[12:], img[12:], color))
    b = host(vol.blocks)
    assert b.min() < 0 and not np.array_equal(np.argsort(imo.packed_keys(b), kind="stable"), np.arange(b.shape[0]))
    want = sparse_want(vol)
    got = check(vol.indexed_mesh(), want)
    assert got["faces"].shape[0] > 1000
    # mesh() is the same triangles with each block's run in pool order: sort the key-ordered triangles by pool index
    tri_v = got["vertices"][got["faces"]]
    sv = host(vol.mesh()[0]).reshape(-1, 3, 3)
    runs = _runs(sv, b, vol)   # the soup triangles of each pool block
    perm = np.concatenate([runs[q] for q in np.argsort(imo.packed_keys(b), kind="stable")])
    assert same(tri_v, sv[perm])
    _lib.check_errors()


def _runs(sv, b, vol):
    """The soup triangles of each pool block, as index arrays, from the soup's run lengths (mesh() of the volume with only
    that block's cubes counted: the range entry on one block)."""
    lib, pool = _lib.load(), vol._pool
    keys, values, _ = vol._table
    m = b.shape[0]
    scratch = torch.empty((lib.demon_sparse_tsdf_mesh_scratch_bytes(1),), dtype=torch.uint8, device="cuda")
    total = torch.empty((1,), dtype=torch.int64, device="cuda")
    counts = []
    for q in range(m):
        _lib.check(lib.demon_sparse_tsdf_mesh_range_count_f32(pool["tsdf"].data_ptr(), pool["weight"].data_ptr(), pool["blocks"].data_ptr(), m,
                                                              q, 1, keys.data_ptr(), values.data_ptr(), keys.numel(), scratch.data_ptr(),
                                                              total.data_ptr(), sequence._stream()))
        counts.append(int(total.item()))
    first = np.cumsum(counts) - counts
    assert sum(counts) == sv.shape[0]
    return [np.arange(first[q], first[q] + counts[q]) for q in range(m)]


def test_sparse_sphere_of_9000_blocks_equals_the_oracle():
    views = fb.varied_sphere_views(24, 192, 256)
    vol = sequence.SparseTsdfVolume(0.005, (-0.75, -0.75, -0.75))
    vol.integrate(*frames(*views))
    assert vol.blocks.shape[0] > 4 * 1024
    got = check(vol.indexed_mesh(), sparse_want(vol))
    assert got["faces"].shape[0] > 100000
    _lib.check_errors()


@pytest.mark.parametrize("color", [True, False])
def test_budgeted_ring_walk_gives_the_unbudgeted_bytes(color):
    walk, per_call = sm.scene("A")
    budgets = sm.budgets(walk, per_call)
    ref = sequence.SparseTsdfVolume(sm.VS, sm.ORIGIN, color=color)
    vols = {k: sequence.SparseTsdfVolume(sm.VS, sm.ORIGIN, color=color, max_device_blocks=budgets[k]) for k in ("one", "below_peak", "tenth")}
    for d, K, R, t, img in sm.chunks(walk, per_call):
        for v in [ref] + list(vols.values()):
            v.integrate(*frames(d, K, R, t, img, color))
    want = {k: host(v) for k, v in ref.indexed_mesh().items()}
    check(ref.indexed_mesh(), want)   # two calls, identical bytes
    oracle = sparse_want(ref)
    check(ref.indexed_mesh(), oracle)
    assert want["faces"].shape[0] > 1000
    for name, v in vols.items():
        assert v._host_blocks() > 0, name
        before = state(v)
        check(v.indexed_mesh(), want)
        check(v.indexed_mesh(normals=False), want, normals=False)
        after = state(v)
        assert all(same(before[k], after[k]) for k in before), name
    _lib.check_errors()


def test_empty_volumes_give_empty_outputs():
    for vol in (sequence.SparseTsdfVolume(0.05), sequence.SparseTsdfVolume(0.05, color=False, max_device_blocks=2)):
        out = vol.indexed_mesh()
        assert out["vertices"].shape == (0, 3) and out["faces"].shape == (0, 3) and out["normals"].shape == (0, 3)
    # blocks (or voxels), but no surface
    dense = sequence.TsdfVolume((9, 10, 11), (0, 0, 0), 0.1)
    dense.weight.fill_(1.0)
    dense.tsdf.fill_(0.5)
    out = dense.indexed_mesh()
    assert all(out[k].shape[0] == 0 for k in KEYS)
    d, K, R, t, img = so.sphere_views(n=2)
    sp = sequence.SparseTsdfVolume(0.043)
    sp.integrate(*frames(d, K, R, t, img))
    sp._pool["tsdf"].abs_()   # keep the blocks, remove the surface
    out = sp.indexed_mesh()
    assert sp.blocks.shape[0] > 0 and all(out[k].shape[0] == 0 for k in KEYS)
    _lib.check_errors()


def test_write_ply_with_normals_reads_back(tmp_path, sphere_box):
    vol, _ = sphere_box[True]
    out = {k: host(v) for k, v in vol.indexed_mesh().items()}
    path = str(tmp_path / "m.ply")
    vis.write_ply(path, out["vertices"], out["colors"], out["faces"], out["normals"])
    raw = open(path, "rb").read()
    head, body = raw.split(b"end_header\n", 1)
    assert b"property float z\nproperty float nx\nproperty float ny\nproperty float nz\nproperty uchar red" in head
    nv, nf = out["vertices"].shape[0], out["faces"].shape[0]
    rec = np.frombuffer(body[:nv * 27], dtype=np.dtype([("p", "<f4", (3,)), ("n", "<f4", (3,)), ("c", "u1", (3,))]))
    frec = np.frombuffer(body[nv * 27:], dtype=np.dtype([("k", "u1"), ("i", "<i4", (3,))]))
    assert same(rec["p"], out["vertices"]) and same(rec["n"], out["normals"]) and same(rec["c"], out["colors"])
    assert frec.shape[0] == nf and (frec["k"] == 3).all() and np.array_equal(frec["i"], out["faces"])
    p2 = str(tmp_path / "m2.ply")
    vis.write_ply(p2, out["vertices"], out["colors"], out["faces"])
    vis.write_ply(p2 + ".n", out["vertices"], out["colors"], out["faces"], None)
    assert open(p2, "rb").read() == open(p2 + ".n", "rb").read() and b" nx" not in open(p2, "rb").read().split(b"end_header")[0]


def test_reconstruct_with_indexed_mesh(synthetic_weights):
    from demon_b200.networks_original import DemonPipeline, Session
    sess = Session(precision="3xtf32")
    sess.load_weights(synthetic_weights)
    pipe = DemonPipeline(sess, batch_size=2, iterations=1)
    rng = np.random.RandomState(3)
    base = np.kron(rng.randint(0, 256, (60, 100, 3)).astype(np.uint8), np.ones((8, 8, 1), np.uint8))
    frames = cuda(np.stack([base[:, 16 * k:16 * k + 640] for k in range(4)]))
    K = np.array([[520.0, 0, 318.0], [0, 515.0, 243.0], [0, 0, 1]])
    soup = sequence.reconstruct(pipe, frames, K, min_ratios=1)
    res = sequence.reconstruct(pipe, frames, K, min_ratios=1, indexed_mesh=True)
    want = res["volume"].indexed_mesh()
    for k in KEYS:
        assert same(host(res[k]), host(want[k])), k
    assert set(res) == set(soup) | {"normals"}
    for k in soup:
        if k in ("vertices", "colors", "faces", "volume"):
            continue
        a, b = soup[k], res[k]
        assert (torch.equal(a, b) if isinstance(a, torch.Tensor) else np.array_equal(a, b)), k
    for k in ("tsdf", "weight", "color"):
        assert torch.equal(getattr(soup["volume"], k), getattr(res["volume"], k)), k
    v, c, f = soup["volume"].mesh()
    assert torch.equal(v, soup["vertices"]) and torch.equal(c, soup["colors"]) and torch.equal(f, soup["faces"])
    _lib.check_errors()
