"""GPU: the connected components of an indexed mesh and the removal of the small ones (demon_b200.mesh; csrc/mesh.cu) bit
for bit against tests/mesh_components_oracle.py: fused meshes (a dense two-sphere field, a sparse sphere with outlier
depths), strips whose unions build the deepest trees, a fan on one root, a million isolated triangles, a component of
more than 2^24 vertices, degenerate faces, unused vertices and empty meshes.  Every call runs twice and must give the same
bytes."""
import numpy as np
import pytest
import torch

import fusion_boundary_scenes as fb
import mesh_components_oracle as mco
from demon_b200 import _lib, mesh, sequence, vis

pytestmark = pytest.mark.gpu
f32 = np.float32
KEYS = ("vertices", "normals", "colors", "faces")


def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(x):
    return None if x is None else x.cpu().numpy()


def same(a, b):
    """Equal shape, dtype kind and bytes (None matching None)."""
    if a is None or b is None:
        return a is None and b is None
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and a.dtype.itemsize == b.dtype.itemsize and a.tobytes() == b.tobytes()


def check_components(faces, nv):
    """components() of faces on the device, twice, equal to the oracle; returns the oracle's."""
    want = mco.components(faces, nv)
    f = cuda(faces)
    for _ in range(2):
        got = mesh.components(f, nv)
        assert got["labels"].dtype == torch.int32 and got["triangles"].dtype == torch.int64
        for k in ("labels", "triangles", "vertices"):
            assert same(host(got[k]), want[k]), k
    return want


def check_filter(m, **kw):
    """remove_small_components() of the dict of numpy arrays m, twice, equal to the oracle's filter; returns it."""
    want = mco.remove_small_components(m, **kw)
    dm = {k: None if m.get(k) is None else cuda(m[k]) for k in KEYS}
    for _ in range(2):
        got = mesh.remove_small_components(dm, **kw)
        assert set(got) == set(KEYS)
        for k in KEYS:
            assert same(host(got[k]), want[k]), (k, kw)
    return want


def attributes(nv, seed=0):
    """Vertices, normals with NaNs of several payloads, and colours of nv vertices."""
    rng = np.random.RandomState(seed)
    v = rng.standard_normal((nv, 3)).astype(f32)
    n = rng.standard_normal((nv, 3)).astype(f32)
    bits = n.view(np.uint32)
    nan = rng.rand(nv, 3) < 0.05
    bits[nan] = 0x7fc00000 | rng.randint(0, 1 << 22, nan.sum()).astype(np.uint32)
    return v, n, rng.randint(0, 256, (nv, 3)).astype(np.uint8)


@pytest.fixture(scope="module")
def two_spheres_box():
    """fb.two_spheres on an odd 61x53x47 box: its indexed mesh with colour."""
    dims, origin, vs = (61, 53, 47), (0.1, -0.2, 0.3), 0.01
    s, w, c = fb.two_spheres(dims)
    vol = sequence.TsdfVolume(dims, origin, vs)
    vol.tsdf.copy_(cuda(s))
    vol.weight.copy_(cuda(w))
    vol.color.copy_(cuda(c))
    return vol


@pytest.mark.parametrize("normals", [True, False])
@pytest.mark.parametrize("color", [True, False])
def test_indexed_mesh_of_two_spheres(two_spheres_box, color, normals):
    m = {k: host(v) for k, v in two_spheres_box.indexed_mesh(normals=normals).items()}
    if not color:
        m["colors"] = None
    comps = check_components(m["faces"], m["vertices"].shape[0])
    assert comps["triangles"].size >= 2 and m["faces"].shape[0] > 1000
    big = int(np.sort(comps["triangles"])[-2])   # the second largest: min_triangles exactly at its size keeps it
    for kw in (dict(), dict(min_triangles=big), dict(min_triangles=big + 1), dict(keep_largest=1), dict(min_triangles=0, keep_largest=3)):
        check_filter(m, **kw)
    _lib.check_errors()


def test_sparse_sphere_with_outliers_has_floaters():
    """varied_sphere_views with 2 % of its 2x2 pixel cells at a random depth: an outlier that no other view sees as free
    space (most of those on the background) survives fusion as a floater."""
    d, K, R, t, img = fb.varied_sphere_views(24, 96, 128, seed=1)
    rng = np.random.RandomState(5)
    cell = np.ones((1, 2, 2))
    out = np.kron(rng.rand(24, 48, 64) < 0.02, cell).astype(bool)
    d[out] = np.kron(rng.uniform(0.3, 4.0, (24, 48, 64)), cell).astype(f32)[out]
    vol = sequence.SparseTsdfVolume(0.01, (-0.75, -0.75, -0.75))
    vol.integrate(cuda(d), cuda(K), cuda(R), cuda(t), cuda(img))
    m = {k: host(v) for k, v in vol.indexed_mesh().items()}
    comps = check_components(m["faces"], m["vertices"].shape[0])
    tri = comps["triangles"]
    assert tri.size > 10 and (tri < 50).sum() > 5 and tri.max() > 10000
    for kw in (dict(), dict(min_triangles=50), dict(min_triangles=int(tri.max())), dict(keep_largest=1), dict(keep_largest=5, min_triangles=2)):
        check_filter(m, **kw)
    clean = check_filter(m, min_triangles=200)
    assert mco.components(clean["faces"], clean["vertices"].shape[0])["triangles"].min() >= 200
    _lib.check_errors()


@pytest.mark.parametrize("order", ["random", "descending", "ascending"])
def test_strips(order):
    n = (1 << 20) + 3
    f = mco.strip(n, order)
    check_components(f, n)
    v, nrm, col = attributes(n)
    check_filter({"vertices": v, "faces": f, "normals": nrm, "colors": col}, min_triangles=n - 2)
    check_filter({"vertices": v, "faces": f, "normals": nrm, "colors": col}, min_triangles=n - 1)
    _lib.check_errors()


def test_one_component_past_2_24_vertices():
    n = (1 << 24) + 4099
    f = mco.strip(n, "random", seed=3)
    want = check_components(f, n)
    assert want["vertices"].tolist() == [n]
    v = np.random.RandomState(1).standard_normal((n, 3)).astype(f32)
    check_filter({"vertices": v, "faces": f})
    _lib.check_errors()


def test_fan_of_a_million_faces():
    n = 1000003
    f = mco.fan(n)
    want = check_components(f, n + 7)   # 5 unused vertices past the fan
    assert want["triangles"].tolist() == [n] + [0] * 5
    v, nrm, col = attributes(n + 7, seed=2)
    check_filter({"vertices": v, "faces": f, "normals": nrm, "colors": col}, min_triangles=0, keep_largest=4)
    _lib.check_errors()


def test_a_million_isolated_triangles():
    n = 1000001
    f = mco.isolated_triangles(n, seed=4)
    want = check_components(f, 3 * n)
    assert want["triangles"].size == n
    v, nrm, col = attributes(3 * n, seed=3)
    m = {"vertices": v, "faces": f, "normals": nrm, "colors": col}
    check_filter(m)
    check_filter(m, min_triangles=2)
    check_filter(m, keep_largest=1000)   # all tie: the 1000 smallest labels
    check_filter(m, keep_largest=n + 5)
    _lib.check_errors()


def test_degenerate_faces_and_unused_vertices():
    rng = np.random.RandomState(7)
    nv = 30011
    f = rng.randint(0, nv // 2, (20000, 3)).astype(np.int32) * 2   # the odd vertices are unused
    f[::7, 1] = f[::7, 0]
    f[::11, :] = f[::11, :1]
    f = f.astype(np.int64)   # int64 faces are taken too
    want = check_components(f, nv)
    assert (want["triangles"] == 0).sum() >= nv // 2 and (want["vertices"] > 1).any()
    v, nrm, col = attributes(nv, seed=5)
    m = {"vertices": v, "faces": f, "normals": nrm, "colors": col}
    for kw in (dict(), dict(min_triangles=0), dict(min_triangles=0, keep_largest=3), dict(min_triangles=2), dict(keep_largest=2)):
        check_filter(m, **kw)
    _lib.check_errors()


def test_empty_meshes():
    got = mesh.components(np.zeros((0, 3), np.int32), 0)
    assert all(got[k].shape == (0,) for k in ("labels", "triangles", "vertices"))
    check_components(np.zeros((0, 3), np.int32), 17)
    v, nrm, col = attributes(17)
    m = {"vertices": v, "faces": np.zeros((0, 3), np.int32), "normals": nrm, "colors": col}
    check_filter(m)   # nothing has a triangle: empty
    check_filter(m, min_triangles=0)
    check_filter(m, min_triangles=0, keep_largest=2)
    e = {"vertices": np.zeros((0, 3), f32), "faces": np.zeros((0, 3), np.int32)}
    out = mesh.remove_small_components(e, min_triangles=0)
    assert out["vertices"].shape == (0, 3) and out["faces"].shape == (0, 3) and out["normals"] is None and out["colors"] is None
    _lib.check_errors()


def test_out_of_range_faces_are_refused_on_the_host():
    lib = _lib.load()
    n0 = lib.demon_launch_count()
    for f in (cuda(np.array([[0, 1, 5]], np.int32)), cuda(np.array([[0, -1, 2]], np.int64)), cuda(np.array([[0, 1, 2 ** 33]], np.int64))):
        with pytest.raises(ValueError, match="index"):
            mesh.components(f, 5)
        with pytest.raises(ValueError, match="index"):
            mesh.remove_small_components({"vertices": torch.zeros((5, 3), device="cuda"), "faces": f})
    assert lib.demon_launch_count() == n0


def test_write_ply_of_the_filtered_mesh_reads_back(tmp_path, two_spheres_box):
    m = two_spheres_box.indexed_mesh()
    out = {k: host(v) for k, v in mesh.remove_small_components(m, keep_largest=1).items()}
    assert same(out["faces"], mco.remove_small_components({k: host(v) for k, v in m.items()}, keep_largest=1)["faces"])
    path = str(tmp_path / "clean.ply")
    vis.write_ply(path, out["vertices"], out["colors"], out["faces"], out["normals"])
    head, body = open(path, "rb").read().split(b"end_header\n", 1)
    nv, nf = out["vertices"].shape[0], out["faces"].shape[0]
    assert b"element vertex %d\n" % nv in head and b"element face %d\n" % nf in head
    rec = np.frombuffer(body[:nv * 27], dtype=np.dtype([("p", "<f4", (3,)), ("n", "<f4", (3,)), ("c", "u1", (3,))]))
    frec = np.frombuffer(body[nv * 27:], dtype=np.dtype([("k", "u1"), ("i", "<i4", (3,))]))
    assert same(rec["p"].copy(), out["vertices"]) and same(rec["n"].copy(), out["normals"]) and same(rec["c"].copy(), out["colors"])
    assert frec.shape[0] == nf and (frec["k"] == 3).all() and np.array_equal(frec["i"], out["faces"])


def test_reconstruct_result(tmp_path, synthetic_weights):
    from demon_b200.networks_original import DemonPipeline, Session
    sess = Session(precision="3xtf32")
    sess.load_weights(synthetic_weights)
    pipe = DemonPipeline(sess, batch_size=2, iterations=1)
    rng = np.random.RandomState(3)
    base = np.kron(rng.randint(0, 256, (60, 100, 3)).astype(np.uint8), np.ones((8, 8, 1), np.uint8))
    frames = cuda(np.stack([base[:, 16 * k:16 * k + 640] for k in range(4)]))
    K = np.array([[520.0, 0, 318.0], [0, 515.0, 243.0], [0, 0, 1]])
    res = sequence.reconstruct(pipe, frames, K, min_ratios=1, indexed_mesh=True)
    m = {k: host(res[k]) for k in KEYS}
    comps = check_components(m["faces"], m["vertices"].shape[0])
    assert m["faces"].shape[0] > 0
    k = int(np.sort(comps["triangles"])[-min(3, comps["triangles"].size)])
    clean = check_filter(m, min_triangles=k)
    got = mesh.remove_small_components(res, min_triangles=k)
    sequence.export_sequence_to_ply(str(tmp_path / "seq"), dict(res, **got))
    head = open(str(tmp_path / "seq_mesh.ply"), "rb").read().split(b"end_header")[0]
    assert b"element vertex %d\n" % clean["vertices"].shape[0] in head and b"element face %d\n" % clean["faces"].shape[0] in head
    _lib.check_errors()
