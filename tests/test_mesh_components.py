"""CPU: the mesh-components oracle (tests/mesh_components_oracle.py) against a plain union-find and meshes of known
answer, the topology of each sphere of a two-sphere field's indexed mesh, and the argument checks of demon_b200.mesh."""
import numpy as np
import pytest
import torch

import indexed_mesh_oracle as imo
import mesh_components_oracle as mco
from demon_b200 import _lib, mesh

f32 = np.float32


def test_oracle_equals_a_plain_union_find():
    rng = np.random.RandomState(0)
    for trial in range(20):
        nv = int(rng.randint(1, 200))
        nf = int(rng.randint(0, 120))
        f = rng.randint(0, nv, (nf, 3)).astype(np.int32)
        got = mco.components(f, nv)
        want = mco.union_find(f, nv)
        assert np.array_equal(got["labels"], want), trial
        assert got["labels"][0] == 0 and np.array_equal(np.unique(got["labels"]), np.arange(got["triangles"].size))
        assert got["triangles"].sum() == nf and got["vertices"].sum() == nv


def test_hand_built_meshes():
    # two tetrahedra (vertices 0..3 and 4..7, the second listed first), a fan on vertex 8, a degenerate face on 16,
    # a face (17, 17, 18), and unused vertices 19, 20
    tet = np.array([[0, 1, 2], [0, 3, 1], [1, 3, 2], [2, 3, 0]])
    fan = np.array([[8, 9, 10], [8, 10, 11], [8, 11, 12], [8, 12, 13], [8, 13, 14], [8, 14, 15]])
    f = np.concatenate([tet + 4, tet, fan, [[16, 16, 16]], [[17, 18, 17]]]).astype(np.int32)
    got = mco.components(f, 21)
    want = np.array([0] * 4 + [1] * 4 + [2] * 8 + [3, 4, 4, 5, 6], np.int32)
    assert np.array_equal(got["labels"], want)
    assert np.array_equal(got["triangles"], [4, 4, 6, 1, 1, 0, 0])
    assert np.array_equal(got["vertices"], [4, 4, 8, 1, 2, 1, 1])
    assert np.array_equal(mco.union_find(f, 21), want)

    v = np.arange(63, dtype=f32).reshape(21, 3)
    col = np.arange(63, dtype=np.uint8).reshape(21, 3)
    m = {"vertices": v, "faces": f, "normals": -v, "colors": col}
    out = mco.remove_small_components(m, min_triangles=4)   # the tetrahedra and the fan
    assert np.array_equal(out["vertices"], v[:16]) and np.array_equal(out["normals"], -v[:16]) and np.array_equal(out["colors"], col[:16])
    assert np.array_equal(out["faces"], f[:14])
    out = mco.remove_small_components(m, min_triangles=4, keep_largest=1)   # the fan
    assert np.array_equal(out["faces"], fan - 8) and np.array_equal(out["vertices"], v[8:16])
    out = mco.remove_small_components(m, min_triangles=0, keep_largest=2)   # the fan, then the first tetrahedron (a tie)
    assert np.array_equal(out["vertices"], v[:4].tolist() + v[8:16].tolist())
    assert np.array_equal(out["faces"], np.concatenate([tet, fan - 4]))
    out = mco.remove_small_components(m, min_triangles=0)   # everything, unused vertices too
    assert np.array_equal(out["vertices"], v) and np.array_equal(out["faces"], f)
    out = mco.remove_small_components(m, min_triangles=7)
    assert out["vertices"].shape == (0, 3) and out["faces"].shape == (0, 3)


def test_oracle_on_the_generated_meshes():
    for order in ("ascending", "descending", "random"):
        f = mco.strip(50, order)
        got = mco.components(f, 50)
        assert (got["labels"] == 0).all() and got["triangles"].tolist() == [48]
    got = mco.components(mco.fan(30), 35)
    assert got["triangles"].tolist() == [30, 0, 0, 0] and got["vertices"].tolist() == [32, 1, 1, 1]
    f = mco.isolated_triangles(40)
    got = mco.components(f, 120)
    assert (got["triangles"] == 1).all() and (got["vertices"] == 3).all()
    assert np.array_equal(got["labels"], mco.union_find(f, 120))
    for nv in (0, 5):
        got = mco.components(np.zeros((0, 3), np.int32), nv)
        assert np.array_equal(got["labels"], np.arange(nv)) and got["triangles"].tolist() == [0] * nv


def two_spheres(dims=(44, 30, 31)):
    """The tsdf (signed distance in voxels over 3, clamped to [-1, 1]) of two disjoint spheres in a dense box, weight 1."""
    nx, ny, nz = dims
    k, j, i = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    a = np.sqrt((i - 11.3) ** 2 + (j - 14.6) ** 2 + (k - 15.2) ** 2) - 8.17
    b = np.sqrt((i - 31.7) ** 2 + (j - 15.1) ** 2 + (k - 14.9) ** 2) - 6.93
    s = np.clip(np.minimum(a, b) / 3.0, -1.0, 1.0).astype(f32)
    return s, np.ones_like(s)


def test_each_sphere_of_a_two_sphere_field_is_closed():
    s, w = two_spheres()
    m = imo.dense(s, w, None, (0, 0, 0), 1.0, normals=False)
    f = m["faces"].astype(np.int64)
    got = mco.components(f, m["vertices"].shape[0])
    assert got["triangles"].size == 2 and (got["vertices"] > 100).all()
    x = m["vertices"][:, 0]
    for c in range(2):
        on = got["labels"] == c
        assert (x[on] < 21.5).all() if c == 0 else (x[on] > 21.5).all()   # component 0 holds vertex 0: the sphere at lower x
        fc = f[got["labels"][f[:, 0]] == c]
        e = np.sort(np.concatenate([fc[:, [0, 1]], fc[:, [1, 2]], fc[:, [2, 0]]]), axis=1)
        _, counts = np.unique(e, axis=0, return_counts=True)
        assert (counts == 2).all()
        assert on.sum() - counts.size + fc.shape[0] == 2   # V - E + F
        assert fc.shape[0] == got["triangles"][c] and on.sum() == got["vertices"][c]
    out = mco.remove_small_components({"vertices": m["vertices"], "faces": m["faces"]}, keep_largest=1)
    assert out["faces"].shape[0] == got["triangles"].max()


def test_arguments_are_checked_before_any_device(monkeypatch):
    def no_device(*a, **k):
        raise AssertionError("a device was touched")
    monkeypatch.setattr(mesh, "_device", no_device)
    monkeypatch.setattr(_lib, "load", no_device)
    f = np.array([[0, 1, 2]], np.int32)
    for faces, nv, what in ((f, 2, "index"), (-f, 3, "index"), (f, -1, "num_vertices"), (f, 2 ** 31, "num_vertices"),
                            (f, 3.0, "num_vertices"), (f, True, "num_vertices"), (f.astype(f32), 3, "int32"),
                            (f.astype(np.int16), 3, "int32"), (f.reshape(3), 3, r"\[F,3\]"), (f.reshape(1, 1, 3), 3, r"\[F,3\]"),
                            (np.zeros((2, 4), np.int32), 4, r"\[F,3\]"), (np.array([[0, 1, 2 ** 40]]), 3, "index"),
                            (torch.tensor([[0, 1, 3]]), 3, "index"), (torch.tensor([[0.0, 1, 2]]), 3, "int32"), (f, 0, "index")):
        with pytest.raises(ValueError, match=what):
            mesh.components(faces, nv)
    v = np.zeros((3, 3), f32)
    good = {"vertices": v, "faces": f}
    for m, kw, what in ((good, dict(min_triangles=-1), "min_triangles"), (good, dict(min_triangles=1.5), "min_triangles"),
                        (good, dict(min_triangles=True), "min_triangles"), (good, dict(keep_largest=0), "keep_largest"),
                        (good, dict(keep_largest=2.0), "keep_largest"), ([v, f], {}, "dict"), ({"vertices": v}, {}, "dict"),
                        ({"vertices": v[:2], "faces": f}, {}, "index"), ({"vertices": v.astype(np.float64), "faces": f}, {}, "float32"),
                        ({"vertices": v.reshape(9), "faces": f}, {}, r"\[V,3\]"),
                        (dict(good, normals=np.zeros((2, 3), f32)), {}, "normals"),
                        (dict(good, colors=np.zeros((3, 3), f32)), {}, "colors")):
        with pytest.raises(ValueError, match=what):
            mesh.remove_small_components(m, **kw)
