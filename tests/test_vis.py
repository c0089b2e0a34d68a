"""CPU: the host side of the point clouds (demon_b200/vis.py): the numpy restatement of compute_point_cloud_from_depthmap
against the reference's own Cython (oracle/vis.py; stored digests where the reference tree is absent), the argument checks,
the K and camera-mesh construction, numpy's float-to-uint8 cast the kernel emulates, and the PLY files."""
import math

import numpy as np
import pytest

from demon_b200 import vis
from demon_b200.evaluation import intrinsics_vector_to_K
from oracle import vis as ov

CASES = ov.edge_cases()


@pytest.mark.parametrize("case", range(len(CASES)))
def test_numpy_point_cloud_matches_reference_cython(case):
    if not ov.available():
        pytest.skip("neither the reference tree nor the stored digests are present")
    ops = ov.case_operands(CASES[case])
    ref = ov.reference_point_cloud(*ops)
    mine = ov.point_cloud_numpy(*ops)
    assert set(mine) == set(ref)
    for k, v in ref.items():
        if isinstance(v, ov.Recorded):
            assert v.matches(mine[k]), k
        else:
            assert v.shape == mine[k].shape and v.dtype == mine[k].dtype, k
            assert ov.digest(v) == ov.digest(mine[k]), k


def test_edge_cases_cover_what_they_claim():
    shapes = {ov.case_operands(c)[0].shape for c in CASES}
    assert {(1, 1), (7, 9), (31, 17), (48, 64), (192, 256), (768, 1024)} <= shapes
    depths = [c['depth'] for c in CASES if c.get('depth') is not None]
    flat = np.concatenate([d.ravel() for d in depths])
    fmax = np.finfo(np.float32).max
    assert np.isnan(flat).any() and np.isposinf(flat).any() and np.isneginf(flat).any() and (flat < 0).any()
    assert (np.signbit(flat) & (flat == 0)).any() and (~np.signbit(flat) & (flat == 0)).any()
    assert ((flat > 0) & (flat < np.finfo(np.float32).tiny)).any() and (flat == fmax).any()
    counts = [ov.point_cloud_numpy(*ov.case_operands(c))['points'].shape[0] for c in CASES]
    sizes = [ov.case_operands(c)[0].size for c in CASES]
    assert 0 in counts and any(n == s for n, s in zip(counts, sizes))
    # FLT_MAX depths overflow into infinite and NaN points
    big = ov.point_cloud_numpy(*ov.case_operands(CASES[5]))['points']
    assert np.isinf(big).any() and np.isnan(big).any()
    inv = np.concatenate([c['inverse_depth'].ravel() for c in CASES if c.get('inverse_depth') is not None])
    assert (inv == 0).any() and (np.signbit(inv) & (inv == 0)).any() and (inv < 0).any()
    with np.errstate(over='ignore'):
        assert np.isinf(1 / inv[(inv > 0) & (inv < np.finfo(np.float32).tiny)]).any()
    img = np.concatenate([c['image'].ravel() for c in CASES if c.get('image') is not None])
    assert (img < -0.5).any() and (img > 0.5 + 1 / 255).any() and np.isnan(img).any()
    assert any(np.isnan(c['normals']).any() for c in CASES if c.get('normals') is not None)
    assert any(not np.array_equal(c['R'], np.eye(3)) and np.any(c['t'] != 0) for c in CASES)


def cvttss2si_low_byte(x):
    """What the kernel computes for ((image+0.5)*255).astype(uint8): int32 truncation as x86 cvttss2si does it (NaN and
    values out of int32 range give 0x80000000), then the low byte."""
    x = np.asarray(x, dtype=np.float32).astype(np.float64)
    out = np.full(x.shape, -2 ** 31, dtype=np.int64)
    ok = (x > -2147483649.0) & (x < 2147483648.0)
    out[ok] = np.trunc(x[ok]).astype(np.int64)
    return (out & 0xff).astype(np.uint8)


def test_numpy_float_to_uint8_cast_is_the_truncations_low_byte():
    vals = np.array([-1, -300, 300, 256, 255.9, -0.5, 0.0, -0.0, np.nan, np.inf, -np.inf, 1e10, -1e10, 2147483520.0, -2147483648.0,
                     65791.7, -65791.7], dtype=np.float32)
    with np.errstate(all='ignore'):
        assert np.array_equal(vals.astype(np.uint8), cvttss2si_low_byte(vals))
        assert list(vals[:4].astype(np.uint8)) == [255, 212, 44, 0]
        img = np.random.RandomState(5).uniform(-600, 600, (3, 50, 50)).astype(np.float32)
        assert np.array_equal(ov.image_to_colors(img), cvttss2si_low_byte((img + np.float32(0.5)) * np.float32(255)))


def bad_calls():
    d = np.ones((4, 5), dtype=np.float32)
    K, R, t = np.eye(3), np.eye(3), np.zeros(3)
    return [
        (AssertionError, (d, K, R, t, None, np.zeros((3, 4, 5), dtype=np.float32))),
        (ValueError, (np.ones((2, 1, 4, 5), dtype=np.float32), K, R, t)),
        (ValueError, (d, K, R, t, np.zeros((3, 5, 4), dtype=np.float32))),
        (ValueError, (d, K, R, t, None, np.zeros((3, 4, 6), dtype=np.uint8))),
        (ZeroDivisionError, (d, np.diag([0.0, 3.0, 1.0]), R, t)),
        (ZeroDivisionError, (d, np.diag([3.0, 0.0, 1.0]), R, t)),
    ]


@pytest.mark.parametrize("i", range(len(bad_calls())))
def test_argument_checks_match_the_reference(i):
    exc, args = bad_calls()[i]
    with pytest.raises(exc) as mine:
        vis.compute_point_cloud_from_depthmap(*args)
    if ov.have_module():
        with pytest.raises(exc) as ref:
            ov.module().compute_point_cloud_from_depthmap(*args)
        assert str(mine.value) == str(ref.value)


def test_messages_name_the_shapes():
    with pytest.raises(ValueError, match=r"shape mismatch: colors \(3, 4, 6\), depth \(4, 5\)"):
        vis.compute_point_cloud_from_depthmap(np.ones((4, 5), np.float32), np.eye(3), np.eye(3), np.zeros(3), None,
                                              np.zeros((3, 4, 6), np.uint8))
    with pytest.raises(ValueError, match="wrong number of dimensions for depth"):
        vis.compute_point_cloud_from_depthmap(np.ones((2, 3, 4), np.float32), np.eye(3), np.eye(3), np.zeros(3))


def vis_py_K(intrinsics, w, h):
    """vis.py:251-258 as written there: float64 eye, the products of intrinsics[i] and the Python ints w, h stored."""
    if intrinsics is None:
        intrinsics = np.array([0.89115971, 1.18821287, 0.5, 0.5])
    K = np.eye(3)
    K[0, 0] = intrinsics[0] * w
    K[1, 1] = intrinsics[1] * h
    K[0, 2] = intrinsics[2] * w
    K[1, 2] = intrinsics[3] * h
    return K


def test_prediction_K_equals_vis_py_construction():
    rng = np.random.RandomState(9)
    for h, w in ((48, 64), (192, 256), (480, 640), (768, 1024), (7, 9)):
        assert np.array_equal(vis.prediction_K(None, 1, h, w)[0], vis_py_K(None, w, h).astype(np.float32))
        for dt in (np.float32, np.float64):
            intr = rng.uniform(0.3, 1.5, (3, 4)).astype(dt)
            got = vis.prediction_K(intr, 3, h, w)
            for i in range(3):
                assert np.array_equal(got[i], vis_py_K(intr[i], w, h).astype(np.float32)), (h, w, dt)
                assert np.array_equal(intrinsics_vector_to_K(intr[i], w, h).astype(np.float32), vis_py_K(intr[i], w, h).astype(np.float32))
            assert np.array_equal(vis.prediction_K(intr[1], 2, h, w)[1], got[1])


def rodrigues(aa):
    aa = np.asarray(aa, dtype=np.float64)
    th = np.linalg.norm(aa)
    k = aa / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + math.sin(th) * Kx + (1 - math.cos(th)) * Kx.dot(Kx)


def test_rodrigues_and_camera_mesh():
    rng = np.random.RandomState(4)
    for _ in range(20):
        aa = rng.normal(0, 0.8, 3)
        R = vis.angleaxis_to_rotation_matrix(aa)
        assert R.dtype == np.float64
        np.testing.assert_allclose(R, rodrigues(aa), rtol=0, atol=1e-14)
        R32 = vis.angleaxis_to_rotation_matrix(aa.astype(np.float32))
        assert R32.dtype == np.float64
        np.testing.assert_allclose(R32, rodrigues(aa.astype(np.float32)), rtol=0, atol=1e-6)
    assert np.array_equal(vis.angleaxis_to_rotation_matrix(np.array([3e-7, 0, 4e-7])), np.eye(3))
    assert not np.array_equal(vis.angleaxis_to_rotation_matrix(np.array([3e-6, 0, 4e-6])), np.eye(3))
    cam = np.array([[0, 0, 0], [-1, -1, 1.5], [1, -1, 1.5], [1, 1, 1.5], [-1, 1, 1.5], [-0.5, 1, 1.5], [0.5, 1, 1.5], [0, 1.2, 1.5],
                    [1, -0.5, 1.5], [1, 0.5, 1.5], [1.2, 0, 1.5]])
    R, t = rodrigues(np.array([0.1, -0.4, 0.2])), np.array([0.3, -1.0, 2.0])
    v, f = vis.camera_mesh(R, t)
    assert np.array_equal(v, (0.25 * cam - t).dot(R))
    assert f.dtype == np.int32 and f.tolist() == [[0, 1, 4], [0, 3, 2], [0, 4, 3], [0, 2, 1], [8, 10, 9], [5, 6, 7]]


def read_ply(path):
    """A minimal binary little-endian PLY reader: header lines, then {element: structured array}."""
    data = open(path, "rb").read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    header = data[:end].decode("ascii").split("\n")[:-1]
    assert header[0] == "ply" and header[1] == "format binary_little_endian 1.0" and header[-1] == "end_header"
    types = {"float": "<f4", "uchar": "u1", "int": "<i4"}
    elements = []
    for line in header[2:-1]:
        words = line.split()
        if words[0] == "element":
            elements.append((words[1], int(words[2]), []))
        elif words[0] == "property" and words[1] == "list":
            assert (words[2], words[3]) == ("uchar", "int")
            elements[-1][2].append(("n", "u1"))
            elements[-1][2].append((words[4], "<i4", (3,)))
        else:
            assert words[0] == "property"
            elements[-1][2].append((words[2], types[words[1]]))
    out, pos = {}, end
    for name, count, fields in elements:
        dt = np.dtype(fields)
        out[name] = np.frombuffer(data, dtype=dt, count=count, offset=pos)
        pos += dt.itemsize * count
    assert pos == len(data)
    return header, out


def test_ply_round_trip(tmp_path):
    rng = np.random.RandomState(2)
    pts = rng.normal(0, 3, (1000, 3)).astype(np.float32)
    pts[5] = [np.nan, np.inf, -0.0]
    col = rng.randint(0, 256, (1000, 3)).astype(np.uint8)
    vis.write_ply(str(tmp_path / "c.ply"), pts, col)
    header, el = read_ply(str(tmp_path / "c.ply"))
    assert header == ["ply", "format binary_little_endian 1.0", "element vertex 1000", "property float x", "property float y",
                      "property float z", "property uchar red", "property uchar green", "property uchar blue", "end_header"]
    v = el["vertex"]
    assert v.dtype.itemsize == 15
    got = np.stack([v["x"], v["y"], v["z"]], axis=1)
    assert got.tobytes() == pts.tobytes()
    assert np.array_equal(np.stack([v["red"], v["green"], v["blue"]], axis=1), col)
    # an empty cloud is a valid file too
    vis.write_ply(str(tmp_path / "e.ply"), np.zeros((0, 3), np.float32), np.zeros((0, 3), np.uint8))
    header, el = read_ply(str(tmp_path / "e.ply"))
    assert header[2] == "element vertex 0" and len(el["vertex"]) == 0
    # the camera mesh: float vertices and six triangles
    verts, faces = vis.camera_mesh(vis.angleaxis_to_rotation_matrix(np.array([0.2, 0.1, -0.3])), np.array([1.0, 0.5, -0.25]))
    vis.write_ply(str(tmp_path / "cam.ply"), verts, faces=faces)
    header, el = read_ply(str(tmp_path / "cam.ply"))
    assert header[2:] == ["element vertex 11", "property float x", "property float y", "property float z", "element face 6",
                          "property list uchar int vertex_indices", "end_header"]
    v = el["vertex"]
    assert np.array_equal(np.stack([v["x"], v["y"], v["z"]], axis=1), verts.astype(np.float32))
    assert (el["face"]["n"] == 3).all() and np.array_equal(el["face"]["vertex_indices"], faces)
    assert (tmp_path / "cam.ply").stat().st_size == len("\n".join(header)) + 1 + 11 * 12 + 6 * 13
