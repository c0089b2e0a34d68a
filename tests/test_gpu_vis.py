"""GPU: the point clouds on the device (csrc/vis.cu, demon_b200/vis.py) against the numpy restatement of the reference's
compute_point_cloud_from_depthmap and the reference's Cython or its stored digests (oracle/vis.py), in every variant
(camera z or inverse depth; uint8 colours or a float image), batched with different counts, captured in a CUDA graph,
end to end behind the network, and through the PLY export."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from demon_b200 import vis
from oracle import vis as ov

CASES = ov.edge_cases()


def same(a, b):
    """Bit equality up to NaN payloads (the digest's rule)."""
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and ov.digest(a) == ov.digest(b)


def check_against_oracles(case, got):
    ops = ov.case_operands(case)
    want = ov.point_cloud_numpy(*ops)
    assert set(got) == set(want)
    for k in want:
        assert same(got[k], want[k]), k
    if ov.available():
        ref = ov.reference_point_cloud(*ops)
        for k, v in ref.items():
            assert v.matches(got[k]) if isinstance(v, ov.Recorded) else same(got[k], v), k


def trimmed(pc, i=0):
    m = int(pc['counts'][i])
    return {k: v[i, :m].cpu().numpy() for k, v in pc.items() if k != 'counts'}


def device_case(case, inverse):
    """One case through point_clouds: with `inverse`, the inverse depth and the float image go to the device as they are;
    otherwise the host's 1/inverse depth and uint8 colours do."""
    K, R, t = (np.asarray(case[k], dtype=np.float32) for k in ('K', 'R', 't'))
    nrm = case.get('normals')
    nrm = None if nrm is None else torch.from_numpy(nrm[None]).cuda()
    if inverse:
        img = case.get('image')
        col = case.get('colors')
        return vis.point_clouds(torch.from_numpy(case['inverse_depth'][None]).cuda(), K, R, t, normals=nrm,
                                colors=None if col is None else torch.from_numpy(col[None]).cuda(),
                                image=None if img is None else torch.from_numpy(img[None]).cuda(), inverse_depth=True)
    depth, _, _, _, _, col = ov.case_operands(case)
    return vis.point_clouds(torch.from_numpy(np.ascontiguousarray(depth, dtype=np.float32)[None]).cuda(), K, R, t, normals=nrm,
                            colors=None if col is None else torch.from_numpy(col[None]).cuda())


@pytest.mark.parametrize("case", range(len(CASES)))
def test_device_equals_numpy_and_reference(case):
    c = CASES[case]
    check_against_oracles(c, trimmed(device_case(c, inverse=False)))
    if c.get('inverse_depth') is not None:
        check_against_oracles(c, trimmed(device_case(c, inverse=True)))


@pytest.mark.parametrize("case", [0, 2, 6, 7, 15, 16])
def test_one_view_api_numpy_and_tensors(case):
    depth, K, R, t, nrm, col = ov.case_operands(CASES[case])
    got = vis.compute_point_cloud_from_depthmap(depth, K, R, t, nrm, col)
    assert all(isinstance(v, np.ndarray) for v in got.values())
    check_against_oracles(CASES[case], got)
    tg = vis.compute_point_cloud_from_depthmap(torch.from_numpy(depth).cuda(), torch.from_numpy(K), R, t,
                                               None if nrm is None else torch.from_numpy(nrm).cuda(),
                                               None if col is None else torch.from_numpy(col).cuda())
    assert all(isinstance(v, torch.Tensor) and v.is_cuda for v in tg.values())
    for k in got:
        assert same(tg[k].cpu().numpy(), got[k]), k


def batch(seed, n, h, w):
    rng = np.random.RandomState(seed)
    depth = rng.uniform(0.2, 5.0, (n, h, w)).astype(np.float32)
    depth[0] = np.nan                          # count 0
    if n > 2:
        depth[2][rng.rand(h, w) < 0.3] = -1.0   # some
        depth[3][rng.rand(h, w) < 0.001] = 0.0
    K = np.stack([vis.prediction_K(rng.uniform(0.7, 1.2, 4), 1, h, w)[0] for _ in range(n)])
    R = np.stack([vis.angleaxis_to_rotation_matrix(rng.normal(0, 0.3, 3)).astype(np.float32) for _ in range(n)])
    t = rng.normal(0, 0.5, (n, 3)).astype(np.float32)
    nrm = rng.normal(0, 1, (n, 3, h, w)).astype(np.float32)
    img = rng.uniform(-0.6, 0.6, (n, 3, h, w)).astype(np.float32)
    return depth, K, R, t, nrm, img


@pytest.mark.parametrize("hw", [(48, 64), (192, 256), (480, 640)])
def test_batch_with_different_counts(hw):
    h, w = hw
    n = 5
    depth, K, R, t, nrm, img = batch(1, n, h, w)
    pc = vis.point_clouds(torch.from_numpy(depth).cuda(), torch.from_numpy(K).cuda(), torch.from_numpy(R).cuda(),
                          torch.from_numpy(t).cuda(), normals=torch.from_numpy(nrm).cuda(), image=torch.from_numpy(img).cuda())
    counts = pc['counts'].cpu().numpy()
    assert counts[0] == 0 and counts[1] == h * w and 0 < counts[2] < h * w and counts.dtype == np.int32
    for i in range(n):
        want = ov.point_cloud_numpy(depth[i], K[i], R[i], t[i], nrm[i], ov.image_to_colors(img[i]))
        got = trimmed(pc, i)
        assert counts[i] == want['points'].shape[0]
        for k in want:
            assert same(got[k], want[k]), (i, k)


def test_graph_capture_replays_with_new_inputs():
    h, w, n = 192, 256, 4
    depth, K, R, t, nrm, img = batch(2, n, h, w)
    with np.errstate(divide='ignore'):
        inv = (1 / depth).astype(np.float32)
    static = {k: torch.from_numpy(v).cuda() for k, v in dict(d=inv, K=K, R=R, t=t, n=nrm, i=img).items()}

    def call():
        return vis.point_clouds(static['d'], static['K'], static['R'], static['t'], normals=static['n'], image=static['i'],
                                inverse_depth=True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        call()   # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = call()
    for seed in (3, 4):
        d2, K2, R2, t2, n2, i2 = batch(seed, n, h, w)
        d2[1, :7] = 0.0   # infinite depth: dropped
        with np.errstate(divide='ignore'):
            new = dict(d=(1 / d2).astype(np.float32), K=K2, R=R2, t=t2, n=n2, i=i2)
        for k, v in new.items():
            static[k].copy_(torch.from_numpy(v))
        g.replay()
        torch.cuda.synchronize()
        eager = vis.point_clouds(*(torch.from_numpy(new[k]).cuda() for k in ('d', 'K', 'R', 't')),
                                 normals=torch.from_numpy(n2).cuda(), image=torch.from_numpy(i2).cuda(), inverse_depth=True)
        assert torch.equal(out['counts'], eager['counts'])
        for i in range(n):
            a, b = trimmed(out, i), trimmed(eager, i)
            for k in b:
                assert same(a[k], b[k]), (seed, i, k)
            with np.errstate(all='ignore'):
                want = ov.point_cloud_numpy(1 / new['d'][i], K2[i], R2[i], t2[i], n2[i], ov.image_to_colors(i2[i]))
            for k in want:
                assert same(a[k], want[k]), (seed, i, k)


def test_end_to_end_behind_the_network(synthetic_weights):
    from demon_b200.networks_original import DemonPipeline, Session
    sess = Session()
    sess.load_weights(synthetic_weights)
    B = 2
    pipe = DemonPipeline(sess, batch_size=B, iterations=1)
    g = torch.Generator().manual_seed(5)
    ip = (torch.rand(B, 6, 192, 256, generator=g) - 0.5).cuda()
    out = pipe.forward(ip)
    inv = out['predict_depth0']
    pc = vis.prediction_point_clouds(inv, None, ip[:, 0:3])
    intr = np.array([[0.9, 1.2, 0.48, 0.52], [0.85, 1.1, 0.5, 0.5]], dtype=np.float32)
    pc2 = vis.prediction_point_clouds(inv, torch.from_numpy(intr), ip[:, 0:3])
    inv_h, img_h = inv.cpu().numpy(), ip[:, 0:3].cpu().numpy()
    for i in range(B):
        for p, K in ((pc, vis.SUN3D_INTRINSICS), (pc2, intr[i])):
            # visualize_prediction (vis.py:246-278) on the host copies
            depth = (1 / inv_h[i]).squeeze()
            Kh = np.eye(3)
            Kh[0, 0], Kh[1, 1], Kh[0, 2], Kh[1, 2] = K[0] * 256, K[1] * 192, K[2] * 256, K[3] * 192
            ops = (depth, Kh, np.eye(3), np.zeros((3,)), None, ((img_h[i] + 0.5) * 255).astype(np.uint8))
            got = trimmed(p, i)
            want = ov.point_cloud_numpy(*ops)
            assert got['points'].shape[0] > 0
            for k in want:
                assert same(got[k], want[k]), (i, k)
            if ov.have_module():
                ref = ov.reference_point_cloud(*ops)
                for k in ref:
                    assert same(got[k], ref[k]), (i, k)


def test_ply_export_from_tensors_equals_numpy(tmp_path):
    rng = np.random.RandomState(8)
    h, w = 48, 64
    inv = rng.uniform(0.1, 2.0, (1, h, w)).astype(np.float32)
    inv[0, :3] = 0.0
    img = rng.uniform(-0.5, 0.5, (3, h, w)).astype(np.float32)
    nrm = rng.normal(0, 1, (3, h, w)).astype(np.float32)
    rot, tr = np.array([0.1, -0.2, 0.05], dtype=np.float32), np.array([0.3, 0.0, -0.1], dtype=np.float32)
    intr = np.array([0.9, 1.2, 0.5, 0.5], dtype=np.float32)
    vis.export_prediction_to_ply(str(tmp_path / "np_"), inv, intr, nrm, rot, tr, img)
    vis.export_prediction_to_ply(str(tmp_path / "t_"), torch.from_numpy(inv).cuda(), torch.from_numpy(intr).cuda(),
                                 torch.from_numpy(nrm).cuda(), torch.from_numpy(rot), torch.from_numpy(tr), torch.from_numpy(img).cuda())
    for name in ("points.ply", "cam1.ply", "cam2.ply"):
        assert (tmp_path / ("np_" + name)).read_bytes() == (tmp_path / ("t_" + name)).read_bytes(), name
    # the cloud in the file is the reference's
    data = (tmp_path / "np_points.ply").read_bytes()
    body = data[data.index(b"end_header\n") + 11:]
    with np.errstate(divide='ignore'):
        depth = (1 / inv).squeeze()
    ops = (depth, vis.prediction_K(intr, 1, h, w)[0], np.eye(3), np.zeros(3), None, ov.image_to_colors(img))
    want = ov.point_cloud_numpy(*ops)
    rec = np.frombuffer(body, dtype=np.dtype([('p', '<f4', (3,)), ('c', 'u1', (3,))]))
    assert len(rec) == want['points'].shape[0] == h * w - 3 * w
    assert same(rec['p'], want['points']) and np.array_equal(rec['c'], want['colors'])
    # without an image the cloud has no colours; without a motion cam2 is cam1
    vis.export_prediction_to_ply(str(tmp_path / "plain_"), inv)
    assert b"property uchar red" not in (tmp_path / "plain_points.ply").read_bytes()
    assert (tmp_path / "plain_cam1.ply").read_bytes() == (tmp_path / "plain_cam2.ply").read_bytes()


def test_bad_arguments_raise():
    d = torch.ones((1, 4, 5), device="cuda")
    with pytest.raises(ValueError):
        vis.point_clouds(d, np.eye(3), np.eye(3), np.zeros(3), colors=torch.zeros((1, 3, 4, 5), dtype=torch.uint8, device="cuda"),
                         image=torch.zeros((1, 3, 4, 5), device="cuda"))
    with pytest.raises(ValueError):
        vis.point_clouds(d, np.eye(3), np.eye(3), np.zeros(3), normals=torch.zeros((1, 3, 5, 4), device="cuda"))
    with pytest.raises(ValueError):   # the C ABI rejects an empty view
        vis.point_clouds(torch.ones((1, 0, 5), device="cuda"), np.eye(3), np.eye(3), np.zeros(3))
    empty = vis.point_clouds(torch.ones((0, 4, 5), device="cuda"), np.zeros((0, 3, 3)), np.zeros((0, 3, 3)), np.zeros((0, 3)))
    assert empty['points'].shape == (0, 20, 3) and empty['counts'].shape == (0,)
