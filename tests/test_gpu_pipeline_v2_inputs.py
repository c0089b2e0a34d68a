"""GPU: the v2 pipeline's input paths (DemonPipelineV2: uint8, resized photos, calibrated views, host buffers, snapshots),
image2_2='area' (tf.image.resize_area, images.resize_area) against the numpy oracle, the handle-kind and mode refusals of
the pipeline's C entries, and Evaluator on a v2 Session.  Synthetic v2 weights at 3xTF32; every comparison is bit for bit except
the evaluation table's non-depth columns (1e-12, as for v1)."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from demon_b200 import _lib, images
from demon_b200 import evaluation as ev
from demon_b200.v2 import weights as W2
from oracle import resize_area as ra
from test_gpu_evaluation import compare_tables, oracle_table, synthetic_gt

B, ITER = 2, 2
FILTERS = ("nearest", "bilinear", "bicubic")
MODES = ("resize", "median", "area")
KEYS = ("predict_depth0", "predict_normal0", "predict_rotation", "predict_translation", "predict_flow2", "predict_depth2",
        "predict_normal2")


@pytest.fixture(scope="module")
def weights():
    return W2.synthetic_weights(0)


@pytest.fixture(scope="module")
def session(weights):
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    from demon_b200.v2.networks import Session
    s = Session(precision="3xtf32")
    s.load_weights(weights)
    return s


def pipeline(session, batch=B, iterations=ITER):
    from demon_b200.v2.networks import DemonPipelineV2
    return DemonPipelineV2(session, batch_size=batch, iterations=iterations)


def rand_images(seed, *shape):
    return torch.from_numpy(np.random.default_rng(seed).integers(0, 256, shape + (3,), dtype=np.uint8)).cuda()


def cameras(b, seed):
    rng = np.random.default_rng(seed)
    f = rng.uniform(380, 700, (b, 2))
    return np.stack([f, f * rng.uniform(0.95, 1.05, (b, 2)), rng.uniform(250, 390, (b, 2)), rng.uniform(180, 300, (b, 2))], -1)


def planes(u8):
    """uint8 [..., h, w, 3] -> x/255 - 0.5 as float32 NCHW, numpy's two operations"""
    return images.to_float(u8).movedim(-1, -3).contiguous()


def fresh(pipe):
    return {k: torch.empty_like(v) for k, v in pipe.own_outputs().items()}


def cloned(out):
    return {k: v.clone() for k, v in out.items()}


def assert_same(got, ref, *what):
    torch.cuda.synchronize()
    assert set(got) >= set(ref) and ref
    for k in ref:
        assert torch.equal(got[k], ref[k]), (k,) + what


def test_forward_u8_equals_forward_on_floats(session):
    pipe = pipeline(session)
    u8 = rand_images(1, B, 2, 192, 256)
    u22 = rand_images(2, B, 48, 64)
    ip = torch.cat([planes(u8[:, 0]), planes(u8[:, 1])], 1)
    for i22_u8, i22 in ((u22, planes(u22)), (None, None), ("area", "area")):
        ref = cloned(pipe.forward(ip, i22, outputs=fresh(pipe)))
        for call in range(3):   # eager, capture, replay
            assert_same(pipe.forward_u8(u8, i22_u8), ref, i22_u8 if isinstance(i22_u8, str) else type(i22_u8), call)
    # 'area' is resize_area of the second image's float planes: the same as passing it in
    ref = cloned(pipe.forward(ip, images.resize_area(ip[:, 3:6], (48, 64)), outputs=fresh(pipe)))
    assert_same(pipe.forward(ip, "area"), ref)
    assert_same(pipe.forward(ip, "area", stage_inputs=False), ref)


@pytest.mark.parametrize("batch, h, w, crop", [(1, 480, 640, False), (4, 480, 640, True), (4, 192, 256, False)])
def test_forward_images_equals_forward_u8_on_resized_bytes(session, batch, h, w, crop):
    pipe = pipeline(session, batch)
    src = rand_images(20 + batch, batch, 2, h + 40, w + 24) if crop else rand_images(20 + batch, batch, 2, h, w)
    x = src[:, :, 17:17 + h, 5:5 + w] if crop else src
    for resample in FILTERS:
        resized = torch.stack([images.resize(x[:, i], (256, 192), resample) for i in range(2)], 1).contiguous()
        for mode in MODES:
            i22 = {"resize": images.resize(resized[:, 1], (64, 48), resample), "median": None, "area": "area"}[mode]
            ref = cloned(pipe.forward_u8(resized, i22, outputs=fresh(pipe)))
            for call in range(2):   # eager, capture + replay
                assert_same(pipe.forward_images(x, resample=resample, image2_2=mode), ref, resample, mode, call)
    _lib.check_errors()


def test_forward_views_equals_forward_u8_on_adapted_bytes(session):
    pipe = pipeline(session)
    h, w = 480, 640
    x = rand_images(31, B, 2, h + 40, w + 24)[:, :, 17:17 + h, 5:5 + w]
    K = torch.from_numpy(cameras(B, 1)).cuda()
    for resample in ("bicubic", "nearest"):
        for mode in MODES:
            for call in range(3):
                if call == 2:
                    K.copy_(torch.from_numpy(cameras(B, 7)))   # same tensor, new values: the replay must see them
                adapted, _, status = images.adjust_intrinsics(x.reshape(B * 2, h, w, 3), K.reshape(-1, 4))
                adapted = adapted.reshape(B, 2, 192, 256, 3).contiguous()
                i22 = {"resize": images.resize(adapted[:, 1], (64, 48), resample), "median": None, "area": "area"}[mode]
                ref = cloned(pipe.forward_u8(adapted, i22, outputs=fresh(pipe)))
                got = pipe.forward_views(x, K, resample=resample, image2_2=mode)
                assert_same(got, ref, resample, mode, call)
                assert torch.equal(got["status"].reshape(-1), status), (resample, mode, call)
    _lib.check_errors()


GUARD = 4096
SENTINEL = -12345.5


def guarded(shape):
    """A pinned host tensor of `shape` inside a sentinel-filled buffer; returns (view, the whole buffer)."""
    n = int(np.prod(shape))
    whole = torch.full((n + 2 * GUARD,), SENTINEL, dtype=torch.float32).pin_memory()
    return whole[GUARD:GUARD + n].view(shape), whole


def test_host_entries_equal_device_entries(session):
    pipe = pipeline(session)
    rng = np.random.default_rng(5)
    u8 = rng.integers(0, 256, (B, 2, 192, 256, 3), dtype=np.uint8)
    u22 = rng.integers(0, 256, (B, 48, 64, 3), dtype=np.uint8)
    ip = torch.cat([planes(torch.from_numpy(u8[:, 0]).cuda()), planes(torch.from_numpy(u8[:, 1]).cuda())], 1)
    i22f = planes(torch.from_numpy(u22).cuda())
    h_ip, h_i22 = ip.cpu().pin_memory(), i22f.cpu().pin_memory()
    h_u8, h_u22 = torch.from_numpy(u8).pin_memory(), torch.from_numpy(u22).pin_memory()
    stream = torch.cuda.Stream()
    for src in ("given", "median", "area"):
        ref = cloned(pipe.forward(ip, {"given": i22f, "median": None, "area": "area"}[src], outputs=fresh(pipe)))
        torch.cuda.synchronize()
        for entry in ("host", "host_async", "host_u8", "host_u8_async"):
            for with_normal0 in (True, False):
                u = entry.startswith("host_u8")
                i22 = {"given": h_u22 if u else h_i22, "median": None, "area": "area"}[src]
                outs = {k: guarded(s) for k, s in (("predict_depth0", (B, 1, 192, 256)), ("predict_normal0", (B, 3, 192, 256)),
                                                    ("predict_rotation", (B, 3)), ("predict_translation", (B, 3)))}
                if not with_normal0:
                    outs.pop("predict_normal0")
                o = {k: v[0] for k, v in outs.items()}
                args = (i22, o["predict_depth0"], o["predict_rotation"], o["predict_translation"])
                if entry == "host":
                    pipe.forward_host(h_ip, *args, normal0=o.get("predict_normal0"))
                elif entry == "host_async":
                    pipe.forward_host_async(h_ip, *args, stream=stream, normal0=o.get("predict_normal0"))
                else:
                    pipe.forward_host_u8(h_u8, *args, stream=stream, sync=entry == "host_u8", normal0=o.get("predict_normal0"))
                stream.synchronize()
                torch.cuda.synchronize()
                for k, (view, whole) in outs.items():
                    assert torch.equal(view, ref[k].cpu()), (src, entry, k)
                    assert (whole[:GUARD] == SENTINEL).all() and (whole[-GUARD:] == SENTINEL).all(), (src, entry, k)
    _lib.check_errors()


def stagewise(session, ip, i22, iterations=ITER):
    """examples/evaluation.py:225-255 with v2's per-stage entries: snapshots k = 0..iterations, refined depth and normals
    of each."""
    from demon_b200.v2.networks import BootstrapNet, IterativeNet, RefinementNet
    n = ip.shape[0]
    boot, it, ref = BootstrapNet(session, batch_size=n), IterativeNet(session, batch_size=n), RefinementNet(session, batch_size=n)
    snaps = []
    r = boot.eval(ip, i22)
    for k in range(iterations + 1):
        if k:
            r = it.eval(ip, i22, r["predict_depth2"], r["predict_normal2"], r["predict_rotation"], r["predict_translation"])
        r = cloned(r)
        r.update(cloned(ref.eval(ip[:, 0:3].contiguous(), r["predict_depth2"], r["predict_normal2"])))
        snaps.append(r)
    torch.cuda.synchronize()
    return snaps


def random_pair(seed, n=B):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(n, 6, 192, 256, generator=g) - 0.5).cuda()


def median_i22(ip):
    from demon_b200 import lmbspecialops as sops
    return sops.median3x3_downsample(sops.median3x3_downsample(ip[:, 3:6].contiguous()))


def test_pipeline_snapshots_equal_stagewise_forward_and_area_mode(session):
    pipe = pipeline(session)
    ip = random_pair(11)
    plain = cloned(pipe.forward(ip, None))
    pipe.forward(ip, None)
    torch.cuda.synchronize()
    plain_launches = pipe.launches()
    want = stagewise(session, ip, median_i22(ip))
    for call in range(3):   # eager, capture, replay
        out = cloned(pipe.forward_snapshots(ip, None))
        torch.cuda.synchronize()
        assert set(out) == set(KEYS) and out["predict_normal0"].shape == (ITER + 1, B, 3, 192, 256)
        for k in range(ITER + 1):
            for key in KEYS:
                assert torch.equal(out[key][k], want[k][key]), (call, k, key)
    for key in KEYS:   # the last snapshot is the plain pipeline's output
        assert torch.equal(out[key][ITER], plain[key]), key
    ip2 = random_pair(12)   # new content through the same staging buffers: a replay
    out = pipe.forward_snapshots(ip2, None)
    torch.cuda.synchronize()
    want2 = stagewise(session, ip2, median_i22(ip2))
    for k in range(ITER + 1):
        for key in KEYS:
            assert torch.equal(out[key][k], want2[k][key]), (k, key)
    out = pipe.forward_snapshots(ip2, None, refine=False)
    torch.cuda.synchronize()
    assert "predict_depth0" not in out and "predict_normal0" not in out
    for key in KEYS[2:]:
        assert torch.equal(out[key], torch.stack([want2[k][key] for k in range(ITER + 1)])), key
    # 'area' staged by resize_area equals the C entry's own image2_2_mode 2
    a = cloned(pipe.forward_snapshots(ip2, "area"))
    want3 = stagewise(session, ip2, images.resize_area(ip2[:, 3:6], (48, 64)))
    for k in range(ITER + 1):
        for key in KEYS:
            assert torch.equal(a[key][k], want3[k][key]), ("area", k, key)
    own = pipe.own_snapshot_outputs(True)
    c = {key: torch.empty_like(v) for key, v in own.items()}
    args = _lib.PipelineArgs(input=_lib.INPUT_F32, images=pipe._ip.data_ptr(), image2_2_mode=2, iterations=ITER, snapshots=1,
                             **{key[len("predict_"):]: c[key].data_ptr() for key in KEYS})
    _lib.check(_lib.load().demon_pipeline_run(pipe.net.ptr, args, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    assert_same(c, a)
    assert pipe.launches() == plain_launches and pipe.snapshot_launches() > 0


def test_interleaved_call_kinds_equal_their_eager_results(session):
    pipe = pipeline(session)
    rng = np.random.default_rng(3)
    x = {"image_pair": torch.from_numpy(rng.uniform(-0.5, 0.5, (B, 6, 192, 256)).astype(np.float32)).cuda(),
         "u8": rand_images(4, B, 2, 192, 256), "photos": rand_images(5, B, 2, 480, 640), "K": torch.from_numpy(cameras(B, 6)).cuda()}
    kinds = {
        "forward": lambda o: pipe.forward(x["image_pair"], None, outputs=o),
        "forward_area": lambda o: pipe.forward(x["image_pair"], "area", outputs=o),
        "u8": lambda o: pipe.forward_u8(x["u8"], None, outputs=o),
        "u8_area": lambda o: pipe.forward_u8(x["u8"], "area", outputs=o),
        "images_resize": lambda o: pipe.forward_images(x["photos"], image2_2="resize", outputs=o),
        "images_median": lambda o: pipe.forward_images(x["photos"], image2_2="median", outputs=o),
        "images_area": lambda o: pipe.forward_images(x["photos"], image2_2="area", outputs=o),
        "views": lambda o: pipe.forward_views(x["photos"], x["K"], outputs=o),
        "snapshots": lambda o: pipe.forward_snapshots(x["image_pair"], None, refine=False, outputs=o),
        "snapshots_refined": lambda o: pipe.forward_snapshots(x["image_pair"], None, refine=True, outputs=o),
    }
    snap = ("snapshots", "snapshots_refined")

    def own(kind):
        return pipe.own_snapshot_outputs(kind == "snapshots_refined") if kind in snap else pipe.own_outputs()

    refs, counts, keep = {}, {}, []
    for kind, call in kinds.items():
        keep.append({k: torch.empty_like(v) for k, v in own(kind).items()})
        refs[kind] = cloned(call(keep[-1]))
        counts[kind] = pipe.snapshot_launches() if kind in snap else pipe.launches()
    order = ("views", "snapshots_refined", "u8_area", "forward", "images_area", "snapshots", "images_median", "u8", "forward_area",
             "images_resize")
    for rnd in range(3):   # the pipeline's own outputs: eager, capture, replay
        for kind in order:
            got = cloned(kinds[kind](None))
            assert (pipe.snapshot_launches() if kind in snap else pipe.launches()) == counts[kind], (kind, rnd)
            assert set(got) == set(refs[kind]), (kind, rnd)
            assert_same(got, refs[kind], kind, rnd)
    _lib.check_errors()


def test_pipeline_args_refusals_launch_nothing(session, synthetic_weights):
    from demon_b200.networks_original import DemonPipeline, Session as SessionV1
    lib = _lib.load()
    v2 = session.net(1)
    s1 = SessionV1("3xtf32")
    s1.load_weights(synthetic_weights)
    v1 = s1.net(1)
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    f = torch.zeros(1, 6, 192, 256, device="cuda")
    u8 = torch.zeros(1, 2, 192, 256, 3, dtype=torch.uint8, device="cuda")
    u22 = torch.zeros(1, 48, 64, 3, dtype=torch.uint8, device="cuda")
    K = torch.full((1, 2, 4), 300.0, dtype=torch.float64, device="cuda")
    st = torch.zeros(1, 2, dtype=torch.uint8, device="cuda")
    o = dict(zip(("depth0", "normal0", "rotation", "translation", "flow2", "depth2", "normal2"),
                 (torch.zeros(4, 3, 192, 256, device="cuda").data_ptr() for _ in range(7))))
    h_f, h_u8 = np.zeros((1, 6, 192, 256), np.float32), np.zeros((1, 2, 192, 256, 3), np.uint8)
    h_o = {k: np.zeros((1, 3, 192, 256), np.float32).ctypes.data for k in ("depth0", "normal0", "rotation", "translation")}
    sizes = dict(zip(("sn", "si", "sy"), u8.stride()[:3]), h=192, w=256, resample=3)
    run = lambda n, a: lib.demon_pipeline_run(n, a, s)
    run_host = lambda sync: lambda n, a: lib.demon_pipeline_run_host(n, a, sync, s)
    calls = {   # call kind -> (entry, the fields of its PipelineArgs)
        "snapshots": (run, dict(input=_lib.INPUT_F32, images=f.data_ptr(), snapshots=1, **o)),
        "u8": (run, dict(input=_lib.INPUT_U8, images=u8.data_ptr(), **o)),
        "images": (run, dict(input=_lib.INPUT_RESIZE_U8, images=u8.data_ptr(), **sizes, **o)),
        "views": (run, dict(input=_lib.INPUT_VIEWS_U8, images=u8.data_ptr(), K=K.data_ptr(), status=st.data_ptr(), **sizes, **o)),
        "host": (run_host(1), dict(input=_lib.INPUT_F32, images=h_f.ctypes.data, **h_o)),
        "host_async": (run_host(0), dict(input=_lib.INPUT_F32, images=h_f.ctypes.data, **h_o)),
        "host_u8": (run_host(1), dict(input=_lib.INPUT_U8, images=h_u8.ctypes.data, **h_o)),
        "host_u8_async": (run_host(0), dict(input=_lib.INPUT_U8, images=h_u8.ctypes.data, **h_o)),
    }

    def call(name, net, mode, i22=None, **change):
        entry, fields = calls[name]
        return entry(net, _lib.PipelineArgs(image2_2=i22, image2_2_mode=mode, iterations=1, **dict(fields, **change)))

    n0 = lib.demon_launch_count()
    for name in calls:
        assert call(name, v1.ptr, 0) == -1, name                     # normal0 on a v1 handle
        assert "normal0" in lib.demon_last_error().decode(), name
        assert call(name, v1.ptr, 2, normal0=None) == -1, name       # area on a v1 handle
        assert "image2_2_mode" in lib.demon_last_error().decode(), name
        assert call(name, v2.ptr, 7) == -1, name                     # no such mode
        if name not in ("images", "views"):
            assert call(name, v2.ptr, 1) == -1, name                 # resize: images / views only
            assert call(name, v2.ptr, 2, u22.data_ptr()) == -1, name  # area and a given image2_2
    # snapshots: normal0 needs depth0
    assert call("snapshots", v2.ptr, 0, depth0=None) == -1
    # a field the input kind does not read, and what the host entry does not take
    assert call("u8", v2.ptr, 0, K=K.data_ptr()) == -1
    assert call("snapshots", v2.ptr, 0, sn=1) == -1
    assert call("images", v2.ptr, 0, u22.data_ptr()) == -1
    assert call("u8", v2.ptr, 0, snapshots=2) == -1
    for change in (dict(snapshots=1), dict(flow2=o["flow2"]), dict(depth0=None), dict(input=_lib.INPUT_RESIZE_U8, **sizes)):
        assert call("host_u8", v2.ptr, 0, **change) == -1, change
    assert lib.demon_launch_count() == n0                            # nothing was launched
    pipe1 = DemonPipeline(s1, batch_size=1, iterations=1)
    for call in (lambda: pipe1.forward(f, "area"), lambda: pipe1.forward_snapshots(f, "area"), lambda: pipe1.forward_u8(u8, "area"),
                 lambda: pipe1.forward_images(u8, image2_2="area"), lambda: pipe1.forward_views(u8, K, image2_2="area"),
                 lambda: pipe1.forward_host(h_f, "area", *[np.zeros((1, 1, 192, 256), np.float32), None, None]),
                 lambda: ev.Evaluator(s1, 1, 1).add(f, np.zeros((1, 48, 64), np.float32), np.zeros((1, 6), np.float32), image2_2="area")):
        with pytest.raises(ValueError):
            call()
    with pytest.raises(ValueError):
        pipeline(session, 1, 1).forward_images(u8, image2_2="lanczos")


@pytest.mark.parametrize("depthmask,crop,area", ((True, False, False), (False, True, False), (False, False, True)))
def test_evaluator_v2_table_equals_oracle_table(session, depthmask, crop, area):
    ip = random_pair(31)
    i22 = images.resize_area(ip[:, 3:6], (48, 64)) if area else median_i22(ip)
    inv, motion, intr = synthetic_gt(4, B, 480, 640)
    motion[1, 3] = np.nan if crop else motion[1, 3]
    evaluator = ev.Evaluator(session, B, ITER, depthmask=depthmask, eigen_crop_gt_and_pred=crop)
    assert evaluator.v2
    got = evaluator.add(ip, inv, motion, intr, image2_2="area" if area else None)
    labels, want = oracle_table(stagewise(session, ip, i22), inv, motion, intr, depthmask, crop)
    compare_tables(got, labels, want)
    part = evaluator.add(ip[:1], inv[:1], motion[:1], intr[:1], image2_2="area" if area else i22[:1])   # padded last batch
    compare_tables(part, labels, want[:, :, :1])
    assert evaluator.result().coords['sample'] == ['0', '1', '2']


def area_cases():
    rng = np.random.RandomState(8)
    special = rng.uniform(-0.5, 0.5, (2, 3, 192, 256)).astype(np.float32)
    flat = special.reshape(-1)
    for v, frac in ((np.nan, 0.002), (np.inf, 0.002), (-np.inf, 0.002), (-0.0, 0.05)):
        flat[rng.rand(flat.size) < frac] = v
    return [(rng.uniform(-0.5, 0.5, (32, 3, 192, 256)).astype(np.float32), (48, 64)),
            (rng.uniform(-0.5, 0.5, (1, 3, 192, 256)).astype(np.float32), (48, 64)),
            (rng.uniform(-1, 1, (3, 2, 96, 130)).astype(np.float32), (48, 65)),      # factor 2
            (rng.uniform(-1, 1, (2, 3, 144, 192)).astype(np.float32), (48, 64)),     # factor 3
            (rng.uniform(-1, 1, (4, 1, 5, 256)).astype(np.float32), (5, 1)),         # 1 x w
            (special, (48, 64))]


def same_bits(got, want):
    """bit for bit, except that a NaN's payload is free (numpy on the host keeps an operand's, the device makes its own)"""
    nan = np.isnan(want)
    return np.array_equal(np.isnan(got), nan) and np.array_equal(got[~nan].view(np.uint32), want[~nan].view(np.uint32))


@pytest.mark.parametrize("case", range(6))
def test_resize_area_equals_oracle(case):
    x, size = area_cases()[case]
    want = ra.resize_area(x, size)
    got = images.resize_area(x, size)                              # numpy in, numpy out
    assert isinstance(got, np.ndarray) and got.dtype == np.float32
    assert same_bits(got, want)
    t = images.resize_area(torch.from_numpy(x).cuda(), size)       # torch in, torch out
    assert t.is_cuda and same_bits(t.cpu().numpy(), want)
    single = images.resize_area(torch.from_numpy(x[0]).cuda(), size)
    assert single.shape == want.shape[1:] and same_bits(single.cpu().numpy(), want[0])


def test_resize_area_reads_channel_slices_in_place_and_refuses_other_sizes():
    ip = random_pair(5, 4)
    n0 = _lib.load().demon_launch_count()
    got = images.resize_area(ip[:, 3:6], (48, 64))
    assert _lib.load().demon_launch_count() - n0 == 1               # no copy of the strided slice
    want = ra.resize_area(ip[:, 3:6].cpu().numpy(), (48, 64))
    assert np.array_equal(got.cpu().numpy().view(np.uint32), want.view(np.uint32))
    for size in ((47, 64), (48, 60), (96, 100)):
        with pytest.raises(ValueError):
            images.resize_area(ip, size)
    lib = _lib.load()
    out = torch.empty(4, 3, 48, 64, device="cuda")
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    assert lib.demon_resize_area_f32(ip.data_ptr(), 6 * 192 * 256, out.data_ptr(), 4, 3, 192, 256, 47, 64, s) == -1
    assert lib.demon_resize_area_f32(ip.data_ptr(), 100, out.data_ptr(), 4, 3, 192, 256, 48, 64, s) == -1
