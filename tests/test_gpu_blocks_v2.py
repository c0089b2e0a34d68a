"""GPU: the block entries of demon_b200.v2.blocks on a training batch of datareader.build_batch, whose rot180 and mirror_x
give every sample its own camera: each block against the float64 oracle on the batch's INTRINSICS, one sample's camera
moving only that sample's outputs, the networks' constant camera reproducing BootstrapNet / IterativeNet bit for bit, and
the refusal of arguments the scope's weights cannot take."""
import numpy as np
import pytest
import torch

from demon_b200 import datareader as dr, images
from demon_b200.dataset_tools import View
from demon_b200.v2 import blocks
from demon_b200.v2 import weights as W2
from oracle import datareader as od
from oracle.network import Weights
from oracle.network_v2 import depthmotion_block, flow_block, refine_block

from objective_oracle import CameraOps

pytestmark = pytest.mark.gpu

BARS = {"fp32": 1e-4, "3xtf32": 1e-4, "tf32": 3e-2}   # test_gpu_network_v2.py's
K_NET = np.array([0.89115971, 1.18821287, 0.5, 0.5], np.float32)
COMBOS = ((False, False), (True, False), (False, True), (True, True))


def training_batch(b, seed):
    """training.py's reader at batch b: ANGLEAXIS6, inverse depth, normalised translation, every rot180 / mirror_x pair."""
    pool = dr.ViewPool(256, 192)
    pool.add([View(*v) for v in od.synthetic_views(6, 480, 640, seed)])
    rng = np.random.default_rng(seed)
    pairs = [tuple(int(i) for i in rng.choice(6, 2, replace=False)) for _ in range(b)]
    params = {'batch_size': b, 'motion_format': 'ANGLEAXIS6', 'inverse_depth': True, 'norm_trans_scale_depth': True,
              'scaled_width': 256, 'scaled_height': 192, 'top_output': ('IMAGE_PAIR', 'MOTION', 'DEPTH', 'INTRINSICS')}
    aug = dr.Augmentation(np.array([COMBOS[i % 4][0] for i in range(b)]), np.array([COMBOS[i % 4][1] for i in range(b)]))
    return dr.build_batch(pool, pairs, params, aug)


@pytest.fixture(scope="module")
def weights():
    return W2.synthetic_weights(0)


@pytest.fixture(scope="module")
def sessions(weights):
    from demon_b200.v2.networks import Session
    out = {}
    for prec in BARS:
        out[prec] = Session(precision=prec)
        out[prec].load_weights(weights)
    return out


@pytest.fixture(scope="module")
def batch():
    b = training_batch(4, 5)
    K = b['INTRINSICS'].cpu().numpy()
    assert len({tuple(r) for r in K}) == 4, K   # each sample has its own camera
    ip = b['IMAGE_PAIR']
    return {"ip": ip, "i22": images.resize_area(ip[:, 3:6], (48, 64)), "K": b['INTRINSICS']}


@pytest.fixture(scope="module")
def oracle(weights, batch):
    """The float64 oracle's blocks, each fed the previous oracle block's float32-rounded outputs (what the device block
    gets in the test)."""
    W = Weights(weights, torch.float64)
    t = lambda a: torch.as_tensor(np.asarray(a.cpu() if isinstance(a, torch.Tensor) else a, np.float64))
    f32 = lambda x: x.to(torch.float32).to(torch.float64)
    ip, i22, K = t(batch["ip"]), t(batch["i22"]), batch["K"].cpu().numpy().astype(np.float64)
    ops = CameraOps(K)
    f1 = flow_block(W, "netFlow1", ip)
    fc2 = f32(f1["predict_flowconf2"])
    dm1 = depthmotion_block(W, "netDM1", ip, i22, fc2[:, 0:2].contiguous(), fc2)
    prev = {k: f32(dm1[k]) for k in ("predict_depth2", "predict_normal2", "predict_rotation", "predict_translation")}
    f2 = flow_block(W, "netFlow2", ip, i22, prev, ops=ops)
    fc2b = f32(f2["predict_flowconf2"])
    dm2 = depthmotion_block(W, "netDM2", ip, i22, fc2b[:, 0:2].contiguous(), fc2b, prev["predict_rotation"], prev["predict_translation"],
                            ops=ops)
    ref = refine_block(W, "netRefine", ip[:, 0:3], f32(dm2["predict_depth2"]))
    n = lambda d: {k: v.numpy() for k, v in d.items()}
    return {"netFlow1": n(f1), "netDM1": n(dm1), "netFlow2": n(f2), "netDM2": n(dm2), "netRefine": n(ref), "prev": n(prev),
            "fc2": fc2.numpy(), "fc2b": fc2b.numpy()}


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


def check_flowconf(out, ref, bar):
    for k in ("predict_flowconf5", "predict_flowconf2"):
        o, r = out[k].cpu().numpy(), ref[k]
        assert o.shape == r.shape
        epe = np.sqrt(((o[:, 0:2] - r[:, 0:2]) ** 2).sum(axis=1)).mean()
        conf = np.abs(o[:, 2:4] - r[:, 2:4]).mean()
        assert epe < bar and conf < bar, (k, epe, conf)


def check_dm(out, ref, bar):
    o = {k: v.cpu().numpy() for k, v in out.items()}
    d = np.abs(o["predict_depth2"] - ref["predict_depth2"]).sum() / np.abs(ref["predict_depth2"]).sum()
    assert d < bar, d
    assert np.abs(o["predict_normal2"] - ref["predict_normal2"]).mean() < bar
    for k in ("predict_rotation", "predict_translation", "predict_scale"):
        assert o[k].shape == ref[k].shape and np.abs(o[k] - ref[k]).max() < bar, k


@pytest.mark.parametrize("prec", list(BARS))
def test_blocks_against_fp64_oracle_on_each_samples_camera(sessions, batch, oracle, prec):
    s, bar = sessions[prec], BARS[prec]
    ip, i22, K = batch["ip"], batch["i22"], batch["K"]
    check_flowconf(blocks.flow_block(ip, scope="netFlow1", session=s), oracle["netFlow1"], bar)
    fc2 = _dev(oracle["fc2"])
    check_dm(blocks.depthmotion_block(ip, i22, fc2[:, 0:2], fc2, scope="netDM1", session=s), oracle["netDM1"], bar)
    prev = {k: _dev(v) for k, v in oracle["prev"].items()}
    check_flowconf(blocks.flow_block(ip, i22, K, prev, scope="netFlow2", session=s), oracle["netFlow2"], bar)
    fc2b = _dev(oracle["fc2b"])
    out = blocks.depthmotion_block(ip, i22, fc2b[:, 0:2], fc2b, prev["predict_rotation"], prev["predict_translation"], K,
                                   scope="netDM2", session=s)
    check_dm(out, oracle["netDM2"], bar)
    r = blocks.depth_refine_block(ip[:, 0:3], {"predict_depth2": _dev(oracle["netDM2"]["predict_depth2"])}, session=s)
    ref = oracle["netRefine"]
    d0 = r["predict_depth0"].cpu().numpy()
    assert np.abs(d0 - ref["predict_depth0"]).sum() / np.abs(ref["predict_depth0"]).sum() < bar
    assert np.abs(r["predict_normal0"].cpu().numpy() - ref["predict_normal0"]).mean() < bar


def test_one_samples_camera_moves_only_its_outputs(sessions, batch, oracle):
    s = sessions["3xtf32"]
    ip, i22, K = batch["ip"], batch["i22"], batch["K"]
    prev = {k: _dev(v) for k, v in oracle["prev"].items()}
    fc2 = _dev(oracle["fc2b"])
    K2 = K.clone()
    K2[2, 2] += 0.03
    K2[2, 0] *= 1.05

    def run(k):
        f = blocks.flow_block(ip, i22, k, prev, scope="netFlow2", session=s)
        d = blocks.depthmotion_block(ip, i22, fc2[:, 0:2], fc2, prev["predict_rotation"], prev["predict_translation"], k,
                                     scope="netDM2", session=s)
        return dict(f, **d)
    a, b = run(K), run(K2)
    for key in a:
        for n in range(4):
            same = torch.equal(a[key][n], b[key][n])
            assert same == (n != 2), (key, n)


def test_constant_camera_equals_the_networks_bit_for_bit(sessions, batch):
    """With the networks' constant camera the blocks are BootstrapNet / IterativeNet stage by stage."""
    from demon_b200.v2.networks import BootstrapNet, IterativeNet
    s = sessions["3xtf32"]
    ip, i22 = batch["ip"], batch["i22"]
    K = _dev(np.tile(K_NET, (4, 1)))
    boot = BootstrapNet(s, batch_size=4).eval(ip, i22)
    f1 = blocks.flow_block(ip, scope="netFlow1", session=s)
    fc2 = f1["predict_flowconf2"]
    dm1 = blocks.depthmotion_block(ip, i22, fc2[:, 0:2], fc2, scope="netDM1", session=s)
    assert torch.equal(f1["predict_flowconf5"][:, 0:2], boot["predict_flow5"])
    assert torch.equal(fc2[:, 0:2], boot["predict_flow2"])
    for k in ("predict_depth2", "predict_normal2", "predict_rotation", "predict_translation"):
        assert torch.equal(dm1[k], boot[k]), k
    it = IterativeNet(s, batch_size=4).eval(ip, i22, dm1["predict_depth2"], dm1["predict_normal2"], dm1["predict_rotation"],
                                            dm1["predict_translation"])
    f2 = blocks.flow_block(ip, i22, K, dm1, scope="netFlow2", session=s)
    fc2 = f2["predict_flowconf2"]
    dm2 = blocks.depthmotion_block(ip, i22, fc2[:, 0:2], fc2, dm1["predict_rotation"], dm1["predict_translation"], K,
                                   scope="netDM2", session=s)
    assert torch.equal(f2["predict_flowconf5"][:, 0:2], it["predict_flow5"])
    assert torch.equal(fc2[:, 0:2], it["predict_flow2"])
    for k in ("predict_depth2", "predict_normal2", "predict_rotation", "predict_translation"):
        assert torch.equal(dm2[k], it[k]), k


def test_scope_and_argument_mismatches_are_refused(sessions, batch):
    s = sessions["fp32"]
    ip, i22, K = batch["ip"], batch["i22"], batch["K"]
    z = lambda *shape: torch.zeros(shape, device="cuda")
    prev = {"predict_depth2": z(4, 1, 48, 64), "predict_normal2": z(4, 3, 48, 64), "predict_rotation": z(4, 3),
            "predict_translation": z(4, 3)}
    fc2 = z(4, 4, 48, 64)
    cases = [
        (lambda: blocks.flow_block(ip, i22, K, scope="netFlow1", session=s), "intrinsics"),
        (lambda: blocks.flow_block(ip, i22, None, prev, scope="netFlow1", session=s), "predict_depth2"),
        (lambda: blocks.flow_block(ip, i22, None, prev, scope="netFlow2", session=s), "intrinsics"),
        (lambda: blocks.flow_block(ip, i22, K, None, scope="netFlow2", session=s), "predict_depth2"),
        (lambda: blocks.flow_block(ip, None, K, prev, scope="netFlow2", session=s), "image2_2"),
        (lambda: blocks.flow_block(ip, i22, K, {"predict_depth2": prev["predict_depth2"]}, scope="netFlow2", session=s),
         "predict_normal2"),
        (lambda: blocks.flow_block(ip, scope="netDM1", session=s), "scope"),
        (lambda: blocks.depthmotion_block(ip, i22, fc2[:, :2], fc2, z(4, 3), scope="netDM1", session=s), "prev_rotation"),
        (lambda: blocks.depthmotion_block(ip, i22, fc2[:, :2], fc2, None, None, K, scope="netDM1", session=s), "intrinsics"),
        (lambda: blocks.depthmotion_block(ip, i22, fc2[:, :2], fc2, z(4, 3), z(4, 3), scope="netDM2", session=s), "intrinsics"),
        (lambda: blocks.depthmotion_block(ip, i22, fc2[:, :2], fc2, z(4, 3), None, K, scope="netDM2", session=s), "prev_translation"),
        (lambda: blocks.depthmotion_block(ip, i22, fc2[:, :2], fc2, scope="netFlow1", session=s), "scope"),
        (lambda: blocks.depthmotion_block(ip, i22, fc2[:, :2], fc2, z(4, 3), z(4, 3), z(3, 4), scope="netDM2", session=s),
         "intrinsics"),
        (lambda: blocks.depth_refine_block(ip[:, 0:3], prev, scope="netDM2", session=s), "scope"),
    ]
    for fn, name in cases:
        with pytest.raises(ValueError, match=name.replace("[", r"\[")):
            fn()
