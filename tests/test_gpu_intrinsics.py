"""GPU: demon_b200.images.adjust_intrinsics returns Pillow's bytes and the reference's status for every fixture case, invalid
intrinsics give fill and status 2, and DemonPipeline.forward_views equals forward_u8 on the adapted bytes, bit for bit."""
import importlib.util
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from demon_b200 import _lib, images

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def golden_module():
    spec = importlib.util.spec_from_file_location("make_intrinsics_golden", os.path.join(GOLDEN, "make_intrinsics_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def rand_images(seed, *shape):
    return torch.from_numpy(np.random.default_rng(seed).integers(0, 256, shape + (3,), dtype=np.uint8)).cuda()


def cameras(b, seed):
    """[b,2,4] plausible cameras for 480x640 images, different per image; some leave the resized image"""
    rng = np.random.default_rng(seed)
    f = rng.uniform(380, 700, (b, 2))
    return np.stack([f, f * rng.uniform(0.95, 1.05, (b, 2)), rng.uniform(250, 390, (b, 2)), rng.uniform(180, 300, (b, 2))], -1)


def test_adjust_intrinsics_matches_every_pillow_digest():
    """Every case of tests/golden/intrinsics_digests.json with K on the device: realistic cameras, a crop view read in
    place, a batch with a K per image, the LANCZOS scans, both filter mixes, skipped passes, windows leaving each side or
    the whole image, round()'s ties and int()'s truncation; the status included."""
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    committed = json.load(open(os.path.join(GOLDEN, "intrinsics_digests.json")))
    committed.pop("_pillow")

    def adjust(x, K, K_new, ow, oh):
        out, _, status = images.adjust_intrinsics(x, torch.from_numpy(K).cuda(), K_new, ow, oh)
        return out, status

    got = golden_module().digests(adjust, put=lambda a: torch.from_numpy(a).cuda(), get=lambda t: t.cpu().numpy())
    assert set(got) == set(committed)
    assert [k for k in got if got[k] != committed[k]] == []
    _lib.check_errors()


def test_host_and_device_intrinsics_agree_and_single_image():
    x = rand_images(3, 2, 600, 800)
    view = x[:, 53:533, 37:677]
    K = np.array([[[525.0, 0, 319.5], [0, 525, 239.5], [0, 0, 1]], [[480.0, 0.3, 300], [0, 470, 250], [0, 0, 1]]])
    a, K_new, sa = images.adjust_intrinsics(view, K)
    b, _, sb = images.adjust_intrinsics(view.contiguous(), torch.from_numpy(K).cuda().float().double())
    c, _, sc = images.adjust_intrinsics(view[1], K[1])
    assert torch.equal(a, b) and torch.equal(sa, sb) and torch.equal(a[1], c) and int(sc) == int(sa[1])
    assert a.shape == (2, 192, 256, 3) and c.shape == (192, 256, 3)
    assert np.array_equal(K_new, images.demon_intrinsics())
    d = images.intrinsics_window(images.intrinsics4(K, (2,), "K"), images.intrinsics4(K_new, (), "K_new"), 640, 480, 256, 192)
    assert sa.cpu().numpy().tolist() == d["status"].tolist()


def test_invalid_device_intrinsics_give_fill_and_status_2():
    """Values the host check would refuse, passed on the device: every output byte is the fill and the status is 2, and the
    valid images of the same batch are unaffected."""
    x = rand_images(4, 9, 480, 640)
    good = [525.0, 525.0, 319.5, 239.5]
    bad = [[np.nan, 525, 319.5, 239.5], [0, 525, 319.5, 239.5], [525, -1, 319.5, 239.5], [525, 525, np.inf, 239.5],
           [525, 525, 319.5, -np.nan], [1e-3, 525, 319.5, 239.5], [525, 1e7, 319.5, 239.5], [525, 525, 1e12, 239.5]]
    K = torch.tensor([good] + bad, dtype=torch.float64, device="cuda")
    out, _, status = images.adjust_intrinsics(x, K)
    assert status.cpu().tolist() == [0] + [2] * len(bad)
    assert bool((out[1:] == 127).all())
    ref, _, _ = images.adjust_intrinsics(x[:1], K[:1])
    assert torch.equal(out[:1], ref)
    _lib.check_errors()


@pytest.fixture(scope="module")
def session(synthetic_weights):
    from demon_b200.networks_original import Session
    s = Session(precision="3xtf32")
    s.load_weights(synthetic_weights)
    return s


@pytest.mark.parametrize("batch, crop", [(1, False), (4, True)])
def test_forward_views_equals_forward_u8_on_adapted_bytes(session, batch, crop):
    """Both image2_2 modes; eager, capture and replay calls, the replays after rewriting the SAME intrinsics tensor with new
    values, which the outputs must follow."""
    from demon_b200.networks_original import DemonPipeline
    pipe = DemonPipeline(session, batch_size=batch, iterations=2)
    h, w = 480, 640
    src = rand_images(30 + batch, batch, 2, h + 40, w + 24) if crop else rand_images(30 + batch, batch, 2, h, w)
    x = src[:, :, 17:17 + h, 5:5 + w] if crop else src
    K = torch.from_numpy(cameras(batch, 1)).cuda()
    for resample, mode in (("bicubic", "resize"), ("bicubic", "median"), ("nearest", "resize")):
        f = images.resample_code(resample)
        for call in range(4):
            if call == 3:
                K.copy_(torch.from_numpy(cameras(batch, 2 + call)))   # same tensor, new values: the replay must see them
            adapted, _, status = images.adjust_intrinsics(x.reshape(batch * 2, h, w, 3), K.reshape(-1, 4))
            adapted = adapted.reshape(batch, 2, 192, 256, 3)
            i22 = images.resize(adapted[:, 1], (64, 48), f) if mode == "resize" else None
            ref_out = {k: v.clone() for k, v in pipe.own_outputs().items()}
            ref = pipe.forward_u8(adapted.contiguous(), i22, outputs=ref_out)
            torch.cuda.synchronize()
            ref = {k: v.clone() for k, v in ref.items()}
            got = pipe.forward_views(x, K, resample=resample, image2_2=mode)
            torch.cuda.synchronize()
            for k in ref:
                assert torch.equal(got[k], ref[k]), (k, resample, mode, call)
            assert torch.equal(got["status"].reshape(-1), status), (resample, mode, call)
    _lib.check_errors()


def test_forward_views_host_intrinsics_and_errors(session):
    from demon_b200.networks_original import DemonPipeline
    pipe = DemonPipeline(session, batch_size=2, iterations=1)
    x = rand_images(7, 2, 2, 480, 640)
    K = cameras(2, 9)
    a = {k: v.clone() for k, v in pipe.forward_views(x, K).items()}
    b = pipe.forward_views(x, torch.from_numpy(K).cuda())
    torch.cuda.synchronize()
    assert all(torch.equal(a[k], b[k]) for k in a)
    K33 = np.zeros((2, 2, 3, 3))
    K33[..., 0, 0], K33[..., 1, 1], K33[..., 0, 2], K33[..., 1, 2], K33[..., 2, 2] = K[..., 0], K[..., 1], K[..., 2], K[..., 3], 1
    c = pipe.forward_views(x, K33)
    torch.cuda.synchronize()
    assert all(torch.equal(a[k], c[k]) for k in a)
    bad = K.copy()
    bad[1, 0, 0] = 0.0
    with pytest.raises(ValueError):
        pipe.forward_views(x, bad)
    with pytest.raises(ValueError):
        pipe.forward_views(x, K[:1])
    with pytest.raises(ValueError):
        pipe.forward_views(x, K, image2_2="nearest")
    with pytest.raises(ValueError):
        pipe.forward_views(rand_images(1, 2, 2, 800, 7), K)   # more than 100 times taller than wide
    _lib.check_errors()
