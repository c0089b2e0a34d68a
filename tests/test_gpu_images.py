"""GPU: demon_b200.images.resize returns Pillow's bytes, prepare_input_data equals examples/example.py:15-42 on them, and
DemonPipeline.forward_images equals forward_u8 on the resized images, bit for bit."""
import importlib.util
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from demon_b200 import images

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def golden_module():
    spec = importlib.util.spec_from_file_location("make_resize_golden", os.path.join(GOLDEN, "make_resize_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def rand_images(seed, *shape):
    return torch.from_numpy(np.random.default_rng(seed).integers(0, 256, shape + (3,), dtype=np.uint8)).cuda()


def test_resize_matches_every_pillow_digest():
    """Every case of tests/golden/resize_digests.json: the 2-D sizes and their 64x48 second resize, the exhaustive width and
    height scans, the crop view (read in place), a batch of different images, the extreme downscales and tall images."""
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    committed = json.load(open(os.path.join(GOLDEN, "resize_digests.json")))
    committed.pop("_pillow")
    got = golden_module().digests(lambda x, size, f: images.resize(x, size, f),
                                  put=lambda a: torch.from_numpy(a).cuda(), get=lambda t: t.cpu().numpy())
    assert set(got) == set(committed)
    assert [k for k in got if got[k] != committed[k]] == []


def test_resize_single_image_and_crop_view_in_place():
    x = rand_images(3, 2, 600, 800)
    view = x[:, 53:533, 37:677]
    assert not view.is_contiguous()
    a = images.resize(view, (256, 192))
    b = images.resize(view.contiguous(), (256, 192))
    c = images.resize(view[1], (256, 192))
    assert torch.equal(a, b) and torch.equal(a[1], c) and c.shape == (192, 256, 3)


@pytest.mark.parametrize("data_format", ["channels_first", "channels_last"])
def test_prepare_input_data_equals_the_reference_arithmetic(data_format):
    """examples/example.py:15-42 applied with numpy to the device-resized bytes; one pair already 256x192 (not resized)."""
    for (h1, w1), (h2, w2), batch in (((480, 640), (480, 640), None), ((192, 256), (1080, 1920), 3)):
        shp = lambda h, w: (h, w) if batch is None else (batch, h, w)
        img1, img2 = rand_images(5, *shp(h1, w1)), rand_images(6, *shp(h2, w2))
        for resample in ("bicubic", "nearest"):
            got = images.prepare_input_data(img1, img2, data_format, resample)
            f = images.resample_code(resample)
            b1 = img1[None] if batch is None else img1
            b2 = img2[None] if batch is None else img2
            r1 = b1 if (h1, w1) == (192, 256) else images.resize(b1, (256, 192), f)
            r2 = b2 if (h2, w2) == (192, 256) else images.resize(b2, (256, 192), f)
            r22 = images.resize(r2, (64, 48), f)
            a1, a2, a22 = (t.cpu().numpy().astype(np.float32) / 255 - 0.5 for t in (r1, r2, r22))
            if data_format == "channels_first":
                a1, a2, a22 = (a.transpose(0, 3, 1, 2) for a in (a1, a2, a22))
                pair = np.concatenate((a1, a2), axis=1)
            else:
                pair = np.concatenate((a1, a2), axis=-1)
            ref = {"image_pair": pair, "image1": a1, "image2_2": a22}
            for k in ref:
                assert got[k].dtype == torch.float32 and got[k].is_cuda
                assert np.array_equal(got[k].cpu().numpy(), ref[k]), (k, resample)


@pytest.fixture(scope="module")
def session(synthetic_weights):
    from demon_b200.networks_original import Session
    s = Session(precision="3xtf32")
    s.load_weights(synthetic_weights)
    return s


@pytest.mark.parametrize("batch, h, w, crop", [(1, 480, 640, False), (4, 480, 640, True), (4, 192, 256, False)])
def test_forward_images_equals_forward_u8_on_resized_bytes(session, batch, h, w, crop):
    """Both image2_2 modes, three calls each with the same arguments (eager, graph capture, replay)."""
    from demon_b200.networks_original import DemonPipeline
    pipe = DemonPipeline(session, batch_size=batch, iterations=3)
    src = rand_images(20 + batch, batch, 2, h + 40, w + 24) if crop else rand_images(20 + batch, batch, 2, h, w)
    x = src[:, :, 17:17 + h, 5:5 + w] if crop else src
    for resample, mode in (("bicubic", "resize"), ("bicubic", "median"), ("nearest", "resize")):
        f = images.resample_code(resample)
        resized = torch.stack([images.resize(x[:, i], (256, 192), f) for i in range(2)], 1)   # [B,2,192,256,3]
        i22 = images.resize(resized[:, 1], (64, 48), f) if mode == "resize" else None
        ref_out = {k: v.clone() for k, v in pipe.own_outputs().items()}
        ref = pipe.forward_u8(resized.contiguous(), i22, outputs=ref_out)
        torch.cuda.synchronize()
        ref = {k: v.clone() for k, v in ref.items()}
        for call in range(3):
            got = pipe.forward_images(x, resample=resample, image2_2=mode)
            torch.cuda.synchronize()
            for k in ref:
                assert torch.equal(got[k], ref[k]), (k, resample, mode, call)
    from demon_b200 import _lib
    _lib.check_errors()


def test_forward_images_argument_errors(session):
    from demon_b200.networks_original import DemonPipeline
    pipe = DemonPipeline(session, batch_size=1, iterations=1)
    ok = rand_images(1, 1, 2, 48, 64)
    with pytest.raises(ValueError):
        pipe.forward_images(ok.float())
    with pytest.raises(ValueError):
        pipe.forward_images(ok[:, 0])                            # not a pair
    with pytest.raises(ValueError):
        pipe.forward_images(rand_images(1, 2, 2, 48, 64))        # batch 2 for a batch-1 pipeline
    with pytest.raises(ValueError):
        pipe.forward_images(ok, resample="lanczos")
    with pytest.raises(ValueError):
        pipe.forward_images(ok, image2_2="nearest")
    with pytest.raises(ValueError):
        pipe.forward_images(ok.cpu())
    with pytest.raises(ValueError):
        pipe.forward_images(ok[:, :, :, ::2])                    # pixel stride 6
    with pytest.raises(ValueError):
        images.resize(ok[0], (0, 10))
    with pytest.raises(ValueError):
        images.resize(ok[0], (64, 48), 1)
