"""CPU: the resize fixture still is what Pillow computes, and demon_b200.images / the C entries refuse bad arguments before
any device work."""
import ctypes
import importlib.util
import json
import os

import numpy as np
import pytest
import torch

from demon_b200 import _lib, build as dbuild, images

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def load_golden_module():
    spec = importlib.util.spec_from_file_location("make_resize_golden", os.path.join(GOLDEN, "make_resize_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_resize_digests_match_pillow():
    """Regenerates every digest with the installed Pillow: guards the committed fixture against Pillow changing its
    arithmetic (the fixture was written with the version stored under "_pillow")."""
    pytest.importorskip("PIL")
    committed = json.load(open(os.path.join(GOLDEN, "resize_digests.json")))
    committed.pop("_pillow")
    fresh = load_golden_module().pillow_digests()
    assert set(fresh) == set(committed)
    assert [k for k in fresh if fresh[k] != committed[k]] == []


def test_resample_names_and_pillow_values():
    assert images.resample_code("bicubic") == images.BICUBIC == 3
    assert images.resample_code("Nearest") == images.NEAREST == 0
    assert images.resample_code(2) == images.BILINEAR
    pil = pytest.importorskip("PIL.Image")
    assert images.resample_code(pil.Resampling.BICUBIC) == 3
    for bad in ("lanczos", "box", "hamming", "area", 1, 4, 5, -1, 2.0, True, None):
        with pytest.raises(ValueError):
            images.resample_code(bad)


@pytest.mark.parametrize("x, size, resample", [
    (np.zeros((1, 8, 8, 3), np.uint8), (4, 4), "bicubic"),                 # not a tensor
    (torch.zeros(1, 8, 8, 3), (4, 4), "bicubic"),                          # float32
    (torch.zeros(1, 8, 8, 4, dtype=torch.uint8), (4, 4), "bicubic"),       # 4 channels
    (torch.zeros(1, 3, 8, 8, dtype=torch.uint8), (4, 4), "bicubic"),       # CHW: 8 channels
    (torch.zeros(1, 8, 16, 3, dtype=torch.uint8)[:, :, ::2], (4, 4), "bicubic"),    # pixel stride 6
    (torch.zeros(1, 8, 3, 8, dtype=torch.uint8).transpose(2, 3), (4, 4), "bicubic"),   # channel stride 8
    (torch.zeros(8, 8, 8, 8, 3, dtype=torch.uint8), (4, 4), "bicubic"),    # 5 dimensions
    (torch.zeros(1, 8, 8, 3, dtype=torch.uint8), (0, 4), "bicubic"),       # size out of range
    (torch.zeros(1, 8, 8, 3, dtype=torch.uint8), (4, 8193), "bicubic"),
    (torch.zeros(1, 8, 8, 3, dtype=torch.uint8), (4,), "bicubic"),
    (torch.zeros(1, 8193, 1, 3, dtype=torch.uint8), (4, 4), "bicubic"),    # source out of range
    (torch.zeros(1, 8, 8, 3, dtype=torch.uint8), (4, 4), "lanczos"),       # filter
    (torch.zeros(1, 8, 8, 3, dtype=torch.uint8), (4, 4), 1),
    (torch.zeros(1, 8, 8, 3, dtype=torch.uint8), (4, 4), "bicubic"),       # a CPU tensor
])
def test_resize_argument_errors(x, size, resample):
    with pytest.raises(ValueError):
        images.resize(x, size, resample)


def test_prepare_input_data_argument_errors():
    ok = torch.zeros(192, 256, 3, dtype=torch.uint8)
    with pytest.raises(ValueError):
        images.prepare_input_data(ok, ok, data_format="NCHW")
    with pytest.raises(ValueError):
        images.prepare_input_data(ok, ok, resample="lanczos")
    with pytest.raises(ValueError):
        images.prepare_input_data(ok.numpy(), ok)
    with pytest.raises(ValueError):
        images.prepare_input_data(ok.float(), ok)
    with pytest.raises(ValueError):   # a CPU tensor
        images.prepare_input_data(ok, ok)


def test_resize_and_pipeline_args_reject_bad_arguments_before_any_device_work():
    dbuild.build()
    lib = _lib.load()
    buf = (ctypes.c_uint8 * 16)()
    p = ctypes.addressof(buf)
    calls = [
        (p, 24, 24, 1, 8, 8, p, 4, 4, 1),        # LANCZOS
        (p, 24, 24, 1, 8, 8, p, 4, 4, 4),        # BOX
        (p, 24, 24, 1, 8, 8, p, 4, 4, 5),        # HAMMING
        (p, 24, 24, 1, 0, 8, p, 4, 4, 3),        # empty source
        (p, 24, 24, 1, 8, 8193, p, 4, 4, 3),     # source too wide
        (p, 24, 24, 1, 8, 8, p, 8193, 4, 3),     # output too tall
        (p, 24, 24, -1, 8, 8, p, 4, 4, 3),       # n
        (p, -24, 24, 1, 8, 8, p, 4, 4, 3),       # negative stride
        (None, 24, 24, 1, 8, 8, p, 4, 4, 3),     # null source
    ]
    for args in calls:
        assert lib.demon_resize_u8(*args, None) == -1, args
    assert lib.demon_resize_u8(p, 24, 24, 1, 8, 8, p, 4, 4, 1, None) == -1
    assert "resample 1" in lib.demon_last_error().decode()
    args = _lib.PipelineArgs(input=_lib.INPUT_RESIZE_U8, images=p, h=480, w=640, resample=3, image2_2_mode=1, iterations=3)
    assert lib.demon_pipeline_run(None, args, None) == -1
