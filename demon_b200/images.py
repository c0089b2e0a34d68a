"""Input preparation on the device: `PIL.Image.resize` and `prepare_input_data` of examples/example.py:15-42.

    from demon_b200 import images
    small = images.resize(frames, (256, 192))                    # CUDA uint8 [N,h,w,3] -> [N,192,256,3]
    input_data = images.prepare_input_data(img1, img2)           # the dict examples/example.py builds, as CUDA tensors

`resize` returns Pillow's bytes exactly for NEAREST, BILINEAR and BICUBIC (the kernel is resize_u8_kernel in
csrc/images.cu).  Inputs are CUDA uint8 RGB tensors in HWC order, as `torch.from_numpy(np.array(pil_image)).cuda()` gives
them; a cropped view such as `x[..., y0:y1, x0:x1, :]` is read in place.
"""
import ctypes

import torch

from . import _lib

NEAREST, BILINEAR, BICUBIC = 0, 2, 3   # PIL.Image.Resampling values
RESAMPLE = {"nearest": NEAREST, "bilinear": BILINEAR, "bicubic": BICUBIC}
MAX_SIDE = 8192


def resample_code(resample):
    """'nearest' | 'bilinear' | 'bicubic', or Pillow's enum value (PIL.Image.Resampling.BICUBIC, 3, ...)."""
    if isinstance(resample, str):
        if resample.lower() not in RESAMPLE:
            raise ValueError("resample must be one of %s, got %r" % (sorted(RESAMPLE), resample))
        return RESAMPLE[resample.lower()]
    if isinstance(resample, bool) or not isinstance(resample, int) or int(resample) not in RESAMPLE.values():
        raise ValueError("resample %r is not supported: NEAREST (0), BILINEAR (2) and BICUBIC (3) are" % (resample,))
    return int(resample)


def check_images(x, name, ndim):
    """CUDA uint8 RGB images of `ndim` dimensions, [..., h, w, 3] with pixel stride 3 and channel stride 1."""
    if not isinstance(x, torch.Tensor):
        raise ValueError("%s: expected a torch tensor, got %s" % (name, type(x).__name__))
    if x.dtype != torch.uint8:
        raise ValueError("%s: expected dtype uint8, got %s" % (name, x.dtype))
    if x.dim() != ndim:
        raise ValueError("%s: expected %d dimensions, got shape %s" % (name, ndim, tuple(x.shape)))
    if x.shape[-1] != 3:
        raise ValueError("%s: expected 3 channels (RGB) in the last dimension, got shape %s" % (name, tuple(x.shape)))
    if x.stride(-1) != 1 or (x.shape[-2] > 1 and x.stride(-2) != 3):   # the stride of a size-1 dimension is never used
        raise ValueError("%s: the pixel and channel strides must be 3 and 1, got %s" % (name, x.stride()[-2:]))
    if any(s < 0 for s in x.stride()):
        raise ValueError("%s: negative strides are not supported" % name)
    h, w = x.shape[-3], x.shape[-2]
    if not (1 <= h <= MAX_SIDE and 1 <= w <= MAX_SIDE):
        raise ValueError("%s: image size %dx%d (width x height) outside 1..%d" % (name, w, h, MAX_SIDE))
    if not x.is_cuda:
        raise ValueError("%s: expected a CUDA tensor" % name)


def _check_size(size):
    try:
        ow, oh = (int(v) for v in size)
    except (TypeError, ValueError):
        raise ValueError("size must be (width, height), got %r" % (size,))
    if not (1 <= ow <= MAX_SIDE and 1 <= oh <= MAX_SIDE):
        raise ValueError("size %dx%d (width x height) outside 1..%d" % (ow, oh, MAX_SIDE))
    return ow, oh


def resize(images, size, resample="bicubic"):
    """`PIL.Image.resize(size, resample)` of every image: images CUDA uint8 [N,h,w,3] (or one [h,w,3]), size (width, height)
    like Pillow's -> a new contiguous CUDA uint8 [N,height,width,3] (or [height,width,3]), asynchronous on the current
    stream.  The default filter is current Pillow's (BICUBIC); the Pillow 2.0 the reference used defaulted to NEAREST."""
    ow, oh = _check_size(size)
    code = resample_code(resample)
    single = isinstance(images, torch.Tensor) and images.dim() == 3
    x = images.unsqueeze(0) if single else images
    check_images(x, "images", 4)
    n, h, w = x.shape[0], x.shape[1], x.shape[2]
    if n > 65535:
        raise ValueError("images: at most 65535 images per call, got %d" % n)
    out = torch.empty((n, oh, ow, 3), dtype=torch.uint8, device=x.device)
    if n:
        with torch.cuda.device(x.device):
            _lib.check(_lib.load().demon_resize_u8(x.data_ptr(), x.stride(0), x.stride(1), n, h, w, out.data_ptr(), oh, ow, code,
                                                   ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    return out[0] if single else out


def to_float(images):
    """`np.array(img).astype(np.float32) / 255 - 0.5` (examples/example.py:25-27) on CUDA uint8 HWC images.  The divisor is a
    device tensor: with a Python number torch multiplies by its reciprocal instead, which is not numpy's division."""
    x = images.to(torch.float32)
    return x / torch.tensor(255.0, dtype=torch.float32, device=x.device) - 0.5


def prepare_input_data(img1, img2, data_format="channels_first", resample="bicubic"):
    """examples/example.py:15-42 on the device: img1, img2 CUDA uint8 [h,w,3] (or batches [N,h,w,3]) of any size ->
    {'image_pair': [N,6,192,256], 'image1': [N,3,192,256], 'image2_2': [N,3,48,64]} CUDA float32 (channels_last: HWC order,
    [N,192,256,6] ...).  Like the reference, an image already 256x192 is not resized, and image2_2 is the resized second
    image resized again to 64x48."""
    if data_format not in ("channels_first", "channels_last"):
        raise ValueError("data_format must be 'channels_first' or 'channels_last'")
    code = resample_code(resample)
    prepared = []
    for name, img in (("img1", img1), ("img2", img2)):
        if not isinstance(img, torch.Tensor) or img.dim() not in (3, 4):
            raise ValueError("%s: expected a CUDA uint8 tensor [h,w,3] or [N,h,w,3]" % name)
        x = img.unsqueeze(0) if img.dim() == 3 else img
        check_images(x, name, 4)
        prepared.append(x if tuple(x.shape[1:3]) == (192, 256) else resize(x, (256, 192), code))
    a, b = prepared
    if a.shape[0] != b.shape[0]:
        raise ValueError("img1 and img2 hold %d and %d images" % (a.shape[0], b.shape[0]))
    img2_2 = resize(b, (64, 48), code)
    i1, i2, i22 = to_float(a), to_float(b), to_float(img2_2)
    if data_format == "channels_first":
        i1, i2, i22 = (t.permute(0, 3, 1, 2) for t in (i1, i2, i22))
        pair = torch.cat((i1, i2), dim=1)
    else:
        pair = torch.cat((i1, i2), dim=-1)
    return {"image_pair": pair.contiguous(), "image1": i1.contiguous(), "image2_2": i22.contiguous()}
