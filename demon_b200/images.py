"""Input preparation on the device: `PIL.Image.resize` and `prepare_input_data` of examples/example.py:15-42, and the image
part of `adjust_intrinsics` (dataset_tools/view_tools.py:97-172) for photos from other cameras.

    from demon_b200 import images
    small = images.resize(frames, (256, 192))                    # CUDA uint8 [N,h,w,3] -> [N,192,256,3]
    input_data = images.prepare_input_data(img1, img2)           # the dict examples/example.py builds, as CUDA tensors
    adapted, K_new, status = images.adjust_intrinsics(frames, K) # to the intrinsics DeMoN was trained for, 256x192

`resize` returns Pillow's bytes exactly for NEAREST, BILINEAR and BICUBIC (the kernel is resize_u8_kernel in
csrc/images.cu).  Inputs are CUDA uint8 RGB tensors in HWC order, as `torch.from_numpy(np.array(pil_image)).cuda()` gives
them; a cropped view such as `x[..., y0:y1, x0:x1, :]` is read in place.
"""
import ctypes

import numpy as np
import torch

from . import _lib

NEAREST, BILINEAR, BICUBIC = 0, 2, 3   # PIL.Image.Resampling values
RESAMPLE = {"nearest": NEAREST, "bilinear": BILINEAR, "bicubic": BICUBIC}
MAX_SIDE = 8192
# The intrinsics DeMoN was trained for, normalised (fx, fy, cx, cy); examples/example.py:51-61 asks for images adapted to them
NETWORK_INTRINSICS = (0.89115971, 1.18821287, 0.5, 0.5)
MAX_OFFSET = 2 ** 24   # largest crop offset adjust_intrinsics accepts


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


def _check_area(x, size):
    """The checks of resize_area that need no device: x torch or numpy float32 [N,C,h,w] or [C,h,w], size (oh, ow) dividing
    (h, w).  Returns (oh, ow)."""
    if not isinstance(x, (torch.Tensor, np.ndarray)):
        raise ValueError("images: expected a torch CUDA tensor or a numpy array, got %s" % type(x).__name__)
    if x.dtype != (torch.float32 if isinstance(x, torch.Tensor) else np.float32):
        raise ValueError("images: expected float32, got %s" % x.dtype)
    if x.ndim not in (3, 4):
        raise ValueError("images: expected [N,C,h,w] or [C,h,w], got shape %s" % (tuple(x.shape),))
    if isinstance(x, torch.Tensor) and not x.is_cuda:
        raise ValueError("images: a torch tensor must be on a CUDA device (or pass a numpy array)")
    try:
        oh, ow = (int(v) for v in size)
    except (TypeError, ValueError):
        raise ValueError("size must be (height, width), got %r" % (size,))
    h, w = x.shape[-2:]
    if not (1 <= oh <= h and 1 <= ow <= w and h % oh == 0 and w % ow == 0):
        raise ValueError("resize_area: %dx%d -> %dx%d (height x width) is not a downsampling by integer factors" % (h, w, oh, ow))
    if x.shape[-3] * h * w >= 2 ** 31 or (x.ndim == 4 and x.shape[0] >= 2 ** 31):
        raise ValueError("images: shape %s too large" % (tuple(x.shape),))
    return oh, ow


def _resize_area_into(x, out):
    """resize_area of CUDA float32 [N,C,h,w] (rows and planes packed, any sample stride) into `out` [N,C,oh,ow] contiguous,
    on the current stream."""
    n, c, h, w = x.shape
    if x.stride()[1:] != (h * w, w, 1) or (n > 1 and x.stride(0) < c * h * w):
        x = x.contiguous()
    with torch.cuda.device(x.device):
        _lib.check(_lib.load().demon_resize_area_f32(x.data_ptr(), x.stride(0) if n > 1 else c * h * w, out.data_ptr(), n, c, h, w,
                                                     out.shape[2], out.shape[3], ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    return out


def resize_area(images, size):
    """`tf.image.resize_area(images, size)` (align_corners=False) for integer factors, the image2_2 of
    training/v2/training.py:179 (`resize_area(image2, (48, 64))`): images float32 [N,C,h,w] or [C,h,w] (NCHW, unlike TF's
    NHWC), size (height, width) as TF takes it, h and w multiples of them; other sizes raise ValueError.  A torch CUDA tensor
    gives a new torch CUDA tensor (asynchronous, current stream; a channel slice such as image_pair[:, 3:6] is read in place),
    a numpy array a numpy array.  Every output is the fy x fx block's rows summed left to right, the row sums top to bottom,
    times float32(1 / (fy fx)), in float32 (this project's definition; DESIGN.md §3.6)."""
    oh, ow = _check_area(images, size)
    was_np = isinstance(images, np.ndarray)
    if was_np:
        if not torch.cuda.is_available():
            raise RuntimeError("resize_area needs a CUDA device (there is no CPU fallback)")
        x = torch.from_numpy(np.ascontiguousarray(images)).cuda()
    else:
        x = images
    single = x.dim() == 3
    x4 = x.unsqueeze(0) if single else x
    out = torch.empty((x4.shape[0], x4.shape[1], oh, ow), dtype=torch.float32, device=x4.device)
    _resize_area_into(x4, out)
    out = out[0] if single else out
    return out.cpu().numpy() if was_np else out


def demon_intrinsics(width=256, height=192):
    """The intrinsics DeMoN was trained for in pixels of a width x height image: numpy float64 K [3,3]."""
    fx, fy, cx, cy = NETWORK_INTRINSICS
    return np.array([[fx * width, 0.0, cx * width], [0.0, fy * height, cy * height], [0.0, 0.0, 1.0]])


def intrinsics4(K, lead, name):
    """K as [*lead,3,3] (the skew K[0,1] is ignored, as in the reference), [*lead,4] (fx, fy, cx, cy) or one [3,3] for all,
    from numpy, a CPU or a CUDA tensor -> float64 [*lead,4]: a numpy array for host input, a CUDA tensor for CUDA input."""
    cuda = isinstance(K, torch.Tensor) and K.is_cuda
    try:
        k = K.to(torch.float64) if cuda else np.asarray(K.cpu() if isinstance(K, torch.Tensor) else K, dtype=np.float64)
    except (TypeError, ValueError):
        raise ValueError("%s: expected a numpy array or a tensor of intrinsics, got %s" % (name, type(K).__name__))
    shape = tuple(k.shape)
    if shape == (3, 3) or shape == tuple(lead) + (3, 3):
        k = k[..., [0, 1, 0, 1], [0, 1, 2, 2]]
    elif shape != tuple(lead) + (4,):
        raise ValueError("%s: expected shape %s, %s or (3, 3), got %s" % (name, tuple(lead) + (3, 3), tuple(lead) + (4,), shape))
    if cuda:
        return k.expand(tuple(lead) + (4,)).contiguous()
    return np.ascontiguousarray(np.broadcast_to(k, tuple(lead) + (4,)))


def intrinsics_window(K, K_new, w, h, width_new, height_new):
    """What csrc/images.cu (window_of) computes for every image, on the host: K [...,4] and K_new [4] float64 numpy
    (fx, fy, cx, cy), a w x h source, a width_new x height_new output -> dict of int64 arrays rw, rh (size of the resize),
    x0, y0 (window offset in it), bilinear (1: BILINEAR, 0: LANCZOS) and status (0 ok, 1 fill added, 2 invalid)."""
    K = np.asarray(K, dtype=np.float64)
    fx, fy, cx, cy = (K[..., i] for i in range(4))
    with np.errstate(all="ignore"):
        sx, sy = K_new[0] / fx, K_new[1] / fy
        rw, rh = w * sx, h * sy
        x0, y0 = np.rint(cx * sx - K_new[2]), np.rint(cy * sy - K_new[3])
        ok = (np.isfinite(fx) & (fx > 0) & np.isfinite(fy) & (fy > 0) & np.isfinite(cx) & np.isfinite(cy) & (rw >= 1) & (rw < MAX_SIDE + 1)
              & (rh >= 1) & (rh < MAX_SIDE + 1) & (np.abs(x0) <= MAX_OFFSET) & (np.abs(y0) <= MAX_OFFSET))
        z = lambda a: np.where(ok, a, 0).astype(np.int64)
        rw, rh, x0, y0 = z(rw), z(rh), z(x0), z(y0)
        leaves = (x0 < 0) | (y0 < 0) | (x0 + width_new > rw) | (y0 + height_new > rh)
    return {"rw": rw, "rh": rh, "x0": x0, "y0": y0, "bilinear": z(sx > 1), "status": np.where(ok, leaves.astype(np.int64), 2)}


def _check_adjust_source(h, w, name):
    if h > 100 * w:
        raise ValueError("%s: a source more than 100 times taller than wide (%dx%d, width x height) is not supported" % (name, w, h))


def _device_intrinsics(K, lead, name, w, h, knew, width_new, height_new, device):
    """intrinsics4 on `device`; host K is checked first (ValueError for what the kernel would mark invalid, status 2)."""
    k = intrinsics4(K, lead, name)
    if isinstance(k, np.ndarray):
        bad = np.flatnonzero(intrinsics_window(k, knew, w, h, width_new, height_new)["status"].reshape(-1) == 2)
        if bad.size:
            raise ValueError("%s: the intrinsics %s of image %d give no valid resize of a %dx%d image: the focal lengths must be "
                             "finite and positive, the principal point finite, the resized size within 1..%d and the offset within "
                             "+-2^24" % (name, k.reshape(-1, 4)[bad[0]].tolist(), bad[0], w, h, MAX_SIDE))
        k = torch.from_numpy(k).to(device)
    return k


def adjust_intrinsics(images, K, K_new=None, width_new=256, height_new=192):
    """The image part of the reference's `adjust_intrinsics(view, K_new, width_new, height_new)` on the device: every image
    (CUDA uint8 [N,h,w,3], or one [h,w,3]) with intrinsics K ([N,3,3], [3,3] or [N,4] = fx, fy, cx, cy in pixels; numpy,
    CPU or CUDA) is resized so that its focal lengths become K_new's (BILINEAR if fx_new / fx > 1, else LANCZOS, bit for bit
    with Pillow) and cropped so that its principal point and size become K_new's and width_new x height_new, with
    (127, 127, 127) where the crop leaves the resized image.  K_new (host [3,3] or [4]) defaults to demon_intrinsics(width_new,
    height_new).  Returns (images [N,height_new,width_new,3], K_new numpy [3,3], status CUDA uint8 [N]): 0 ok, 1 fill was
    added (where the reference prints a warning), 2 invalid K (only for CUDA K; host K is checked here: ValueError).
    Asynchronous on the current stream.  Unlike the reference's safe_crop_image, the crop is also right when the box leaves
    the image with a positive offset (DESIGN.md section 7)."""
    ow, oh = _check_size((width_new, height_new))
    single = isinstance(images, torch.Tensor) and images.dim() == 3
    x = images.unsqueeze(0) if single else images
    check_images(x, "images", 4)
    n, h, w = x.shape[0], x.shape[1], x.shape[2]
    if n > 65535:
        raise ValueError("images: at most 65535 images per call, got %d" % n)
    _check_adjust_source(h, w, "images")
    knew = intrinsics4(demon_intrinsics(ow, oh) if K_new is None else K_new, (), "K_new")
    if not isinstance(knew, np.ndarray):
        knew = knew.cpu().numpy()
    if not (np.all(np.isfinite(knew)) and knew[0] > 0 and knew[1] > 0):
        raise ValueError("K_new: the focal lengths must be finite and positive and the principal point finite, got %s" % knew.tolist())
    k = _device_intrinsics(K, (n,), "K", w, h, knew, ow, oh, x.device)
    out = torch.empty((n, oh, ow, 3), dtype=torch.uint8, device=x.device)
    status = torch.empty((n,), dtype=torch.uint8, device=x.device)
    if n:
        with torch.cuda.device(x.device):
            _lib.check(_lib.load().demon_adjust_intrinsics_u8(
                x.data_ptr(), x.stride(0), x.stride(1), n, h, w, k.data_ptr(), *(float(v) for v in knew), out.data_ptr(), oh, ow,
                status.data_ptr(), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    K_out = np.array([[knew[0], 0.0, knew[2]], [0.0, knew[1], knew[3]], [0.0, 0.0, 1.0]])
    return (out[0], K_out, status[0]) if single else (out, K_out, status)
