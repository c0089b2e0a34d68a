"""Mirror of `depthmotionnet.networks_original` (python/depthmotionnet/networks_original.py) over
the CUDA network plan in libdemon_b200.so.

    session = Session(); session.load_weights(tf_named_weights)        # examples/example.py:70-83
    bootstrap_net = BootstrapNet(session, data_format)                  # examples/example.py:75-77
    iterative_net = IterativeNet(session, data_format)
    refine_net = RefinementNet(session, data_format)
    result = bootstrap_net.eval(image_pair, image2_2)                   # examples/example.py:87-99
    ...

Same class names, constructor arguments, `eval` signatures and result-dict keys as the reference;
numpy (or torch) arrays in, a dict of numpy arrays out (torch CUDA tensors out if the inputs were
torch CUDA tensors).  `Session` stands in for the `tf.Session` that owns the variables in the
reference: it owns the TF-named weights and the device network handle.  `DemonPipeline` is the
fused bootstrap -> N x iterative -> refinement call that never leaves the device.
"""
import ctypes

import numpy as np
import torch

from . import _lib
from ._lib import check_errors  # noqa: F401  (re-exported: networks_original.check_errors())

PRECISIONS = {"fp32": 0, "3xtf32": 1, "tf32": 2}
DEFAULT_PRECISION = "3xtf32"


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


class _NetHandle:
    """RAII wrapper of a finalized `demon_net*`."""

    _create = "demon_net_create"   # the C entry that lays out the plan (demon_b200.v2.networks: demon_net_create_v2)

    def __init__(self, weights, batch, refine_hw, precision):
        if not torch.cuda.is_available():
            raise RuntimeError("demon_b200 networks need a CUDA device (there is no CPU fallback)")
        lib = _lib.load()
        self._lib = lib
        self.ptr = ctypes.c_void_p()
        self.batch, self.refine_hw, self.precision = batch, refine_hw, precision
        _lib.check(getattr(lib, self._create)(ctypes.byref(self.ptr), batch, refine_hw[0], refine_hw[1], PRECISIONS[precision]))
        for i in range(lib.demon_net_num_variables(self.ptr)):
            name = lib.demon_net_variable_name(self.ptr, i).decode()
            if name not in weights:
                raise KeyError("weights are missing variable %r" % name)
            a = np.ascontiguousarray(weights[name], dtype=np.float32)
            shape = (ctypes.c_int64 * a.ndim)(*a.shape)
            _lib.check(lib.demon_net_set_weight(self.ptr, name.encode(), a.ctypes.data_as(ctypes.c_void_p),
                                                ctypes.cast(shape, ctypes.c_void_p), a.ndim))
        _lib.check(lib.demon_net_finalize(self.ptr))

    def variable_names(self):
        return [self._lib.demon_net_variable_name(self.ptr, i).decode()
                for i in range(self._lib.demon_net_num_variables(self.ptr))]

    def uses_tensor_cores(self, layer):
        return bool(self._lib.demon_net_layer_uses_tensor_cores(self.ptr, layer.encode()))

    def __del__(self):
        try:
            if getattr(self, "ptr", None) is not None and self.ptr.value:
                self._lib.demon_net_destroy(self.ptr)
                self.ptr = ctypes.c_void_p()
        except Exception:
            pass


class Session:
    """Owner of the variables, in place of the tf.Session of the reference (examples/example.py:70-83)."""

    _handle = _NetHandle   # the network the session's handles run (demon_b200.v2.networks: v2)

    def __init__(self, precision=DEFAULT_PRECISION):
        if precision not in PRECISIONS:
            raise ValueError("precision must be one of %s" % sorted(PRECISIONS))
        self.precision = precision
        self.weights = None
        self._nets = {}

    def load_weights(self, weights):
        """weights: dict TF variable name -> numpy array in TF layout (see demon_b200.weights, demon_b200.v2.weights)."""
        self.weights = weights
        self._nets = {}

    def restore(self, save_path):
        """`tf.train.Saver().restore(session, save_path)` of examples/example.py:82-83: reads the TensorFlow checkpoint
        `save_path` (prefix of the .index / .data-0000x-of-0000y files, e.g. 'weights/demon_original') with the
        pure-Python bundle reader.  A dict of arrays is accepted as well (same as load_weights)."""
        if isinstance(save_path, dict):
            return self.load_weights(save_path)
        from . import checkpoint
        self.load_weights(checkpoint.load_demon_weights(str(save_path)))

    def net(self, batch, refine_hw=(192, 256)):
        if self.weights is None:
            raise RuntimeError("Session.load_weights() has not been called")
        key = (int(batch), tuple(refine_hw))
        if key not in self._nets:
            self._nets[key] = self._handle(self.weights, key[0], key[1], self.precision)
        return self._nets[key]


_default_session = None


def default_session():
    global _default_session
    if _default_session is None:
        _default_session = Session()
    return _default_session


def _check_format(data_format):
    if data_format not in ("channels_first", "channels_last"):
        raise ValueError("data_format must be 'channels_first' or 'channels_last'")
    return 0 if data_format == "channels_first" else 1


def _require_cuda():
    if not torch.cuda.is_available():
        raise RuntimeError("demon_b200 networks need a CUDA device (there is no CPU fallback)")


def _to_dev(x, shape, name):
    _require_cuda()
    was_torch = isinstance(x, torch.Tensor)
    if was_torch:
        t = x if x.is_cuda else x.cuda()
        t = t.to(torch.float32)
    else:
        t = torch.from_numpy(np.ascontiguousarray(np.asarray(x), dtype=np.float32)).cuda()
    if tuple(t.shape) != tuple(shape):
        raise ValueError("%s: expected shape %s, got %s" % (name, tuple(shape), tuple(t.shape)))
    return t.contiguous(), (was_torch and x.is_cuda)


def _shape(fmt, b, c, h, w):
    return (b, c, h, w) if fmt == 0 else (b, h, w, c)


def _ptr(x):
    """The address of a torch tensor (host or device) or of a numpy array; None for None."""
    if x is None:
        return None
    return x.data_ptr() if isinstance(x, torch.Tensor) else x.ctypes.data


# the output pointers of the fused-pipeline entries, in C ABI order
_OUTPUTS = ("predict_depth0", "predict_rotation", "predict_translation", "predict_flow2", "predict_depth2", "predict_normal2")
_SNAPSHOT_OUTPUTS = ("predict_flow2", "predict_depth2", "predict_normal2", "predict_rotation", "predict_translation", "predict_depth0")


class _NetBase:
    def __init__(self, session, data_format="channels_first", batch_size=1):
        self.session = session if session is not None else default_session()
        self.data_format = data_format
        self._fmt = _check_format(data_format)
        self.batch_size = int(batch_size)

    def _outputs(self, dev):
        b, f = self.batch_size, self._fmt
        mk = lambda *s: torch.empty(s, dtype=torch.float32, device=dev)
        return {
            "predict_flow5": mk(*_shape(f, b, 2, 6, 8)),
            "predict_flow2": mk(*_shape(f, b, 2, 48, 64)),
            "predict_depth2": mk(*_shape(f, b, 1, 48, 64)),
            "predict_normal2": mk(*_shape(f, b, 3, 48, 64)),
            "predict_rotation": mk(b, 3),
            "predict_translation": mk(b, 3),
        }

    @staticmethod
    def _finish(out, keep_torch):
        """numpy in -> numpy out like the reference's session.run (synchronises and checks the device error flag);
        torch CUDA tensors in -> torch CUDA tensors out, asynchronous: call `check_errors()` after synchronising."""
        if keep_torch:
            return out
        torch.cuda.current_stream().synchronize()
        _lib.check_errors()
        return {k: v.cpu().numpy() for k, v in out.items()}


class BootstrapNet(_NetBase):
    """networks_original.py:22-88."""

    def eval(self, image_pair, image2_2):
        b, f = self.batch_size, self._fmt
        ip, t1 = _to_dev(image_pair, _shape(f, b, 6, 192, 256), "image_pair")
        i2, t2 = _to_dev(image2_2, _shape(f, b, 3, 48, 64), "image2_2")
        net = self.session.net(b)
        out = self._outputs(ip.device)
        _lib.check(_lib.load().demon_bootstrap_forward(
            net.ptr, ip.data_ptr(), i2.data_ptr(), out["predict_flow5"].data_ptr(), out["predict_flow2"].data_ptr(),
            out["predict_depth2"].data_ptr(), out["predict_normal2"].data_ptr(), out["predict_rotation"].data_ptr(),
            out["predict_translation"].data_ptr(), f, _stream()))
        return self._finish(out, t1 and t2)


class IterativeNet(_NetBase):
    """networks_original.py:92-198.  The intrinsics are the constant of networks_original.py:108."""

    def eval(self, image_pair, image2_2, depth2, normal2, rotation, translation):
        b, f = self.batch_size, self._fmt
        ip, t1 = _to_dev(image_pair, _shape(f, b, 6, 192, 256), "image_pair")
        i2, t2 = _to_dev(image2_2, _shape(f, b, 3, 48, 64), "image2_2")
        d2, t3 = _to_dev(depth2, _shape(f, b, 1, 48, 64), "depth2")
        n2, t4 = _to_dev(normal2, _shape(f, b, 3, 48, 64), "normal2")
        r, t5 = _to_dev(rotation, (b, 3), "rotation")
        t, t6 = _to_dev(translation, (b, 3), "translation")
        net = self.session.net(b)
        out = self._outputs(ip.device)
        _lib.check(_lib.load().demon_iterative_forward(
            net.ptr, ip.data_ptr(), i2.data_ptr(), d2.data_ptr(), n2.data_ptr(), r.data_ptr(), t.data_ptr(),
            out["predict_flow5"].data_ptr(), out["predict_flow2"].data_ptr(), out["predict_depth2"].data_ptr(),
            out["predict_normal2"].data_ptr(), out["predict_rotation"].data_ptr(), out["predict_translation"].data_ptr(),
            f, _stream()))
        return self._finish(out, t1 and t2 and t3 and t4 and t5 and t6)   # torch out only if every input was a CUDA tensor


class RefinementNet(_NetBase):
    """networks_original.py:202-255.  `image_size` = (H, W) of image1; the reference fixes (192, 256),
    the block itself is size generic (blocks_original.py:466-475)."""

    def __init__(self, session, data_format="channels_first", batch_size=1, image_size=(192, 256)):
        super().__init__(session, data_format, batch_size)
        self.image_size = (int(image_size[0]), int(image_size[1]))
        if self.image_size[0] % 4 or self.image_size[1] % 4:
            raise ValueError("image_size must be a multiple of 4")

    def eval(self, image1, depth2):
        b, f = self.batch_size, self._fmt
        H, W = self.image_size
        im, t1 = _to_dev(image1, _shape(f, b, 3, H, W), "image1")
        d2, t2 = _to_dev(depth2, _shape(f, b, 1, H // 4, W // 4), "depth2")
        net = self.session.net(b, (H, W))
        out = {"predict_depth0": torch.empty(_shape(f, b, 1, H, W), dtype=torch.float32, device=im.device)}
        _lib.check(_lib.load().demon_refine_forward(net.ptr, im.data_ptr(), d2.data_ptr(), out["predict_depth0"].data_ptr(),
                                                    f, _stream()))
        return self._finish(out, t1 and t2)


class DemonPipeline:
    """examples/example.py:87-99 as one device-resident call (channels_first only)."""

    def __init__(self, session=None, batch_size=1, iterations=3, private_net=False):
        self.session = session if session is not None else default_session()
        self.batch_size = int(batch_size)
        self.iterations = int(iterations)
        # private_net: an own network handle (own workspace), so that two pipelines can be in flight on two streams
        self.net = (_NetHandle(self.session.weights, self.batch_size, (192, 256), self.session.precision) if private_net
                    else self.session.net(self.batch_size))
        # The C call replays ONE CUDA graph per set of pointer arguments, so the pipeline owns persistent input staging
        # and output buffers: the graph key is then the same for every call, whatever tensors the caller passes.
        self._ip = self._i22 = self._out = None
        self._snap = self._snap_refined = None
        self._K = self._status = None   # forward_views: intrinsics staging [B,2,4] float64 and status [B,2] uint8

    def stage(self, image_pair, image2_2=None):
        """Copies the inputs into the pipeline's own device buffers (asynchronous, current stream) and returns them."""
        b = self.batch_size
        ip, _ = _to_dev(image_pair, (b, 6, 192, 256), "image_pair")
        if self._ip is None:
            self._ip = torch.empty((b, 6, 192, 256), dtype=torch.float32, device=ip.device)
            self._i22 = torch.empty((b, 3, 48, 64), dtype=torch.float32, device=ip.device)
        if ip.data_ptr() != self._ip.data_ptr():
            self._ip.copy_(ip, non_blocking=True)
        i2 = None
        if image2_2 is not None:
            i2, _ = _to_dev(image2_2, (b, 3, 48, 64), "image2_2")
            if i2.data_ptr() != self._i22.data_ptr():
                self._i22.copy_(i2, non_blocking=True)
            i2 = self._i22
        return self._ip, i2

    def _own(self, attr, shapes):
        """The persistent float32 buffers `attr` of the pipeline (name -> shape), made on the first call."""
        if getattr(self, attr) is None:
            dev = self._ip.device if self._ip is not None else torch.device("cuda", torch.cuda.current_device())
            setattr(self, attr, {k: torch.empty(s, dtype=torch.float32, device=dev) for k, s in shapes.items()})
        return getattr(self, attr)

    def own_outputs(self):
        b = self.batch_size
        return self._own("_out", {"predict_depth0": (b, 1, 192, 256), "predict_rotation": (b, 3), "predict_translation": (b, 3),
                                  "predict_flow2": (b, 2, 48, 64), "predict_depth2": (b, 1, 48, 64), "predict_normal2": (b, 3, 48, 64)})

    def _run(self, entry, args, outputs=None, keys=_OUTPUTS):
        """Calls the C entry `entry` on the net with `args`, the iteration count, the pointers of `outputs` (default: the
        pipeline's own) in the order of `keys` (null for a missing one) and the current stream; raises on an error code."""
        if outputs is None:
            outputs = self.own_outputs()
        fn = getattr(_lib.load(), entry)
        _lib.check(fn(self.net.ptr, *args, self.iterations, *(_ptr(outputs.get(k)) for k in keys), _stream()))
        return outputs

    def forward(self, image_pair, image2_2=None, outputs=None, stage_inputs=True):
        """image_pair: torch CUDA [B,6,192,256]; image2_2: torch CUDA [B,3,48,64] or None (then it is
        median3x3_downsample applied twice to the second image, examples/evaluation.py:170-173).
        Returns dict of torch CUDA tensors; no host synchronisation.  With `outputs=None` the result tensors belong to
        the pipeline and are overwritten by the next call (clone them to keep them).  `stage_inputs=False` skips the
        device-to-device copy into the pipeline's own input buffers; pass the same tensors every call then, or every
        new pointer set costs an eager ~270-launch pass plus a graph capture."""
        b = self.batch_size
        if stage_inputs:
            ip, i2 = self.stage(image_pair, image2_2)
        else:
            ip, _ = _to_dev(image_pair, (b, 6, 192, 256), "image_pair")
            i2 = None
            if image2_2 is not None:
                i2, _ = _to_dev(image2_2, (b, 3, 48, 64), "image2_2")
        return self.forward_staged(outputs, ip, i2)

    def forward_staged(self, outputs=None, ip=None, i2=None, use_image2_2=False):
        """The pipeline on inputs that are already in place: by default the pipeline's own staging buffers (filled by
        `stage()`; image2_2 only if `use_image2_2`).  This is the part a caller captures in a CUDA graph of its own
        (bench.py captures it together with the all-gather that follows)."""
        if ip is None:
            if self._ip is None:
                raise RuntimeError("forward_staged() before stage()")
            ip, i2 = self._ip, (self._i22 if use_image2_2 else None)
        return self._run("demon_pipeline_forward", (ip.data_ptr(), _ptr(i2)), outputs)

    def own_snapshot_outputs(self, refine=True):
        """The persistent output buffers of forward_snapshots (S = iterations + 1 snapshots); one set per `refine`."""
        b, s = self.batch_size, self.iterations + 1
        shapes = {"predict_flow2": (s, b, 2, 48, 64), "predict_depth2": (s, b, 1, 48, 64), "predict_normal2": (s, b, 3, 48, 64),
                  "predict_rotation": (s, b, 3), "predict_translation": (s, b, 3)}
        if refine:
            shapes["predict_depth0"] = (s, b, 1, 192, 256)
        return self._own("_snap_refined" if refine else "_snap", shapes)

    def forward_snapshots(self, image_pair, image2_2=None, refine=True, outputs=None):
        """The pipeline keeping every intermediate prediction, as examples/evaluation.py:225-255 stores them: snapshot 0
        is the bootstrap net's output, snapshot k the output after iteration k.  Returns a dict of torch CUDA tensors
        [S, B, ...] with S = iterations + 1: predict_flow2 [S,B,2,48,64], predict_depth2 [S,B,1,48,64], predict_normal2
        [S,B,3,48,64], predict_rotation / predict_translation [S,B,3], and with `refine` predict_depth0 [S,B,1,192,256]
        (the refinement net on every snapshot's depth, evaluation.py:249).  Inputs are staged like forward(); with
        `outputs=None` the results are the pipeline's own buffers, overwritten by the next call."""
        ip, i2 = self.stage(image_pair, image2_2)
        if outputs is None:
            outputs = self.own_snapshot_outputs(refine)
        # without `refine` no depth0 pointer, which is what skips the refinement
        self._run("demon_pipeline_forward_snapshots", (ip.data_ptr(), _ptr(i2)),
                  outputs if refine else dict(outputs, predict_depth0=None), _SNAPSHOT_OUTPUTS)
        return outputs

    def snapshot_launches(self):
        return _lib.load().demon_net_snapshot_launches(self.net.ptr, self.iterations)

    def forward_u8(self, images, image2_2=None, outputs=None):
        """The pipeline on uint8 images (torch CUDA uint8): images [B,2,192,256,3] = image 1 and image 2 of every pair as
        PIL gives them (HWC RGB), image2_2 [B,48,64,3] or None (median3x3_downsample twice).  /255 - 0.5 and the pair
        concat run on the device (examples/example.py:15-42); same outputs as forward(), bit for bit."""
        b = self.batch_size
        if not (isinstance(images, torch.Tensor) and images.is_cuda and images.dtype == torch.uint8 and tuple(images.shape) == (b, 2, 192, 256, 3)):
            raise ValueError("images: expected a CUDA uint8 tensor of shape %s" % ((b, 2, 192, 256, 3),))
        if image2_2 is not None and not (isinstance(image2_2, torch.Tensor) and image2_2.is_cuda and image2_2.dtype == torch.uint8
                                          and tuple(image2_2.shape) == (b, 48, 64, 3)):
            raise ValueError("image2_2: expected a CUDA uint8 tensor of shape %s" % ((b, 48, 64, 3),))
        images = images.contiguous()
        if image2_2 is not None:
            image2_2 = image2_2.contiguous()
        return self._run("demon_pipeline_forward_u8", (images.data_ptr(), _ptr(image2_2)), outputs)

    def _check_pairs(self, images, resample, image2_2):
        """The checks of forward_images / forward_views; returns h, w, the resample code and the image2_2 mode."""
        from .images import check_images, resample_code
        code = resample_code(resample)
        if image2_2 not in ("resize", "median"):
            raise ValueError("image2_2 must be 'resize' or 'median', got %r" % (image2_2,))
        check_images(images, "images", 5)
        if tuple(images.shape[:2]) != (self.batch_size, 2):
            raise ValueError("images: expected shape (%d, 2, h, w, 3), got %s" % (self.batch_size, tuple(images.shape)))
        return images.shape[2], images.shape[3], code, 1 if image2_2 == "resize" else 0

    def forward_images(self, images, resample="bicubic", image2_2="resize", outputs=None):
        """The pipeline on image pairs of any size (examples/example.py:15-42 and :87-99 in one call): images CUDA uint8
        [B,2,h,w,3] (HWC RGB, pixel stride 3 and channel stride 1; a cropped view is read in place).  Both images are resized
        to 256x192 on the device exactly like PIL.Image.resize with `resample` ('nearest', 'bilinear', 'bicubic' or Pillow's
        enum value); image2_2 is 'resize' (the resized second image resized to 64x48 with the same filter, example.py:22) or
        'median' (median3x3_downsample twice, examples/evaluation.py:170-173).  Same outputs as forward_u8 on the resized
        bytes, bit for bit."""
        h, w, code, mode = self._check_pairs(images, resample, image2_2)
        return self._run("demon_pipeline_forward_images_u8", (images.data_ptr(), *images.stride()[:3], h, w, code, mode), outputs)

    def forward_views(self, images, intrinsics, resample="bicubic", image2_2="resize", outputs=None):
        """The pipeline on photos from any calibrated camera: images CUDA uint8 [B,2,h,w,3] as in forward_images, intrinsics
        [B,2,3,3] or [B,2,4] (fx, fy, cx, cy in pixels) or one [3,3] for all, from numpy, CPU or CUDA.  Every image is first
        adapted to the intrinsics DeMoN was trained for at 256x192 (images.adjust_intrinsics with its defaults, the step
        examples/example.py:51-61 asks for); image2_2 is then made from the adapted second image as in forward_images.  The
        intrinsics are copied into a buffer of the pipeline, so the call replays one CUDA graph for new values.  Returns the
        outputs of forward_u8 on the adapted bytes, bit for bit, plus 'status' CUDA uint8 [B,2] (adjust_intrinsics' status;
        host intrinsics are checked here instead: ValueError)."""
        from .images import _check_adjust_source, _device_intrinsics, demon_intrinsics, intrinsics4
        b = self.batch_size
        h, w, code, mode = self._check_pairs(images, resample, image2_2)
        _check_adjust_source(h, w, "images")
        k = _device_intrinsics(intrinsics, (b, 2), "intrinsics", w, h, intrinsics4(demon_intrinsics(), (), "K_new"), 256, 192,
                               images.device)
        if self._K is None:
            self._K = torch.empty((b, 2, 4), dtype=torch.float64, device=images.device)
            self._status = torch.empty((b, 2), dtype=torch.uint8, device=images.device)
        self._K.copy_(k, non_blocking=True)
        out = self._run("demon_pipeline_forward_views_u8",
                        (images.data_ptr(), *images.stride()[:3], h, w, self._K.data_ptr(), self._status.data_ptr(), code, mode), outputs)
        return dict(out, status=self._status)

    def forward_host_u8(self, images, image2_2, depth0, rotation, translation, stream=None, sync=True):
        """End to end from HOST uint8 images [B,2,192,256,3] (numpy or pinned torch CPU uint8): H2D of the bytes, the
        pipeline, D2H of depth0 / rotation / translation.  sync=False: asynchronous on `stream` like forward_host_async."""
        s = ctypes.c_void_p((stream or torch.cuda.current_stream()).cuda_stream)
        fn = _lib.load().demon_pipeline_forward_host_u8 if sync else _lib.load().demon_pipeline_forward_host_u8_async
        _lib.check(fn(self.net.ptr, _ptr(images), _ptr(image2_2), self.iterations, _ptr(depth0), _ptr(rotation), _ptr(translation), s))

    def forward_host(self, image_pair, image2_2, depth0, rotation, translation):
        """End-to-end call on HOST buffers (pinned torch CPU tensors or numpy arrays): H2D, pipeline, D2H and a
        stream synchronise inside the C call."""
        _lib.check(_lib.load().demon_pipeline_forward_host(
            self.net.ptr, _ptr(image_pair), _ptr(image2_2), self.iterations, _ptr(depth0), _ptr(rotation), _ptr(translation), _stream()))
        # (the C call synchronises and returns DEMON_E_STATE itself if a tensor-core pipeline wait timed out)

    def forward_host_async(self, image_pair, image2_2, depth0, rotation, translation, stream=None):
        """forward_host without the final synchronisation, on `stream` (a torch.cuda.Stream; default: current).  The host
        buffers must be pinned and are valid after `stream.synchronize()`.  Two DemonPipeline objects on two Sessions'
        nets and two streams overlap one batch's copies with the other's compute."""
        s = ctypes.c_void_p((stream or torch.cuda.current_stream()).cuda_stream)
        _lib.check(_lib.load().demon_pipeline_forward_host_async(
            self.net.ptr, _ptr(image_pair), _ptr(image2_2), self.iterations, _ptr(depth0), _ptr(rotation), _ptr(translation), s))

    def launches(self):
        return _lib.load().demon_net_pipeline_launches(self.net.ptr, self.iterations)
