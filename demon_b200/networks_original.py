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

    def __init__(self, weights, batch, refine_hw, precision):
        if not torch.cuda.is_available():
            raise RuntimeError("demon_b200 networks need a CUDA device (there is no CPU fallback)")
        lib = _lib.load()
        self._lib = lib
        self.ptr = ctypes.c_void_p()
        self.batch, self.refine_hw, self.precision = batch, refine_hw, precision
        _lib.check(lib.demon_net_create(ctypes.byref(self.ptr), batch, refine_hw[0], refine_hw[1], PRECISIONS[precision]))
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

    def __init__(self, precision=DEFAULT_PRECISION):
        if precision not in PRECISIONS:
            raise ValueError("precision must be one of %s" % sorted(PRECISIONS))
        self.precision = precision
        self.weights = None
        self._nets = {}

    def load_weights(self, weights):
        """weights: dict TF variable name -> numpy array in TF layout (see demon_b200.weights)."""
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
            self._nets[key] = _NetHandle(self.weights, key[0], key[1], self.precision)
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

    def own_outputs(self):
        if self._out is None:
            b = self.batch_size
            dev = self._ip.device if self._ip is not None else torch.device("cuda", torch.cuda.current_device())
            mk = lambda *s: torch.empty(s, dtype=torch.float32, device=dev)
            self._out = {"predict_depth0": mk(b, 1, 192, 256), "predict_rotation": mk(b, 3), "predict_translation": mk(b, 3),
                         "predict_flow2": mk(b, 2, 48, 64), "predict_depth2": mk(b, 1, 48, 64), "predict_normal2": mk(b, 3, 48, 64)}
        return self._out

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
        if outputs is None:
            outputs = self.own_outputs()
        ptr = lambda k: outputs[k].data_ptr() if outputs.get(k) is not None else None
        _lib.check(_lib.load().demon_pipeline_forward(
            self.net.ptr, ip.data_ptr(), None if i2 is None else i2.data_ptr(), self.iterations,
            ptr("predict_depth0"), ptr("predict_rotation"), ptr("predict_translation"),
            ptr("predict_flow2"), ptr("predict_depth2"), ptr("predict_normal2"), _stream()))
        return outputs

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
        if outputs is None:
            outputs = self.own_outputs()
        ptr = lambda k: outputs[k].data_ptr() if outputs.get(k) is not None else None
        _lib.check(_lib.load().demon_pipeline_forward_u8(
            self.net.ptr, images.data_ptr(), None if image2_2 is None else image2_2.data_ptr(), self.iterations,
            ptr("predict_depth0"), ptr("predict_rotation"), ptr("predict_translation"),
            ptr("predict_flow2"), ptr("predict_depth2"), ptr("predict_normal2"), _stream()))
        return outputs

    def forward_host_u8(self, images, image2_2, depth0, rotation, translation, stream=None, sync=True):
        """End to end from HOST uint8 images [B,2,192,256,3] (numpy or pinned torch CPU uint8): H2D of the bytes, the
        pipeline, D2H of depth0 / rotation / translation.  sync=False: asynchronous on `stream` like forward_host_async."""
        def hp(x):
            if x is None:
                return None
            return x.data_ptr() if isinstance(x, torch.Tensor) else x.ctypes.data
        s = ctypes.c_void_p((stream or torch.cuda.current_stream()).cuda_stream)
        fn = _lib.load().demon_pipeline_forward_host_u8 if sync else _lib.load().demon_pipeline_forward_host_u8_async
        _lib.check(fn(self.net.ptr, hp(images), hp(image2_2), self.iterations, hp(depth0), hp(rotation), hp(translation), s))

    def forward_host(self, image_pair, image2_2, depth0, rotation, translation):
        """End-to-end call on HOST buffers (pinned torch CPU tensors or numpy arrays): H2D, pipeline, D2H and a
        stream synchronise inside the C call."""
        def hp(x):
            if x is None:
                return None
            return x.data_ptr() if isinstance(x, torch.Tensor) else x.ctypes.data
        _lib.check(_lib.load().demon_pipeline_forward_host(
            self.net.ptr, hp(image_pair), hp(image2_2), self.iterations, hp(depth0), hp(rotation), hp(translation), _stream()))
        # (the C call synchronises and returns DEMON_E_STATE itself if a tensor-core pipeline wait timed out)

    def forward_host_async(self, image_pair, image2_2, depth0, rotation, translation, stream=None):
        """forward_host without the final synchronisation, on `stream` (a torch.cuda.Stream; default: current).  The host
        buffers must be pinned and are valid after `stream.synchronize()`.  Two DemonPipeline objects on two Sessions'
        nets and two streams overlap one batch's copies with the other's compute."""
        def hp(x):
            if x is None:
                return None
            return x.data_ptr() if isinstance(x, torch.Tensor) else x.ctypes.data
        s = ctypes.c_void_p((stream or torch.cuda.current_stream()).cuda_stream)
        _lib.check(_lib.load().demon_pipeline_forward_host_async(
            self.net.ptr, hp(image_pair), hp(image2_2), self.iterations, hp(depth0), hp(rotation), hp(translation), s))

    def launches(self):
        return _lib.load().demon_net_pipeline_launches(self.net.ptr, self.iterations)
