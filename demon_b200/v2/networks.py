"""Mirror of `depthmotionnet.v2.networks` (python/depthmotionnet/v2/networks.py) over the v2 plan in libdemon_b200.so.

    session = Session(); session.restore('checkpoints/snapshot-250000')   # a checkpoint of training/v2/training.py
    bootstrap_net = BootstrapNet(session)
    iterative_net = IterativeNet(session)
    refine_net = RefinementNet(session)
    result = bootstrap_net.eval(image_pair, image2_2)                  # examples/example_v2.py
    ...

Same class names, constructor and `eval` arguments and result-dict keys as the reference, and the same conventions as
demon_b200.networks_original (numpy or torch in; numpy out, or torch CUDA out when every input was a torch CUDA tensor;
`data_format` and `batch_size` as extensions).  `DemonPipelineV2` is bootstrap -> N x iterative -> refinement in one call
that never leaves the device.
"""
import ctypes

import numpy as np
import torch

from .. import _lib
from .. import networks_original as _v1
from .._lib import check_errors  # noqa: F401  (re-exported like networks_original.check_errors)
from . import weights as W

PRECISIONS = _v1.PRECISIONS
_stream, _to_dev, _shape, _ptr = _v1._stream, _v1._to_dev, _v1._shape, _v1._ptr


class _NetHandleV2(_v1._NetHandle):
    _create = "demon_net_create_v2"


class Session(_v1.Session):
    """Owner of the v2 variables, in place of the reference's tf.Session.  `restore` reads a TensorFlow checkpoint of the
    v2 graph (e.g. one written by training/v2/training.py); `load_weights` takes a dict of TF-named arrays."""

    _handle = _NetHandleV2

    def load_weights(self, weights):
        super().load_weights(weights)
        self._kernel_l2 = None

    def kernel_l2(self):
        """v2.weights.kernel_l2 of the loaded weights, computed once per load_weights (v2.objective's regularisation)."""
        if self.weights is None:
            raise RuntimeError("Session.load_weights() has not been called")
        if getattr(self, "_kernel_l2", None) is None:
            self._kernel_l2 = W.kernel_l2(self.weights)
        return self._kernel_l2

    def restore(self, save_path):
        if isinstance(save_path, dict):
            return self.load_weights(save_path)
        from .. import checkpoint
        specs = W.variable_specs()
        got = checkpoint.load_checkpoint(str(save_path), names=list(specs))
        for name, (_, shape) in specs.items():
            if tuple(got[name].shape) != tuple(shape):
                raise ValueError("checkpoint variable %s has shape %s, the v2 graph needs %s" % (name, got[name].shape, shape))
            got[name] = np.ascontiguousarray(got[name], dtype=np.float32)
        self.load_weights(got)


_default_session = None


def default_session():
    global _default_session
    if _default_session is None:
        _default_session = Session()
    return _default_session


class _NetBase(_v1._NetBase):
    def __init__(self, session, data_format="channels_first", batch_size=1):
        super().__init__(session if session is not None else default_session(), data_format, batch_size)


class BootstrapNet(_NetBase):
    """v2/networks.py:20-75."""

    def eval(self, image_pair, image2_2):
        b, f = self.batch_size, self._fmt
        ip, t1 = _to_dev(image_pair, _shape(f, b, 6, 192, 256), "image_pair")
        i2, t2 = _to_dev(image2_2, _shape(f, b, 3, 48, 64), "image2_2")
        net = self.session.net(b)
        out = self._outputs(ip.device)
        _lib.check(_lib.load().demon_bootstrap_forward_v2(
            net.ptr, ip.data_ptr(), i2.data_ptr(), *(out[k].data_ptr() for k in _STAGE_OUTPUTS), f, _stream()))
        return self._finish(out, t1 and t2)


class IterativeNet(_NetBase):
    """v2/networks.py:80-172.  The intrinsics are the constant of v2/networks.py:90."""

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
        _lib.check(_lib.load().demon_iterative_forward_v2(
            net.ptr, ip.data_ptr(), i2.data_ptr(), d2.data_ptr(), n2.data_ptr(), r.data_ptr(), t.data_ptr(),
            *(out[k].data_ptr() for k in _STAGE_OUTPUTS), f, _stream()))
        return self._finish(out, t1 and t2 and t3 and t4 and t5 and t6)


class RefinementNet(_NetBase):
    """v2/networks.py:177-228: eval(image1, depth2, normal2) -> predict_depth0, predict_normal0.  normal2 is taken and
    not used, as by the reference.  `image_size` as in networks_original.RefinementNet (a multiple of 4)."""

    def __init__(self, session, data_format="channels_first", batch_size=1, image_size=(192, 256)):
        super().__init__(session, data_format, batch_size)
        self.image_size = (int(image_size[0]), int(image_size[1]))
        if self.image_size[0] % 4 or self.image_size[1] % 4:
            raise ValueError("image_size must be a multiple of 4")

    def eval(self, image1, depth2, normal2):
        b, f = self.batch_size, self._fmt
        H, W_ = self.image_size
        im, t1 = _to_dev(image1, _shape(f, b, 3, H, W_), "image1")
        d2, t2 = _to_dev(depth2, _shape(f, b, 1, H // 4, W_ // 4), "depth2")
        net = self.session.net(b, (H, W_))
        out = {"predict_depth0": torch.empty(_shape(f, b, 1, H, W_), dtype=torch.float32, device=im.device),
               "predict_normal0": torch.empty(_shape(f, b, 3, H, W_), dtype=torch.float32, device=im.device)}
        _lib.check(_lib.load().demon_refine_forward_v2(net.ptr, im.data_ptr(), d2.data_ptr(), None, out["predict_depth0"].data_ptr(),
                                                       out["predict_normal0"].data_ptr(), f, _stream()))
        return self._finish(out, t1 and t2)


# output pointers of the stage-wise entries and of demon_pipeline_forward_v2, in C ABI order
_STAGE_OUTPUTS = ("predict_flow5", "predict_flow2", "predict_depth2", "predict_normal2", "predict_rotation", "predict_translation")
_OUTPUTS = ("predict_depth0", "predict_normal0", "predict_rotation", "predict_translation", "predict_flow2", "predict_depth2",
            "predict_normal2")


class DemonPipelineV2(_v1._Pipeline):
    """examples/example_v2.py's bootstrap -> iterations -> refinement as one device-resident call (channels_first), with
    every method of networks_original.DemonPipeline (stage, forward_staged, forward_snapshots, forward_u8, forward_images,
    forward_views, the host entries) and v2's outputs: predict_normal0 [B,3,192,256] comes with predict_depth0 wherever the
    refinement block runs.  Like DemonPipeline it owns its input staging and output buffers, so every call replays one CUDA
    graph.

    image2_2 may also be 'area': tf.image.resize_area of the second image to 48x64 (images.resize_area), the input
    training/v2/training.py:179 trains v2 on.  forward / forward_snapshots stage it with images.resize_area, the uint8,
    images, views and host entries compute it inside the pipeline from image 2's float planes (x/255 - 0.5 for uint8)."""

    _handle = _NetHandleV2
    _suffix = "_v2"
    _keys = _snapshot_keys = _OUTPUTS
    _host_keys = ("predict_depth0", "predict_normal0", "predict_rotation", "predict_translation")
    _modes = {"resize": 1, "median": 0, "area": 2}
    _area = True

    def __init__(self, session=None, batch_size=1, iterations=3, private_net=False):
        super().__init__(session if session is not None else default_session(), batch_size, iterations, private_net)

    def _mode_args(self, mode):
        return (mode,)

    def _output_shapes(self):
        return dict(super()._output_shapes(), predict_normal0=(self.batch_size, 3, 192, 256))

    def own_outputs(self, device=None):
        return self._own("_out", self._output_shapes(), device)

    def forward(self, image_pair, image2_2=None, iterations=None, outputs=None, stage_inputs=True):
        """image_pair [B,6,192,256], image2_2 [B,3,48,64], None (median3x3_downsample twice of the second image) or 'area';
        torch CUDA tensors or host arrays.  Returns a dict of torch CUDA tensors: predict_depth0, predict_normal0,
        predict_flow2, predict_depth2, predict_normal2, predict_rotation, predict_translation; no host synchronisation.
        With `outputs=None` they belong to the pipeline and are overwritten by the next call.  `stage_inputs` as in
        DemonPipeline.forward."""
        return self._forward(image_pair, image2_2, outputs, stage_inputs, iterations)

    def forward_host_u8(self, images, image2_2, depth0, rotation, translation, stream=None, sync=True, normal0=None):
        """DemonPipeline.forward_host_u8 with v2's optional normal0 [B,3,192,256] host buffer; image2_2 may be 'area'."""
        self._host("demon_pipeline_forward_host_u8" if sync else "demon_pipeline_forward_host_u8_async", images, image2_2,
                   {"predict_depth0": depth0, "predict_normal0": normal0, "predict_rotation": rotation, "predict_translation": translation},
                   stream)

    def forward_host(self, image_pair, image2_2, depth0, rotation, translation, normal0=None):
        """DemonPipeline.forward_host with v2's optional normal0 [B,3,192,256] host buffer; image2_2 may be 'area'."""
        self._host("demon_pipeline_forward_host", image_pair, image2_2,
                   {"predict_depth0": depth0, "predict_normal0": normal0, "predict_rotation": rotation, "predict_translation": translation},
                   None)

    def forward_host_async(self, image_pair, image2_2, depth0, rotation, translation, stream=None, normal0=None):
        """DemonPipeline.forward_host_async with v2's optional normal0 [B,3,192,256] host buffer; image2_2 may be 'area'."""
        self._host("demon_pipeline_forward_host_async", image_pair, image2_2,
                   {"predict_depth0": depth0, "predict_normal0": normal0, "predict_rotation": rotation, "predict_translation": translation},
                   stream)

    def launches(self, iterations=None):
        return _lib.load().demon_net_pipeline_launches(self.net.ptr, self.iterations if iterations is None else int(iterations))
