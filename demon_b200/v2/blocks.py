"""Mirror of `depthmotionnet.v2.blocks` (python/depthmotionnet/v2/blocks.py) over the v2 plan in libdemon_b200.so: one block
at a time, under a variable scope of training/v2/training.py, on each sample's own camera.

    session = Session(); session.restore('training/training/checkpoints/snapshot-250000')
    flow1 = flow_block(image_pair, scope='netFlow1', session=session)
    dm1 = depthmotion_block(image_pair, image2_2, flow1['predict_flowconf2'][:, 0:2], flow1['predict_flowconf2'],
                            scope='netDM1', session=session)
    flow2 = flow_block(image_pair, image2_2, INTRINSICS, dm1, scope='netFlow2', session=session)   # training.py:329-335

Same function names, arguments and result keys as the reference.  `scope` selects the weights as tf.variable_scope does
in training.py ('netFlow1' / 'netFlow2', 'netDM1' / 'netDM2', 'netRefine'), and `session` is the v2 Session that holds
them (default: v2.networks.default_session()).  There is no `kernel_regularizer`: the regularisation is a function of the
checkpoint alone (Session.kernel_l2, v2.objective).  The iterative scopes need every previous prediction and the
intrinsics [B,4] (normalised fx, fy, cx, cy per sample, as datareader.build_batch's INTRINSICS); the bootstrap scopes take
none of them, because their weights have no conv2_extra_inputs for them.  A mismatch raises ValueError naming the argument.

Conventions as in v2.networks: numpy or torch in; numpy out, or torch CUDA out (asynchronous, current stream) when every
input is a torch CUDA tensor.  The batch size is the inputs' first dimension.
"""
import torch

from .. import _lib
from .. import networks_original as _v1
from . import networks as _nets

_stream, _to_dev, _shape = _v1._stream, _v1._to_dev, _v1._shape
_PREV = ("predict_depth2", "predict_normal2", "predict_rotation", "predict_translation")


def _session(session):
    return session if session is not None else _nets.default_session()


def _batch(x, name):
    if x is None or len(getattr(x, "shape", ())) < 1:
        raise ValueError("%s must be a batch of arrays" % name)
    return int(x.shape[0])


def _opt(x, shape, name):
    """(device tensor or None, whether x was a torch CUDA tensor or absent)"""
    if x is None:
        return None, True
    return _to_dev(x, shape, name)


def _empty(dev, *shape):
    return torch.empty(shape, dtype=torch.float32, device=dev)


def _ptr(t):
    return None if t is None else t.data_ptr()


def flow_block(image_pair, image2_2=None, intrinsics=None, prev_predictions=None, data_format='channels_first', scope='netFlow1',
               session=None):
    """flow_block (v2/blocks.py:120-253) -> {'predict_flowconf5': [B,4,6,8], 'predict_flowconf2': [B,4,48,64]}: flow x, y
    and confidence x, y.  prev_predictions: a dict with predict_depth2, predict_normal2, predict_rotation and
    predict_translation (netFlow2 only; e.g. depthmotion_block's result)."""
    f = _v1._check_format(data_format)
    b = _batch(image_pair, "image_pair")
    prev = {} if prev_predictions is None else prev_predictions
    missing = [k for k in _PREV if k not in prev] if prev_predictions is not None else []
    if missing:
        raise ValueError("flow_block: prev_predictions has no %s" % missing[0])
    ip, t0 = _to_dev(image_pair, _shape(f, b, 6, 192, 256), "image_pair")
    i2, t1 = _opt(image2_2, _shape(f, b, 3, 48, 64), "image2_2")
    k, t2 = _opt(intrinsics, (b, 4), "intrinsics")
    d2, t3 = _opt(prev.get("predict_depth2"), _shape(f, b, 1, 48, 64), "prev_predictions['predict_depth2']")
    n2, t4 = _opt(prev.get("predict_normal2"), _shape(f, b, 3, 48, 64), "prev_predictions['predict_normal2']")
    r, t5 = _opt(prev.get("predict_rotation"), (b, 3), "prev_predictions['predict_rotation']")
    t, t6 = _opt(prev.get("predict_translation"), (b, 3), "prev_predictions['predict_translation']")
    net = _session(session).net(b)
    out = {"predict_flowconf5": _empty(ip.device, *_shape(f, b, 4, 6, 8)),
           "predict_flowconf2": _empty(ip.device, *_shape(f, b, 4, 48, 64))}
    _lib.check(_lib.load().demon_flow_block_forward_v2(
        net.ptr, str(scope).encode(), ip.data_ptr(), _ptr(i2), _ptr(k), _ptr(d2), _ptr(n2), _ptr(r), _ptr(t),
        out["predict_flowconf5"].data_ptr(), out["predict_flowconf2"].data_ptr(), f, _stream()))
    return _v1._NetBase._finish(out, t0 and t1 and t2 and t3 and t4 and t5 and t6)


def depthmotion_block(image_pair, image2_2, prev_flow2, prev_flowconf2, prev_rotation=None, prev_translation=None, intrinsics=None,
                      data_format='channels_first', scope='netDM1', session=None):
    """depthmotion_block (v2/blocks.py:317-494) -> predict_depth2 [B,1,48,64], predict_normal2 [B,3,48,64],
    predict_rotation [B,3], predict_translation [B,3] and predict_scale [B,1].  prev_flow2 [B,2,48,64] is the flow the
    extra inputs warp with (and netDM2 turns into depth), prev_flowconf2 [B,4,48,64] the flow block's full output."""
    f = _v1._check_format(data_format)
    b = _batch(image_pair, "image_pair")
    ip, t0 = _to_dev(image_pair, _shape(f, b, 6, 192, 256), "image_pair")
    i2, t1 = _to_dev(image2_2, _shape(f, b, 3, 48, 64), "image2_2")
    fl, t2 = _to_dev(prev_flow2, _shape(f, b, 2, 48, 64), "prev_flow2")
    fc, t3 = _to_dev(prev_flowconf2, _shape(f, b, 4, 48, 64), "prev_flowconf2")
    r, t4 = _opt(prev_rotation, (b, 3), "prev_rotation")
    t, t5 = _opt(prev_translation, (b, 3), "prev_translation")
    k, t6 = _opt(intrinsics, (b, 4), "intrinsics")
    net = _session(session).net(b)
    dev = ip.device
    out = {"predict_depth2": _empty(dev, *_shape(f, b, 1, 48, 64)), "predict_normal2": _empty(dev, *_shape(f, b, 3, 48, 64)),
           "predict_rotation": _empty(dev, b, 3), "predict_translation": _empty(dev, b, 3), "predict_scale": _empty(dev, b, 1)}
    _lib.check(_lib.load().demon_depthmotion_block_forward_v2(
        net.ptr, str(scope).encode(), ip.data_ptr(), i2.data_ptr(), fl.data_ptr(), fc.data_ptr(), _ptr(r), _ptr(t), _ptr(k),
        *(out[key].data_ptr() for key in ("predict_depth2", "predict_normal2", "predict_rotation", "predict_translation",
                                          "predict_scale")), f, _stream()))
    return _v1._NetBase._finish(out, t0 and t1 and t2 and t3 and t4 and t5 and t6)


def depth_refine_block(image1, depthmotion_predictions, data_format='channels_first', scope='netRefine', session=None):
    """depth_refine_block (v2/blocks.py:499-560): image1 [B,3,H,W] (H, W multiples of 4) and depthmotion_predictions'
    predict_depth2 [B,1,H/4,W/4] -> predict_depth0 [B,1,H,W] and predict_normal0 [B,3,H,W]."""
    if scope != "netRefine":
        raise ValueError("depth_refine_block: scope must be netRefine, got %r" % (scope,))
    if "predict_depth2" not in depthmotion_predictions:
        raise ValueError("depth_refine_block: depthmotion_predictions has no predict_depth2")
    f = _v1._check_format(data_format)
    b = _batch(image1, "image1")
    H, W = (int(image1.shape[2]), int(image1.shape[3])) if f == 0 else (int(image1.shape[1]), int(image1.shape[2]))
    if H % 4 or W % 4:
        raise ValueError("depth_refine_block: image1 must be a multiple of 4 in height and width, got %dx%d" % (H, W))
    im, t0 = _to_dev(image1, _shape(f, b, 3, H, W), "image1")
    d2, t1 = _to_dev(depthmotion_predictions["predict_depth2"], _shape(f, b, 1, H // 4, W // 4),
                     "depthmotion_predictions['predict_depth2']")
    net = _session(session).net(b, (H, W))
    out = {"predict_depth0": _empty(im.device, *_shape(f, b, 1, H, W)), "predict_normal0": _empty(im.device, *_shape(f, b, 3, H, W))}
    _lib.check(_lib.load().demon_refine_forward_v2(net.ptr, im.data_ptr(), d2.data_ptr(), None, out["predict_depth0"].data_ptr(),
                                                   out["predict_normal0"].data_ptr(), f, _stream()))
    return _v1._NetBase._finish(out, t0 and t1)
