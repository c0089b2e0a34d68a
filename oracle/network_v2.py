"""ORACLE (test infrastructure) -- CPU restatement of the DeMoN v2 inference graphs (python/depthmotionnet/v2/blocks.py,
networks.py) with torch-CPU convolutions, in float32 or float64.

Same conventions as oracle/network.py, whose helpers it reuses: NCHW tensors, `force` (layer_name, x) -> y taps for the
layer trace, `ops` for the geometry ops between the blocks.  What differs from the original network:

  * every convolution is tf.layers.conv2d(padding='same') (v2/helpers.py:24-91): per axis out = ceil(in / s),
    pad_total = max((out - 1) s + k - in, 0), pad_before = pad_total // 2, the rest after (`conv2d_same`);
  * dense5 (v2/blocks.py:198-215): the first 96 channels of conv5_1, flattened NCHW, a 4608 -> 4608 dense layer with
    leaky ReLU, reshaped to [96, 6, 8] and concatenated after conv5_1;
  * the motion branch (v2/blocks.py:417-456) and the clip of depth_from_flow to [0, 50] (v2/blocks.py:379), restated as
    TF 1.4's clip_by_value computes it: minimum(x, 50) then maximum(., 0), so NaN stays NaN (`clip_by_value`);
  * the refinement block predicts depth0 and normal0 (v2/blocks.py:557-560).

No trained v2 weights are published, so the reference's graphs were never run on any; this file is pinned by its
restatement of the reference and by tests/test_v2_plan.py, which checks `conv2d_same` against a numpy loop written from
TensorFlow's documented 'SAME' definition.
"""
import numpy as np
import torch
import torch.nn.functional as F

from . import ops as oops
from .network import INTRINSICS, Weights, _np, _ops_dtype, _upconv, dense, my_leaky_relu


def same_pads(n, k, s):
    """(before, after) of tf.nn.conv2d padding='SAME' along one axis of size n."""
    out = -(-n // s)
    total = max((out - 1) * s + k - n, 0)
    return total // 2, total - total // 2


def conv2d_same(W, name, x, stride=(1, 1), activation=False, force=None):
    """tf.layers.conv2d(padding='same') (v2/helpers.py:24-43), leaky ReLU if `activation`."""
    if force is not None:
        return force(name, x)
    k, b = W.conv(name)
    sy, sx = stride
    py, px = same_pads(x.shape[2], k.shape[2], sy), same_pads(x.shape[3], k.shape[3], sx)
    y = F.conv2d(F.pad(x, (px[0], px[1], py[0], py[1])), k, b, stride=(sy, sx))
    return my_leaky_relu(y) if activation else y


def convrelu(W, name, x, stride=1, force=None):
    return conv2d_same(W, name, x, (stride, stride), activation=True, force=force)


def convrelu2(W, name, x, stride, force=None):
    """v2/helpers.py:46-91: (k x 1) conv strided in H, leaky, (1 x k) conv strided in W, leaky."""
    y = conv2d_same(W, name + "y", x, (stride, 1), activation=True, force=force)
    return conv2d_same(W, name + "x", y, (1, stride), activation=True, force=force)


def refine(W, scope, inp, features_direct, upsampled_prediction=None, force=None):
    """_refine, v2/blocks.py:80-116."""
    up = force(scope + "/upconv", inp) if force is not None else my_leaky_relu(_upconv(W, scope + "/upconv", inp))
    return torch.cat([up, features_direct] + ([upsampled_prediction] if upsampled_prediction is not None else []), dim=1)


def clip_by_value(x, lo, hi):
    """tf.clip_by_value of TF 1.4: maximum(minimum(x, hi), lo) with std::min / std::max compare order: NaN passes."""
    t = torch.where(x > hi, torch.full_like(x, hi), x)
    return torch.where(t < lo, torch.full_like(t, lo), t)


def dense5(W, s, conv5_1, force=None):
    """v2/blocks.py:198-215: conv5_1 ++ reshape(dense(flatten(conv5_1[:, :96])), [96, H, W])."""
    B, _, h, w = conv5_1.shape
    d = dense(W, s + "dense5", conv5_1[:, 0:96].reshape(B, -1), True, force=force)
    return torch.cat((conv5_1, d.reshape(B, 96, h, w)), dim=1)


def trunk(W, s, image_pair, extra_fn, flow, force=None):
    """The contracting part shared by the two blocks; `extra_fn(conv2)` returns conv2_1's input (conv2 ++ the extra inputs'
    convolution) or None for the bootstrap flow block."""
    f = force
    conv1 = convrelu2(W, s + "conv1", image_pair, 2, force=f)
    conv2 = convrelu2(W, s + "conv2", conv1, 2, force=f)
    cat = extra_fn(conv2)
    conv2_1 = convrelu2(W, s + "conv2_1", conv2 if cat is None else cat, 1, force=f)
    conv3 = convrelu2(W, s + "conv3", conv2_1, 2, force=f)
    conv3_1 = convrelu2(W, s + "conv3_1", conv3, 1, force=f)
    conv4 = convrelu2(W, s + "conv4", conv3_1, 2, force=f)
    conv4_1 = convrelu2(W, s + "conv4_1", conv4, 1, force=f)
    conv5 = convrelu2(W, s + "conv5", conv4_1, 2, force=f)
    conv5_1 = convrelu2(W, s + "conv5_1", conv5, 1, force=f)
    return conv2_1, conv3_1, conv4_1, conv5_1, dense5(W, s, conv5_1, force=f)


def flow_block(W, scope, image_pair, image2_2=None, prev=None, force=None, ops=oops):
    """flow_block, v2/blocks.py:120-253."""
    s = scope + "/"
    f = force
    extras = {}

    def extra_fn(conv2):
        if prev is None:
            return None
        npdt = _ops_dtype(image_pair)
        intr = np.broadcast_to(np.asarray([INTRINSICS], npdt), (image_pair.shape[0], 4))
        flow_dm = torch.from_numpy(ops.depth_to_flow(_np(prev["predict_depth2"]), intr, _np(prev["predict_rotation"]),
                                                     _np(prev["predict_translation"]), inverse_depth=True, normalize_flow=True))
        norm = torch.sqrt(flow_dm[:, 0:1] * flow_dm[:, 0:1] + flow_dm[:, 1:2] * flow_dm[:, 1:2])
        flow_dm = torch.where(norm < 1.0, flow_dm, torch.zeros_like(flow_dm))
        warped = torch.from_numpy(ops.warp2d(_np(image2_2), _np(flow_dm), normalized=True, border_mode="value"))
        extra = torch.cat((warped, flow_dm, prev["predict_depth2"], prev["predict_normal2"]), dim=1)
        extras.update({"flow_from_depth_motion": flow_dm, "image2_2_warped": warped})
        return torch.cat((conv2, convrelu2(W, s + "conv2_extra_inputs", extra, 1, force=f)), dim=1)

    conv2_1, conv3_1, conv4_1, conv5_1, c5d = trunk(W, s, image_pair, extra_fn, True, force=f)
    flowconf5 = conv2d_same(W, s + "predict_flow5/conv2", convrelu(W, s + "predict_flow5/conv1", c5d, force=f), force=f)
    flowconf5to4 = _upconv(W, s + "upsample_flow5to4/upconv", flowconf5, force=f)
    concat4 = refine(W, s + "refine4", c5d, conv4_1, flowconf5to4, force=f)
    concat3 = refine(W, s + "refine3", concat4, conv3_1, force=f)
    concat2 = refine(W, s + "refine2", concat3, conv2_1, force=f)
    flowconf2 = conv2d_same(W, s + "predict_flow2/conv2", convrelu(W, s + "predict_flow2/conv1", concat2, force=f), force=f)
    out = {"predict_flowconf5": flowconf5, "predict_flowconf2": flowconf2, "conv5_1_dense5": c5d}
    out.update(extras)
    return out


def depthmotion_block(W, scope, image_pair, image2_2, prev_flow2, prev_flowconf2, prev_rotation=None, prev_translation=None,
                      force=None, ops=oops):
    """depthmotion_block, v2/blocks.py:317-494.  Forced, predict_depth2 is predict_depthnormal2/conv2's forced output."""
    s = scope + "/"
    f = force
    dbg = {}

    def extra_fn(conv2):
        warped = torch.from_numpy(ops.warp2d(_np(image2_2), _np(prev_flow2), normalized=True, border_mode="value"))
        extra = [warped, prev_flowconf2]
        dbg["image2_2_warped"] = warped
        if prev_rotation is not None and prev_translation is not None:
            intr = np.broadcast_to(np.asarray([INTRINSICS], _ops_dtype(image_pair)), (image_pair.shape[0], 4))
            dff = torch.from_numpy(ops.flow_to_depth(_np(prev_flow2), intr, _np(prev_rotation), _np(prev_translation),
                                                     normalized_flow=True, inverse_depth=True, nowarning=True))
            dbg["depth_from_flow_unclipped"] = dff
            dff = clip_by_value(dff, 0.0, 50.0)
            extra.append(dff)
            dbg["depth_from_flow"] = dff
        return torch.cat((conv2, convrelu2(W, s + "conv2_extra_inputs", torch.cat(extra, dim=1), 1, force=f)), dim=1)

    conv2_1, conv3_1, conv4_1, conv5_1, c5d = trunk(W, s, image_pair, extra_fn, False, force=f)
    m3 = convrelu2(W, s + "motion_conv3", conv2_1, 2, force=f)
    m4 = convrelu2(W, s + "motion_conv4", m3, 2, force=f)
    m5a = convrelu2(W, s + "motion_conv5a", m4, 2, force=f)
    m5b = convrelu(W, s + "motion_conv5b", c5d, force=f)
    m51 = torch.cat((m5a, m5b), dim=1)
    fc1 = dense(W, s + "motion_fc1", m51.reshape(m51.shape[0], -1), True, force=f)
    fc2 = dense(W, s + "motion_fc2", fc1, True, force=f)
    motion = dense(W, s + "motion_fc3", fc2, False, force=f)
    rotation, translation, scale = motion[:, 0:3], motion[:, 3:6], motion[:, 6:7]
    concat4 = refine(W, s + "refine4", conv5_1, conv4_1, force=f)
    concat3 = refine(W, s + "refine3", concat4, conv3_1, force=f)
    concat2 = refine(W, s + "refine2", concat3, conv2_1, force=f)
    tmp2 = conv2d_same(W, s + "predict_depthnormal2/conv2", convrelu(W, s + "predict_depthnormal2/conv1", concat2, force=f), force=f)
    depth = scale.reshape(-1, 1, 1, 1) * tmp2[:, 0:1] if f is None else tmp2[:, 0:1]
    out = {"predict_depth2": depth, "predict_normal2": tmp2[:, 1:4], "predict_rotation": rotation.contiguous(),
           "predict_translation": translation.contiguous(), "predict_scale": scale.contiguous(), "motion_conv5_1": m51,
           "conv5_1_dense5": c5d}
    out.update(dbg)
    return out


def refine_block(W, scope, image1, depth2, force=None):
    """depth_refine_block, v2/blocks.py:499-560."""
    s = scope + "/"
    f = force
    H, Wd = image1.shape[-2:]
    h, w = depth2.shape[-2:]
    iy = torch.div(torch.arange(H) * h, H, rounding_mode="floor")
    ix = torch.div(torch.arange(Wd) * w, Wd, rounding_mode="floor")
    x = torch.cat((image1, depth2[:, :, iy][:, :, :, ix]), dim=1)
    conv0 = convrelu(W, s + "conv0", x, 1, force=f)
    conv1 = convrelu(W, s + "conv1", conv0, 2, force=f)
    conv1_1 = convrelu(W, s + "conv1_1", conv1, 1, force=f)
    conv2 = convrelu(W, s + "conv2", conv1_1, 2, force=f)
    conv2_1 = convrelu(W, s + "conv2_1", conv2, 1, force=f)
    concat1 = refine(W, s + "refine1", conv2_1, conv1_1, force=f)
    concat0 = refine(W, s + "refine0", concat1, conv0, force=f)
    tmp2 = conv2d_same(W, s + "predict_depth0/conv2", convrelu(W, s + "predict_depth0/conv1", concat0, force=f), force=f)
    return {"predict_depth0": tmp2[:, 0:1].contiguous(), "predict_normal0": tmp2[:, 1:4].contiguous()}


class OracleNetsV2:
    """CPU twin of v2's BootstrapNet / IterativeNet / RefinementNet (v2/networks.py)."""

    def __init__(self, tf_weights, dtype=torch.float32):
        self.dtype = dtype
        self.W = Weights(tf_weights, dtype)

    def _t(self, a):
        return torch.as_tensor(np.asarray(a)).to(self.dtype)

    @staticmethod
    def _outputs(f, d, full):
        fc2 = f["predict_flowconf2"]
        out = {"predict_flow5": f["predict_flowconf5"][:, 0:2], "predict_flow2": fc2[:, 0:2],
               "predict_depth2": d["predict_depth2"], "predict_normal2": d["predict_normal2"],
               "predict_rotation": d["predict_rotation"], "predict_translation": d["predict_translation"]}
        if full:
            out.update({k: v for k, v in f.items() if k not in out})
            out.update({k: v for k, v in d.items() if k not in out and k != "conv5_1_dense5"})
            out["flow_conv5_1_dense5"], out["dm_conv5_1_dense5"] = f["conv5_1_dense5"], d["conv5_1_dense5"]
        return {k: v.contiguous() for k, v in out.items()}

    @torch.no_grad()
    def bootstrap(self, image_pair, image2_2, full=False, force=None, ops=oops):
        image_pair, image2_2 = self._t(image_pair), self._t(image2_2)
        f = flow_block(self.W, "netFlow1", image_pair, force=force, ops=ops)
        fc2 = f["predict_flowconf2"]
        d = depthmotion_block(self.W, "netDM1", image_pair, image2_2, fc2[:, 0:2].contiguous(), fc2, force=force, ops=ops)
        return self._outputs(f, d, full)

    @torch.no_grad()
    def iterative(self, image_pair, image2_2, depth2, normal2, rotation, translation, full=False, force=None, ops=oops):
        image_pair, image2_2 = self._t(image_pair), self._t(image2_2)
        prev = {"predict_depth2": self._t(depth2), "predict_normal2": self._t(normal2),
                "predict_rotation": self._t(rotation), "predict_translation": self._t(translation)}
        f = flow_block(self.W, "netFlow2", image_pair, image2_2, prev, force=force, ops=ops)
        fc2 = f["predict_flowconf2"]
        d = depthmotion_block(self.W, "netDM2", image_pair, image2_2, fc2[:, 0:2].contiguous(), fc2,
                              prev["predict_rotation"], prev["predict_translation"], force=force, ops=ops)
        return self._outputs(f, d, full)

    @torch.no_grad()
    def refine(self, image1, depth2, normal2=None, force=None):
        """RefinementNet.eval(image1, depth2, normal2): normal2 is not used (v2/networks.py:204-228)."""
        return refine_block(self.W, "netRefine", self._t(image1), self._t(depth2), force=force)

    @torch.no_grad()
    def pipeline(self, image_pair, image2_2, iterations=3):
        """examples/example_v2.py: bootstrap, `iterations` x iterative, refinement."""
        r = self.bootstrap(image_pair, image2_2)
        for _ in range(iterations):
            r = self.iterative(image_pair, image2_2, r["predict_depth2"], r["predict_normal2"], r["predict_rotation"],
                               r["predict_translation"])
        out = dict(r)
        out.update(self.refine(self._t(image_pair)[:, 0:3].contiguous(), r["predict_depth2"], r["predict_normal2"]))
        return out
