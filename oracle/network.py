"""ORACLE (test infrastructure) -- CPU restatement of the DeMoN
`networks_original` inference graphs with torch-CPU convolutions.

PARITY UNPINNED at the network level: the reference holds no test, golden
output or checkpoint for its TensorFlow graphs (SURVEY.md section 8c), and
TensorFlow 1.4 cannot be installed here.  What pins this file is (a) the
line-by-line restatement below, every function citing the reference, and (b)
tests/test_oracle_network.py (test_*_matches_tf_definition), which checks the torch calls used here against naive numpy loops
written directly from TensorFlow's documented definitions of conv2d /
conv2d_transpose / dense / resize_nearest_neighbor.  The geometry ops this
file threads between the blocks (oracle/ops.py) ARE pinned: bit for bit against
the reference's own sources compiled here (oracle/ref.py, tests/test_oracle_ref.py).

All tensors are NCHW (the reference's `channels_first` graph; the
`channels_last` graph is the same arithmetic behind transposes,
blocks_original.py:150-179,335-360,466-482).  `dtype` float32 is the timed
"reference CPU path", float64 is the truth both it and the CUDA path are
measured against.

Forcing (tests/test_gpu_layer_trace.py): every block function and OracleNets entry takes `force`, a callable
(layer_name, x) -> y that every conv, transposed conv and dense layer calls instead of computing its own output (after
its activation, if it has one).  `x` is the input the oracle built from the layers before, in the reference's own order:
its concats, nearest-neighbour upsampling, NCHW flatten and the geometry ops between the blocks.  `ops` is the module
those geometry ops come from (default oracle.ops).  With both at their defaults nothing changes.

Only tests/, __graft_entry__.smoke() and bench.py's CPU legs may import this.
"""
import numpy as np
import torch
import torch.nn.functional as F

from . import ops as oops

# IterativeNet hard-wires these normalized intrinsics (networks_original.py:108)
INTRINSICS = (0.89115971, 1.18821287, 0.5, 0.5)


class Weights:
    """Name -> torch tensor view of a TF-layout weight dict, converted lazily
    to the layouts torch wants (SURVEY.md appendix A.2)."""

    def __init__(self, tf_weights, dtype=torch.float32):
        self.w = tf_weights
        self.dtype = dtype
        self._cache = {}

    def conv(self, name):  # [kh,kw,cin,cout] -> [cout,cin,kh,kw]
        if name not in self._cache:
            k = torch.from_numpy(np.ascontiguousarray(self.w[name + "/kernel"])).to(self.dtype)
            self._cache[name] = (k.permute(3, 2, 0, 1).contiguous(),
                                 torch.from_numpy(self.w[name + "/bias"]).to(self.dtype))
        return self._cache[name]

    def deconv(self, name):  # [kh,kw,cout,cin] -> [cin,cout,kh,kw]
        if name not in self._cache:
            k = torch.from_numpy(np.ascontiguousarray(self.w[name + "/kernel"])).to(self.dtype)
            self._cache[name] = (k.permute(3, 2, 0, 1).contiguous(),
                                 torch.from_numpy(self.w[name + "/bias"]).to(self.dtype))
        return self._cache[name]

    def dense(self, name):  # [in,out]
        if name not in self._cache:
            self._cache[name] = (torch.from_numpy(self.w[name + "/kernel"]).to(self.dtype),
                                 torch.from_numpy(self.w[name + "/bias"]).to(self.dtype))
        return self._cache[name]


def my_leaky_relu(x):
    """helpers.py:60-63 -> sops.leaky_relu(x, leak=0.1) = max(0.1f*x, x) (leakyrelu.cc:79).
    The leak is a float attr converted to T (leakyrelu.cc:55-59)."""
    leak = torch.tensor(np.float32(0.1), dtype=x.dtype)
    return torch.maximum(leak * x, x)


def conv2d_caffe_padding(W, name, x, stride=1, activation=False, force=None):
    """helpers.py:70-94: explicit zero tf.pad of k//2, then VALID conv, bias on."""
    if force is not None:
        return force(name, x)
    k, b = W.conv(name)
    kh, kw = k.shape[2], k.shape[3]
    x = F.pad(x, (kw // 2, kw // 2, kh // 2, kh // 2))
    y = F.conv2d(x, k, b, stride=stride)
    return my_leaky_relu(y) if activation else y


def convrelu_caffe_padding(W, name, x, stride=1, force=None):
    """helpers.py:97-102."""
    return conv2d_caffe_padding(W, name, x, stride, activation=True, force=force)


def convrelu2_caffe_padding(W, name, x, stride, force=None):
    """helpers.py:105-153: (k x 1) conv strided in H, leaky, (1 x k) conv strided in W, leaky."""
    if force is not None:
        return force(name + "x", force(name + "y", x))
    ky, by = W.conv(name + "y")
    kx, bx = W.conv(name + "x")
    pad = ky.shape[2] // 2
    t = my_leaky_relu(F.conv2d(F.pad(x, (0, 0, pad, pad)), ky, by, stride=(stride, 1)))
    return my_leaky_relu(F.conv2d(F.pad(t, (pad, pad, 0, 0)), kx, bx, stride=(1, stride)))


def _upconv(W, name, x, force=None):
    """conv2d_transpose k4 s2 VALID then slice [1:1+2n] (blocks_original.py:97-110), and
    'same' (blocks_original.py:64-74): both are torch's ConvTranspose2d(k=4,s=2,p=1)."""
    if force is not None:
        return force(name, x)
    k, b = W.deconv(name)
    return F.conv_transpose2d(x, k, b, stride=2, padding=1)


def refine_caffe_padding(W, scope, inp, features_direct, upsampled_prediction=None, force=None):
    """blocks_original.py:79-117; concat order [upsampled_features, features_direct, upsampled_prediction]."""
    up = force(scope + "/upconv", inp) if force is not None else my_leaky_relu(_upconv(W, scope + "/upconv", inp))
    parts = [up, features_direct] + ([upsampled_prediction] if upsampled_prediction is not None else [])
    return torch.cat(parts, dim=1)


def dense(W, name, x, activation, force=None):
    """tf.layers.dense (blocks_original.py:390-410): x @ kernel + bias, leaky ReLU if `activation`."""
    if force is not None:
        return force(name, x)
    k, b = W.dense(name)
    y = x @ k + b
    return my_leaky_relu(y) if activation else y


def _np(t):
    return t.detach().numpy()


def _ops_dtype(t):
    return np.float64 if t.dtype == torch.float64 else np.float32


def flow_block(W, scope, image_pair, image2_2=None, prev=None, force=None, ops=oops):
    """flow_block_demon_original, blocks_original.py:121-235."""
    s = scope + "/"
    f = force
    conv1 = convrelu2_caffe_padding(W, s + "conv1", image_pair, 2, force=f)
    extras = {}
    if prev is None:
        conv2 = convrelu2_caffe_padding(W, s + "conv2", conv1, 2, force=f)
        conv2_1 = convrelu2_caffe_padding(W, s + "conv2_1", conv2, 1, force=f)
    else:
        conv2 = convrelu2_caffe_padding(W, s + "conv2", conv1, 2, force=f)
        npdt = _ops_dtype(image_pair)
        B = image_pair.shape[0]
        intr = np.broadcast_to(np.asarray([INTRINSICS], npdt), (B, 4))
        flow_dm = ops.depth_to_flow(_np(prev["predict_depth2"]), intr, _np(prev["predict_rotation"]),
                                    _np(prev["predict_translation"]), inverse_depth=True, normalize_flow=True)
        flow_dm = torch.from_numpy(flow_dm)
        # tf.norm(axis=1) then where(norm < 1, flow, 0)   (blocks_original.py:165-168)
        norm = torch.sqrt(flow_dm[:, 0:1] * flow_dm[:, 0:1] + flow_dm[:, 1:2] * flow_dm[:, 1:2])
        flow_dm = torch.where(norm < 1.0, flow_dm, torch.zeros_like(flow_dm))
        warped = torch.from_numpy(ops.warp2d(_np(image2_2), _np(flow_dm), normalized=True, border_mode="value"))
        extra = torch.cat((warped, flow_dm, prev["predict_depth2"], prev["predict_normal2"]), dim=1)
        conv_extra = convrelu2_caffe_padding(W, s + "conv2_extra_inputs", extra, 1, force=f)
        conv2_1 = convrelu2_caffe_padding(W, s + "conv2_1", torch.cat((conv2, conv_extra), dim=1), 1, force=f)
        extras = {"flow_from_depth_motion": flow_dm, "image2_2_warped": warped}
    conv3 = convrelu2_caffe_padding(W, s + "conv3", conv2_1, 2, force=f)
    conv3_1 = convrelu2_caffe_padding(W, s + "conv3_1", conv3, 1, force=f)
    conv4 = convrelu2_caffe_padding(W, s + "conv4", conv3_1, 2, force=f)
    conv4_1 = convrelu2_caffe_padding(W, s + "conv4_1", conv4, 1, force=f)
    conv5 = convrelu2_caffe_padding(W, s + "conv5", conv4_1, 2, force=f)
    conv5_1 = convrelu2_caffe_padding(W, s + "conv5_1", conv5, 1, force=f)

    def predict_flow(prefix, x):  # _predict_flow_caffe_padding, blocks_original.py:23-51
        return conv2d_caffe_padding(W, prefix + "/conv2", convrelu_caffe_padding(W, prefix + "/conv1", x, force=f), force=f)

    flowconf5 = predict_flow(s + "predict_flow5", conv5_1)
    flowconf5to4 = _upconv(W, s + "upsample_flow5to4/upconv", flowconf5, force=f)  # no activation (blocks_original.py:70)
    concat4 = refine_caffe_padding(W, s + "refine4", conv5_1, conv4_1, flowconf5to4, force=f)
    concat3 = refine_caffe_padding(W, s + "refine3", concat4, conv3_1, force=f)
    concat2 = refine_caffe_padding(W, s + "refine2", concat3, conv2_1, force=f)
    flowconf2 = predict_flow(s + "predict_flow2", concat2)
    out = {"predict_flowconf5": flowconf5, "predict_flowconf2": flowconf2, "conv1": conv1, "conv5_1": conv5_1}
    out.update(extras)
    return out


def depthmotion_block(W, scope, image_pair, image2_2, prev_flow2, prev_flowconf2,
                      prev_rotation=None, prev_translation=None, force=None, ops=oops):
    """depthmotion_block_demon_original, blocks_original.py:299-448.  Forced, predict_depth2 is the forced output of
    predict_depthnormal2/conv2 itself: the layer that computes it includes the scale."""
    s = scope + "/"
    f = force
    conv1 = convrelu2_caffe_padding(W, s + "conv1", image_pair, 2, force=f)
    conv2 = convrelu2_caffe_padding(W, s + "conv2", conv1, 2, force=f)
    warped = torch.from_numpy(ops.warp2d(_np(image2_2), _np(prev_flow2), normalized=True, border_mode="value"))
    extra = [warped, prev_flowconf2]
    dbg = {"image2_2_warped": warped}
    if prev_rotation is not None and prev_translation is not None:
        npdt = _ops_dtype(image_pair)
        intr = np.broadcast_to(np.asarray([INTRINSICS], npdt), (image_pair.shape[0], 4))
        dff = ops.flow_to_depth(_np(prev_flow2), intr, _np(prev_rotation), _np(prev_translation),
                                normalized_flow=True, inverse_depth=True, nowarning=True)
        dff = torch.from_numpy(dff)
        extra.append(dff)
        dbg["depth_from_flow"] = dff
    conv_extra = convrelu2_caffe_padding(W, s + "conv2_extra_inputs", torch.cat(extra, dim=1), 1, force=f)
    conv2_1 = convrelu2_caffe_padding(W, s + "conv2_1", torch.cat((conv2, conv_extra), dim=1), 1, force=f)
    conv3 = convrelu2_caffe_padding(W, s + "conv3", conv2_1, 2, force=f)
    conv3_1 = convrelu2_caffe_padding(W, s + "conv3_1", conv3, 1, force=f)
    conv4 = convrelu2_caffe_padding(W, s + "conv4", conv3_1, 2, force=f)
    conv4_1 = convrelu2_caffe_padding(W, s + "conv4_1", conv4, 1, force=f)
    conv5 = convrelu2_caffe_padding(W, s + "conv5", conv4_1, 2, force=f)
    conv5_1 = convrelu2_caffe_padding(W, s + "conv5_1", conv5, 1, force=f)

    motion_conv1 = convrelu_caffe_padding(W, s + "motion_conv1", conv5_1, force=f)
    flat = motion_conv1.reshape(motion_conv1.shape[0], -1)  # NCHW flatten (blocks_original.py:388-392)
    fc1 = dense(W, s + "motion_fc1", flat, True, force=f)
    fc2 = dense(W, s + "motion_fc2", fc1, True, force=f)
    motion = dense(W, s + "motion_fc3", fc2, False, force=f)
    rotation, translation, scale = motion[:, 0:3], motion[:, 3:6], motion[:, 6:7]

    concat4 = refine_caffe_padding(W, s + "refine4", conv5_1, conv4_1, force=f)
    concat3 = refine_caffe_padding(W, s + "refine3", concat4, conv3_1, force=f)
    concat2 = refine_caffe_padding(W, s + "refine2", concat3, conv2_1, force=f)
    # _predict_depthnormal_caffe_padding, blocks_original.py:238-294
    tmp = convrelu_caffe_padding(W, s + "predict_depthnormal2/conv1", concat2, force=f)
    tmp2 = conv2d_caffe_padding(W, s + "predict_depthnormal2/conv2", tmp, force=f)
    depth = scale.reshape(-1, 1, 1, 1) * tmp2[:, 0:1] if f is None else tmp2[:, 0:1]
    normal = tmp2[:, 1:4]
    out = {"predict_depth2": depth, "predict_normal2": normal, "predict_rotation": rotation.contiguous(),
           "predict_translation": translation.contiguous(), "predict_scale": scale.contiguous()}
    out.update(dbg)
    return out


def refine_block(W, scope, image1, depth2, force=None):
    """depth_refine_block_demon_original, blocks_original.py:452-513."""
    s = scope + "/"
    f = force
    H, Wd = image1.shape[-2:]
    h, w = depth2.shape[-2:]
    # tf.image.resize_nearest_neighbor(align_corners=False): src = floor(dst * in / out)
    iy = torch.div(torch.arange(H) * h, H, rounding_mode="floor")
    ix = torch.div(torch.arange(Wd) * w, Wd, rounding_mode="floor")
    up = depth2[:, :, iy][:, :, :, ix]
    x = torch.cat((image1, up), dim=1)
    conv0 = convrelu_caffe_padding(W, s + "conv0", x, 1, force=f)
    conv1 = convrelu_caffe_padding(W, s + "conv1", conv0, 2, force=f)
    conv1_1 = convrelu_caffe_padding(W, s + "conv1_1", conv1, 1, force=f)
    conv2 = convrelu_caffe_padding(W, s + "conv2", conv1_1, 2, force=f)
    conv2_1 = convrelu_caffe_padding(W, s + "conv2_1", conv2, 1, force=f)
    concat1 = refine_caffe_padding(W, s + "refine1", conv2_1, conv1_1, force=f)
    concat0 = refine_caffe_padding(W, s + "refine0", concat1, conv0, force=f)
    tmp = convrelu_caffe_padding(W, s + "predict_depth0/conv1", concat0, force=f)
    return {"predict_depth0": conv2d_caffe_padding(W, s + "predict_depth0/conv2", tmp, force=f)}


class OracleNets:
    """CPU twin of BootstrapNet / IterativeNet / RefinementNet (networks_original.py:22-255).  `force` and `ops`: see the
    module docstring."""

    def __init__(self, tf_weights, dtype=torch.float32):
        self.dtype = dtype
        self.W = Weights(tf_weights, dtype)

    def _t(self, a):
        return torch.as_tensor(np.asarray(a)).to(self.dtype)

    @torch.no_grad()
    def bootstrap(self, image_pair, image2_2, full=False, force=None, ops=oops):
        image_pair, image2_2 = self._t(image_pair), self._t(image2_2)
        f = flow_block(self.W, "netFlow1", image_pair, force=force, ops=ops)
        fc2 = f["predict_flowconf2"]
        d = depthmotion_block(self.W, "netDM1", image_pair, image2_2, fc2[:, 0:2].contiguous(), fc2, force=force, ops=ops)
        out = {"predict_flow5": f["predict_flowconf5"][:, 0:2], "predict_flow2": fc2[:, 0:2],
               "predict_depth2": d["predict_depth2"], "predict_normal2": d["predict_normal2"],
               "predict_rotation": d["predict_rotation"], "predict_translation": d["predict_translation"]}
        if full:
            out.update({"predict_flowconf2": fc2, "predict_flowconf5": f["predict_flowconf5"],
                        "predict_scale": d["predict_scale"]})
        return {k: v.contiguous() for k, v in out.items()}

    @torch.no_grad()
    def iterative(self, image_pair, image2_2, depth2, normal2, rotation, translation, full=False, force=None, ops=oops):
        image_pair, image2_2 = self._t(image_pair), self._t(image2_2)
        prev = {"predict_depth2": self._t(depth2), "predict_normal2": self._t(normal2),
                "predict_rotation": self._t(rotation), "predict_translation": self._t(translation)}
        f = flow_block(self.W, "netFlow2", image_pair, image2_2, prev, force=force, ops=ops)
        fc2 = f["predict_flowconf2"]
        d = depthmotion_block(self.W, "netDM2", image_pair, image2_2, fc2[:, 0:2].contiguous(), fc2,
                              prev["predict_rotation"], prev["predict_translation"], force=force, ops=ops)
        out = {"predict_flow5": f["predict_flowconf5"][:, 0:2], "predict_flow2": fc2[:, 0:2],
               "predict_depth2": d["predict_depth2"], "predict_normal2": d["predict_normal2"],
               "predict_rotation": d["predict_rotation"], "predict_translation": d["predict_translation"]}
        if full:
            out.update({"predict_flowconf2": fc2, "flow_from_depth_motion": f["flow_from_depth_motion"],
                        "depth_from_flow": d["depth_from_flow"], "predict_scale": d["predict_scale"]})
        return {k: v.contiguous() for k, v in out.items()}

    @torch.no_grad()
    def refine(self, image1, depth2, force=None):
        return refine_block(self.W, "netRefine", self._t(image1), self._t(depth2), force=force)

    @torch.no_grad()
    def pipeline(self, image_pair, image2_2, iterations=3):
        """examples/example.py:87-99."""
        r = self.bootstrap(image_pair, image2_2)
        for _ in range(iterations):
            r = self.iterative(image_pair, image2_2, r["predict_depth2"], r["predict_normal2"],
                               r["predict_rotation"], r["predict_translation"])
        image1 = self._t(image_pair)[:, 0:3].contiguous()
        out = dict(r)
        out.update(self.refine(image1, r["predict_depth2"]))
        return out
