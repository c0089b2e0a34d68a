"""Mirror of `depthmotionnet.evaluation.metrics` (python/depthmotionnet/evaluation/metrics.py) over the device
reductions in libdemon_b200.so (csrc/metrics.cu): same function names, arguments and result dictionaries, numpy or torch
arrays in, Python floats out -- plus batched forms that keep everything on the GPU.

    errs, errs_scaled = evaluate_depth(translation_gt, depth_gt, depth_pred)        # metrics.py:321-372
    errs = compute_errors(depth_pred, depth_gt)                                    # metrics.py:240-280
    epe = compute_flow_epe(flow_pred, flow_gt)                                     # metrics.py:377-387
    rot_deg, t_dist, t_deg = compute_motion_errors(pred6, gt6, True)               # metrics.py:390-445 (host, 6 numbers)

One streaming pass over prediction and ground truth yields all sums the eleven distances and the least-squares scale
factor need; the scale factor itself is computed on the device, so `evaluate_depth` is two kernel passes and one
[n,16]-double copy.  Tolerance against the numpy reference: 1e-5 relative (float32 pairwise summation there, double
accumulation here; `logf` vs numpy's log).  Mixed scalar / array arithmetic follows NumPy 1.x promotion: the
ground truth's divide and the scaled prediction are float32, and the ratio thresholds compare the float32 |log ratio|
with float32(log t) (DESIGN.md §3.4).  There is no CPU fallback.
"""
import ctypes
import math

import numpy as np
import torch

from . import _lib

DISTANCES = ['l1', 'l1_inverse', 'scale_invariant', 'abs_relative', 'sq_relative', 'avg_log10', 'rmse_log', 'rmse',
             'ratio_threshold_1.25', 'ratio_threshold_1.5625', 'ratio_threshold_1.953125']
_SCALING = {'abs': 0, 'log': 1, 'inv': 2}


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _dev(x):
    if not torch.cuda.is_available():
        raise RuntimeError("demon_b200.evaluation needs a CUDA device (there is no CPU fallback)")
    t = x if isinstance(x, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(np.asarray(x), dtype=np.float32))
    return t.to(device="cuda", dtype=torch.float32).contiguous()


def depth_error_sums(pred, gt, inverse_pred=False, inverse_gt=False, gt_div=None, pred_scale=None):
    """pred, gt: [n, ...] (all trailing dims are pixels) -> CUDA float64 tensor [n, 16] of masked sums
    (include/demon_b200.h: demon_depth_error_sums_f32)."""
    p, g = _dev(pred), _dev(gt)
    if p.shape != g.shape:
        raise ValueError("prediction %s and ground truth %s differ in shape" % (tuple(p.shape), tuple(g.shape)))
    n = p.shape[0]
    hw = p[0].numel() if n else 0
    lib = _lib.load()
    sums = torch.empty((n, 16), dtype=torch.float64, device=p.device)
    ws = torch.empty(max(1, lib.demon_metric_workspace_bytes(n, hw) // 8), dtype=torch.float64, device=p.device)
    gd = None if gt_div is None else _dev(gt_div).reshape(n)
    ps = None if pred_scale is None else _dev(pred_scale).reshape(n)
    _lib.check(lib.demon_depth_error_sums_f32(p.data_ptr(), g.data_ptr(), n, hw, int(bool(inverse_pred)), int(bool(inverse_gt)),
                                              None if gd is None else gd.data_ptr(), None if ps is None else ps.data_ptr(),
                                              sums.data_ptr(), ws.data_ptr(), _stream()))
    return sums


def depth_scale_factor(sums, depth_scaling='abs'):
    """CUDA float32 [n]: the factor for the prediction that minimises the squared error (metrics.py:283-318)."""
    if depth_scaling not in _SCALING:
        raise Exception('Unknown depth scaling method')
    n = sums.shape[0]
    scale = torch.empty(n, dtype=torch.float32, device=sums.device)
    _lib.check(_lib.load().demon_depth_scale_factor(sums.data_ptr(), n, _SCALING[depth_scaling], scale.data_ptr(), _stream()))
    return scale


def errors_from_sums(row, distances_to_compute=None):
    """One row of sums (16 numbers on the host) -> the result dictionary of compute_errors (metrics.py:240-280)."""
    s = [float(v) for v in row]
    num = s[0]
    nan = float('nan')

    def dist(name):
        if num == 0:
            return nan
        if name == 'l1':
            return s[1] / num
        if name == 'l1_inverse':
            return s[2] / num
        if name == 'scale_invariant':
            return math.sqrt(max(0.0, s[4] / num - (s[3] * s[3]) / (num * num)))
        if name == 'abs_relative':
            return s[5] / num
        if name == 'sq_relative':
            return s[6] / num
        if name == 'avg_log10':
            return s[7] / num
        if name == 'rmse_log':
            return math.sqrt(s[4] / num)
        if name == 'rmse':
            return math.sqrt(s[8] / num)
        if name.startswith('ratio_threshold'):
            t = float(name.split('_')[-1])
            idx = {1.25: 9, 1.5625: 10, 1.953125: 11}.get(t)
            if idx is None:
                raise ValueError("ratio thresholds on the device are 1.25, 1.5625 and 1.953125 (got %r)" % t)
            return s[idx] / num
        raise KeyError(name)
    out = {'num_valid': int(num)}
    for name in (DISTANCES if distances_to_compute is None else distances_to_compute):
        out[name] = dist(name)
    return out


def compute_errors(depth_pred, depth_gt, distances_to_compute=None):
    """metrics.py:240-280 for one pair of depth maps (any shape)."""
    p, g = _dev(depth_pred).reshape(1, -1), _dev(depth_gt).reshape(1, -1)
    return errors_from_sums(depth_error_sums(p, g)[0].cpu().numpy(), distances_to_compute)


def evaluate_depth_batch(translation_gt, depth_gt_in, depth_pred_in, inverse_gt=True, inverse_pred=True, depth_scaling='abs'):
    """Batched evaluate_depth on the device: translation_gt [n,3], depths [n,...] -> (sums, sums_scaled, scale), CUDA
    tensors [n,16] / [n,16] / [n]; nothing leaves the GPU."""
    t = np.asarray(translation_gt.detach().cpu() if isinstance(translation_gt, torch.Tensor) else translation_gt, dtype=np.float64).reshape(-1, 3)
    norm = np.sqrt((t * t).sum(axis=1))
    gt_div = None if np.all(np.isclose(1.0, norm)) else np.where(np.isclose(1.0, norm), 1.0, norm).astype(np.float32)
    sums = depth_error_sums(depth_pred_in, depth_gt_in, inverse_pred, inverse_gt, gt_div)
    scale = depth_scale_factor(sums, depth_scaling)
    sums_scaled = depth_error_sums(depth_pred_in, depth_gt_in, inverse_pred, inverse_gt, gt_div, scale)
    return sums, sums_scaled, scale


def evaluate_depth(translation_gt, depth_gt_in, depth_pred_in, distances_to_compute=None, inverse_gt=True, inverse_pred=True,
                   depth_scaling='abs', depth_pred_max=np.inf):
    """metrics.py:321-372: (errs, errs_pred_scaled) for one sample."""
    p, g = _dev(depth_pred_in).reshape(1, -1), _dev(depth_gt_in).reshape(1, -1)
    sums, sums_scaled, _ = evaluate_depth_batch(np.asarray(translation_gt, dtype=np.float64).reshape(1, 3), g, p, inverse_gt, inverse_pred, depth_scaling)
    both = torch.stack([sums[0], sums_scaled[0]]).cpu().numpy()
    return errors_from_sums(both[0], distances_to_compute), errors_from_sums(both[1], distances_to_compute)


def flow_epe_sums(flow1, flow2):
    """flow [n,2,...] -> CUDA float64 [n,2] = (sum of the valid end point errors, count)."""
    a, b = _dev(flow1), _dev(flow2)
    if a.shape != b.shape or a.dim() < 3 or a.shape[1] != 2:
        raise ValueError("flows must be [n,2,...] of equal shape")
    n = a.shape[0]
    hw = a[0, 0].numel() if n else 0
    lib = _lib.load()
    sums = torch.empty((n, 2), dtype=torch.float64, device=a.device)
    ws = torch.empty(max(1, lib.demon_metric_workspace_bytes(n, hw) // 8), dtype=torch.float64, device=a.device)
    _lib.check(lib.demon_flow_epe_sums_f32(a.data_ptr(), b.data_ptr(), n, hw, sums.data_ptr(), ws.data_ptr(), _stream()))
    return sums


def compute_flow_epe(flow1, flow2):
    """metrics.py:377-387: average end point error between two flow fields [2,h,w]."""
    a, b = _dev(flow1), _dev(flow2)
    s = flow_epe_sums(a.reshape((1,) + tuple(a.shape)), b.reshape((1,) + tuple(b.shape)))[0].cpu().numpy()
    return float(s[0] / s[1]) if s[1] > 0 else float('nan')


def compute_motion_errors(predicted_motion, gt_motion, normalize_translations):
    """metrics.py:390-445 (six numbers per sample: host arithmetic in float64; minieigen's Quaternion(angle, axis) and
    angularDistance restated: 2 * acos(min(1, |q1 . q2|)))."""
    def quat(aa):
        aa = np.asarray(aa, dtype=np.float64)
        angle = math.sqrt(float(aa.dot(aa)))
        if angle < 1e-6:
            angle, axis = 0.0, np.array([1.0, 0.0, 0.0])
        else:
            axis = aa / angle
            axis = axis / math.sqrt(float(axis.dot(axis)))
        return np.concatenate([[math.cos(angle / 2)], math.sin(angle / 2) * axis])
    pm, gm = np.asarray(predicted_motion, dtype=np.float64), np.asarray(gt_motion, dtype=np.float64)
    d = abs(float(quat(gm[0:3]).dot(quat(pm[0:3]))))
    rotation_angle_dist = 0.0 if d >= 1.0 else 2.0 * math.acos(d)
    gt_trans, pred_trans = gm[3:6].copy(), pm[3:6].copy()
    if normalize_translations:
        gt_trans = gt_trans / math.sqrt(float(gt_trans.dot(gt_trans)))
        if math.sqrt(float(pred_trans.dot(pred_trans))) > 1e-6:
            pred_trans = pred_trans / math.sqrt(float(pred_trans.dot(pred_trans)))
    diff = gt_trans - pred_trans
    translation_dist = math.sqrt(float(diff.dot(diff)))
    translation_angle_diff = math.acos(float(np.clip(gt_trans.dot(pred_trans), -1, 1)))
    return float(np.rad2deg(rotation_angle_dist)), translation_dist, float(np.rad2deg(translation_angle_diff))


# ---------------------------------------------------------------------------------------------------------------------
# The evaluation run of examples/evaluation.py / evaluation/evaluate_to_xarray.py on the device
# ---------------------------------------------------------------------------------------------------------------------
SUN3D_INTRINSICS = (0.891, 1.188, 0.5, 0.5)        # evaluate_to_xarray.py:114 (not the network's 0.89115971 constant)
EIGEN_CROP = (23, 27, 436, 588)                    # (y0, x0, h, w): depth_gt[23:459, 27:615] (evaluate_to_xarray.py:207-211)
MOTION_ERRORS = ['rot_err', 'tran_err', 'tran_angle_err']
ERRORS = MOTION_ERRORS + ['depth_' + d for d in DISTANCES] + ['flow_epe', 'camera_baseline']


def iteration_sort_key(label):
    """Order of the iteration labels (evaluate_to_xarray.py:74): '0', '0_refined', '1', ..."""
    return (int(label.split('_')[0]), len(label.split('_')))


def nearest_index(n_in, n_out):
    """int32 [n_out]: the input index skimage.transform.resize(order=0) reads for every output index along one axis, -1
    where it reads its cval.  Since skimage 0.19 that resize is scipy.ndimage.zoom(order=0, grid_mode=True,
    mode='grid-constant'): output pixel centre o + 0.5 maps to c = (o + 0.5) * n_in / n_out - 0.5, rounded half up (scipy
    rounds the exact .5 ties of 192 -> 480 and 256 -> 640 up)."""
    o = np.arange(n_out, dtype=np.float64)
    idx = np.floor((o + 0.5) * (n_in / n_out) - 0.5 + 0.5).astype(np.int64)
    idx[(idx < 0) | (idx >= n_in)] = -1
    return idx.astype(np.int32)


def angleaxis_to_rotation_matrix(aa, epsilon=1e-6):
    """evaluation/helpers.py:22-77 without minieigen: Quaternion(AngleAxis(angle, axis)).toRotationMatrix() in float64,
    Eigen's formulas (the ones oracle/ref_stub/eigen_stub.h restates for depth_to_flow)."""
    x, y, z = (float(v) for v in np.asarray(aa, dtype=np.float64).reshape(3))
    angle = math.sqrt((x * x + y * y) + z * z)
    if angle < epsilon:
        angle, axis = 0.0, (1.0, 0.0, 0.0)
    else:
        axis = (x / angle, y / angle, z / angle)        # Eigen normalized(): v / norm()
    ha = 0.5 * angle
    s = math.sin(ha)
    qw, qx, qy, qz = math.cos(ha), s * axis[0], s * axis[1], s * axis[2]
    tx, ty, tz = 2.0 * qx, 2.0 * qy, 2.0 * qz
    twx, twy, twz = tx * qw, ty * qw, tz * qw
    txx, txy, txz = tx * qx, ty * qx, tz * qx
    tyy, tyz, tzz = ty * qy, tz * qy, tz * qz
    return np.array([[1.0 - (tyy + tzz), txy - twz, txz + twy],
                     [txy + twz, 1.0 - (txx + tzz), tyz - twx],
                     [txz - twy, tyz + twx, 1.0 - (txx + tyy)]], dtype=np.float64)


def motion_vector_to_Rt(motion, epsilon=1e-6):
    """evaluation/helpers.py:81-100: (R float64 [3,3], t float64 [3]) of an angle-axis-6 motion vector."""
    tmp = np.asarray(motion).squeeze().astype(np.float64)
    return angleaxis_to_rotation_matrix(tmp[0:3], epsilon), tmp[3:].copy()


def intrinsics_vector_to_K(intrinsics, width, height):
    """evaluation/helpers.py:103-120: float64 K from the normalised [fx, fy, cx, cy]."""
    tmp = np.asarray(intrinsics).squeeze().astype(np.float64)
    return np.array([tmp[0] * width, 0, tmp[2] * width, 0, tmp[1] * height, tmp[3] * height, 0, 0, 1], dtype=np.float64).reshape((3, 3))


def projection_matrix(K, R, t):
    """P2 of compute_visible_points_mask (view_tools_cython.pyx:81-84, 98): K . [R|t], with [R|t] stored as float32 first
    and the float64 product cast to float32."""
    P2 = np.empty((3, 4), dtype=np.float32)
    P2[:, 0:3] = R
    P2[:, 3:4] = np.asarray(t).reshape((3, 1))
    return np.asarray(K).dot(P2).astype(np.float32)


def visible_points_operands(motion, intrinsics, height, width):
    """The float32 operands invalidate_points_not_visible_in_second_image hands compute_visible_points_mask, per sample
    (evaluate_to_xarray.py:110-119): view 1 at the origin, view 2 at (R, t) of the motion, both with K of the intrinsics
    (the sun3d default where `intrinsics` is None).  motion [n,6], intrinsics [n,4] or None -> (K1 [n,3,3], R1 [n,3,3],
    t1 [n,3], P2 [n,3,4])."""
    motion = np.asarray(motion, dtype=np.float32).reshape(-1, 6)
    n = motion.shape[0]
    intr = (np.tile(np.array([SUN3D_INTRINSICS], dtype=np.float32), (n, 1)) if intrinsics is None
            else np.asarray(intrinsics, dtype=np.float32).reshape(n, 4))
    K1, R1, t1, P2 = (np.empty((n,) + s, dtype=np.float32) for s in ((3, 3), (3, 3), (3,), (3, 4)))
    for i in range(n):
        R, t = motion_vector_to_Rt(motion[i])
        K = intrinsics_vector_to_K(intr[i], width, height)
        K1[i], R1[i], t1[i] = K.astype(np.float32), np.eye(3).astype(np.float32), np.zeros((3,)).astype(np.float32)
        P2[i] = projection_matrix(K, R, t)
    return K1, R1, t1, P2


def visible_points_mask(depth, K1, R1, t1, P2, width2=None, height2=None, borderx=0, bordery=0, inverse_depth=False):
    """compute_visible_points_mask (view_tools_cython.pyx:9-58) on the device for n views: depth [n,h,w] (camera z, or
    inverse depth with `inverse_depth`), operands as visible_points_operands returns them -> CUDA uint8 [n,h,w]."""
    d = _dev(depth)
    if d.dim() == 2:
        d = d.unsqueeze(0)
    n, h, w = d.shape
    ops = [_dev(np.asarray(a, dtype=np.float32).reshape((n,) + s)) for a, s in ((K1, (3, 3)), (R1, (3, 3)), (t1, (3,)), (P2, (3, 4)))]
    mask = torch.empty((n, h, w), dtype=torch.uint8, device=d.device)
    fn = _lib.load().demon_visible_points_mask_inverse_f32 if inverse_depth else _lib.load().demon_visible_points_mask_f32
    _lib.check(fn(d.data_ptr(), *[o.data_ptr() for o in ops], n, h, w, w if width2 is None else int(width2),
                  h if height2 is None else int(height2), int(borderx), int(bordery), mask.data_ptr(), _stream()))
    return mask


def invalidate_points_not_visible_in_second_image(depth, motion, intrinsics=None):
    """evaluate_to_xarray.py:93-124 for a batch: sets the INVERSE depth of every pixel that is not visible in the second
    view to NaN, in place.  depth [n,h,w] (or [h,w]) numpy float32 or torch CUDA float32, motion [n,6], intrinsics [n,4]
    or None (sun3d).  The mask runs on the device; returns it (CUDA uint8 [n,h,w], 1 = visible)."""
    h, w = depth.shape[-2:]
    K1, R1, t1, P2 = visible_points_operands(motion, intrinsics, h, w)
    mask = visible_points_mask(depth, K1, R1, t1, P2, inverse_depth=True)
    if isinstance(depth, torch.Tensor):
        depth.masked_fill_((mask == 0).reshape(depth.shape), float('nan'))
    else:
        depth[(mask == 0).cpu().numpy().reshape(depth.shape)] = np.nan
    return mask


def motion_errors(pred_rotation, pred_translation, gt_motion):
    """compute_motion_errors for n samples on the device (demon_motion_errors): -> (CUDA float64 [n,4] = rot_err,
    tran_err, tran_angle_err, camera_baseline; CUDA float32 [n] gt_div, the divisor of the gt depth)."""
    r, t, g = _dev(pred_rotation).reshape(-1, 3), _dev(pred_translation).reshape(-1, 3), _dev(gt_motion).reshape(-1, 6)
    n = g.shape[0]
    out = torch.empty((n, 4), dtype=torch.float64, device=g.device)
    gt_div = torch.empty(n, dtype=torch.float32, device=g.device)
    _lib.check(_lib.load().demon_motion_errors(r.data_ptr(), t.data_ptr(), g.data_ptr(), n, out.data_ptr(), gt_div.data_ptr(), _stream()))
    return out, gt_div


class _Resampler:
    """Index tables of one prediction size onto the ground truth window, on the device."""

    def __init__(self, ph, pw, gh, gw, window, device):
        y0, x0, oh, ow = window
        self.ph, self.pw, self.gh, self.gw, self.window = ph, pw, gh, gw, window
        self.rows = torch.from_numpy(nearest_index(ph, gh)[y0:y0 + oh].copy()).to(device)
        self.cols = torch.from_numpy(nearest_index(pw, gw)[x0:x0 + ow].copy()).to(device)

    def depth_sums(self, pred, gt, gt_valid, gt_div, pred_scale=None):
        n = gt.shape[0]
        y0, x0, oh, ow = self.window
        lib = _lib.load()
        sums = torch.empty((n, 16), dtype=torch.float64, device=gt.device)
        ws = torch.empty(max(1, lib.demon_metric_workspace_bytes(n, oh * ow) // 8), dtype=torch.float64, device=gt.device)
        _lib.check(lib.demon_depth_error_sums_resampled_f32(
            pred.data_ptr(), self.ph, self.pw, gt.data_ptr(), None if gt_valid is None else gt_valid.data_ptr(), self.gh, self.gw,
            n, y0, x0, oh, ow, self.rows.data_ptr(), self.cols.data_ptr(), 1, 1, gt_div.data_ptr(),
            None if pred_scale is None else pred_scale.data_ptr(), sums.data_ptr(), ws.data_ptr(), _stream()))
        return sums

    def flow_sums(self, pred, gt):
        n = gt.shape[0]
        y0, x0, oh, ow = self.window
        lib = _lib.load()
        sums = torch.empty((n, 2), dtype=torch.float64, device=gt.device)
        ws = torch.empty(max(1, lib.demon_metric_workspace_bytes(n, oh * ow) // 8), dtype=torch.float64, device=gt.device)
        _lib.check(lib.demon_flow_epe_sums_resampled_f32(
            pred.data_ptr(), self.ph, self.pw, gt.data_ptr(), self.gh, self.gw, n, y0, x0, oh, ow, self.rows.data_ptr(),
            self.cols.data_ptr(), sums.data_ptr(), ws.data_ptr(), _stream()))
        return sums


class EvaluationResult:
    """The table evaluate_to_xarray.evaluate returns, without xarray: `values` float64 [snapshot, iteration, sample,
    errors, scaled] and its coordinates.  to_dict() is xarray.DataArray.to_dict()'s layout, so the reference's
    read_xarray_json (evaluate_to_xarray.py:38-41) and printing code (examples/evaluation.py:296-321) read what
    write_xarray_json writes."""
    DIMS = ('snapshot', 'iteration', 'sample', 'errors', 'scaled')

    def __init__(self, values, snapshots, iterations, samples, attrs):
        self.values = values
        self.coords = {'snapshot': list(snapshots), 'iteration': list(iterations), 'sample': list(samples), 'errors': list(ERRORS),
                       'scaled': [False, True]}
        self.attrs = dict(attrs)

    def sel(self, iteration, error, scaled=False, snapshot=0):
        """values[snapshot, iteration, :, error, scaled] by label: one number per sample."""
        return self.values[snapshot, self.coords['iteration'].index(iteration), :, ERRORS.index(error), int(bool(scaled))]

    def to_dict(self):
        def var(dim):
            return {'dims': (dim,), 'attrs': {}, 'data': list(self.coords[dim])}
        return {'dims': self.DIMS, 'attrs': dict(self.attrs), 'data': self.values.tolist(),
                'coords': {d: var(d) for d in self.DIMS}, 'name': None}

    @staticmethod
    def concatenate(results):
        """Results of consecutive batches -> one result, samples renumbered '0', '1', ..."""
        values = np.concatenate([r.values for r in results], axis=2)
        first = results[0]
        return EvaluationResult(values, first.coords['snapshot'], first.coords['iteration'], [str(i) for i in range(values.shape[2])],
                                first.attrs)


def write_xarray_json(data, out_file):
    """evaluate_to_xarray.py:33-36: the table as JSON (NaN written as NaN, like json.dump does there)."""
    import json
    with open(out_file, 'w') as f:
        json.dump(data.to_dict(), f)


def evaluate_batch(predictions, depth_gt, motion_gt, intrinsics=None, flow_gt=None, depthmask=False, eigen_crop_gt_and_pred=False,
                   depth_scaling='abs', snapshot='snapshot_1', first_sample=0):
    """evaluate_to_xarray.evaluate (lines 216-316) for one batch of predictions that never left the device.

    predictions: DemonPipeline.forward_snapshots' dict (or DemonPipelineV2's; keys it does not use are ignored) (predict_flow2 [S,B,2,h,w], predict_depth2 [S,B,1,h,w],
        predict_rotation / predict_translation [S,B,3], optional predict_depth0 [S,B,1,H,W]); the first n samples are used
    depth_gt: [n,gh,gw] INVERSE depth (the ground-truth file's 'depth'), motion_gt [n,6] ('motion', angle axis |
        translation), intrinsics [n,4] normalised ('intrinsics') or None for the sun3d default, flow_gt [n,2,gh,gw]
        ('flow') or None: then it is depth_to_flow of the unmasked depth (examples/evaluation.py:81)
    depthmask: inverse depth of the points not visible in the second view is ignored (invalidate_points_not_visible_...)
    eigen_crop_gt_and_pred: depth errors on [23:459, 27:615] of a 480x640 ground truth

    Predictions are resized to the ground truth's size by nearest neighbour inside the sum kernels (nearest_index);
    the depth mask applies before that resize, the crop after it, both to depth only.  Returns an EvaluationResult with
    iterations '0', '0_refined', ..., one snapshot, the reference's errors and fill rules: motion, flow and baseline in
    both `scaled` slots, '_refined' rows carry depth errors and the baseline only."""
    from . import lmbspecialops as sops
    if depth_scaling not in _SCALING:
        raise Exception('Unknown depth scaling method')
    gt = _dev(depth_gt)
    if gt.dim() == 2:
        gt = gt.unsqueeze(0)
    n, gh, gw = gt.shape
    d2 = predictions['predict_depth2']
    S = d2.shape[0]
    if d2.shape[1] < n:
        raise ValueError("predictions hold %d samples, the ground truth %d" % (d2.shape[1], n))
    motion = _dev(motion_gt).reshape(n, 6)
    intr_host = (np.tile(np.array([SUN3D_INTRINSICS], dtype=np.float32), (n, 1)) if intrinsics is None
                 else np.asarray(intrinsics.detach().cpu() if isinstance(intrinsics, torch.Tensor) else intrinsics, dtype=np.float32).reshape(n, 4))
    if eigen_crop_gt_and_pred and (gh, gw) != (436, 588):
        if (gh, gw) != (480, 640):
            raise ValueError("eigen_crop_gt_and_pred needs a 480x640 ground truth, got %dx%d" % (gh, gw))
        window = EIGEN_CROP
    else:
        window = (0, 0, gh, gw)
    # flow first: from the depth before the visibility mask
    if flow_gt is None:
        flow = sops.depth_to_flow(gt.reshape(n, 1, gh, gw), _dev(intr_host), motion[:, 0:3].contiguous(), motion[:, 3:6].contiguous(),
                                  rotation_format="angleaxis3", inverse_depth=True, normalize_flow=True)
    else:
        flow = _dev(flow_gt).reshape(n, 2, gh, gw)
    valid = None
    if depthmask:
        K1, R1, t1, P2 = visible_points_operands(motion.cpu().numpy(), intr_host, gh, gw)
        valid = visible_points_mask(gt, K1, R1, t1, P2, inverse_depth=True)
    refined = predictions.get('predict_depth0') is not None
    dev = gt.device
    rs2 = _Resampler(d2.shape[-2], d2.shape[-1], gh, gw, window, dev)
    f2 = predictions['predict_flow2']
    rsf = _Resampler(f2.shape[-2], f2.shape[-1], gh, gw, (0, 0, gh, gw), dev)
    if refined:
        d0 = predictions['predict_depth0']
        rs0 = _Resampler(d0.shape[-2], d0.shape[-1], gh, gw, window, dev)
    rows = []   # per iteration label: (label, motion [n,4] or None, depth sums, scaled sums, flow sums or None)
    gt_div = None
    for k in range(S):
        mot, div = motion_errors(predictions['predict_rotation'][k, :n], predictions['predict_translation'][k, :n], motion)
        if gt_div is None:
            gt_div = div   # it depends on the ground truth only
        targets = [(str(k), rs2, d2[k, :n])]
        if refined:
            targets.append(('%d_refined' % k, rs0, d0[k, :n]))
        for label, rs, pred in targets:
            sums = rs.depth_sums(pred, gt, valid, gt_div)
            scaled = rs.depth_sums(pred, gt, valid, gt_div, depth_scale_factor(sums, depth_scaling))
            rows.append((label, mot, sums, scaled, rsf.flow_sums(f2[k, :n], flow) if rs is rs2 else None))
    # one copy of the whole table's inputs to the host
    packed = torch.cat([torch.cat([r[1].reshape(-1), r[2].reshape(-1), r[3].reshape(-1)] + ([r[4].reshape(-1)] if r[4] is not None else []))
                        for r in rows]).cpu().numpy()
    labels = sorted((r[0] for r in rows), key=iteration_sort_key)
    values = np.full((1, len(labels), n, len(ERRORS), 2), np.nan, dtype=np.float64)
    off = 0
    for label, _, _, _, fl in rows:
        mot = packed[off:off + 4 * n].reshape(n, 4); off += 4 * n
        sums = packed[off:off + 16 * n].reshape(n, 16); off += 16 * n
        scaled = packed[off:off + 16 * n].reshape(n, 16); off += 16 * n
        it = labels.index(label)
        v = values[0, it]
        for i in range(n):
            e, es = errors_from_sums(sums[i]), errors_from_sums(scaled[i])
            for j, d in enumerate(DISTANCES):
                v[i, 3 + j, 0], v[i, 3 + j, 1] = e[d], es[d]
        v[:, ERRORS.index('camera_baseline'), :] = mot[:, 3:4]
        if fl is not None:
            f = packed[off:off + 2 * n].reshape(n, 2); off += 2 * n
            with np.errstate(invalid='ignore', divide='ignore'):
                epe = np.where(f[:, 1] > 0, f[:, 0] / np.where(f[:, 1] > 0, f[:, 1], 1.0), np.nan)
            v[:, ERRORS.index('flow_epe'), :] = epe[:, None]
            v[:, 0:3, :] = mot[:, 0:3, None]
    attrs = {'depthmask': bool(depthmask), 'depth_scaling': depth_scaling, 'depth_pred_max': str(np.inf),
             'eigen_crop_gt_and_pred': bool(eigen_crop_gt_and_pred), 'iterations': labels}
    return EvaluationResult(values, [snapshot], labels, [str(first_sample + i) for i in range(n)], attrs)


class Evaluator:
    """examples/evaluation.py's create_prediction_file + evaluate, batch by batch on the device:

        ev = Evaluator(session, batch_size=64, depthmask=True)
        for image_pair, depth, motion, intrinsics in batches:        # the ground-truth file's groups, see DESIGN.md §1
            ev.add(image_pair, depth, motion, intrinsics)
        write_xarray_json(ev.result(), 'sun3d_eval.json')

    Every batch is one forward_snapshots call (bootstrap, `iterations` iterations, the refinement net on every snapshot)
    and one evaluate_batch; only the table's numbers leave the GPU.  A last, smaller batch is padded to the batch size
    and only its real samples are evaluated.  A v2 Session (demon_b200.v2.networks, e.g. restored from a checkpoint of
    training/v2/training.py) is evaluated with DemonPipelineV2; its predict_normal0 is not part of the table."""

    def __init__(self, session, batch_size, iterations=3, depthmask=False, eigen_crop_gt_and_pred=False, depth_scaling='abs',
                 refine=True):
        from .networks_original import DemonPipeline
        from .v2.networks import DemonPipelineV2, Session as SessionV2
        self.v2 = isinstance(session, SessionV2)
        self.pipeline = (DemonPipelineV2 if self.v2 else DemonPipeline)(session, batch_size, iterations)
        self.batch_size = int(batch_size)
        self.options = dict(depthmask=depthmask, eigen_crop_gt_and_pred=eigen_crop_gt_and_pred, depth_scaling=depth_scaling)
        self.refine = refine
        self._parts = []
        self._count = 0

    def add(self, image_pair, depth_gt, motion_gt, intrinsics=None, flow_gt=None, image2_2=None):
        """image_pair [m,6,192,256] (m <= batch size), image2_2 [m,3,48,64], None (median3x3 twice) or, for a v2 session,
        'area' (tf.image.resize_area of the second image, the input training/v2/training.py trains v2 on); ground truth as
        evaluate_batch takes it.  Returns this batch's EvaluationResult."""
        if isinstance(image2_2, str) and not (self.v2 and image2_2 == 'area'):
            raise ValueError("image2_2 must be a tensor, None%s, got %r (v1 was never trained on resize_area's image2_2)"
                             % (" or 'area'" if self.v2 else "", image2_2))
        ip = _dev(image_pair)
        m = ip.shape[0]
        if m > self.batch_size:
            raise ValueError("%d pairs in a batch of %d" % (m, self.batch_size))
        i2 = image2_2 if image2_2 is None or isinstance(image2_2, str) else _dev(image2_2)
        if m < self.batch_size:
            pad = self.batch_size - m
            ip = torch.cat([ip, ip[-1:].expand(pad, -1, -1, -1)])
            i2 = i2 if i2 is None or isinstance(i2, str) else torch.cat([i2, i2[-1:].expand(pad, -1, -1, -1)])
        preds = self.pipeline.forward_snapshots(ip, i2, refine=self.refine)
        r = evaluate_batch(preds, depth_gt, motion_gt, intrinsics, flow_gt, first_sample=self._count, **self.options)
        self._parts.append(r)
        self._count += m
        return r

    def result(self):
        if not self._parts:
            raise RuntimeError("Evaluator.result() before add()")
        return EvaluationResult.concatenate(self._parts)
