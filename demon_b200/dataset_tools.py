"""Mirror of the compute in `depthmotionnet.dataset_tools` (python/depthmotionnet/dataset_tools): choosing the multi-view
samples DeMoN trains and tests on from RGB-D sequences, on the device (csrc/dataset_tools.cu), bit for bit with the
reference's helpers, Cython and greedy grouping.

    s = measure_sharpness(pil_image)                          # np.float32, helpers.measure_sharpness
    s = measure_sharpness(frames)                             # CUDA uint8 [N,h,w,3] -> CUDA float32 [N]
    depth, valid = sun3d_depth(raw)                           # sun3d_utils.read_depth on decoded uint16 PNGs
    dr = compute_depth_ratios(view1, view2)                   # view_tools_cython.compute_depth_ratios
    ok = check_depth_consistency(view, [v2, v3])              # view_tools.check_depth_consistency, one launch
    groups = sequence_view_groups(sharpness, R, t, K, depth, (0.05, 0.5))   # create_samples_from_sequence's grouping
    groups = sun3d_view_groups(sun3d_path, 'mit_32_d463/d463_1', (0.05, 0.5), compute_sharpness(sun3d_path, seq))

Writing the HDF5 groups is not part of this module: each group comes back as its frames, its viewpoint_pairs and its name.
There is no CPU fallback.
"""
import ctypes
import itertools
import math
import os
from collections import namedtuple

import numpy as np
import torch

from . import _lib
from .evaluation import projection_matrix

# dataset_tools/view.py:25
View = namedtuple('View', ['R', 't', 'K', 'image', 'depth', 'depth_metric'])

MAX_PIXELS = 2 ** 24      # h*w must stay below this: the pixel count must be exact in float32
UPLOAD_FRAMES = 64        # frames read from disk and sent to the device per launch


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _device():
    if not torch.cuda.is_available():
        raise RuntimeError("demon_b200.dataset_tools needs a CUDA device (there is no CPU fallback)")
    return torch.device("cuda", torch.cuda.current_device())


def _check_pixels(h, w, name):
    if h * w >= MAX_PIXELS:
        raise ValueError("%s: %dx%d pixels is too many (h*w must be below 2^24)" % (name, h, w))


# ---- sharpness ----------------------------------------------------------------------------------------------------
def sharpness(frames):
    """measure_sharpness of every frame on the device: frames CUDA uint8 [N,h,w,3] RGB (pixel stride 3, channel stride 1;
    a cropped view is read in place) -> CUDA float32 [N], asynchronous on the current stream."""
    if not isinstance(frames, torch.Tensor) or not frames.is_cuda:
        raise ValueError("frames: expected a CUDA tensor")
    if frames.dtype != torch.uint8:
        raise ValueError("frames: expected dtype uint8, got %s" % (frames.dtype,))
    if frames.dim() != 4 or frames.shape[-1] != 3:
        raise ValueError("frames: expected [N,h,w,3] RGB, got shape %s" % (tuple(frames.shape),))
    n, h, w = frames.shape[:3]
    if h < 1 or w < 1:
        raise ValueError("frames: empty frames %dx%d" % (h, w))
    _check_pixels(h, w, "frames")
    if frames.stride(-1) != 1 or (w > 1 and frames.stride(-2) != 3) or any(s < 0 for s in frames.stride()):
        raise ValueError("frames: the pixel and channel strides must be 3 and 1, got %s" % (frames.stride()[-2:],))
    out = torch.empty((n,), dtype=torch.float32, device=frames.device)
    if n:
        with torch.cuda.device(frames.device):
            _lib.check(_lib.load().demon_sharpness_u8(frames.data_ptr(), frames.stride(0), frames.stride(1), n, h, w,
                                                      out.data_ptr(), _stream()))
    return out


def _rgb_array(img):
    """A PIL image or an HWC uint8 array as contiguous uint8 [h,w,3] RGB: convert('L') of any of Pillow's colour modes equals
    convert('RGB') then convert('L'), and grey replicated to RGB gives the same grey back."""
    if hasattr(img, "convert"):
        img = np.array(img.convert('RGB'))
    a = np.asarray(img)
    if a.dtype != np.uint8:
        raise ValueError("img: expected uint8, got %s" % (a.dtype,))
    if a.ndim == 2:
        a = np.repeat(a[:, :, None], 3, axis=2)
    if a.ndim != 3 or a.shape[2] != 3:
        raise ValueError("img: expected [h,w,3] RGB, got shape %s" % (a.shape,))
    return np.ascontiguousarray(a)


def measure_sharpness(img):
    """helpers.py:23-31: the variance of the Laplacian of the grey image, bit for bit.  A PIL image or an HWC uint8 array
    gives the np.float32 the reference returns; a CUDA uint8 [N,h,w,3] tensor gives a CUDA float32 [N] (see `sharpness`)."""
    if isinstance(img, torch.Tensor) and img.is_cuda:
        return sharpness(img)
    a = _rgb_array(img.cpu().numpy() if isinstance(img, torch.Tensor) else img)
    return np.float32(sharpness(torch.from_numpy(a).to(_device())[None]).item())


def compute_sharpness(sun3d_data_path, seq_name):
    """sun3d_utils.compute_sharpness: the sharpness of every image/*.jpg of the sequence in file-name order, float32 [F]
    (the reference returns the same values as an array of np.float32).  Images are decoded on the host and measured on the
    device UPLOAD_FRAMES at a time."""
    image_dir = os.path.join(sun3d_data_path, seq_name, 'image')
    files = [f for f in sorted(os.listdir(image_dir)) if f.endswith('.jpg')]
    out = np.empty((len(files),), dtype=np.float32)
    dev = _device()
    i = 0
    while i < len(files):
        first = _rgb_array(_read_image(os.path.join(image_dir, files[i])))
        batch = [first]
        while i + len(batch) < len(files) and len(batch) < UPLOAD_FRAMES:
            a = _rgb_array(_read_image(os.path.join(image_dir, files[i + len(batch)])))
            if a.shape != first.shape:
                break
            batch.append(a)
        out[i:i + len(batch)] = sharpness(torch.from_numpy(np.stack(batch)).to(dev)).cpu().numpy()
        i += len(batch)
    return out


# ---- SUN3D depth --------------------------------------------------------------------------------------------------
def sun3d_depth(raw):
    """sun3d_utils.read_depth's arithmetic on decoded depth PNGs: raw uint16 [N,h,w] (or [h,w]; numpy or torch) ->
    (CUDA float32 depth [N,h,w], CUDA int64 [N] count of finite depths > 0), bit for bit."""
    if isinstance(raw, torch.Tensor):
        if raw.dtype not in (torch.uint16, torch.int16):
            raise ValueError("raw: expected uint16, got %s" % (raw.dtype,))
        r = raw.to(_device()).contiguous()
    else:
        a = np.asarray(raw)
        if a.dtype != np.uint16:
            raise ValueError("raw: expected uint16, got %s" % (a.dtype,))
        r = torch.from_numpy(np.ascontiguousarray(a).view(np.int16)).to(_device())
    single = r.dim() == 2
    if single:
        r = r[None]
    if r.dim() != 3:
        raise ValueError("raw: expected [N,h,w], got shape %s" % (tuple(r.shape),))
    n, h, w = r.shape
    if n > 65535:
        raise ValueError("raw: at most 65535 frames per call, got %d" % n)
    depth = torch.empty((n, h, w), dtype=torch.float32, device=r.device)
    valid = torch.empty((n,), dtype=torch.int64, device=r.device)
    with torch.cuda.device(r.device):
        _lib.check(_lib.load().demon_sun3d_depth_u16(r.data_ptr(), n, h, w, depth.data_ptr(), valid.data_ptr(), _stream()))
    return (depth[0], valid[0]) if single else (depth, valid)


# ---- depth ratios and consistency -----------------------------------------------------------------------------------
def view_operands(views):
    """The float32 operands the .pyx wrapper builds for each view (view_tools_cython.pyx:180-191), stacked: K, R, t and
    P = K.dot([R|t] as float32), as CUDA tensors [n,3,3], [n,3,3], [n,3], [n,3,4]."""
    dev = _device()
    K = np.stack([np.asarray(v.K).astype(np.float32) for v in views])
    R = np.stack([np.asarray(v.R).astype(np.float32) for v in views])
    t = np.stack([np.asarray(v.t).astype(np.float32).reshape(3) for v in views])
    P = np.stack([projection_matrix(v.K, v.R, v.t) for v in views])
    return tuple(torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (K, R, t, P))


def _depth_stack(depths):
    """Camera-z depths of one size (numpy arrays or tensors [h,w]), or one [n,h,w] tensor -> contiguous CUDA float32."""
    dev = _device()
    if isinstance(depths, torch.Tensor):
        d = depths
    else:
        maps = [x if isinstance(x, torch.Tensor) else torch.from_numpy(np.asarray(x)) for x in depths]
        shapes = {tuple(m.shape) for m in maps}
        if len(shapes) != 1:
            raise ValueError("depth maps of different sizes: %s" % sorted(shapes))
        if any(m.dtype != torch.float32 for m in maps):
            raise ValueError("depth maps must be float32")
        d = torch.stack([m.to(dev) for m in maps])
    if d.dtype != torch.float32:
        raise ValueError("depth maps must be float32, got %s" % (d.dtype,))
    if d.dim() != 3:
        raise ValueError("depth maps must be [h,w], got %s" % (tuple(d.shape[1:]),))
    _check_pixels(d.shape[1], d.shape[2], "depth")
    return d.to(dev).contiguous()


def _pairs(pairs, n_views):
    p = np.asarray(pairs, dtype=np.int64).reshape(-1, 2)
    if p.size and (p.min() < 0 or p.max() >= n_views):
        raise ValueError("pair index outside 0..%d" % (n_views - 1))
    if p.shape[0] > 2 ** 31 - 1:
        raise ValueError("too many pairs")
    return torch.from_numpy(p.astype(np.int32)).to(_device())


def depth_ratios(depth, K, R, t, P, pairs):
    """compute_depth_ratios of ordered view pairs on the device: depth CUDA float32 [n,h,w] camera z, K/R/t/P the
    `view_operands`, pairs [p,2] (i, j) -> CUDA float32 [p,h,w], the ratio map of view i against view j, bit for bit the
    .pyx's (NaN where the .pyx reads past depth j, DESIGN.md §7)."""
    d = _depth_stack(depth)
    n, h, w = d.shape
    pr = _pairs(pairs, n)
    out = torch.empty((pr.shape[0], h, w), dtype=torch.float32, device=d.device)
    _lib.check(_lib.load().demon_depth_ratios_f32(d.data_ptr(), K.data_ptr(), R.data_ptr(), t.data_ptr(), P.data_ptr(), n, h, w,
                                                  pr.data_ptr(), pr.shape[0], out.data_ptr(), _stream()))
    return out


def ratio_thresholds(depth_ratio_threshold):
    """check_depth_consistency's (min, max) of (th, 1/th), 1/th in double, as the float32 values numpy 2 compares a float32
    ratio array with."""
    th = float(depth_ratio_threshold)
    return np.float32(min(th, 1 / th)), np.float32(max(th, 1 / th))


def consistency_counts(depth, K, R, t, P, pairs, depth_ratio_threshold=0.9):
    """The counts check_depth_consistency needs from each ratio map, without writing the maps: int64 CUDA [p,2] =
    (finite ratios, finite ratios strictly between the float32 thresholds), one launch for every pair."""
    d = _depth_stack(depth)
    n, h, w = d.shape
    pr = _pairs(pairs, n)
    lo, hi = ratio_thresholds(depth_ratio_threshold)
    out = torch.empty((pr.shape[0], 2), dtype=torch.int64, device=d.device)
    _lib.check(_lib.load().demon_depth_consistency_counts_f32(d.data_ptr(), K.data_ptr(), R.data_ptr(), t.data_ptr(), P.data_ptr(), n,
                                                              h, w, pr.data_ptr(), pr.shape[0], float(lo), float(hi), out.data_ptr(),
                                                              _stream()))
    return out


def consistent_from_counts(n_finite, n_consistent, size, min_valid_threshold=0.5, min_depth_consistent=0.7):
    """check_depth_consistency's two tests for one view pair in its order, with its operand types: False if
    n_finite / size < min_valid (int / int), False if n_consistent / n_finite < min_consistent, else True.  The reference's
    n_consistent is np.count_nonzero's np.int64, so with no finite ratio (reachable with min_valid_threshold <= 0) the
    second test is 0/0 = nan with numpy's RuntimeWarning, not a ZeroDivisionError, and the pair passes."""
    n_finite, size = int(n_finite), int(size)
    if n_finite / size < min_valid_threshold:
        return False
    if np.int64(n_consistent) / n_finite < min_depth_consistent:
        return False
    return True


def _check_views(views):
    for v in views:
        assert v.depth_metric == 'camera_z', "Depth metric must be 'camera_z'"


def compute_depth_ratios(view1, view2):
    """view_tools.compute_depth_ratios: the ratio map of view1 against view2 (View tuples with camera-z float32 depths of
    one size).  numpy depths give a numpy float32 [h,w]; a CUDA tensor depth gives a CUDA tensor."""
    _check_views([view1, view2])
    K, R, t, P = view_operands([view1, view2])
    out = depth_ratios([view1.depth, view2.depth], K, R, t, P, [[0, 1]])[0]
    return out if isinstance(view1.depth, torch.Tensor) else out.cpu().numpy()


def check_depth_consistency(view, rest_of_the_views, depth_ratio_threshold=0.9, min_valid_threshold=0.5, min_depth_consistent=0.7):
    """view_tools.check_depth_consistency: True if view's depth is consistent with every view of rest_of_the_views.  The
    counts of every pair come from one launch; the tests run on the host in the reference's order, so the first
    inconsistent view decides."""
    views = [view] + list(rest_of_the_views)
    _check_views(views)
    if len(views) == 1:
        return True
    K, R, t, P = view_operands(views)
    d = _depth_stack([v.depth for v in views])
    counts = consistency_counts(d, K, R, t, P, [[0, j] for j in range(1, len(views))], depth_ratio_threshold).cpu().numpy()
    size = d.shape[1] * d.shape[2]
    for n_finite, n_consistent in counts:
        if not consistent_from_counts(n_finite, n_consistent, size, min_valid_threshold, min_depth_consistent):
            return False
    return True


# ---- grouping of a sequence (sun3d_utils.create_samples_from_sequence) -------------------------------------------------
SEQUENCE_CHECK = {'min_valid_threshold': 0.4, 'min_depth_consistent': 0.7}   # sun3d_utils.py:204


def sharp_frames(sharpness, sharpness_window=30):
    """The frames kept by the non-maximum suppression of sun3d_utils.py:163-164, in order."""
    from scipy.ndimage import maximum_filter1d
    s = np.asarray(sharpness)
    return np.where(s == maximum_filter1d(s, size=sharpness_window, mode='constant', cval=0))[0]


def _geometry_ok(R1, t1, R2, t2, baseline_range):
    """sun3d_utils.py:189-195 in float64: the baseline between the camera centres in range, the optical axes within 70 deg."""
    baseline = np.linalg.norm((-R1.transpose().dot(t1)) - (-R2.transpose().dot(t2)))
    if baseline < baseline_range[0] or baseline > baseline_range[1]:
        return False
    return not np.dot(R1[2, :], R2[2, :]) < math.cos(math.radians(70))


def group_views(sharp, R, t, valid, size, baseline_range, consistent, max_views_num=10, img_ids=None):
    """The greedy grouping of create_samples_from_sequence (sun3d_utils.py:166-232) on the host, with its quirks: a frame
    already taken as i2 is skipped as i1 but never as i2; an i1 with too little valid depth is skipped without being
    marked used; the loop breaks after the append, so a group holds up to max_views_num + 1 views; the viewpoint_pairs
    baseline test is always true; the name uses img_ids[i1], i1 being the position in the sharp list.

    sharp: frame indices kept by the NMS; R [F,3,3], t [F,3] float64 (read_Rt's); valid [F] valid-depth counts of size
    pixels; consistent(i1, i2) -> bool, both directions' check_depth_consistency for sharp positions i1 < i2.  Returns a
    list of {'frames': frame indices, 'viewpoint_pairs': int32 [2k], 'suffix': '-%07d'}."""
    img_ids = np.arange(len(R)) if img_ids is None else img_ids
    groups = []
    used = set()
    for i1, f1 in enumerate(sharp):
        if i1 in used:
            continue
        if valid[f1] < 0.5 * size:
            continue
        views = [f1]
        used.add(i1)
        for i2 in range(i1 + 1, len(sharp)):
            f2 = sharp[i2]
            if not _geometry_ok(R[f1], t[f1], R[f2], t[f2], baseline_range):
                continue
            if valid[f2] < 0.5 * size:
                continue
            if consistent(i1, i2):
                views.append(f2)
                used.add(i2)
            if len(views) > max_views_num:
                break
        if len(views) > 1:
            pairs = []
            for a, b in itertools.product(range(len(views)), repeat=2):
                if a != b:
                    baseline = np.linalg.norm(t[views[a]] - t[views[b]])
                    if baseline >= baseline_range[0] or baseline <= baseline_range[1]:
                        pairs.extend((a, b))
            groups.append({'frames': [int(f) for f in views], 'viewpoint_pairs': np.array(pairs, dtype=np.int32),
                           'suffix': '-{:07d}'.format(img_ids[i1])})
    return groups


def _device_consistency(sharp, R, t, K, depth_of, valid, size, baseline_range):
    """consistent(i1, i2) for group_views from one counts launch over every pair the greedy loop can reach, both
    directions.  depth_of(positions) -> CUDA float32 [len(positions),h,w], the depths of those sharp positions."""
    cand = []
    for i1, f1 in enumerate(sharp):
        if valid[f1] < 0.5 * size:
            continue
        for i2 in range(i1 + 1, len(sharp)):
            f2 = sharp[i2]
            if valid[f2] >= 0.5 * size and _geometry_ok(R[f1], t[f1], R[f2], t[f2], baseline_range):
                cand.append((i1, i2))
    if not cand:
        return lambda i1, i2: False
    pos = sorted({i for p in cand for i in p})
    row = {p: k for k, p in enumerate(pos)}
    views = [View(R=R[sharp[p]], t=t[sharp[p]], K=K, image=None, depth=None, depth_metric='camera_z') for p in pos]
    Kd, Rd, td, Pd = view_operands(views)
    pairs = [(row[a], row[b]) for i1, i2 in cand for a, b in ((i1, i2), (i2, i1))]
    counts = consistency_counts(depth_of(pos), Kd, Rd, td, Pd, pairs).cpu().numpy()
    index = {c: k for k, c in enumerate(cand)}

    def consistent(i1, i2):
        k = index[(i1, i2)]
        fwd, bwd = counts[2 * k], counts[2 * k + 1]
        return (consistent_from_counts(fwd[0], fwd[1], size, **SEQUENCE_CHECK)
                and consistent_from_counts(bwd[0], bwd[1], size, **SEQUENCE_CHECK))
    return consistent


def sequence_view_groups(sharpness, R, t, K, depth, baseline_range, sharpness_window=30, max_views_num=10, img_ids=None):
    """The grouping of create_samples_from_sequence (sun3d_utils.py:112-235) without file I/O: sharpness [F] per frame,
    R [F,3,3], t [F,3] (read_Rt's float64 world-to-camera), K [3,3] float64, depth [F,h,w] per frame, either camera-z
    float32 (numpy or CUDA) or SUN3D's raw uint16 (decoded by sun3d_depth), baseline_range (lo, hi), img_ids [F] the frame
    ids of the group names (default 0..F-1).  The NMS and the geometric filters run on the host in float64, the valid
    depth counts and every consistency check on the device; see group_views for the result and its quirks."""
    R, t = np.asarray(R, dtype=np.float64), np.asarray(t, dtype=np.float64)
    sharp = sharp_frames(sharpness, sharpness_window)
    if isinstance(depth, torch.Tensor) and depth.dtype == torch.float32:
        d = depth.to(_device())
        valid = torch.count_nonzero(torch.isfinite(d) & (d > 0), dim=(1, 2)).cpu().numpy() if len(d) else np.zeros(0)
    elif isinstance(depth, torch.Tensor) or np.asarray(depth).dtype == np.uint16:
        d, valid = sun3d_depth(depth)
        valid = valid.cpu().numpy()
    else:
        a = np.asarray(depth)
        if a.dtype != np.float32:
            raise ValueError("depth must be float32 camera z or uint16 SUN3D depth, got %s" % (a.dtype,))
        valid = np.count_nonzero(np.isfinite(a) & (a > 0), axis=(1, 2))
        d = torch.from_numpy(np.ascontiguousarray(a)).to(_device())
    if d.dim() != 3 or d.shape[0] != len(R):
        raise ValueError("depth must be [F,h,w] for the F = %d frames, got %s" % (len(R), tuple(d.shape)))
    size = d.shape[1] * d.shape[2]
    _check_pixels(d.shape[1], d.shape[2], "depth")
    index = torch.from_numpy(np.asarray(sharp, dtype=np.int64)).to(d.device)
    consistent = _device_consistency(sharp, R, t, np.asarray(K, dtype=np.float64), lambda pos: d[index[pos]].contiguous(), valid,
                                     size, baseline_range)
    return group_views(sharp, R, t, valid, size, baseline_range, consistent, max_views_num, img_ids)


# ---- SUN3D directories (sun3d_utils.py) ---------------------------------------------------------------------------------
def _read_image(filename):
    from PIL import Image
    image = Image.open(filename)
    image.load()
    return image


def _read_frameid_timestamp(files):
    ids = [f[:-4].split('-') for f in files]
    return np.asarray([int(i[0]) for i in ids]), np.asarray([int(i[1]) for i in ids])


def read_Rt(extrinsics, frame):
    """sun3d_utils.read_Rt: (R, t) world-to-camera of frame from the camera-to-world rows of the extrinsics file."""
    Rt = extrinsics[3 * frame:3 * frame + 3]
    R = Rt[0:3, 0:3].transpose()
    return R, -np.dot(R, Rt[0:3, 3])


def sun3d_view_groups(sun3d_data_path, seq_name, baseline_range, sharpness, sharpness_window=30, max_views_num=10):
    """The groups create_samples_from_sequence would write for a SUN3D sequence (image/*.jpg, depthTSDF/*.png,
    extrinsics/*.txt, intrinsics.txt), each as group_views' dict plus 'name' (the HDF5 group name).  The files are read
    with Pillow and np.loadtxt like the reference; only the depth maps of the sharp frames are read, and they go to the
    device UPLOAD_FRAMES at a time.  A sequence without extrinsics has no groups."""
    from PIL import Image
    seq_path = os.path.join(sun3d_data_path, seq_name)
    prefix = seq_name.replace('/', '.')
    if not os.path.exists(os.path.join(seq_path, 'extrinsics')):
        return []
    image_files = [f for f in sorted(os.listdir(os.path.join(seq_path, 'image'))) if f.endswith('.jpg')]
    depth_files = [f for f in sorted(os.listdir(os.path.join(seq_path, 'depthTSDF'))) if f.endswith('.png')]
    extrinsics_files = [f for f in sorted(os.listdir(os.path.join(seq_path, 'extrinsics'))) if f.endswith('.txt')]
    K = np.loadtxt(os.path.join(seq_path, 'intrinsics.txt'))
    extrinsics = np.loadtxt(os.path.join(seq_path, 'extrinsics', extrinsics_files[-1]))
    img_ids, img_timestamps = _read_frameid_timestamp(image_files)
    _, depth_timestamps = _read_frameid_timestamp(depth_files)
    idx_img2depth = [np.argmin(abs(depth_timestamps[:] - ts)) for ts in img_timestamps]
    sharpness = np.asarray(sharpness)
    assert sharpness.size == len(image_files)
    sharp = sharp_frames(sharpness, sharpness_window)
    F = len(image_files)
    Rt = [read_Rt(extrinsics, f) if 3 * f + 3 <= len(extrinsics) else (None, None) for f in range(F)]
    R = np.full((F, 3, 3), np.nan)
    t = np.full((F, 3), np.nan)
    for f in sharp:
        R[f], t[f] = Rt[f]
    # the sharp frames' depths, decoded on the device in chunks; `rows` maps a sharp position to its row
    chunks, valid = [], np.zeros((F,), dtype=np.int64)
    for s in range(0, len(sharp), UPLOAD_FRAMES):
        part = sharp[s:s + UPLOAD_FRAMES]
        raw = np.stack([np.array(Image.open(os.path.join(seq_path, 'depthTSDF', depth_files[idx_img2depth[f]]))).astype(np.uint16)
                        for f in part])
        dd, vv = sun3d_depth(raw)
        chunks.append(dd)
        valid[part] = vv.cpu().numpy()
    if not chunks:
        return []
    d = torch.cat(chunks)
    size = d.shape[1] * d.shape[2]
    _check_pixels(d.shape[1], d.shape[2], "depth")
    consistent = _device_consistency(sharp, R, t, K, lambda pos: d[torch.as_tensor(pos, device=d.device)].contiguous(), valid, size,
                                     baseline_range)
    groups = group_views(sharp, R, t, valid, size, baseline_range, consistent, max_views_num, img_ids)
    for g in groups:
        g['name'] = prefix + g['suffix']
    return groups
