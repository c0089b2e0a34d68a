"""ORACLE (test infrastructure, not product code): the per-pixel compute and the pose math of the reference's multi-view
training reader (multivih5datareaderop/multivih5datareader.cpp) restated in numpy.

The reader itself cannot be built here (it needs Eigen, OpenCV, HDF5, webp and lz4), so this is a restatement, not a
run of the reference: every float step follows the reader's float32 operation order (line numbers at each step) with
numpy's IEEE float32 element-wise ops, which are not contracted into FMAs, as the reference's x86 build is not.  Where
the reader calls into Eigen or OpenCV, the published algorithm is restated and says so:
  - Matrix products sum left to right, the 3x3 inverse is cofactors times 1/det (as oracle/ref_stub/eigen_stub.h);
  - the 4x4 determinant, Quaternion(Matrix3d) and AngleAxis(Quaternion) are Eigen 3.3's formulas;
  - cv::resize INTER_AREA for downscaling is OpenCV's three paths (below; DESIGN.md section 3.8) and INTER_NEAREST is
    sx = floor(x * (1 / (dw / sw))), clamped.  Both are held bit for bit to OpenCV 4.13.0's results
    (tests/test_datareader_opencv.py and tests/golden/datareader_resize_digests.json); the reference's build used
    OpenCV 2.4.9, whose resize code is believed to be the same but has not been run against this.
The pose math is float64.  The flips are applied as the reader applies them: the whole plane reversed, rows reversed.
"""
import math

import numpy as np

f32 = np.float32
_NAN = np.array([0x7fc00000], np.uint32).view(np.float32)[0]   # the C macro NAN


# ---- prepareScene (:1384-1520) -----------------------------------------------------------------------------------------
# cv::resize(INTER_AREA) of uint8 images, downscaling only (imgproc/src/resize.cpp), in one of three paths per view:
#   '2x2'      both axes at the integer factor 2: (a + b + c + d + 2) >> 2, half up (ResizeAreaFastVec);
#   'fast'     both axes at an integer factor, any other pair: float(int block sum) * (1.f / area), cvRound (resizeAreaFast_);
#   'general'  otherwise: computeResizeAreaTab's float weights, float accumulation (ResizeArea_Invoker).
# An axis takes an integer factor when |scale - cvRound(scale)| < DBL_EPSILON for scale = 1 / (dsize / (double)ssize):
# not the same as "ssize divisible by dsize" (98 -> 2 is divisible, and its scale 49.00000000000001 is not integral).
DBL_EPSILON = float(np.finfo(np.float64).eps)


def area_scale(n, m):
    """cv::resize's scale along an axis of n source cells -> m output cells: 1 / inv_scale, inv_scale = m / (double)n."""
    return 1.0 / (m / float(n))


def area_factor(n, m):
    """The integer factor of n -> m when INTER_AREA's integer test passes along that axis, else None."""
    s = area_scale(n, m)
    k = round(s)   # saturate_cast<int>(double) is cvRound: half to even, as Python's round
    return k if abs(s - k) < DBL_EPSILON else None


def area_path(sh, sw, h, w):
    """'2x2', 'fast' or 'general': which of INTER_AREA's paths an sh x sw -> h x w downscale takes."""
    ky, kx = area_factor(sh, h), area_factor(sw, w)
    if ky is None or kx is None:
        return 'general'
    return '2x2' if (ky, kx) == (2, 2) else 'fast'


def area_table(n, m):
    """computeResizeAreaTab for n -> m as [m, K] source indices and float32 weights: row d holds output d's entries in the
    table's order (the leading partial cell, the full cells, the trailing partial cell; consecutive source cells), padded
    with (0, +0).  Every step is the double arithmetic of the table, element-wise."""
    scale = area_scale(n, m)
    fs1 = np.arange(m) * scale
    fs2 = fs1 + scale
    cell = np.minimum(scale, n - fs1)
    s2 = np.minimum(np.floor(fs2), n - 1)
    s1 = np.minimum(np.ceil(fs1), s2)
    lead, trail = s1 - fs1 > 1e-3, fs2 - s2 > 1e-3
    lo = np.where(lead, s1 - 1, s1).astype(np.int64)
    hi = np.where(trail, s2, s2 - 1).astype(np.int64)
    k = int((hi - lo).max()) + 1
    idx = lo[:, None] + np.arange(k)[None, :]
    wt = np.broadcast_to((1.0 / cell).astype(np.float32)[:, None], (m, k)).copy()
    wt[lead, 0] = ((s1 - fs1) / cell).astype(np.float32)[lead]
    rows = np.nonzero(trail)[0]
    wt[rows, (hi - lo)[rows]] = (np.minimum(np.minimum(fs2 - s2, 1.0), cell) / cell).astype(np.float32)[rows]
    pad = idx > hi[:, None]
    idx[pad], wt[pad] = 0, 0
    return idx, wt


def _area_general(img, h, w):
    sh, sw = img.shape[:2]
    xi, xa = area_table(sw, w)
    yi, ya = area_table(sh, h)
    src = img.astype(np.float32)
    # horizontal: buf[dx] = buf[dx] + S[sx] * alpha per source row, in the x table's order (a padded +0 term adds nothing)
    buf = np.zeros((sh, w, img.shape[2]), np.float32)
    for k in range(xi.shape[1]):
        buf = buf + src[:, xi[:, k]] * xa[None, :, k, None]
    # vertical: sum = beta * buf for an output row's first source row, then sum = sum + beta * buf
    acc = ya[:, 0, None, None] * buf[yi[:, 0]]
    for k in range(1, yi.shape[1]):
        acc = acc + ya[:, k, None, None] * buf[yi[:, k]]
    return np.clip(np.rint(acc), 0, 255).astype(np.uint8)   # saturate_cast<uchar>: cvRound, half to even


def area_downscale(img, h, w):
    """cv::resize(img, (w, h), INTER_AREA) of a uint8 [sh, sw, c] image with h <= sh and w <= sw."""
    img = np.asarray(img, np.uint8)
    sh, sw = img.shape[:2]
    assert h <= sh and w <= sw, "INTER_AREA's upscaling is not restated"
    path = area_path(sh, sw, h, w)
    if path == 'general':
        return _area_general(img, h, w)
    ky, kx = sh // h, sw // w
    blocks = img.reshape(h, ky, w, kx, img.shape[2]).astype(np.int64).sum((1, 3))
    if path == '2x2':
        return ((blocks + 2) >> 2).astype(np.uint8)
    blocks = ((blocks + 2 ** 31) % 2 ** 32 - 2 ** 31).astype(np.int32)   # the sum is an int: it wraps above 2^31 - 1
    scale = f32(1) / f32(kx * ky)   # 1.f / area: above 2^24 the area itself is rounded to float first
    return np.clip(np.rint(blocks.astype(np.float32) * scale), 0, 255).astype(np.uint8)


def nearest_indices(n, m):   # cv::resize INTER_NEAREST: cvFloor(x * ifx), ifx = 1 / (m / (double)n), clamped
    ifx = 1.0 / (m / float(n))
    return np.minimum(np.array([math.floor(x * ifx) for x in range(m)]), n - 1)


def half_to_float(d):
    """float16 -> float32, exact; a NaN keeps sign and payload."""
    h = np.asarray(d, np.float16)
    out = h.astype(np.float32)
    bits = h.view(np.uint16).astype(np.uint32)
    nan = np.isnan(h)
    out_bits = out.view(np.uint32)
    out_bits[nan] = ((bits[nan] & 0x8000) << 16) | 0x7f800000 | ((bits[nan] & 0x3ff) << 13)
    return out


def inverse3(K):
    """Eigen's fixed 3x3 inverse (InverseImpl.h compute_inverse<.,.,3>) in the matrix's precision: cofactors times 1/det."""
    m = K
    def cof(i, j):
        i1, i2, j1, j2 = (i + 1) % 3, (i + 2) % 3, (j + 1) % 3, (j + 2) % 3
        return m[i1, j1] * m[i2, j2] - m[i1, j2] * m[i2, j1]
    c0, c1, c2 = cof(0, 0), cof(1, 0), cof(2, 0)
    det = (c0 * m[0, 0] + c1 * m[1, 0]) + c2 * m[2, 0]
    invdet = m.dtype.type(1) / det
    r = np.empty((3, 3), m.dtype)
    for i in range(3):
        for j in range(3):
            r[i, j] = cof(j, i) * invdet
    return r


def scaled_k(cam, h, w):
    """cam.K.cast<float>() with K(0,0), K(0,2) times the width and K(1,1), K(1,2) times the height (:372-376)."""
    K = np.array([[cam[0], cam[1], cam[2]], [0, cam[3], cam[4]], [0, 0, 1]], np.float64).astype(np.float32)
    K[0, 0] *= f32(w)
    K[1, 1] *= f32(h)
    K[0, 2] *= f32(w)
    K[1, 2] *= f32(h)
    return K


def prepare(image, depth, K, R, t, depth_metric, w, h):
    """prepareScene for one view: (image uint8 [h,w,3], depth float32 [h,w] camera z, cam float64 [17])."""
    sh, sw = image.shape[:2]
    cam = np.zeros(17)
    cam[:5] = (K[0, 0] / sw, K[0, 1], K[0, 2] / sw, K[1, 1] / sh, K[1, 2] / sh)   # :1393-1396
    cam[5:14] = np.asarray(R, np.float64).reshape(-1)
    cam[14:] = np.asarray(t, np.float64).reshape(-1)
    img = area_downscale(np.asarray(image, np.uint8), h, w)
    d = half_to_float(depth) if np.asarray(depth).dtype == np.float16 else np.asarray(depth, np.float32)
    d = d[nearest_indices(sh, h)][:, nearest_indices(sw, w)].copy()
    if depth_metric == 'ray_length':   # :1489-1511
        ik = inverse3(scaled_k(cam, h, w))
        px = ik[0, 0] * (np.arange(w, dtype=np.float32) + f32(0.5)) + ik[0, 2]
        py = ik[1, 1] * (np.arange(h, dtype=np.float32) + f32(0.5)) + ik[1, 2]
        px, py = np.broadcast_to(px[None, :], (h, w)), np.broadcast_to(py[:, None], (h, w))
        norm = np.sqrt((px * px + py * py) + f32(1) * f32(1))
        d = d / norm
    return img, d, cam


# ---- pose math, float64 (:1650-1813) -------------------------------------------------------------------------------------
def _mm(A, B):
    out = np.empty((A.shape[0], B.shape[1]), A.dtype)
    for i in range(A.shape[0]):
        for j in range(B.shape[1]):
            s = A[i, 0] * B[0, j]
            for k in range(1, A.shape[1]):
                s = s + A[i, k] * B[k, j]
            out[i, j] = s
    return out


def _mv(A, v):
    return _mm(A, v.reshape(-1, 1)).reshape(-1)


def _norm(v):
    return math.sqrt(float((v[0] * v[0] + v[1] * v[1]) + v[2] * v[2]))


def _quaternion(m):   # Eigen 3.3 quaternion_assign_impl<Other,3,3>
    q = np.zeros(4)   # x, y, z, w
    t = (m[0, 0] + m[1, 1]) + m[2, 2]
    if t > 0:
        t = math.sqrt(t + 1.0)
        q[3] = 0.5 * t
        t = 0.5 / t
        q[0] = (m[2, 1] - m[1, 2]) * t
        q[1] = (m[0, 2] - m[2, 0]) * t
        q[2] = (m[1, 0] - m[0, 1]) * t
    else:
        i = 0
        if m[1, 1] > m[0, 0]:
            i = 1
        if m[2, 2] > m[i, i]:
            i = 2
        j = (i + 1) % 3
        k = (j + 1) % 3
        t = math.sqrt(((m[i, i] - m[j, j]) - m[k, k]) + 1.0)
        q[i] = 0.5 * t
        t = 0.5 / t
        q[3] = (m[k, j] - m[j, k]) * t
        q[j] = (m[j, i] + m[i, j]) * t
        q[k] = (m[k, i] + m[i, k]) * t
    return q


def _angle_axis(m):   # Eigen 3.3 AngleAxis::operator=(QuaternionBase), then axis()*angle() (:253-260)
    q = _quaternion(m)
    v = q[:3]
    n = _norm(v)
    if n < np.finfo(np.float64).eps:
        s = np.max(np.abs(v))
        n = 0.0 if s == 0 else s * _norm(v / s)
    if n == 0:
        return np.zeros(3)
    angle = 2.0 * math.atan2(n, abs(q[3]))
    if q[3] < 0:
        n = -n
    return (v / n) * angle


def _det4(m):   # Eigen 3.3 Determinant.h determinant_impl<Derived,4>
    def h(j, k, a, b):
        return (m[j, 0] * m[k, 1] - m[k, 0] * m[j, 1]) * (m[a, 2] * m[b, 3] - m[b, 2] * m[a, 3])
    return ((((h(0, 1, 2, 3) - h(0, 2, 1, 3)) + h(0, 3, 1, 2)) + h(1, 2, 0, 3)) - h(1, 3, 0, 2)) + h(2, 3, 0, 1)


def _fundamental(P1, P2):   # computeFundamentalFromCameras (:264-304)
    X = [P1[[1, 2]], P1[[2, 0]], P1[[0, 1]]]
    Y = [P2[[1, 2]], P2[[2, 0]], P2[[0, 1]]]
    F = np.empty((3, 3))
    for i in range(3):
        for j in range(3):
            F[i, j] = _det4(np.concatenate([X[j], Y[i]]))
    return F


def _k(cam):
    return np.array([[cam[0], cam[1], cam[2]], [0, cam[3], cam[4]], [0, 0, 1]], np.float64)


def motion(cam1, cam2, rot180, mirror_x, motion_format, norm_trans_scale_depth):
    """(motion float64, depth_scale_factor) of one pair, or None where the reader `continue`s (:1680, :1765)."""
    R1, t1 = cam1[5:14].reshape(3, 3).copy(), cam1[14:].copy()
    R2, t2 = cam2[5:14].reshape(3, 3).copy(), cam2[14:].copy()
    if rot180:   # rotateCamera180DegAroundZ (:307-313)
        for R, t in ((R1, t1), (R2, t2)):
            C = _mv(-R.T, t)
            R[0] = -R[0]
            R[1] = -R[1]
            t[:] = _mv(-R, C)
    R12 = _mm(R2, R1.T)
    t12 = t2 - _mv(R12, t1)
    if mirror_x:   # :1669-1676
        C2 = _mv(-R12.T, t12)
        C2[0] = -C2[0]
        R12[:, 0] *= -1
        R12[0, :] *= -1
        t12 = _mv(-R12, C2)
    n = _norm(t12)
    if n < 1e-6:
        return None
    dsf = 1.0
    if norm_trans_scale_depth:
        dsf = 1 / n
        t12 = t12 / n
    if motion_format == 'ANGLEAXIS6':
        return np.concatenate([_angle_axis(R12), t12]), dsf
    if motion_format == 'ANGLEAXIS7':
        aa = _angle_axis(R12)
        mag = _norm(aa)
        aa = np.zeros(3) if mag < 1e-6 else aa / mag
        return np.concatenate([[mag], aa, t12]), dsf
    if motion_format == 'QUATERNION':
        q = _quaternion(R12)
        return np.concatenate([[q[3]], q[:3], t12]), dsf
    P1 = _mm(_k(cam1), np.concatenate([R1, t1[:, None]], 1))
    P2 = _mm(_k(cam2), np.concatenate([R2, t2[:, None]], 1))
    F = _fundamental(P1, P2)
    if abs(F[2, 2]) < 1e-6:   # the reader computes normalizer = 1/F(2,2) first; unused when it skips
        return None
    normalizer = 1 / F[2, 2]
    return np.array([F[i, j] * normalizer for j in range(3) for i in range(3)][:8]), dsf


# ---- per-pixel outputs -------------------------------------------------------------------------------------------------
def _min(a, b):
    return np.where(b < a, b, a)


def _max(a, b):
    return np.where(a < b, b, a)


def _saturate(v):
    return _max(f32(0), _min(f32(1), v))


def fast_powf(a, b):   # :633-638 with x86's int wrap and cvttss2si (out of range -> INT_MIN)
    x = a.view(np.int32).astype(np.int64) - 1064866805
    x = ((x + 2 ** 31) % 2 ** 32 - 2 ** 31).astype(np.int32)
    f = f32(b) * x.astype(np.float32) + np.float32(1064866805)
    fd = f.astype(np.float64)
    ok = (fd > -2147483649.0) & (fd < 2147483648.0)
    r = np.where(ok, np.trunc(np.where(ok, fd, 0)), -2 ** 31).astype(np.int32)
    return r.view(np.float32)


def augment(layers, aug):   # augmentImage (:676-711) on one image [3,h,w]
    hue, sat, val, contrast, brightness, gamma = (f32(a) for a in aug)
    r, g, b = layers[2] + f32(0.5), layers[1] + f32(0.5), layers[0] + f32(0.5)
    mn = _min(r, _min(g, b))   # rgb2hsv (:547-559)
    v = _max(r, _max(g, b))
    den = (v - mn) + f32(1e-6)
    h = np.where(r == v, f32(60) * (g - b) / den,
                 np.where(g == v, f32(120) + f32(60) * (r - g) / den, f32(240) + f32(60) * (r - g) / den))
    s = (v - mn) / (v + f32(1e-6))
    h = h + hue
    while np.any(h < 0):
        h = np.where(h < 0, h + f32(360), h)
    while np.any(h >= 360):
        h = np.where(h >= 360, h - f32(360), h)
    s = _saturate(s + sat)
    v = _saturate(v + val)
    hh = h / f32(60)   # hsv2rgb (:561-612)
    i = np.floor(hh).astype(np.int32)
    f = hh - i.astype(np.float32)
    p = v * (f32(1) - s)
    q = v * (f32(1) - s * f)
    t = v * (f32(1) - s * (f32(1) - f))
    cases = [i == 0, i == 1, i == 2, i == 3, i == 4]
    rr = np.select(cases, [v, q, p, p, t], v)
    gg = np.select(cases, [t, v, v, q, p], p)
    bb = np.select(cases, [p, p, t, v, v], q)
    grey = s == 0
    rgb = [np.where(grey, v, rr), np.where(grey, v, gg), np.where(grey, v, bb)]
    for c in range(3):
        value = ((rgb[c] - f32(0.5)) * contrast + brightness) + f32(0.5)
        rgb[c] = _saturate(fast_powf(value, gamma))
    return np.stack([rgb[2] - f32(0.5), rgb[1] - f32(0.5), rgb[0] - f32(0.5)])


def _project(cam1, cam2, depth, h, w):
    """computeFlow / computeDepthmask's p1 and p2 for every pixel of cam1 (:372-418); depth is camera z."""
    ik = inverse3(scaled_k(cam1, h, w))
    K2 = scaled_k(cam2, h, w)
    P2 = _mm(K2, np.concatenate([cam2[5:14].reshape(3, 3), cam2[14:, None]], 1).astype(np.float32))
    t = cam1[14:].astype(np.float32)
    inv_R = cam1[5:14].reshape(3, 3).T.astype(np.float32)
    p1x = np.broadcast_to(np.arange(w, dtype=np.float32)[None, :] + f32(0.5), (h, w))
    p1y = np.broadcast_to(np.arange(h, dtype=np.float32)[:, None] + f32(0.5), (h, w))
    s = depth / f32(1)
    pos = [(ik[0, 0] * p1x + ik[0, 2]) * s, (ik[1, 1] * p1y + ik[1, 2]) * s, f32(1) * s]
    pos = [pos[i] - t[i] for i in range(3)]
    q = [(inv_R[i, 0] * pos[0] + inv_R[i, 1] * pos[1]) + inv_R[i, 2] * pos[2] for i in range(3)]
    p2 = [((P2[i, 0] * q[0] + P2[i, 1] * q[1]) + P2[i, 2] * q[2]) + P2[i, 3] * f32(1) for i in range(3)]
    return p1x, p1y, p2[0] / p2[2], p2[1] / p2[2]


def flow(cam1, cam2, depth, h, w):   # computeFlow (:370-424)
    with np.errstate(all='ignore'):
        p1x, p1y, p2x, p2y = _project(cam1, cam2, depth, h, w)
        bad = (depth <= 0) | ~np.isfinite(depth)
        return np.stack([np.where(bad, _NAN, p2x - p1x), np.where(bad, _NAN, p2y - p1y)]).astype(np.float32)


def depthmask(cam1, cam2, depth, h, w, border1, border2):   # computeDepthmask (:431-498)
    with np.errstate(all='ignore'):
        p1x, p1y, p2x, p2y = _project(cam1, cam2, depth, h, w)
        x = np.arange(w)[None, :]
        y = np.arange(h)[:, None]
        border = (x < border1) | (y < border1) | (x >= w - border1) | (y >= h - border1)
        bad = (depth <= 0) | ~np.isfinite(depth)
        out2 = (p2x < f32(border2)) | (p2y < f32(border2)) | (p2x >= f32(w - border2)) | (p2y >= f32(h - border2))
        return np.where(border | bad | out2, f32(0), f32(1)).astype(np.float32)


def _rotate180(a):   # rotateImageBy180: every plane reversed as a whole
    return a[..., ::-1, ::-1].copy()


def _mirror(a):   # mirrorImageX: every row reversed
    return a[..., ::-1].copy()


def build_batch(views, pairs, params, rot180, mirror_x, colour):
    """The batch loop (:1585-1950) on prepared views [(image, depth, cam)] for a full parameter dict (defaults filled).
    Returns ({name: float32 array}, used pair indices)."""
    b = int(params['batch_size'])
    h, w = views[0][1].shape
    rmin, rmax = f32(params['image_range_min']), f32(params['image_range_max'])
    scale = (rmax - rmin) / f32(255)
    nd = 2 if params['depth_pair'] else 1
    out = {'IMAGE_PAIR': np.empty((b, 6, h, w), np.float32), 'MOTION': None, 'FLOW': np.empty((b, 2, h, w), np.float32),
           'DEPTH': np.empty((b, nd, h, w), np.float32), 'INTRINSICS': np.empty((b, 4), np.float32),
           'DEPTHMASKS': np.empty((b, nd, h, w), np.float32)}
    used = []
    k = 0
    for s in range(b):
        rot, mir = bool(rot180[s]), bool(mirror_x[s])
        while True:
            if k >= len(pairs):
                raise ValueError("too few usable pairs")
            i1, i2 = int(pairs[k][0]), int(pairs[k][1])
            k += 1
            res = motion(views[i1][2], views[i2][2], rot, mir, params['motion_format'], params['norm_trans_scale_depth'])
            if res is not None:
                break
        used.append(k - 1)
        (img1, d1, c1), (img2, d2, c2) = views[i1], views[i2]
        mot, dsf = res
        if out['MOTION'] is None:
            out['MOTION'] = np.empty((b, len(mot)), np.float64)   # float64: the reader's values before the float cast
        out['MOTION'][s] = mot
        # images (:1614-1647): RGB layers (:344-363), rot180, mirror, then the colour step
        ip = np.concatenate([scale * img.transpose(2, 0, 1).astype(np.float32) + rmin for img in (img1, img2)])
        if rot:
            ip = _rotate180(ip)
        if mir:
            ip = _mirror(ip)
        if colour is not None:
            ip = np.concatenate([augment(ip[0:3], colour[s]), augment(ip[3:6], colour[s])])
        out['IMAGE_PAIR'][s] = ip
        # intrinsics (:1784-1814), float
        fx, fy, cx, cy = f32(c1[0]), f32(c1[3]), f32(c1[2]), f32(c1[4])
        if rot:
            cx, cy = f32(1) - cx, f32(1) - cy
        if mir:
            cx = f32(1) - cx
        out['INTRINSICS'][s] = (fx, fy, cx, cy)
        # flow (:1817-1844)
        fl = flow(c1, c2, d1, h, w)
        if rot:
            fl = -_rotate180(fl)
        if mir:
            fl = _mirror(fl)
            fl[0] = -fl[0]
        out['FLOW'][s] = fl
        # depth (:1847-1909)
        dep = np.stack([d1, d2][:nd]).copy()
        with np.errstate(all='ignore'):
            mx, mn = f32(params['max_depth']), f32(params['min_depth'])
            invalid = (dep == 0) | ((mx > 0) & (dep > mx)) | ((mn > 0) & (dep < mn))
            val = (dep.astype(np.float64) * dsf).astype(np.float32)
            if params['inverse_depth']:
                val = f32(1) / val
            dep = np.where(invalid, _NAN, val).astype(np.float32)
        if rot:
            dep = _rotate180(dep)
        if mir:
            dep = _mirror(dep)
        out['DEPTH'][s] = dep
        # depth masks (:1911-1941)
        b1, b2 = int(params['depthmask_border1']), int(params['depthmask_border2'])
        dm = [depthmask(c1, c2, d1, h, w, b1, b2)]
        if params['depth_pair']:
            dm.append(depthmask(c2, c1, d2, h, w, b1, b2))
        dm = np.stack(dm)
        if rot:
            dm = _rotate180(dm)
        if mir:
            dm = _mirror(dm)
        out['DEPTHMASKS'][s] = dm
    return {kk: out[kk] for kk in params['top_output']}, np.asarray(used)


# ---- synthetic scenes for the tests and the benchmark ----------------------------------------------------------------------
def _rotation(axis, angle):
    axis = np.asarray(axis, np.float64)
    axis = axis / np.linalg.norm(axis)
    x, y, z = axis
    c, s = math.cos(angle), math.sin(angle)
    return np.array([[c + x * x * (1 - c), x * y * (1 - c) - z * s, x * z * (1 - c) + y * s],
                     [y * x * (1 - c) + z * s, c + y * y * (1 - c), y * z * (1 - c) - x * s],
                     [z * x * (1 - c) - y * s, z * y * (1 - c) + x * s, c + z * z * (1 - c)]])


def synthetic_views(n, height, width, seed, skew=0.0, centred=False, depth_dtype=np.float32, depth_metric='camera_z'):
    """n (R, t, K, image, depth, depth_metric) tuples of a smooth scene seen from nearby cameras: uint8 images with
    texture, depths in about [1.5, 4.5]."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:height, 0:width].astype(np.float64)
    fx, fy = width * rng.uniform(0.8, 1.0), height * rng.uniform(1.05, 1.35)
    cx, cy = (width / 2, height / 2) if centred else (width * rng.uniform(0.4, 0.6), height * rng.uniform(0.4, 0.6))
    K = np.array([[fx, skew, cx], [0, fy, cy], [0, 0, 1]])   # one camera for the whole sequence
    out = []
    for _ in range(n):
        R = _rotation(rng.normal(size=3), rng.uniform(0.0, 0.15))
        t = rng.normal(scale=0.3, size=3)
        depth = 3 + np.sin(xx / width * rng.uniform(2, 6) + rng.uniform(0, 6)) + 0.5 * np.cos(yy / height * rng.uniform(2, 6))
        img = np.clip(128 + 60 * np.sin(xx / rng.uniform(3, 9))[..., None] * np.cos(yy / rng.uniform(3, 9))[..., None]
                      + rng.normal(scale=25, size=(height, width, 3)), 0, 255).astype(np.uint8)
        out.append((R, t, K, img, depth.astype(depth_dtype), depth_metric))
    return out
