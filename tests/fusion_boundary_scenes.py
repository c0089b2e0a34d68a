"""Scenes for the fusion boundary tests (tests/test_fusion_boundaries.py on the CPU, tests/test_gpu_fusion_boundaries.py
on the device): sphere views with their own intrinsics for every frame, a grid-aligned plane whose fused state is known in
closed form, and an analytic field for meshes of more than 1024 tiles of 2048 cubes."""
import numpy as np

import sequence_oracle as so

f32 = np.float32


def varied_sphere_views(n, h=48, w=64, seed=0):
    """so.sphere_views' cameras, each frame with its own fx, fy, cx and cy, and its depth rendered through them: depth
    [n,h,w], K, R [n,3,3], t [n,3] float32, images [n,h,w,3] uint8.  3 % of the finite depths each are NaN, 0, -1 and inf.
    A mix-up of K, R, t or the depth map between two frames changes voxels."""
    _, _, R, t, img = so.sphere_views(n=n, h=h, w=w, seed=seed)
    rng = np.random.RandomState(seed)
    f = 60.0 * w / 64 * rng.uniform(0.85, 1.15, n)
    K = np.zeros((n, 3, 3))
    K[:, 0, 0], K[:, 1, 1] = f, f * rng.uniform(0.9, 1.1, n)
    K[:, 0, 2], K[:, 1, 2] = w / 2 + rng.uniform(-3, 3, n) * w / 64, h / 2 + rng.uniform(-3, 3, n) * h / 48
    K[:, 2, 2] = 1.0
    K = K.astype(f32)
    d = np.array([so.render_depth(R[k], t[k], K[k], h, w, sphere=((0, 0, 0), 0.6)) for k in range(n)], dtype=f32)
    for bad in (np.nan, 0.0, -1.0, np.inf):
        m = rng.rand(*d.shape) < 0.03
        d[m & np.isfinite(d)] = bad
    return d, K, R, t, img


# ---- the grid-aligned plane -------------------------------------------------------------------------------------------
# Voxel 1/8 and trunc 1/2; cameras with R = I, fx = fy = 16, integer cx and cy, and translations that are multiples of 1/8
# in x and y and 0 in z; every pixel sees the plane world z = 2 at depth 2.  All of it is dyadic with few bits, so every
# float32 operation of integration and allocation is exact.  In the slice z = 2 a voxel projects to u = 8 x + cx, an
# integer, so voxels land exactly on u = 0 and u = w (and v = 0, v = h); elsewhere u is a fraction 16 a / b + cx
# (x = a/8, z = b/8) at least 1/b from an integer, so its rounding never crosses one.  The fused state is the closed form
# of plane_state: tsdf = f(z) = min(1, (2 - z) / trunc), the same in every frame, reaching -1 exactly at z = 2 + trunc.
VOXEL, TRUNC, PLANE_Z = 0.125, 0.5, 2.0
H, W = 24, 32
ORIGIN = (-4.0, -3.0, 0.25)   # voxel planes on multiples of 1/8, block faces on z = 0.25 + integer
DIMS = (65, 49, 23)           # x in [-4, 4], y in [-3, 3], z in [0.25, 3]
_O8 = (-32, -24, 2)           # ORIGIN in units of 1/8


def plane_cameras(n=129):
    """Integer cx [n], cy [n] and translations in units of 1/8, tx8 [n], ty8 [n] (tz = 0): 7 x 7 principal points and
    17 x 13 shifts, so that neighbouring voxels see different numbers of frames."""
    f = np.arange(n)
    return 13 + (3 * f) % 7, 9 + (5 * f) % 7, (7 * f) % 17 - 8, (11 * f) % 13 - 6


def plane_frames(n=129, seed=0):
    """depth [n,h,w] = 2, K, R = I [n,3,3], t [n,3] float32 and random images [n,h,w,3] uint8 of the plane scene."""
    cx, cy, tx8, ty8 = plane_cameras(n)
    K = np.zeros((n, 3, 3), f32)
    K[:, 0, 0] = K[:, 1, 1] = 16.0
    K[:, 0, 2], K[:, 1, 2], K[:, 2, 2] = cx, cy, 1.0
    R = np.broadcast_to(np.eye(3, dtype=f32), (n, 3, 3)).copy()
    t = np.stack([tx8 / 8.0, ty8 / 8.0, np.zeros(n)], axis=1).astype(f32)
    img = np.random.RandomState(seed).randint(0, 256, (n, H, W, 3)).astype(np.uint8)
    return np.full((n, H, W), PLANE_Z, f32), K, R, t, img


def plane_state(g, n=129):
    """The closed form of n plane frames integrated into the voxels at integer grid coordinates g [N,3] (x, y, z) from
    ORIGIN: tsdf and weight float32 [N], and counts of the (voxel, frame) updates that land on a boundary.

    Frame k updates voxel X when z > 0, its pixel (floor(u), floor(v)) is in the image, and sdf = 2 - z >= -trunc; then
    f = min(1, sdf / trunc).  Everything is computed on integers: with x8 = 8 x (camera), z8 = 8 z, u = (16 x8 + cx z8) / z8."""
    g = np.asarray(g, dtype=np.int64).reshape(-1, 3)
    X8 = [g[:, a] + _O8[a] for a in range(3)]
    z8 = X8[2]
    sdf8 = 8 * int(PLANE_Z) - z8                    # 8 (d - z)
    near = sdf8 >= -8 * TRUNC                       # not skipped by sdf < -trunc
    weight = np.zeros(len(g), np.int64)
    edges = {"u=0": 0, "u=w": 0, "v=0": 0, "v=h": 0, "sdf=-trunc": 0}
    for cx, cy, tx8, ty8 in zip(*plane_cameras(n)):
        un, vn = 16 * (X8[0] + tx8) + cx * z8, 16 * (X8[1] + ty8) + cy * z8   # u z8 and v z8
        front = z8 > 0
        zs = np.where(front, z8, 1)
        px, py = un // zs, vn // zs
        seen = front & (px >= 0) & (px < W) & (py >= 0) & (py < H) & near
        weight += seen
        exact = front & near & (py >= 0) & (py < H)
        edges["u=0"] += int((exact & (un == 0)).sum())
        edges["u=w"] += int((exact & (un == W * zs)).sum())
        exact = front & near & (px >= 0) & (px < W)
        edges["v=0"] += int((exact & (vn == 0)).sum())
        edges["v=h"] += int((exact & (vn == H * zs)).sum())
        edges["sdf=-trunc"] += int((seen & (sdf8 == -8 * TRUNC)).sum())
    fv = np.minimum(1.0, sdf8 / (8 * TRUNC))
    return np.where(weight > 0, fv, 0.0).astype(f32), weight.astype(f32), edges


def box_grid(dims=DIMS):
    """Grid coordinates [nz*ny*nx, 3] (x, y, z) of a dense box, in state order."""
    nx, ny, nz = dims
    k, j, i = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    return np.stack([i.reshape(-1), j.reshape(-1), k.reshape(-1)], axis=1)


def block_grid(blocks):
    """Grid coordinates [m*512, 3] of the voxels of blocks [m,3], in state order (block, then z, y, x)."""
    l = np.arange(512)
    local = np.stack([l & 7, (l >> 3) & 7, l >> 6], axis=1)
    return (8 * np.asarray(blocks, dtype=np.int64).reshape(-1, 1, 3) + local[None]).reshape(-1, 3)


def plane_blocks(n=129):
    """The closed form of the blocks the plane frames allocate with ORIGIN as the volume's origin, as a set of
    (bx, by, bz), and the number of range ends that fall exactly on a block face ('lo' and 'hi' over pixels and axes).

    A pixel's band cell has corners (u - cx) / 16 * z at z = 3/2 and 5/2, so in units of 1/32 its AABB is
    [min(3 A, 5 A) - 4 tx8, ...] over A in {px - cx, px + 1 - cx} (likewise y), and [48, 80] in z; the range
    floor(((lo - o) / vs - 2) / 8) .. floor(((hi - o) / vs + 2) / 8) is floor((lo32 - o32 - 8) / 32) ..
    floor((hi32 - o32 + 8) / 32)."""
    o32 = [4 * o for o in _O8]
    py, px = (a.reshape(-1) for a in np.meshgrid(np.arange(H), np.arange(W), indexing="ij"))
    keys, faces = [], {"lo": 0, "hi": 0}
    for cx, cy, tx8, ty8 in zip(*plane_cameras(n)):
        lo, hi = [], []
        for p, c, s8 in ((px, cx, tx8), (py, cy, ty8)):
            A = np.stack([3 * (p - c), 5 * (p - c), 3 * (p + 1 - c), 5 * (p + 1 - c)])
            lo.append(A.min(axis=0) - 4 * s8)
            hi.append(A.max(axis=0) - 4 * s8)
        lo.append(np.full(px.shape, 48))
        hi.append(np.full(px.shape, 80))
        b0 = [(lo[a] - o32[a] - 8) // 32 for a in range(3)]
        b1 = [(hi[a] - o32[a] + 8) // 32 for a in range(3)]
        faces["lo"] += sum(int(((lo[a] - o32[a] - 8) % 32 == 0).sum()) for a in range(3))
        faces["hi"] += sum(int(((hi[a] - o32[a] + 8) % 32 == 0).sum()) for a in range(3))
        assert all((b1[a] - b0[a] < 4).all() for a in range(3))   # no pixel is skipped
        for dz in range(4):
            for dy in range(4):
                for dx in range(4):
                    b = [b0[0] + dx, b0[1] + dy, b0[2] + dz]
                    sel = (b[0] <= b1[0]) & (b[1] <= b1[1]) & (b[2] <= b1[2])
                    keys.append(np.stack([b[0][sel], b[1][sel], b[2][sel]], axis=1))
    return set(map(tuple, np.unique(np.concatenate(keys), axis=0).tolist())), faces


def plane_mesh_cubes(weight):
    """The cubes of the plane scene's dense box that mesh: corner 0 in the slice z = 2 and all 8 corners of weight > 0.
    Their corners read tsdf 0 below and -1/2 above, case 240, two triangles each with every vertex at mu = 0, on a voxel
    of the plane.  No other cube changes sign.  Returns bool [nz-1,ny-1,nx-1]."""
    nz, ny, nx = weight.shape
    seen = weight > 0
    ok = np.ones((nz - 1, ny - 1, nx - 1), bool)
    for dx, dy, dz in so.CORNERS:
        ok &= seen[dz:dz + nz - 1, dy:dy + ny - 1, dx:dx + nx - 1]
    ok[np.arange(nz - 1) != int(round((PLANE_Z - ORIGIN[2]) / VOXEL))] = False
    return ok


def plane_render_cameras():
    """Three cameras for ray casting the plane: R = I, fx = fy = 16, cx = 15.5 and cy = 11.5, so pixel (15, 11) looks
    down the optical axis, and translations on the voxel grid: that ray's samples lie on voxel planes (trilinear weights
    0) and, from a near on one, on the block faces.  K, R [3,3,3], t [3,3] float32."""
    K = np.array([[16.0, 0, 15.5], [0, 16.0, 11.5], [0, 0, 1]], f32)
    t = np.array([[0, 0, 0], [0.375, -0.25, 0], [-0.625, 0.5, 0]], f32)
    return np.broadcast_to(K, (3, 3, 3)).copy(), np.broadcast_to(np.eye(3, dtype=f32), (3, 3, 3)).copy(), t


# ---- meshes past 1024 tiles -------------------------------------------------------------------------------------------
def two_spheres(dims, seed=0):
    """An analytic field on a dense box of dims (nx, ny, nz) voxels: tsdf, weight [nz,ny,nx] and color [nz,ny,nx,3]
    float32.  The tsdf is the signed distance in voxels over 3, clamped to [-1, 1], of the union of a large sphere across
    the box and a small one cut by its +y and +z faces, whose triangles lie in the last 2048-cube tile.  Values within
    0.02 of 0 are +0 or -0 by their sign (mu = 0 or 1, and -0 counts as outside).  Weight is 0 on the x = 0..2 slab and at
    1 % of the voxels, 1 to 4 elsewhere; colours are random in [0, 255]."""
    nx, ny, nz = dims
    k, j, i = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    big = np.sqrt((i - 0.46 * nx) ** 2 + (j - 0.52 * ny) ** 2 + (k - 0.5 * nz) ** 2) - 0.43 * min(dims)
    small = np.sqrt((i - 0.5 * nx) ** 2 + (j - (ny - 3.3)) ** 2 + (k - (nz - 0.7)) ** 2) - 4.2
    s = np.clip(np.minimum(big, small) / 3.0, -1.0, 1.0)
    s = np.where(np.abs(s) < 0.02, np.copysign(0.0, s), s).astype(f32)
    rng = np.random.RandomState(seed)
    w = rng.randint(1, 5, s.shape).astype(f32)
    w[:, :, :3] = 0
    w[rng.rand(*s.shape) < 0.01] = 0
    return s, w, rng.uniform(0, 255, s.shape + (3,)).astype(f32)
