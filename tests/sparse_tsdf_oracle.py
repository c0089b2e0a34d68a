"""numpy restatements of the sparse TSDF volume (demon_b200.sequence.SparseTsdfVolume, csrc/fusion.cu) for the tests: the
block allocation rule in the kernel's float32 order, and the voxel positions of blocks, so that sequence_oracle.integrate's
arithmetic runs on sparse state."""
from unittest import mock

import numpy as np

import sequence_oracle as so

f32 = np.float32
MAX_SPAN = 4              # DEMON_SPARSE_TSDF_MAX_SPAN
MAX_COORD = 2 ** 20 - 1   # DEMON_SPARSE_TSDF_MAX_COORD


def allocate(depth, K, R, t, origin, voxel_size, trunc):
    """The blocks the frames allocate, as a set of (bx, by, bz), and the number of skipped pixels.

    A pixel with finite d > 0 takes its band cell: corners (u, v) in {px, px+1} x {py, py+1}, a = (u - cx)/fx,
    b = (v - cy)/fy, camera points (a zf, b zf, zf) with zf = d + trunc and (a zn, b zn, zn) with zn = d - trunc, or the
    camera centre when zn <= 0; world X = R^T (x - t) as (R_0i e_0 + R_1i e_1) + R_2i e_2; the blocks
    floor(((lo - o)/vs - 2) / 8) .. floor(((hi - o)/vs + 2) / 8) of the AABB, unless a point is not finite, a block is
    past +-MAX_COORD or the range spans more than MAX_SPAN blocks."""
    depth = np.asarray(depth, dtype=f32)
    n, h, w = depth.shape
    K, R, t = (np.broadcast_to(np.asarray(a, dtype=f32), s) for a, s in ((K, (n, 3, 3)), (R, (n, 3, 3)), (t, (n, 3))))
    o, vs, tr = np.asarray(origin, dtype=f32), f32(voxel_size), f32(trunc)
    py, px = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    keys, skipped = [], 0
    with np.errstate(all="ignore"):
        for f in range(n):
            d = depth[f]
            valid = np.isfinite(d) & (d > 0)
            zf, zn = d + tr, d - tr
            near = zn > 0
            pts = []
            for c in range(4):
                a = ((px + (c & 1)).astype(f32) - K[f, 0, 2]) / K[f, 0, 0]
                b = ((py + (c >> 1)).astype(f32) - K[f, 1, 2]) / K[f, 1, 1]
                pts.append((a * zf, b * zf, zf))
                zero = np.zeros_like(d)
                pts.append((np.where(near, a * zn, zero), np.where(near, b * zn, zero), np.where(near, zn, zero)))
            lo, hi, finite = [], [], valid.copy()
            for i in range(3):
                X = [(R[f, 0, i] * (x - t[f, 0]) + R[f, 1, i] * (y - t[f, 1])) + R[f, 2, i] * (z - t[f, 2]) for x, y, z in pts]
                X = np.stack(X)
                finite &= np.isfinite(X).all(axis=0)
                lo.append(X.min(axis=0))
                hi.append(X.max(axis=0))
            b0 = [np.floor(((lo[i] - o[i]) / vs - f32(2)) * f32(0.125)) for i in range(3)]
            b1 = [np.floor(((hi[i] - o[i]) / vs + f32(2)) * f32(0.125)) for i in range(3)]
            ok = finite.copy()
            for i in range(3):
                ok &= (b0[i] >= -MAX_COORD) & (b1[i] <= MAX_COORD)
                ok &= np.where(ok, b1[i] - b0[i], 0) < MAX_SPAN
            skipped += int((valid & ~ok).sum())
            b0 = [np.where(ok, b, 0).astype(np.int64)[ok] for b in b0]
            b1 = [np.where(ok, b, 0).astype(np.int64)[ok] for b in b1]
            for dz in range(MAX_SPAN):
                for dy in range(MAX_SPAN):
                    for dx in range(MAX_SPAN):
                        g = [b0[0] + dx, b0[1] + dy, b0[2] + dz]
                        sel = (g[0] <= b1[0]) & (g[1] <= b1[1]) & (g[2] <= b1[2])
                        keys.append(np.stack([g[0][sel], g[1][sel], g[2][sel]], axis=1))
    allb = np.unique(np.concatenate(keys), axis=0) if keys else np.zeros((0, 3), np.int64)
    return set(map(tuple, allb.tolist())), skipped


def block_points(blocks, origin, voxel_size):
    """float32 X0, X1, X2 of every voxel of blocks [m,3], in state order (block, then z, y, x with x fastest):
    origin + voxel_size * (8 b + l), the kernels' fadd(o, fmul(vs, (float)g)) for any integer g."""
    blocks = np.asarray(blocks, dtype=np.int64).reshape(-1, 3)
    l = np.arange(512)
    local = np.stack([l & 7, (l >> 3) & 7, l >> 6], axis=1)
    g = (8 * blocks[:, None, :] + local[None]).reshape(-1, 3)
    o, vs = np.asarray(origin, dtype=f32), f32(voxel_size)
    return [o[a] + vs * g[:, a].astype(f32) for a in range(3)]


def integrate_blocks(tsdf, weight, color, blocks, origin, voxel_size, trunc, depth, K, R, t, image=None):
    """sequence_oracle.integrate on sparse state (tsdf, weight [m,8,8,8], color [m,8,8,8,3] or None), in place: the same
    per-frame arithmetic with the voxel positions of block_points."""
    m = tsdf.shape[0]
    shape = (m * 8, 8, 8)
    pts = block_points(blocks, origin, voxel_size)
    with mock.patch.object(so, "voxel_points", lambda dims, o, vs: pts):
        so.integrate(tsdf.reshape(shape), weight.reshape(shape), None if color is None else color.reshape(shape + (3,)),
                     origin, voxel_size, trunc, depth, K, R, t, image)
    return tsdf, weight, color


def block_of(g):
    """The block of integer voxel coordinates g [..., 3]."""
    return np.floor_divide(np.asarray(g), 8)
