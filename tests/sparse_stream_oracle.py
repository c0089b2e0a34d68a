"""numpy restatement of the reach rule that streams a sparse TSDF volume's blocks (include/demon_b200.h:
demon_sparse_tsdf_depth_tiles_f32 and demon_sparse_tsdf_reach_f32, csrc/fusion.cu) in the kernels' float32 order, and a
ring corridor scene whose inner walls hide the far side of the loop."""
import numpy as np

import sequence_oracle as so

f32 = np.float32
TILE = 8


def depth_tiles(depth):
    """float32 [n, ceil(h/8), ceil(w/8)]: the largest finite depth > 0 of each 8x8 tile, -inf where there is none."""
    depth = np.asarray(depth, dtype=f32)
    n, h, w = depth.shape
    th, tw = -(-h // TILE), -(-w // TILE)
    pad = np.full((n, th * TILE, tw * TILE), -np.inf, f32)
    with np.errstate(invalid="ignore"):
        pad[:, :h, :w] = np.where(np.isfinite(depth) & (depth > 0), depth, -np.inf)
    return pad.reshape(n, th, TILE, tw, TILE).max(axis=(2, 4))


def reach(blocks, origin, voxel_size, trunc, tiles, K, R, t, h, w):
    """bool [n, m]: frame f reaches block b, by the header's rule in its float32 order."""
    blocks = np.asarray(blocks, dtype=np.int64).reshape(-1, 3)
    tiles = np.asarray(tiles, dtype=f32)
    n, th, tw = tiles.shape
    K, R, t = (np.broadcast_to(np.asarray(a, dtype=f32), s) for a, s in ((K, (n, 3, 3)), (R, (n, 3, 3)), (t, (n, 3))))
    o, vs, tr = np.asarray(origin, dtype=f32), f32(voxel_size), f32(trunc)
    tr2 = tr + tr
    lo = [(o[a] + vs * (8 * blocks[:, a] - 3).astype(f32)) - tr2 for a in range(3)]
    hi = [(o[a] + vs * (8 * blocks[:, a] + 10).astype(f32)) + tr2 for a in range(3)]
    out = np.zeros((n, blocks.shape[0]), bool)
    with np.errstate(all="ignore"):
        for f in range(n):
            Rf, tf = R[f], t[f]
            zs, us, vs_ = [], [], []
            for q in range(8):
                X = [hi[a] if (q >> a) & 1 else lo[a] for a in range(3)]
                cam = [((Rf[r, 0] * X[0] + Rf[r, 1] * X[1]) + Rf[r, 2] * X[2]) + tf[r] for r in range(3)]
                zs.append(cam[2])
                us.append((K[f, 0, 0] * cam[0]) / cam[2] + K[f, 0, 2])
                vs_.append((K[f, 1, 1] * cam[1]) / cam[2] + K[f, 1, 2])
            zs, us, vs_ = np.stack(zs), np.stack(us), np.stack(vs_)
            behind = ~(zs > vs).all(axis=0)
            zmin = np.where(behind, f32(0), zs.min(axis=0))
            u0, u1 = np.floor(us.min(axis=0)) - f32(1), np.floor(us.max(axis=0)) + f32(1)
            v0, v1 = np.floor(vs_.min(axis=0)) - f32(1), np.floor(vs_.max(axis=0)) + f32(1)
            meets = (zs.max(axis=0) > vs) & (behind | ((u1 >= 0) & (u0 <= f32(w - 1)) & (v1 >= 0) & (v0 <= f32(h - 1))))
            x0 = np.where(behind, 0, np.clip(np.nan_to_num(u0), 0, w - 1)).astype(np.int64)
            x1 = np.where(behind, w - 1, np.clip(np.nan_to_num(u1), 0, w - 1)).astype(np.int64)
            y0 = np.where(behind, 0, np.clip(np.nan_to_num(v0), 0, h - 1)).astype(np.int64)
            y1 = np.where(behind, h - 1, np.clip(np.nan_to_num(v1), 0, h - 1)).astype(np.int64)
            tx0, tx1, ty0, ty1 = x0 // TILE, x1 // TILE, y0 // TILE, y1 // TILE
            hit = np.zeros(blocks.shape[0], bool)
            for ty in range(th):
                for tx in range(tw):
                    under = (ty >= ty0) & (ty <= ty1) & (tx >= tx0) & (tx <= tx1)
                    hit |= under & (tiles[f, ty, tx] + tr >= zmin)
            out[f] = meets & hit
    return out


def raycast_tiles(far, h, w):
    """The tiles a ray cast tests with: every tile of frame f at far[f]."""
    far = np.asarray(far, dtype=f32).reshape(-1)
    return np.broadcast_to(far[:, None, None], (far.size, -(-h // TILE), -(-w // TILE))).copy()


# ---- the ring corridor ------------------------------------------------------------------------------------------------
# The inside of the box [-L, L]^2 x [0, H] minus the pillar [-L + W, L - W]^2 (full height): a square loop of corridor of
# width W.  The pillar's walls hide the far side of the loop from every camera on its centre line.
def render_ring(R, t, K, h, w, L, W, H):
    """float64 camera z [h,w] of pixel centres: the nearest hit of the outer box's inside and the pillar's outside."""
    R, t, K = (np.asarray(a, dtype=np.float64) for a in (R, t, K))
    lam = so.render_depth(R, t, K, h, w, box=((-L, -L, 0.0), (L, L, H)))
    x, y = np.meshgrid(np.arange(w) + 0.5, np.arange(h) + 0.5)
    d = np.stack([(x - K[0, 2]) / K[0, 0], (y - K[1, 2]) / K[1, 1], np.ones_like(x)], axis=-1).dot(R)
    o = -R.T.dot(t)
    lo, hi = np.array([-L + W, -L + W, -1.0]), np.array([L - W, L - W, H + 1.0])
    with np.errstate(divide="ignore", invalid="ignore"):
        a, b = (lo - o) / d, (hi - o) / d
    enter = np.minimum(a, b).max(axis=-1)
    leave = np.maximum(a, b).min(axis=-1)
    pillar = (enter <= leave) & (enter > 0)
    return np.where(pillar, np.minimum(lam, enter), lam)


def ring_path(s, L, W):
    """The point at arc length s along the corridor's centre line (a square of side 2L - W, counter-clockwise)."""
    c = L - W / 2
    side = 2 * c
    s = s % (4 * side)
    k, r = int(s // side), s % side
    corners = [(-c, -c), (c, -c), (c, c), (-c, c)]
    (x0, y0), (x1, y1) = corners[k], corners[(k + 1) % 4]
    return np.array([x0 + (x1 - x0) * r / side, y0 + (y1 - y0) * r / side])


def ring_walk(n, loops=1.3, h=48, w=64, L=2.0, W=1.0, H=1.0, f=40.0, seed=0):
    """n frames walking `loops` times round the ring, each camera on the centre line at mid-height looking along it:
    depth [n,h,w], K, R [n,3,3], t [n,3] float32 and random images [n,h,w,3] uint8."""
    side = 2 * (L - W / 2)
    K = np.array([[f, 0, w / 2], [0, f, h / 2], [0, 0, 1]])
    Rs, ts, ds = [], [], []
    for s in np.linspace(0, loops * 4 * side, n, endpoint=False):
        c = np.append(ring_path(s, L, W), H / 2)
        target = np.append(ring_path(s + 0.5, L, W), H / 2)
        R, tt = so.look_at(c, target)
        Rs.append(R)
        ts.append(tt)
        ds.append(render_ring(R, tt, K, h, w, L, W, H))
    img = np.random.RandomState(seed).randint(0, 256, (n, h, w, 3)).astype(np.uint8)
    return (np.array(ds, dtype=f32), np.broadcast_to(K.astype(f32), (n, 3, 3)).copy(), np.array(Rs, dtype=f32),
            np.array(ts, dtype=f32), img)
