"""A numpy restatement of the indexed mesh (include/demon_b200.h: demon_tsdf_indexed_mesh_f32), by a route of its own:
every corner of marching cubes' soup is tagged with its edge (g, a), the edges are deduplicated with np.unique, which
gives the vertex order and the faces, and each vertex and normal is computed once from its edge in float32, in the
header's order.  A sparse volume is laid into a box (weight 0 outside its blocks), meshed there, and its vertices and
triangles moved into key order."""
import numpy as np

import sequence_oracle as so

f32 = np.float32
TABLE = np.full((256, 15), -1, dtype=np.int64)
for _c, _row in enumerate(so.TRIANGLES):
    TABLE[_c, :len(_row)] = _row
TRI_COUNT = (TABLE >= 0).sum(axis=1) // 3
AXIS = np.array([0, 1, 0, 1, 0, 1, 0, 1, 2, 2, 2, 2])   # the axis of each of the 12 edges
CORNERS = np.asarray(so.CORNERS)
EDGES = np.asarray(so.EDGES)


def soup_edges(tsdf, weight):
    """so.marching_cubes' triangles, in its order, as edges: the corner 0 of each triangle's cube [T,3] (x, y, z), and for
    each of the 3T corners the edge's first voxel g [3T,3] and axis a [3T]."""
    nz, ny, nx = tsdf.shape
    seen, neg = weight > 0, tsdf < 0
    valid = np.ones((nz - 1, ny - 1, nx - 1), bool)
    case = np.zeros((nz - 1, ny - 1, nx - 1), np.int64)
    for q, (dx, dy, dz) in enumerate(CORNERS):
        sl = (slice(dz, dz + nz - 1), slice(dy, dy + ny - 1), slice(dx, dx + nx - 1))
        valid &= seen[sl]
        case |= neg[sl].astype(np.int64) << q
    count = np.where(valid, TRI_COUNT[case], 0).reshape(-1)
    cubes = np.flatnonzero(count)
    k, j, i = np.unravel_index(cubes, (nz - 1, ny - 1, nx - 1))
    cs, n = case.reshape(-1)[cubes], count[cubes]
    cube = np.repeat(np.arange(cubes.size), n)
    m = np.arange(cube.size) - np.repeat(np.cumsum(n) - n, n)   # the triangle's number within its cube
    gc = np.stack([i, j, k], axis=1)[cube]
    edge = np.stack([TABLE[cs[cube], 3 * m + e3] for e3 in range(3)], axis=1).reshape(-1)
    return gc, np.repeat(gc, 3, axis=0) + CORNERS[EDGES[edge, 0]], AXIS[edge]


def _at(field, weight, g):
    """field at voxels g [N,3] and whether each is inside the box with weight > 0 (0 where not)."""
    nz, ny, nx = weight.shape
    ok = (g >= 0).all(axis=1) & (g[:, 0] < nx) & (g[:, 1] < ny) & (g[:, 2] < nz)
    gg = np.where(ok[:, None], g, 0)
    ok &= weight[gg[:, 2], gg[:, 1], gg[:, 0]] > 0
    return field[gg[:, 2], gg[:, 1], gg[:, 0]], ok


def edge_vertices(tsdf, weight, color, origin, voxel_size, g, a, offset=(0, 0, 0), normals=True):
    """The vertex, colour and normal of each edge (g [V,3], a [V]) of the box, its grid coordinates shifted by `offset`."""
    ea = np.eye(3, dtype=np.int64)[a]
    f0, f1 = tsdf[g[:, 2], g[:, 1], g[:, 0]], tsdf[g[:, 2] + ea[:, 2], g[:, 1] + ea[:, 1], g[:, 0] + ea[:, 0]]
    mu = f0 / (f0 - f1)
    o, vs, off = np.asarray(origin, dtype=f32), f32(voxel_size), np.asarray(offset, dtype=np.int64)
    pa, pb = o + vs * (g + off).astype(f32), o + vs * (g + ea + off).astype(f32)
    out = {"vertices": (pa + mu[:, None] * (pb - pa)).astype(f32), "colors": None, "normals": None}
    if color is not None:
        ca, cb = color[g[:, 2], g[:, 1], g[:, 0]], color[g[:, 2] + ea[:, 2], g[:, 1] + ea[:, 1], g[:, 0] + ea[:, 0]]
        out["colors"] = np.clip(np.rint(ca + mu[:, None] * (cb - ca)), 0, 255).astype(np.uint8)
    if normals:
        ok = np.ones(g.shape[0], bool)
        n = []
        for i in range(3):
            ei = np.eye(3, dtype=np.int64)[i]
            d = []
            for p in (g, g + ea):
                fh, oh = _at(tsdf, weight, p + ei)
                fl, ol = _at(tsdf, weight, p - ei)
                ok &= oh & ol
                d.append(fh - fl)
            n.append(d[0] + mu * (d[1] - d[0]))
        length = np.sqrt((n[0] * n[0] + n[1] * n[1]) + n[2] * n[2])
        ok &= length > 0
        with np.errstate(invalid="ignore", divide="ignore"):
            out["normals"] = np.where(ok[:, None], np.stack([c / length for c in n], axis=1), np.nan).astype(f32)
    return out


def dense(tsdf, weight, color, origin, voxel_size, normals=True, offset=(0, 0, 0)):
    """The indexed mesh of a dense box: vertices [V,3] float32, normals [V,3] float32 or None, colors [V,3] uint8 or None,
    faces [T,3] int32, and `cubes` [T,3] (corner 0 of each triangle's cube) and `soup_keys` [3T] (each soup corner's
    edge key 3 (linear index of g) + a) for the tests."""
    nz, ny, nx = tsdf.shape
    gc, g, a = soup_edges(tsdf, weight)
    key = 3 * ((g[:, 2] * ny + g[:, 1]) * nx + g[:, 0]) + a
    uniq, first, inv = np.unique(key, return_index=True, return_inverse=True)
    out = edge_vertices(tsdf, weight, color, origin, voxel_size, g[first], a[first], offset, normals)
    out.update(faces=inv.reshape(-1, 3).astype(np.int32), cubes=gc, soup_keys=key)
    return out


def packed_keys(b):
    """The table's packed key of blocks b [N,3]: 21 bits per axis offset by 2^20, z highest."""
    b = np.asarray(b, dtype=np.int64) + (1 << 20)
    return (b[:, 2] << 42) | (b[:, 1] << 21) | b[:, 0]


def sparse(blocks, tsdf, weight, color, origin, voxel_size, normals=True):
    """The indexed mesh of sparse blocks [m,3] with state [m,8,8,8] (color [m,8,8,8,3] or None): the blocks laid into a
    box, meshed by `dense`, vertices sorted by (block key, local index, axis) and triangles by (block key, local cube
    index), stably."""
    out = {"vertices": np.zeros((0, 3), f32), "normals": np.zeros((0, 3), f32) if normals else None,
           "colors": None if color is None else np.zeros((0, 3), np.uint8), "faces": np.zeros((0, 3), np.int32)}
    blocks = np.asarray(blocks, dtype=np.int64).reshape(-1, 3)
    if blocks.shape[0] == 0:
        return out
    lo = blocks.min(axis=0)
    nx, ny, nz = 8 * (blocks.max(axis=0) - lo + 1)
    bt, bw = np.zeros((nz, ny, nx), f32), np.zeros((nz, ny, nx), f32)
    bc = None if color is None else np.zeros((nz, ny, nx, 3), f32)
    for q, (x, y, z) in enumerate(8 * (blocks - lo)):
        bt[z:z + 8, y:y + 8, x:x + 8] = tsdf[q]
        bw[z:z + 8, y:y + 8, x:x + 8] = weight[q]
        if bc is not None:
            bc[z:z + 8, y:y + 8, x:x + 8] = color[q]
    d = dense(bt, bw, bc, origin, voxel_size, normals, offset=8 * lo)
    nv = d["vertices"].shape[0]
    if nv == 0:
        return out
    uniq = np.unique(d["soup_keys"])
    a, lin = uniq % 3, uniq // 3
    g = np.stack([lin % nx, (lin // nx) % ny, lin // (nx * ny)], axis=1) + 8 * lo
    perm = np.lexsort((3 * (((g[:, 2] & 7) << 6) | ((g[:, 1] & 7) << 3) | (g[:, 0] & 7)) + a, packed_keys(g >> 3)))
    new = np.empty(nv, np.int64)
    new[perm] = np.arange(nv)
    c = d["cubes"] + 8 * lo
    tperm = np.lexsort(((((c[:, 2] & 7) << 6) | ((c[:, 1] & 7) << 3) | (c[:, 0] & 7)), packed_keys(c >> 3)))
    for k in ("vertices", "normals", "colors"):
        out[k] = None if d[k] is None else d[k][perm]
    out["faces"] = new[d["faces"]][tperm].astype(np.int32)
    return out
