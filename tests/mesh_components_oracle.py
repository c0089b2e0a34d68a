"""The connected components of an indexed mesh and the removal of the small ones, restated in numpy and scipy
(include/demon_b200.h: demon_mesh_*).  scipy's connected_components over the vertex adjacency of the faces finds the
classes; they are relabelled by each class's smallest vertex, counted with np.bincount and filtered with boolean masks.
"""
import numpy as np
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components


def components(faces, num_vertices):
    """{"labels": [V] int32, "triangles": [C] int64, "vertices": [C] int64} of faces [F,3] over num_vertices vertices."""
    f = np.asarray(faces, dtype=np.int64).reshape(-1, 3)
    nv = int(num_vertices)
    if nv == 0:
        z = np.zeros(0, np.int64)
        return {"labels": np.zeros(0, np.int32), "triangles": z, "vertices": z.copy()}
    rows = np.concatenate([f[:, 0], f[:, 1]])
    cols = np.concatenate([f[:, 1], f[:, 2]])
    adj = coo_matrix((np.ones(rows.size, np.int8), (rows, cols)), shape=(nv, nv)).tocsr()
    c, lab = connected_components(adj, directed=False)
    first = np.full(c, nv, np.int64)
    np.minimum.at(first, lab, np.arange(nv, dtype=np.int64))
    rank = np.empty(c, np.int64)
    rank[np.argsort(first, kind="stable")] = np.arange(c)
    labels = rank[lab]
    return {"labels": labels.astype(np.int32), "triangles": np.bincount(labels[f[:, 0]], minlength=c).astype(np.int64),
            "vertices": np.bincount(labels, minlength=c).astype(np.int64)}


def kept(triangles, min_triangles=1, keep_largest=None):
    """[C] bool: the components with at least min_triangles triangles, and of those the keep_largest with the most (ties
    to the smaller label)."""
    tri = np.asarray(triangles, np.int64)
    keep = tri >= min_triangles
    if keep_largest is not None and keep_largest < tri.size:
        key = np.where(keep, tri, -1)
        sel = np.zeros(tri.size, bool)
        sel[np.argsort(-key, kind="stable")[:keep_largest]] = True
        keep &= sel
    return keep


def remove_small_components(mesh, min_triangles=1, keep_largest=None):
    """The filtered mesh of a dict of numpy arrays (vertices, faces, and normals / colors or None)."""
    v = np.asarray(mesh["vertices"])
    f = np.asarray(mesh["faces"], dtype=np.int64).reshape(-1, 3)
    comps = components(f, v.shape[0])
    keep = kept(comps["triangles"], min_triangles, keep_largest)
    vmask = keep[comps["labels"]]
    fmask = keep[comps["labels"][f[:, 0]]] if f.shape[0] else np.zeros(0, bool)
    new = np.cumsum(vmask) - 1
    out = {"vertices": v[vmask], "faces": new[f[fmask]].astype(np.int32).reshape(-1, 3)}
    for k in ("normals", "colors"):
        out[k] = None if mesh.get(k) is None else np.asarray(mesh[k])[vmask]
    return out


def union_find(faces, num_vertices):
    """The labels of a plain sequential union-find (smallest vertex as the root), an independent check of components()."""
    parent = list(range(num_vertices))

    def find(x):
        while parent[x] != x:
            x = parent[x]
        return x
    for a, b, c in np.asarray(faces, dtype=np.int64).reshape(-1, 3).tolist():
        for p, q in ((a, b), (b, c)):
            rp, rq = find(p), find(q)
            if rp != rq:
                parent[max(rp, rq)] = min(rp, rq)
    roots = [find(v) for v in range(num_vertices)]
    rank = {r: k for k, r in enumerate(sorted(set(roots)))}
    return np.array([rank[r] for r in roots], dtype=np.int32)


# ---- meshes ---------------------------------------------------------------------------------------------------------
def strip(n, order="random", seed=0):
    """A triangle strip over n vertices, faces (s_i, s_{i+1}, s_{i+2}) of a sequence s: s = 0, 1, ... with order
    'ascending', n-1, n-2, ... with 'descending' (every union hooks a new smaller root: the deepest trees), or a random
    permutation.  One component."""
    if order == "ascending":
        s = np.arange(n)
    elif order == "descending":
        s = np.arange(n)[::-1]
    else:
        s = np.random.RandomState(seed).permutation(n)
    return np.stack([s[:-2], s[1:-1], s[2:]], axis=1).astype(np.int32)


def fan(n):
    """n triangles (0, i+1, i+2) around vertex 0: every union meets the same root."""
    i = np.arange(n)
    return np.stack([np.zeros(n, np.int64), i + 1, i + 2], axis=1).astype(np.int32)


def isolated_triangles(n, seed=0):
    """n disjoint triangles over 3n vertices, shuffled in vertex index and in face order."""
    rng = np.random.RandomState(seed)
    perm = rng.permutation(3 * n)
    return perm.reshape(n, 3)[rng.permutation(n)].astype(np.int32)
