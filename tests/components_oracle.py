"""NumPy oracle of the mesh components (include/sparf_b200.h, mesh components): scipy's connected components of the
vertex graph, relabelled by smallest vertex id, the face counts, the component choice of mesh.keep_components and the
selection with its renumbering."""
import numpy as np
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components


def components(faces, n_verts):
    """(labels [V] int32, face_counts [C] int64): label = the rank of the component's smallest vertex id; a face counts
    under the label of its first vertex"""
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    if n_verts == 0:
        return np.zeros(0, np.int32), np.zeros(0, np.int64)
    rows = np.concatenate([f[:, 0], f[:, 0]])
    cols = np.concatenate([f[:, 1], f[:, 2]])
    g = coo_matrix((np.ones(len(rows), np.int8), (rows, cols)), shape=(n_verts, n_verts))
    n, lab = connected_components(g, directed=False)
    _, first = np.unique(lab, return_index=True)        # first[l] = the smallest vertex with scipy label l
    rank = np.empty(n, np.int64)
    rank[np.argsort(first)] = np.arange(n)
    labels = rank[lab].astype(np.int32)
    counts = np.bincount(labels[f[:, 0]], minlength=n).astype(np.int64)
    return labels, counts


def keep_mask(counts, largest=None, min_faces=1):
    """uint8 [C]: the components with >= min_faces faces, and of those the `largest` first by (count desc, label asc)"""
    idx = np.flatnonzero(counts >= min_faces)
    if largest is not None:
        idx = idx[np.argsort(-counts[idx], kind="stable")][:largest]
    keep = np.zeros(len(counts), np.uint8)
    keep[idx] = 1
    return keep


def select(faces, labels, keep):
    """(vert_ids [V'] int64, faces [F', 3] int64): the kept vertices in order, and the faces whose first vertex is
    kept, in order, renumbered"""
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    kv = np.asarray(keep, bool)[labels] if len(labels) else np.zeros(0, bool)
    new = np.cumsum(kv) - 1
    fk = kv[f[:, 0]] if len(f) else np.zeros(0, bool)
    return np.flatnonzero(kv).astype(np.int64), new[f[fk]].astype(np.int64).reshape(-1, 3)


def bfs_labels(faces, n_verts):
    """labels by a plain breadth-first search from each unvisited vertex in increasing order (the rank rule directly)"""
    adj = [[] for _ in range(n_verts)]
    for a, b, c in np.asarray(faces, np.int64).reshape(-1, 3):
        for x, y in ((a, b), (b, c), (a, c)):
            adj[x].append(y)
            adj[y].append(x)
    labels = np.full(n_verts, -1, np.int32)
    n = 0
    for s in range(n_verts):
        if labels[s] >= 0:
            continue
        labels[s] = n
        queue = [s]
        while queue:
            x = queue.pop()
            for y in adj[x]:
                if labels[y] < 0:
                    labels[y] = n
                    queue.append(y)
        n += 1
    return labels


def random_soup(n_verts, n_faces, seed, n_groups=None):
    """faces over n_verts vertices, each face drawn inside one of n_groups random vertex groups (many components), with
    some degenerate faces"""
    rng = np.random.default_rng(seed)
    n_groups = n_groups or max(1, n_verts // 8)
    group = rng.integers(0, n_groups, n_verts)
    order = np.argsort(group, kind="stable")
    starts = np.searchsorted(group[order], np.arange(n_groups))
    ends = np.searchsorted(group[order], np.arange(n_groups), side="right")
    g = rng.integers(0, n_groups, n_faces)
    ok = ends[g] > starts[g]
    g = g[ok]
    pick = starts[g][:, None] + (rng.random((len(g), 3)) * (ends[g] - starts[g])[:, None]).astype(np.int64)
    return order[pick].astype(np.int64)
