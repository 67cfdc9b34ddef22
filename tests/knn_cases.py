"""numpy restatement of region_graph.knn_graph: float32 squared distances in the contract's rounding order, candidates
(present and finite), each row's first min(k, P_b - 1) other candidates under the (s, j) order, the symmetric union
and the CSR layout."""
import numpy as np


def candidates(points, present=None):
    """bool [B,K]: present and every coordinate finite."""
    ok = np.isfinite(points).all(axis=2)
    return ok if present is None else ok & np.asarray(present, bool)


def sqdist(a, b):
    """s[i, j] for rows a [n,D] and b [m,D]: t_c = a_c - b_c, s = +0, s = s + t_c * t_c for c = 0..D-1, each float32
    operation rounded on its own (numpy does not contract them)."""
    a = np.asarray(a, np.float32)
    b = np.asarray(b, np.float32)
    s = np.zeros((len(a), len(b)), np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        for c in range(a.shape[1]):
            t = a[:, None, c] - b[None, :, c]
            s = s + t * t
    return s


def image_rows(points, mask, k, block=1024):
    """One image's directed rows: {i: (targets ascending, distances)} for every candidate i."""
    cand = np.flatnonzero(mask)
    P = len(cand)
    cnt = min(k, P - 1)
    rows = {}
    if P == 0:
        return rows
    pts = points[cand]
    J = np.broadcast_to(cand[None, :].astype(np.int64), (min(block, P), P))
    for r0 in range(0, P, block):
        r1 = min(P, r0 + block)
        S = sqdist(pts[r0:r1], pts)
        Jb = np.array(J[:r1 - r0])
        ar = np.arange(r1 - r0)
        S[ar, ar + r0] = np.inf  # self last: after every candidate, inf distances included (j < K)
        Jb[ar, ar + r0] = np.iinfo(np.int64).max
        order = np.lexsort((Jb, S), axis=-1)[:, :cnt]
        for a in range(r1 - r0):
            pick = order[a]
            js, ss = Jb[a, pick], S[a, pick]
            o = np.argsort(js, kind="stable")
            rows[int(cand[r0 + a])] = (js[o], ss[o])
    return rows


def csr(n_nodes, src, dst, dist):
    """Edges sorted by (source, target) -> (indptr int64 [n+1], edge_index int64 [2,E], distance float32 [E])."""
    src = np.asarray(src, np.int64)
    dst = np.asarray(dst, np.int64)
    o = np.lexsort((dst, src))
    src, dst, dist = src[o], dst[o], np.asarray(dist, np.float32)[o]
    indptr = np.zeros(n_nodes + 1, np.int64)
    np.cumsum(np.bincount(src, minlength=n_nodes), out=indptr[1:])
    return indptr, np.stack([src, dst]), dist


def ref_knn(points, k, present=None, symmetric=False):
    """points float32 [B,K,D], present bool [B,K] or None -> (indptr, edge_index, distance) as knn_graph returns them."""
    points = np.asarray(points, np.float32)
    B, K, _ = points.shape
    mask = candidates(points, present)
    src, dst, dist = [], [], []
    for b in range(B):
        for i, (js, ss) in image_rows(points[b], mask[b], k).items():
            src.append(np.full(len(js), b * K + i, np.int64))
            dst.append(b * K + js)
            dist.append(ss)
    cat = (lambda x, t: np.concatenate(x).astype(t) if x else np.zeros(0, t))
    src, dst, dist = cat(src, np.int64), cat(dst, np.int64), cat(dist, np.float32)
    ref = csr(B * K, src, dst, dist)
    return union(ref) if symmetric else ref


def union(ref):
    """The symmetric graph of a directed one (indptr, edge_index, distance): every edge in both directions, each
    (source, target) once, as PyG's to_undirected makes it."""
    indptr, (src, dst), dist = ref
    N = len(indptr) - 1
    keys = np.concatenate([src * N + dst, dst * N + src])
    both = np.concatenate([dist, dist])
    keys, first = np.unique(keys, return_index=True)
    return csr(N, keys // N, keys % N, both[first])
