"""numpy restatement of superpixel merging (fast_slic_b200.merging, csrc/merge.cuh): the undirected edge list, its order
by (weight key, lower local id, higher local id), Kruskal with a Python union-find per image, the threshold or
region-count prefix of the forest, the numbering by smallest member and the paint."""
import numpy as np


def wkey(w):
    """float32 weights -> the order-preserving uint32 keys as uint64, -0.0 mapped to +0.0 (NaN is never keyed)."""
    w = np.array(w, np.float32, copy=True).reshape(-1)
    w[w == 0] = 0.0
    u = w.view(np.uint32).astype(np.uint64)
    return np.where(u & 0x80000000, ~u & 0xFFFFFFFF, u | 0x80000000)


def ref_present(labels, K):
    """bool [B,K]: label k occurs in image b."""
    lab = np.asarray(labels).view(np.uint16).astype(np.int64)
    B = lab.shape[0]
    present = np.zeros((B, K), bool)
    for b in range(B):
        v = lab[b].reshape(-1)
        present[b, np.unique(v[v < K])] = True
    return present


def ref_edges(src, dst, weights, present):
    """The entries that count as undirected edges: (image, lo, hi, weight) arrays, in entry order."""
    B, K = present.shape
    n = B * K
    src, dst = np.asarray(src, np.int64), np.asarray(dst, np.int64)
    w = np.asarray(weights, np.float32)
    ok = (src >= 0) & (src < dst) & (dst < n)
    s, d = np.where(ok, src, 0), np.where(ok, dst, 0)
    flat = present.reshape(-1)
    ok &= (s // K == d // K) & flat[s] & flat[d] & ~np.isnan(w)
    b = src[ok] // K
    return b, src[ok] - b * K, dst[ok] - b * K, w[ok]


def _find(parent, x):
    while parent[x] != x:
        parent[x] = parent[parent[x]]
        x = parent[x]
    return x


def _union(parent, a, b):
    """Larger root under the smaller; returns whether a link was made."""
    a, b = _find(parent, a), _find(parent, b)
    if a == b:
        return False
    if a < b:
        a, b = b, a
    parent[a] = b
    return True


def ref_forest(present, src, dst, weights):
    """Kruskal per image over the order (wkey, lo, hi): a list over images of the accepted edges (lo, hi, weight) in
    the order they were accepted."""
    B, K = present.shape
    b, lo, hi, w = ref_edges(src, dst, weights, present)
    order = np.lexsort((hi, lo, wkey(w), b))
    b, lo, hi, w = b[order], lo[order], hi[order], w[order]
    bounds = np.searchsorted(b, np.arange(B + 1))
    forest = []
    for i in range(B):
        s, e = bounds[i], bounds[i + 1]
        parent = list(range(K))
        keep = [j for j, u, v in zip(range(s, e), lo[s:e].tolist(), hi[s:e].tolist()) if _union(parent, u, v)]
        forest.append((lo[keep], hi[keep], w[keep]))
    return forest


def ref_cut(forest, present, threshold=None, num_regions=None):
    """(region int32 [B,K], num_regions int32 [B]) of the forest's prefix: the edges with float64(w) < threshold, or
    the first max(0, P_b - num_regions)."""
    B, K = present.shape
    region = np.full((B, K), -1, np.int32)
    count = np.zeros(B, np.int32)
    for b in range(B):
        lo, hi, w = forest[b]
        if threshold is not None:
            take = int(np.count_nonzero(w.astype(np.float64) < threshold))
            assert (w[:take].astype(np.float64) < threshold).all()  # the forest is sorted: a prefix
        else:
            take = max(0, int(present[b].sum()) - num_regions)
        parent = list(range(K))
        for u, v in zip(lo[:take].tolist(), hi[:take].tolist()):
            _union(parent, u, v)
        root = np.array([_find(parent, k) for k in range(K)], np.int64)
        is_root = present[b] & (root == np.arange(K))
        number = np.cumsum(is_root) - 1
        region[b] = np.where(present[b], number[root], -1)
        count[b] = int(is_root.sum())
    return region, count


def ref_paint(labels, region):
    """int16 [B,H,W]: region[b, label] (as int16) at each pixel, -1 where the label is outside [0, K)."""
    lab = np.asarray(labels).view(np.uint16).astype(np.int64)
    B, K = region.shape
    out = np.full(lab.shape, -1, np.int32)
    for b in range(B):
        inside = lab[b] < K
        out[b][inside] = region[b][lab[b][inside]]
    return (out & 0xFFFF).astype(np.uint16).view(np.int16)


def ref_merge(labels, K, src, dst, weights, threshold=None, num_regions=None, forest=None):
    """(labels int16 [B,H,W], region int32 [B,K], num_regions int32 [B]); pass `forest` (ref_forest of the same
    inputs) to cut one graph several times."""
    present = ref_present(labels, K)
    if forest is None:
        forest = ref_forest(present, src, dst, weights)
    region, count = ref_cut(forest, present, threshold, num_regions)
    return ref_paint(labels, region), region, count
