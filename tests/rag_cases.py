"""fast_slic_b200.region_graph restated in numpy, for the region adjacency graph tests.

Per image: the pixel pairs by array slicing (right and down; with connectivity 8 also down-right and down-left), the
valid pairs with differing labels, np.unique of their (low, high) keys with counts, both directions, lexsorted by
(source, target).  Node ids are b*K + label.
"""
import numpy as np


def pixel_pairs(lab, connectivity):
    """The two ends of every unordered pixel pair of one [H,W] map, flattened."""
    ends = [(lab[:, :-1], lab[:, 1:]), (lab[:-1, :], lab[1:, :])]
    if connectivity == 8:
        ends += [(lab[:-1, :-1], lab[1:, 1:]), (lab[:-1, 1:], lab[1:, :-1])]
    return (np.concatenate([a.ravel() for a, _ in ends]), np.concatenate([c.ravel() for _, c in ends]))


def ref_rag_image(labels, K, connectivity):
    """One int16 [H,W] map -> (source labels, target labels, boundary counts), int64, sorted by (source, target)."""
    lab = np.ascontiguousarray(labels).view(np.uint16).astype(np.int64)
    a, c = pixel_pairs(lab, connectivity)
    ok = (a < K) & (c < K) & (a != c)
    lo, hi = np.minimum(a[ok], c[ok]), np.maximum(a[ok], c[ok])
    keys, counts = np.unique(lo * K + hi, return_counts=True)
    lo, hi = keys // K, keys % K
    src, dst, w = np.concatenate([lo, hi]), np.concatenate([hi, lo]), np.concatenate([counts, counts])
    order = np.lexsort((dst, src))
    return src[order], dst[order], w[order]


def ref_rag(labels, K, connectivity=4):
    """int16 [B,H,W] -> (indptr int64[B*K+1], edge_index int64[2,E], boundary int32[E])."""
    B = labels.shape[0]
    parts = [ref_rag_image(labels[b], K, connectivity) for b in range(B)]
    src = np.concatenate([p[0] + b * K for b, p in enumerate(parts)] + [np.zeros(0, np.int64)])
    dst = np.concatenate([p[1] + b * K for b, p in enumerate(parts)] + [np.zeros(0, np.int64)])
    w = np.concatenate([p[2] for p in parts] + [np.zeros(0, np.int64)])
    indptr = np.zeros(B * K + 1, np.int64)
    indptr[1:] = np.cumsum(np.bincount(src, minlength=B * K))
    return indptr, np.stack([src, dst]).astype(np.int64), w.astype(np.int32)
