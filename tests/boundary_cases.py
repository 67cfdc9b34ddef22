"""fast_slic_b200.region_graph.boundary_stats restated in numpy (DESIGN.md section 4.17), for the boundary tests.

Per image: the pixel pairs by array slicing, as rag_cases.pixel_pairs takes them (right and down; with connectivity 8
also down-right and down-left), each with its ordinal anchor * D + d; the boundary pairs (both labels in [0, K) and
different), lexsorted by (label-pair key, ordinal).  Each run of one key interleaves its anchor and other values; the
sum follows pool_cases.ref_pool's lanes and butterfly, the mean is sum / float32(2n), min / max use the order of
non-NaN floats with -0.0 < +0.0 and NaN when any value is NaN.  Entries look their key up among the runs.
"""
import numpy as np

_NAN = np.float32("nan")


def pair_ends(H, W, connectivity):
    """(anchor, other, ordinal) int64 flat pixel indices and ordinals of every pixel pair of an [H,W] image."""
    idx = np.arange(H * W, dtype=np.int64).reshape(H, W)
    ends = [(idx[:, :-1], idx[:, 1:]), (idx[:-1, :], idx[1:, :])]
    if connectivity == 8:
        ends += [(idx[:-1, :-1], idx[1:, 1:]), (idx[:-1, 1:], idx[1:, :-1])]
    D = len(ends)
    anchor = np.concatenate([a.ravel() for a, _ in ends])
    other = np.concatenate([o.ravel() for _, o in ends])
    d = np.concatenate([np.full(a.size, k, np.int64) for k, (a, _) in enumerate(ends)])
    return anchor, other, anchor * D + d


def okey(x):
    """float32 -> int64 keys of the total order of non-NaN floats with -0.0 < +0.0."""
    i = np.ascontiguousarray(x, np.float32).view(np.int32).astype(np.int64)
    return np.where(i < 0, i ^ 0x7fffffff, i)


def from_okey(k):
    k = np.asarray(k, np.int64)
    return np.where(k < 0, k ^ 0x7fffffff, k).astype(np.int32).view(np.float32)


def lane_sums(vals, run, pos, runs):
    """float32 [C, runs]: per run, the values vals[:, i] at position pos[i] of run run[i], dealt to 32 lanes left to
    right from +0.0 and combined by five butterfly steps (pool_cases.ref_pool's order)."""
    C = vals.shape[0]
    v = np.zeros((C, runs, 32), np.float32)
    if vals.shape[1] == 0:
        return v[:, :, 0]
    row, lane = pos // 32, pos % 32
    with np.errstate(invalid="ignore", over="ignore"):
        for r in range(int(row.max()) + 1):
            sel = row == r  # each (run, lane) at most once per row
            v[:, run[sel], lane[sel]] = v[:, run[sel], lane[sel]] + vals[:, sel]
        lanes = np.arange(32)
        for off in (16, 8, 4, 2, 1):
            v = v + v[:, :, lanes ^ off]
    return v[:, :, 0]


def ref_boundary_image(labels, values, K, connectivity):
    """One int16 [H,W] map and float32 [C,H,W] values -> (keys int64 lo * 65536 + hi [R], mean, min, max f32 [C,R],
    count int64 [R]) of its R runs, in key order."""
    H, W = labels.shape
    lab = np.ascontiguousarray(labels).view(np.uint16).ravel().astype(np.int64)
    feats = np.ascontiguousarray(values, np.float32).reshape(values.shape[0], -1)
    C = feats.shape[0]
    anchor, other, ordinal = pair_ends(H, W, connectivity)
    a, o = lab[anchor], lab[other]
    ok = (a < K) & (o < K) & (a != o)
    anchor, other, ordinal, a, o = anchor[ok], other[ok], ordinal[ok], a[ok], o[ok]
    key = np.minimum(a, o) * 65536 + np.maximum(a, o)
    order = np.lexsort((ordinal, key))
    anchor, other, key = anchor[order], other[order], key[order]
    keys, first, count = np.unique(key, return_index=True, return_counts=True)
    R = keys.size
    if R == 0:
        empty = np.zeros((C, 0), np.float32)
        return keys, empty, empty, empty, count
    # the 2n values of each run: anchor, other of each pair in ordinal order
    pix = np.empty(2 * anchor.size, np.int64)
    pix[0::2], pix[1::2] = anchor, other
    run = np.repeat(np.arange(R), 2 * count)
    pos = np.arange(pix.size) - np.repeat(2 * first, 2 * count)
    vals = feats[:, pix]
    sums = lane_sums(vals, run, pos, R)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        mean = sums / (2 * count).astype(np.float32)
    nan = np.isnan(vals)
    k = okey(vals)
    starts = 2 * first
    lo = np.minimum.reduceat(np.where(nan, np.iinfo(np.int64).max, k), starts, axis=1)
    hi = np.maximum.reduceat(np.where(nan, np.iinfo(np.int64).min, k), starts, axis=1)
    anynan = np.logical_or.reduceat(nan, starts, axis=1)
    mn = np.where(anynan, _NAN, from_okey(np.where(anynan, 0, lo)))
    mx = np.where(anynan, _NAN, from_okey(np.where(anynan, 0, hi)))
    return keys, mean.astype(np.float32), mn.astype(np.float32), mx.astype(np.float32), count


def entry_keys(src, dst, B, K):
    """(image int64 [E], key lo * 65536 + hi int64 [E], valid bool [E]) of graph entries."""
    src, dst = np.asarray(src, np.int64), np.asarray(dst, np.int64)
    n = B * K
    valid = (src >= 0) & (dst >= 0) & (src < n) & (dst < n) & (src != dst)
    s, d = np.where(valid, src, 0), np.where(valid, dst, 0)
    valid &= s // K == d // K
    b = s // K
    ls, ld = s - b * K, d - b * K
    return b, np.minimum(ls, ld) * 65536 + np.maximum(ls, ld), valid


def ref_boundary(labels, K, src, dst, values, connectivity=4):
    """int16 labels [B,H,W], entries src / dst [E], float32 values [B,C,H,W] -> (mean, min, max f32 [E,C],
    count int32 [E])."""
    labels = np.asarray(labels)
    values = np.asarray(values, np.float32)
    B, C = labels.shape[0], values.shape[1]
    E = len(src)
    mean = np.full((E, C), _NAN, np.float32)
    mn, mx = mean.copy(), mean.copy()
    count = np.zeros(E, np.int32)
    b, key, valid = entry_keys(src, dst, B, K)
    for i in range(B):
        sel = np.nonzero(valid & (b == i))[0]
        if sel.size == 0:
            continue
        keys, m, lo, hi, cnt = ref_boundary_image(labels[i], values[i], K, connectivity)
        at = np.searchsorted(keys, key[sel])
        hit = at < keys.size
        hit[hit] &= keys[at[hit]] == key[sel][hit]
        e, r = sel[hit], at[hit]
        mean[e], mn[e], mx[e], count[e] = m[:, r].T, lo[:, r].T, hi[:, r].T, cnt[r]
    return mean, mn, mx, count
