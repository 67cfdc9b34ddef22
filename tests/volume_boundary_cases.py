"""fast_slic_b200.region_graph.boundary_stats_3d and fast_slic_b200.groundtruth.segmentation_scores_3d /
boundaries_3d restated in numpy, for the volume boundary tests.

Boundary statistics per volume: the voxel pairs by array slicing over the forward offsets in RAG3D_OFFSETS order (the
same set as volume_graph_cases.forward_offsets), each with its ordinal anchor * Ndir + d; the boundary pairs (both
labels in [0, K) and different), lexsorted by (label-pair key, ordinal); each run of one key interleaves its anchor
and other values, summed in boundary_cases.lane_sums' lane order, min / max by boundary_cases.okey.  Entries look their
key up among the runs (boundary_cases.entry_keys).

Scores per volume: the overlap fields by groundtruth_cases.ref_scores_image on the [D*H, W] view (the overlap table
does not depend on the layout); the boundary maps by array slicing along x, y and z; the windows by a binary dilation
with the (2rz+1, 2ry+1, 2rx+1) box, scipy.ndimage.maximum_filter of that size.
"""
import numpy as np
from scipy import ndimage

from boundary_cases import entry_keys, from_okey, lane_sums, okey
from groundtruth_cases import FIELDS, gt_valid, ref_scores_image
from volume_graph_cases import forward_offsets

# region_graph.RAG3D_OFFSETS: direction d of a voxel pair, (dz, dy, dx)
OFFSETS = ((0, 0, 1), (0, 1, 0), (1, 0, 0), (0, 1, 1), (0, 1, -1), (1, 1, 0), (1, -1, 0), (1, 0, 1), (1, 0, -1),
           (1, 1, 1), (1, 1, -1), (1, -1, 1), (1, -1, -1))
NDIR = {6: 3, 18: 9, 26: 13}
_NAN = np.float32("nan")


def offsets(connectivity):
    """The forward offsets of a connectivity in RAG3D_OFFSETS order."""
    out = OFFSETS[:NDIR[connectivity]]
    assert sorted(out) == sorted(forward_offsets(connectivity))
    return out


def pair_ends_3d(D, H, W, connectivity):
    """(anchor, other, ordinal) int64 flat voxel indices and ordinals of every voxel pair of a [D,H,W] volume."""
    idx = np.arange(D * H * W, dtype=np.int64).reshape(D, H, W)
    nd = NDIR[connectivity]
    anchors, others, ords = [], [], []
    for d, o in enumerate(offsets(connectivity)):
        a_sl = tuple(slice(max(0, -v), L - max(0, v)) for L, v in zip((D, H, W), o))
        o_sl = tuple(slice(max(0, v), L + min(0, v)) for L, v in zip((D, H, W), o))
        a = idx[a_sl].ravel()
        anchors.append(a)
        others.append(idx[o_sl].ravel())
        ords.append(a * nd + d)
    return np.concatenate(anchors), np.concatenate(others), np.concatenate(ords)


def run_stats(lab, feats, anchor, other, ordinal, K):
    """lab int64 [N] flat labels, feats float32 [C,N], the pairs -> (keys lo * 65536 + hi [R], mean, min, max f32
    [C,R], count int64 [R]) of the R runs of boundary pairs, in key order."""
    C = feats.shape[0]
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


def ref_boundary3d_volume(labels, values, K, connectivity):
    """One int16 [D,H,W] volume and float32 [C,D,H,W] values -> run_stats' runs."""
    D, H, W = labels.shape
    lab = np.ascontiguousarray(labels).view(np.uint16).ravel().astype(np.int64)
    feats = np.ascontiguousarray(values, np.float32).reshape(values.shape[0], -1)
    return run_stats(lab, feats, *pair_ends_3d(D, H, W, connectivity), K)


def ref_boundary3d(labels, K, src, dst, values, connectivity=6):
    """int16 labels [B,D,H,W], entries src / dst [E], float32 values [B,C,D,H,W] -> (mean, min, max f32 [E,C],
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
        keys, m, lo, hi, cnt = ref_boundary3d_volume(labels[i], values[i], K, connectivity)
        at = np.searchsorted(keys, key[sel])
        hit = at < keys.size
        hit[hit] &= keys[at[hit]] == key[sel][hit]
        e, r = sel[hit], at[hit]
        mean[e], mn[e], mx[e], count[e] = m[:, r].T, lo[:, r].T, hi[:, r].T, cnt[r]
    return mean, mn, mx, count


def ref_boundaries_3d(labels):
    """int16 [B,D,H,W] -> bool [B,D,H,W]: the +x, +y or +z neighbour exists and has another label."""
    lab = np.asarray(labels).view(np.uint16)
    out = np.zeros(lab.shape, bool)
    out[..., :-1] |= lab[..., :-1] != lab[..., 1:]
    out[..., :-1, :] |= lab[..., :-1, :] != lab[..., 1:, :]
    out[..., :-1, :, :] |= lab[..., :-1, :, :] != lab[..., 1:, :, :]
    return out


def gt_boundary_map_3d(gt, ignore_index=None):
    """[D,H,W] gt -> bool [D,H,W]: valid voxels whose +x, +y or +z neighbour is valid and has another value."""
    g = gt.astype(np.int64)
    ok = gt_valid(gt, ignore_index)
    out = np.zeros(g.shape, bool)
    out[:, :, :-1] |= ok[:, :, :-1] & ok[:, :, 1:] & (g[:, :, :-1] != g[:, :, 1:])
    out[:, :-1, :] |= ok[:, :-1, :] & ok[:, 1:, :] & (g[:, :-1, :] != g[:, 1:, :])
    out[:-1, :, :] |= ok[:-1, :, :] & ok[1:, :, :] & (g[:-1, :, :] != g[1:, :, :])
    return out


def tolerance_3d(tolerance):
    return tuple(tolerance) if isinstance(tolerance, (tuple, list)) else (tolerance,) * 3


def dilate_3d(mask, tolerance):
    """Binary dilation of a bool [D,H,W] mask by the box |dz| <= rz, |dy| <= ry, |dx| <= rx, clipped to the volume."""
    rz, ry, rx = tolerance_3d(tolerance)
    return ndimage.maximum_filter(mask.astype(np.uint8), size=(2 * rz + 1, 2 * ry + 1, 2 * rx + 1), mode="constant",
                                  cval=0).astype(bool)


def ref_scores_volume(labels, gt, K, tolerance=2, ignore_index=None):
    """One int16 [D,H,W] label volume and its gt -> dict of the seven integer fields."""
    D, H, W = labels.shape
    res = ref_scores_image(labels.reshape(D * H, W), gt.reshape(D * H, W), K, 0, ignore_index)
    ok = gt_valid(gt, ignore_index)
    sp = ref_boundaries_3d(labels[None])[0]
    gb = gt_boundary_map_3d(gt, ignore_index)
    res["gt_boundary"] = int(gb.sum())
    res["gt_boundary_hits"] = int((gb & dilate_3d(sp, tolerance)).sum())
    res["sp_boundary"] = int((sp & ok).sum())
    res["sp_boundary_hits"] = int((sp & ok & dilate_3d(gb, tolerance)).sum())
    return res


def ref_scores_3d(labels, gt, K, tolerance=2, ignore_index=None):
    """int16 [B,D,H,W] labels and their gt -> dict of int64 [B] arrays (the seven integer fields) and the four float64
    ratios (NaN where the denominator is 0)."""
    per = [ref_scores_volume(labels[b], gt[b], K, tolerance, ignore_index) for b in range(labels.shape[0])]
    res = {f: np.array([p[f] for p in per], np.int64) for f in FIELDS}

    def ratio(num, den):
        with np.errstate(invalid="ignore", divide="ignore"):
            return np.where(res[den] > 0, res[num] / np.maximum(res[den], 1), np.nan)

    res["asa"] = ratio("asa_pixels", "pixels")
    res["undersegmentation"] = ratio("ue_pixels", "pixels")
    res["boundary_recall"] = ratio("gt_boundary_hits", "gt_boundary")
    res["boundary_precision"] = ratio("sp_boundary_hits", "sp_boundary")
    return res
