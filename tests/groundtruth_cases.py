"""fast_slic_b200.groundtruth restated in numpy, for the ground-truth score tests.

Per image: the class histogram by np.unique over combined (label, class) keys; the overlap table n_kg by np.unique over
combined (label, gt) keys of the counted pixels; the boundary maps by array slicing; the tolerance windows by a binary
dilation with the (2r+1)^2 square, as scipy.ndimage.maximum_filter of that size (the square is separable, so this stays
fast at r = 32 on large maps; the CPU tests check it against binary_dilation and against scanning every window).
"""
import numpy as np
from scipy import ndimage

FIELDS = ("pixels", "asa_pixels", "ue_pixels", "gt_boundary", "gt_boundary_hits", "sp_boundary", "sp_boundary_hits")


def ref_class_histogram(classes, labels, K, C):
    """[B,H,W] classes (any integer dtype), int16 labels -> int32 [B,K,C]."""
    B = labels.shape[0]
    out = np.zeros((B, K, C), np.int32)
    for b in range(B):
        lab = labels[b].view(np.uint16).astype(np.int64).ravel()
        cls = classes[b].astype(np.int64).ravel()
        ok = (lab < K) & (cls >= 0) & (cls < C)
        keys, counts = np.unique(lab[ok] * C + cls[ok], return_counts=True)
        out[b].reshape(-1)[keys] = counts
    return out


def ref_boundaries(labels):
    """int16 [B,H,W] -> bool [B,H,W]: the right or lower neighbour exists and has another label."""
    lab = labels.view(np.uint16)
    out = np.zeros(lab.shape, bool)
    out[:, :, :-1] |= lab[:, :, :-1] != lab[:, :, 1:]
    out[:, :-1, :] |= lab[:, :-1, :] != lab[:, 1:, :]
    return out


def gt_valid(gt, ignore_index=None):
    g = gt.astype(np.int64)
    ok = (g >= 0) & (g <= 2 ** 31 - 1)
    if ignore_index is not None:
        ok &= g != ignore_index
    return ok


def gt_boundary_map(gt, ignore_index=None):
    """[H,W] gt -> bool [H,W]: valid pixels whose right or lower neighbour is valid and has another value."""
    g = gt.astype(np.int64)
    ok = gt_valid(gt, ignore_index)
    out = np.zeros(g.shape, bool)
    out[:, :-1] |= ok[:, :-1] & ok[:, 1:] & (g[:, :-1] != g[:, 1:])
    out[:-1, :] |= ok[:-1, :] & ok[1:, :] & (g[:-1, :] != g[1:, :])
    return out


def dilate(mask, r):
    """Binary dilation of a bool [H,W] mask by the (2r+1)^2 square, clipped to the map."""
    return ndimage.maximum_filter(mask.astype(np.uint8), size=2 * r + 1, mode="constant", cval=0).astype(bool)


def ref_scores_image(labels, gt, K, tolerance=2, ignore_index=None):
    """One int16 [H,W] label map and its gt -> dict of the seven integer fields."""
    lab = labels.view(np.uint16).astype(np.int64)
    g = gt.astype(np.int64)
    ok = gt_valid(gt, ignore_index)
    counted = ok & (lab < K)
    res = dict.fromkeys(FIELDS, 0)
    res["pixels"] = int(counted.sum())
    if res["pixels"]:
        gv = g[counted]
        # (label, gt) -> n_kg, by unique over combined keys (gt < 2^31)
        keys, n_kg = np.unique(lab[counted] * 2 ** 31 + gv, return_counts=True)
        k_of = keys // 2 ** 31
        n_k = np.bincount(k_of, weights=n_kg, minlength=K).astype(np.int64)
        mx = np.zeros(K, np.int64)
        np.maximum.at(mx, k_of, n_kg)
        res["asa_pixels"] = int(mx.sum())
        res["ue_pixels"] = int(np.minimum(n_kg, n_k[k_of] - n_kg).sum())
    sp = ref_boundaries(labels[None])[0]
    gb = gt_boundary_map(gt, ignore_index)
    res["gt_boundary"] = int(gb.sum())
    res["gt_boundary_hits"] = int((gb & dilate(sp, tolerance)).sum())
    res["sp_boundary"] = int((sp & ok).sum())
    res["sp_boundary_hits"] = int((sp & ok & dilate(gb, tolerance)).sum())
    return res


def ref_scores(labels, gt, K, tolerance=2, ignore_index=None):
    """int16 [B,H,W] labels and their gt -> dict of int64 [B] arrays (the seven integer fields) and the four float64
    ratios (NaN where the denominator is 0)."""
    per = [ref_scores_image(labels[b], gt[b], K, tolerance, ignore_index) for b in range(labels.shape[0])]
    res = {f: np.array([p[f] for p in per], np.int64) for f in FIELDS}

    def ratio(num, den):
        with np.errstate(invalid="ignore", divide="ignore"):
            return np.where(res[den] > 0, res[num] / np.maximum(res[den], 1), np.nan)

    res["asa"] = ratio("asa_pixels", "pixels")
    res["undersegmentation"] = ratio("ue_pixels", "pixels")
    res["boundary_recall"] = ratio("gt_boundary_hits", "gt_boundary")
    res["boundary_precision"] = ratio("sp_boundary_hits", "sp_boundary")
    return res
