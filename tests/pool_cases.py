"""The summation order of fast_slic_b200.pooling restated in numpy (DESIGN.md section 4.12), for the pooling tests.

The members of superpixel k of one image, in raster order m_0, m_1, ..., are dealt to 32 lanes: lane l adds
f[m_l], f[m_{l+32}], ... left to right in float32, starting from +0.0.  Five butterfly steps (o = 16, 8, 4, 2, 1:
v_l = v_l + v_{l xor o}) combine the lanes; the sum is lane 0's value.  The mean is sum / float32(count).
"""
import numpy as np


def ref_pool(features, labels, K):
    """One image: float32 features [C,H,W], int16 labels [H,W] -> (sums f32[C,K], means f32[C,K], counts int64[K])."""
    feats = np.ascontiguousarray(features, np.float32).reshape(features.shape[0], -1)
    lab = np.ascontiguousarray(labels).view(np.uint16).ravel().astype(np.int64)
    C = feats.shape[0]
    pix = np.nonzero(lab < K)[0]
    order = pix[np.argsort(lab[pix], kind="stable")]  # grouped by label, raster order inside each label
    seg_lab = lab[order]
    counts = np.bincount(seg_lab, minlength=K)
    sums = np.zeros((C, K), np.float32)
    if order.size:
        used, first = np.unique(seg_lab, return_index=True)
        seg = np.searchsorted(used, seg_lab)
        pos = np.arange(order.size) - first[seg]
        rows = int(pos.max()) // 32 + 1
        # lanes [C, used, rows, 32], the members past a segment's end padded with +0.0: adding +0.0 to a lane's
        # partial sum (never -0.0, since it starts from +0.0) changes nothing, NaN and inf included
        A = np.zeros((C, used.size, rows, 32), np.float32)
        A[:, seg, pos // 32, pos % 32] = feats[:, order]
        v = np.zeros((C, used.size, 32), np.float32)
        with np.errstate(invalid="ignore", over="ignore"):
            for r in range(rows):
                v = v + A[:, :, r, :]
            lanes = np.arange(32)
            for off in (16, 8, 4, 2, 1):
                v = v + v[:, :, lanes ^ off]
        sums[:, used] = v[:, :, 0]
    means = np.zeros_like(sums)
    nz = counts > 0
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        means[:, nz] = sums[:, nz] / counts[nz].astype(np.float32)
    return sums, means, counts


def ref_pool_batch(features, labels, K):
    """[B,C,H,W], [B,H,W] -> (sums [B,C,K], means [B,C,K], counts int32 [B,K]), image by image."""
    out = [ref_pool(features[b], labels[b], K) for b in range(labels.shape[0])]
    C = features.shape[1]
    if not out:
        return (np.zeros((0, C, K), np.float32), np.zeros((0, C, K), np.float32), np.zeros((0, K), np.int32))
    return (np.stack([o[0] for o in out]), np.stack([o[1] for o in out]),
            np.stack([o[2] for o in out]).astype(np.int32))


def nan_class_equal(a, b):
    """Bit-identical (signed zeros included), except that any NaN equals any NaN."""
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    if not (na == nb).all():
        return False
    return bool((a.view(np.uint32)[~na] == b.view(np.uint32)[~nb]).all())
