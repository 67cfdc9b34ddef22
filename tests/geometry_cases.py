"""fast_slic_b200.geometry restated in numpy, for the superpixel shape tests.

Integer fields by brute force over pixels: np.add.at for the area and the moments, np.minimum.at / np.maximum.at for
the box.  The perimeter from the four shifted neighbour maps of the label map padded with a sentinel that no uint16
label equals, the border from the padded sides alone.  The float fields from the integer ones, one float64 operation
at a time in the documented order.  Node k of image b is row [b, k].
"""
import numpy as np

FIELDS = ("area", "bbox", "moments", "perimeter", "border", "centroid", "covariance")
_SENTINEL = -1  # as int64 no uint16 label equals it


def _sides(lab):
    """Per pixel of int64 [B,H,W] maps: the number of its 4 sides across which the neighbour is outside the image or
    has another label, and the number of those on the image edge."""
    B, H, W = lab.shape
    pad = np.full((B, H + 2, W + 2), _SENTINEL, np.int64)
    pad[:, 1:-1, 1:-1] = lab
    edge = np.ones((H + 2, W + 2), bool)
    edge[1:-1, 1:-1] = False
    diff = np.zeros((B, H, W), np.int64)
    border = np.zeros((H, W), np.int64)
    for dy, dx in ((-1, 0), (1, 0), (0, -1), (0, 1)):
        diff += pad[:, 1 + dy:H + 1 + dy, 1 + dx:W + 1 + dx] != lab
        border += edge[1 + dy:H + 1 + dy, 1 + dx:W + 1 + dx]
    return diff, np.broadcast_to(border, (B, H, W))


def ref_finish(area, moments):
    """centroid float64 [...,2] and covariance float64 [...,3] from int area [...] and int64 moments [...,5]."""
    n = area.astype(np.float64)
    m = moments.astype(np.float64)  # int64 -> float64, round to nearest
    ok = area > 0
    q = np.zeros(m.shape, np.float64)
    np.divide(m, n[..., None], out=q, where=ok[..., None])
    cy, cx = q[..., 0], q[..., 1]
    cov = np.stack([q[..., 2] - cy * cy, q[..., 3] - cy * cx, q[..., 4] - cx * cx], -1)
    cov[~ok] = 0.0
    return np.stack([cy, cx], -1), cov


def ref_properties(labels, K):
    """int16 [B,H,W] -> dict of every field with the dtypes and shapes of region_properties."""
    lab = np.ascontiguousarray(labels).view(np.uint16).astype(np.int64)
    B, H, W = lab.shape
    N = B * K
    bb, yy, xx = (a.astype(np.int64) for a in np.meshgrid(np.arange(B), np.arange(H), np.arange(W), indexing="ij"))
    diff, border = _sides(lab)
    ok = lab < K
    node, y, x = bb[ok] * K + lab[ok], yy[ok], xx[ok]
    area = np.zeros(N, np.int64)
    np.add.at(area, node, 1)
    moments = np.zeros((N, 5), np.int64)
    for f, v in enumerate((y, x, y * y, x * y, x * x)):
        np.add.at(moments[:, f], node, v)
    lo = np.full((N, 2), np.iinfo(np.int64).max)
    hi = np.full((N, 2), -1, np.int64)
    np.minimum.at(lo[:, 0], node, y)
    np.minimum.at(lo[:, 1], node, x)
    np.maximum.at(hi[:, 0], node, y + 1)
    np.maximum.at(hi[:, 1], node, x + 1)
    some = area > 0
    bbox = np.zeros((N, 4), np.int64)
    bbox[some, :2], bbox[some, 2:] = lo[some], hi[some]
    perimeter = np.zeros(N, np.int64)
    bord = np.zeros(N, np.int64)
    np.add.at(perimeter, node, diff[ok])
    np.add.at(bord, node, border[ok])
    out = {"area": area.reshape(B, K).astype(np.int32), "bbox": bbox.reshape(B, K, 4).astype(np.int32),
           "moments": moments.reshape(B, K, 5), "perimeter": perimeter.reshape(B, K).astype(np.int32),
           "border": bord.reshape(B, K).astype(np.int32)}
    out["centroid"], out["covariance"] = ref_finish(out["area"], out["moments"])
    return out


def ref_properties_image(labels, K):
    """One int16 [H,W] map -> dict of every field, [K] / [K,4] / [K,5] / [K,2] / [K,3]."""
    return {f: v[0] for f, v in ref_properties(labels[None], K).items()}
