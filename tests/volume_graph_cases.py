"""fast_slic_b200.region_graph.region_adjacency_3d and fast_slic_b200.geometry.region_properties_3d restated in numpy,
for the volume graph and supervoxel shape tests.

The graph per volume: the voxel pairs by array slicing over the 3 / 9 / 13 forward offsets, the valid pairs with
differing labels, np.unique of their (low, high) keys with counts, both directions, lexsorted by (source, target).
The properties by brute force over voxels: np.add.at for the area and the moments, np.minimum.at / np.maximum.at for
the box, the surface from the six shifted neighbour volumes of the label volume padded with a sentinel that no uint16
label equals, the border from the padded faces alone, the float fields one float64 operation at a time.  Node k of
volume b is row [b, k] (node id b*K + k in the graph).
"""
import itertools

import numpy as np

FIELDS_3D = ("area", "bbox", "moments", "surface", "border", "centroid", "covariance")
_SENTINEL = -1  # as int64 no uint16 label equals it
# (zz, zy, zx, yy, yx, xx): the moment index of each covariance entry and its two axes
_COV = ((3, 0, 0), (4, 0, 1), (5, 0, 2), (6, 1, 1), (7, 1, 2), (8, 2, 2))


def forward_offsets(connectivity):
    """(dz, dy, dx) in {-1, 0, 1}^3 whose first non-zero component is positive, with at most 1 (connectivity 6),
    2 (18) or 3 (26) non-zero components."""
    most = {6: 1, 18: 2, 26: 3}[connectivity]
    out = []
    for o in itertools.product((-1, 0, 1), repeat=3):
        nz = [v for v in o if v]
        if nz and nz[0] > 0 and len(nz) <= most:
            out.append(o)
    return out


def _span(L, o):
    """The anchors' slice along an axis of length L for offset o, and their neighbours' slice."""
    return slice(max(0, -o), L - max(0, o)), slice(max(0, o), L + min(0, o))


def voxel_pairs(lab, connectivity):
    """The two ends of every unordered voxel pair of one [D,H,W] volume, flattened."""
    D, H, W = lab.shape
    a_parts, c_parts = [], []
    for o in forward_offsets(connectivity):
        (az, cz), (ay, cy), (ax, cx) = (_span(L, v) for L, v in zip((D, H, W), o))
        a_parts.append(lab[az, ay, ax].ravel())
        c_parts.append(lab[cz, cy, cx].ravel())
    return np.concatenate(a_parts), np.concatenate(c_parts)


def pair_count(D, H, W, connectivity):
    """P = sum over the forward offsets of (D - |dz|)(H - |dy|)(W - |dx|)."""
    if D * H * W == 0:
        return 0
    return sum((D - abs(dz)) * (H - abs(dy)) * (W - abs(dx)) for dz, dy, dx in forward_offsets(connectivity))


def ref_rag3d_volume(labels, K, connectivity):
    """One int16 [D,H,W] volume -> (source labels, target labels, boundary counts), int64, sorted by (source, target)."""
    lab = np.ascontiguousarray(labels).view(np.uint16).astype(np.int64)
    a, c = voxel_pairs(lab, connectivity)
    ok = (a < K) & (c < K) & (a != c)
    lo, hi = np.minimum(a[ok], c[ok]), np.maximum(a[ok], c[ok])
    keys, counts = np.unique(lo * K + hi, return_counts=True)
    lo, hi = keys // K, keys % K
    src, dst, w = np.concatenate([lo, hi]), np.concatenate([hi, lo]), np.concatenate([counts, counts])
    order = np.lexsort((dst, src))
    return src[order], dst[order], w[order]


def ref_rag3d(labels, K, connectivity=6):
    """int16 [B,D,H,W] -> (indptr int64[B*K+1], edge_index int64[2,E], boundary int32[E])."""
    B = labels.shape[0]
    parts = [ref_rag3d_volume(labels[b], K, connectivity) for b in range(B)]
    src = np.concatenate([p[0] + b * K for b, p in enumerate(parts)] + [np.zeros(0, np.int64)])
    dst = np.concatenate([p[1] + b * K for b, p in enumerate(parts)] + [np.zeros(0, np.int64)])
    w = np.concatenate([p[2] for p in parts] + [np.zeros(0, np.int64)])
    indptr = np.zeros(B * K + 1, np.int64)
    indptr[1:] = np.cumsum(np.bincount(src, minlength=B * K))
    return indptr, np.stack([src, dst]).astype(np.int64), w.astype(np.int32)


def _faces(lab):
    """Per voxel of int64 [B,D,H,W] volumes: the number of its 6 faces across which the neighbour is outside the
    volume or has another label, and the number of those on the volume's edge."""
    B, D, H, W = lab.shape
    pad = np.full((B, D + 2, H + 2, W + 2), _SENTINEL, np.int64)
    pad[:, 1:-1, 1:-1, 1:-1] = lab
    edge = np.ones((D + 2, H + 2, W + 2), bool)
    edge[1:-1, 1:-1, 1:-1] = False
    diff = np.zeros((B, D, H, W), np.int64)
    border = np.zeros((D, H, W), np.int64)
    for dz, dy, dx in ((-1, 0, 0), (1, 0, 0), (0, -1, 0), (0, 1, 0), (0, 0, -1), (0, 0, 1)):
        diff += pad[:, 1 + dz:D + 1 + dz, 1 + dy:H + 1 + dy, 1 + dx:W + 1 + dx] != lab
        border += edge[1 + dz:D + 1 + dz, 1 + dy:H + 1 + dy, 1 + dx:W + 1 + dx]
    return diff, np.broadcast_to(border, (B, D, H, W))


def ref_finish_3d(area, moments):
    """centroid float64 [...,3] and covariance float64 [...,6] from int area [...] and int64 moments [...,9]."""
    n = area.astype(np.float64)
    m = moments.astype(np.float64)  # int64 -> float64, round to nearest
    ok = area > 0
    q = np.zeros(m.shape, np.float64)
    np.divide(m, n[..., None], out=q, where=ok[..., None])
    c = q[..., :3]
    cov = np.stack([q[..., f] - c[..., a] * c[..., b] for f, a, b in _COV], -1)
    cov[~ok] = 0.0
    return c.copy(), cov


def ref_properties_3d(labels, K):
    """int16 [B,D,H,W] -> dict of every field with the dtypes and shapes of region_properties_3d."""
    lab = np.ascontiguousarray(labels).view(np.uint16).astype(np.int64)
    B, D, H, W = lab.shape
    N = B * K
    bb, zz, yy, xx = (a.astype(np.int64) for a in np.meshgrid(np.arange(B), np.arange(D), np.arange(H), np.arange(W),
                                                              indexing="ij"))
    diff, border = _faces(lab)
    ok = lab < K
    node, z, y, x = bb[ok] * K + lab[ok], zz[ok], yy[ok], xx[ok]
    area = np.zeros(N, np.int64)
    np.add.at(area, node, 1)
    moments = np.zeros((N, 9), np.int64)
    for f, v in enumerate((z, y, x, z * z, z * y, z * x, y * y, y * x, x * x)):
        np.add.at(moments[:, f], node, v)
    lo = np.full((N, 3), np.iinfo(np.int64).max)
    hi = np.full((N, 3), -1, np.int64)
    for a, v in enumerate((z, y, x)):
        np.minimum.at(lo[:, a], node, v)
        np.maximum.at(hi[:, a], node, v + 1)
    some = area > 0
    bbox = np.zeros((N, 6), np.int64)
    bbox[some, :3], bbox[some, 3:] = lo[some], hi[some]
    surface = np.zeros(N, np.int64)
    bord = np.zeros(N, np.int64)
    np.add.at(surface, node, diff[ok])
    np.add.at(bord, node, border[ok])
    out = {"area": area.reshape(B, K).astype(np.int32), "bbox": bbox.reshape(B, K, 6).astype(np.int32),
           "moments": moments.reshape(B, K, 9), "surface": surface.reshape(B, K),
           "border": bord.reshape(B, K).astype(np.int32)}
    out["centroid"], out["covariance"] = ref_finish_3d(out["area"], out["moments"])
    return out
