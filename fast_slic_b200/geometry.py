"""Superpixel shapes on the GPU (csrc/props.cuh), for whole batches of the int16 label maps iterate_batch returns:
each superpixel's area, bounding box, raw moments, perimeter, centroid and covariance -- what skimage.measure.regionprops
gives one image at a time.  With pooling.pool it gives a superpixel GNN positions next to its node features::

    x = pool(features, labels, K)                                   # [B,C,K] node features
    p = region_properties(labels, K)
    pos = p.centroid / torch.tensor([H, W], dtype=torch.float64, device=labels.device)   # [B,K,2] in [0, 1)

These describe the returned label map.  Cluster.y / x / num_members do not: they come from the last update over the
row subsample, before connectivity enforcement moved pixels between labels.  No counterpart in the reference.  Cuda
tensors only; every argument is checked (ValueError) before any device work.  Work runs on the labels' device, on its
current stream, with no scratch and nothing read back, so a CUDA graph can capture the call.  DESIGN.md section 4.15
describes the kernels.

region_properties_3d gives the same of supervoxel label volumes [B,D,H,W], with the surface in place of the perimeter
(DESIGN.md section 4.23)::

    p = region_properties_3d(r.labels, K2)                          # r = supervoxel_slic(...); p.centroid [B,K2,3]
    mm = p.centroid * torch.tensor(spacing, dtype=torch.float64, device=p.centroid.device)   # (z, y, x) in mm
"""
import collections

import torch

from . import _lib
from ._labelmaps import MAX_PIXELS, check_K, check_pixels, cuda_device, tensor

# Longest side: with it and MAX_PIXELS every sum fits int64 (sum y^2 of a whole image is at most H W H^2 / 3 < 2^63)
MAX_SIDE = 65535
# Longest side of a volume (supervoxels' limit): with MAX_PIXELS every sum fits int64 (sum z^2 <= N D^2 < 2^59)
MAX_SIDE_3D = 32767

RegionProperties = collections.namedtuple("RegionProperties", [
    "area", "bbox", "moments", "perimeter", "border", "centroid", "covariance"])
RegionProperties3D = collections.namedtuple("RegionProperties3D", [
    "area", "bbox", "moments", "surface", "border", "centroid", "covariance"])


def region_properties(labels, K):
    """Shapes of the superpixels of int16 labels [B,H,W] (read as uint16) -> RegionProperties, every field indexed
    [b, k] for label k of image b (node b*K + k of pool's [B,C,K] and region_adjacency's graph).  Pixel (row y,
    column x) has coordinates (y, x), skimage's convention.  A label outside [0, K) (-1 included) belongs to no
    superpixel.
    - area       int32 [B,K]: pixels labelled k (mask empty superpixels with area > 0);
    - bbox       int32 [B,K,4]: (y0, x0, y1, x1), min inclusive and max exclusive (skimage's bbox); all 0 when empty;
    - moments    int64 [B,K,5]: raw sums (sum y, sum x, sum y^2, sum xy, sum x^2) over k's pixels, exact;
    - perimeter  int32 [B,K]: crack length, the sides of k's pixels whose 4-neighbour across that side lies outside the
      image or has another raw label (-1 and labels >= K count as other labels);
    - border     int32 [B,K]: those of the sides that lie on the image edge;
    - centroid   float64 [B,K,2]: (sum y / n, sum x / n);
    - covariance float64 [B,K,3]: (sum y^2 / n - cy cy, sum xy / n - cy cx, sum x^2 / n - cx cx), the central second
      moments over n (skimage's inertia_tensor entries up to sign and order).
    The float fields come from the integer ones, each step one correctly rounded float64 operation; an empty
    superpixel gets 0.0, never NaN.  1 <= K <= 65534, H, W <= 65535 and H * W <= 2^29; anything else, or a tensor that
    is not a cuda int16 [B,H,W] tensor, raises ValueError before any device work.  B, H or W = 0 gives zeros without a
    launch.  All kernel arithmetic is integer: image b's result depends only on labels[b], not on the batch, the stream
    or the run."""
    tensor("labels", labels, torch.int16, 3)
    K = check_K(K)
    B, H, W = (int(v) for v in labels.shape)
    if H > MAX_SIDE or W > MAX_SIDE:
        raise ValueError("images of %dx%d pixels have a side over %d: a moment could overflow int64" % (H, W, MAX_SIDE))
    check_pixels(H, W, ": a moment could overflow int64")
    dev = cuda_device(labels)
    with torch.cuda.device(dev):
        empty = B == 0 or H == 0 or W == 0
        new = torch.zeros if empty else torch.empty
        out = RegionProperties(new((B, K), dtype=torch.int32, device=dev), new((B, K, 4), dtype=torch.int32, device=dev),
                               new((B, K, 5), dtype=torch.int64, device=dev), new((B, K), dtype=torch.int32, device=dev),
                               new((B, K), dtype=torch.int32, device=dev), new((B, K, 2), dtype=torch.float64, device=dev),
                               new((B, K, 3), dtype=torch.float64, device=dev))
        if not empty:
            lab = labels.contiguous()
            _lib.check(_lib.lib().fslic_b200_props_batch(dev.index, B, H, W, K, lab.data_ptr(),
                                                         *(f.data_ptr() for f in out),
                                                         torch.cuda.current_stream(dev).cuda_stream))
    return out


def region_properties_3d(labels, K):
    """Shapes of the supervoxels of int16 label volumes [B,D,H,W] (read as uint16) -> RegionProperties3D, every field
    indexed [b, k] for label k of volume b (node b*K + k of region_adjacency_3d's graph).  Voxel (slice z, row y,
    column x) has coordinates (z, y, x), skimage's order for 3-D regionprops.  A label outside [0, K) (-1 included)
    belongs to no supervoxel.
    - area       int32 [B,K]: voxels labelled k;
    - bbox       int32 [B,K,6]: (z0, y0, x0, z1, y1, x1), min inclusive and max exclusive; all 0 when empty;
    - moments    int64 [B,K,9]: raw sums (sum z, y, x, z^2, zy, zx, y^2, yx, x^2) over k's voxels, exact;
    - surface    int64 [B,K]: voxel faces of k whose 6-neighbour across that face lies outside the volume or has another
      raw label (-1 and labels >= K count as other labels), the 3-D crack perimeter;
    - border     int32 [B,K]: those of the faces that lie on the volume's edge;
    - centroid   float64 [B,K,3]: (sum z / n, sum y / n, sum x / n);
    - covariance float64 [B,K,6]: (zz, zy, zx, yy, yx, xx), each sum ab / n - c_a c_b, the central second moments.
    The float fields follow region_properties: int64 -> float64 rounded to nearest, then one correctly rounded float64
    operation per step (no FMA); an empty supervoxel gets 0.0.  Coordinates are in voxels: scale centroid and
    covariance by the voxel spacing for physical units.  1 <= K <= 65534, D, H, W <= 32767 and D * H * W <= 2^29;
    anything else, or a tensor that is not a cuda int16 [B,D,H,W] tensor, raises ValueError before any device work.
    B, D, H or W = 0 gives zeros without a launch.  No scratch and nothing read back, so a CUDA graph can capture the
    call.  All kernel arithmetic is integer: volume b's result depends only on labels[b]."""
    tensor("labels", labels, torch.int16, 4)
    K = check_K(K)
    B, D, H, W = (int(v) for v in labels.shape)
    if max(D, H, W) > MAX_SIDE_3D or D * H * W > MAX_PIXELS:
        raise ValueError("volumes must be at most %d voxels on each side and %d voxels in all, got %dx%dx%d: a moment "
                         "could overflow int64" % (MAX_SIDE_3D, MAX_PIXELS, D, H, W))
    dev = cuda_device(labels)
    with torch.cuda.device(dev):
        empty = B * D * H * W == 0
        new = torch.zeros if empty else torch.empty
        out = RegionProperties3D(new((B, K), dtype=torch.int32, device=dev),
                                 new((B, K, 6), dtype=torch.int32, device=dev),
                                 new((B, K, 9), dtype=torch.int64, device=dev),
                                 new((B, K), dtype=torch.int64, device=dev),
                                 new((B, K), dtype=torch.int32, device=dev),
                                 new((B, K, 3), dtype=torch.float64, device=dev),
                                 new((B, K, 6), dtype=torch.float64, device=dev))
        if not empty:
            lab = labels.contiguous()
            _lib.check(_lib.lib().fslic_b200_props3d_batch(dev.index, B, D, H, W, K, lab.data_ptr(),
                                                           *(f.data_ptr() for f in out),
                                                           torch.cuda.current_stream(dev).cuda_stream))
    return out
