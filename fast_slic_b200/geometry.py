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
"""
import collections

import torch

from . import _lib
from ._labelmaps import check_K, check_pixels, cuda_device, tensor

# Longest side: with it and MAX_PIXELS every sum fits int64 (sum y^2 of a whole image is at most H W H^2 / 3 < 2^63)
MAX_SIDE = 65535

RegionProperties = collections.namedtuple("RegionProperties", [
    "area", "bbox", "moments", "perimeter", "border", "centroid", "covariance"])


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
