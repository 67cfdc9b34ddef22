"""SLIC over float feature maps on the GPU (csrc/float_slic.cuh): superpixels of float32 [B,C,H,W] tensors -- RGB-D,
multispectral bands, float Lab, a network's feature maps -- with any number of channels::

    x = torch.cat([lab_float, depth[:, None] * alpha], 1)          # [B,4,H,W] float32 on the GPU
    r = feature_slic(x, K=1600, compactness=10.0)
    means = pool(x, r.labels, 1600)                                # then region_adjacency, region_properties, ...

A new algorithm with its own contract, not a reference port (DESIGN.md section 4.19 gives every float32 operation and
its order): the result is exact and deterministic -- the bits of image b depend only on features[b] and the
arguments, not on the batch, the chunking, the stream or the run.  Cuda tensors only.  Work is enqueued on the features'
device on its current torch stream with no host synchronisation and no read-back, so a CUDA graph can capture it;
every argument is checked (ValueError) before any device work.  Not differentiable.
"""
import collections
import ctypes
import math

import torch

from . import _lib
from ._labelmaps import FLOAT_SLIC_MAX_C as MAX_C
from ._labelmaps import FLOAT_SLIC_MAX_NODES as MAX_NODES
from ._labelmaps import FLOAT_SLIC_MAX_SIDE as MAX_SIDE
from ._labelmaps import FLOAT_SLIC_MAX_STRIDE as MAX_STRIDE
from ._labelmaps import MAX_K, MAX_PIXELS, check_int, check_number, chunk, slic_dispatch, slic_pass_tiles, tensor
from .base_slic import _locked, get_cca_engine

# Device memory one launch takes for its scratch at most (about 16 bytes per pass-row pixel, plus 4 * C + 8 per
# cluster): a batch that needs more runs in chunks of images, with identical results.
FEATURE_SLIC_SCRATCH_CAP = 1 << 30
TILE_W, TILE_R = 32, 8  # MapSlic::TILE_W, TILE_R of float_slic.cuh

FeatureSlic = collections.namedtuple("FeatureSlic", "labels position features count")
FeatureSlic.__doc__ = """labels int16 [B,H,W] after connectivity enforcement; position float32 [B,K,2] (y, x),
features float32 [B,K,C] and count int32 [B,K] of the centres after the last update (the seeds when max_iter == 0,
count 0 then), which describe the map before enforcement."""


def superpixel_size(H, W, K):
    """S = (int)(int16)sqrt((double)(H*W/K)), the grid step and window radius (values up to 23170 fit int16)."""
    return int(math.sqrt((H * W) // K))


def min_size_threshold(S, min_size_factor):
    """round(S^2 * min_size_factor) as the u16 path computes it: min_size_factor as float32, C's round."""
    x = float(S * S) * ctypes.c_float(min_size_factor).value
    t = math.floor(x)
    return int(t + 1 if x - t >= 0.5 else t)


def _check(features, K, compactness, max_iter, subsample_stride, min_size_factor, init):
    tensor("features", features, torch.float32, 4)
    B, C, H, W = (int(v) for v in features.shape)
    if not 1 <= C <= MAX_C:
        raise ValueError("features must have 1 to %d channels, got %d" % (MAX_C, C))
    if not (1 <= H <= MAX_SIDE and 1 <= W <= MAX_SIDE) or H * W > MAX_PIXELS:
        raise ValueError("images must be 1 to %d pixels on each side and at most %d pixels, got %dx%d" % (
            MAX_SIDE, MAX_PIXELS, H, W))
    K = check_int("K", K, 1, min(MAX_K, H * W))
    if B * K > MAX_NODES:
        raise ValueError("B*K must be at most %d, got %d" % (MAX_NODES, B * K))
    compactness = check_number("compactness", compactness)
    if not (math.isfinite(compactness) and compactness > 0) or not math.isfinite(ctypes.c_float(compactness).value):
        raise ValueError("compactness must be finite and > 0, got %r" % compactness)
    max_iter = check_int("max_iter", max_iter, 0, 2 ** 31 - 2)
    subsample_stride = check_int("subsample_stride", subsample_stride, 1, MAX_STRIDE)
    min_size_factor = check_number("min_size_factor", min_size_factor)
    if not min_size_factor >= 0:
        raise ValueError("min_size_factor must be >= 0, got %r" % min_size_factor)
    if init is not None:
        if not isinstance(init, (tuple, list)) or len(init) != 2:
            raise ValueError("init must be (position, features) of an earlier result")
        position, feats = init
        tensor("init position", position, torch.float32, 3)
        tensor("init features", feats, torch.float32, 3)
        if tuple(position.shape) != (B, K, 2) or tuple(feats.shape) != (B, K, C):
            raise ValueError("init must be position [B,K,2] = %s and features [B,K,C] = %s, got %s and %s" % (
                (B, K, 2), (B, K, C), tuple(position.shape), tuple(feats.shape)))
        for name, x in (("init position", position), ("init features", feats)):
            if x.device != features.device:
                raise ValueError("%s is on %s, features on %s" % (name, x.device, features.device))
        init = (position.contiguous(), feats.contiguous())
    if features.device.type != "cuda":
        raise ValueError("features is a %s tensor: pass cuda tensors (torch.from_numpy(...).cuda())" %
                         features.device.type)
    return (B, C, H, W), K, compactness, max_iter, subsample_stride, min_size_factor, init


def _run(features, K, compactness, max_iter, subsample_stride, min_size_factor, init, overflow=None):
    (B, C, H, W), K, compactness, max_iter, stride, min_size_factor, init = _check(
        features, K, compactness, max_iter, subsample_stride, min_size_factor, init)
    dev = features.device
    L = _lib.lib()
    with torch.cuda.device(dev):
        labels = torch.empty((B, H, W), dtype=torch.int16, device=dev)
        position = torch.empty((B, K, 2), dtype=torch.float32, device=dev)
        centroids = torch.empty((B, K, C), dtype=torch.float32, device=dev)
        count = torch.empty((B, K), dtype=torch.int32, device=dev)
        if B == 0:
            return FeatureSlic(labels, position, centroids, count)
        x = features.contiguous()
        f = L.fslic_b200_feature_slic_scratch_bytes
        n = chunk(lambda c: f(c, H, W, C, K, stride, max_iter), FEATURE_SLIC_SCRATCH_CAP, B, limit=65535)
        nbytes = int(f(n, H, W, C, K, stride, max_iter))
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        stream = torch.cuda.current_stream(dev).cuda_stream
        thres = min_size_threshold(superpixel_size(H, W, K), min_size_factor)
        with _locked(lambda: get_cca_engine(H, W, n, dev.index)) as eng:
            for i, b0 in enumerate(range(0, B, n)):
                c = min(n, B - b0)
                _lib.check(L.fslic_b200_feature_slic(
                    dev.index, c, H, W, C, K, compactness, stride, max_iter, x[b0].data_ptr(),
                    None if init is None else init[0][b0].data_ptr(), None if init is None else init[1][b0].data_ptr(),
                    labels[b0].data_ptr(), position[b0].data_ptr(), centroids[b0].data_ptr(), count[b0].data_ptr(),
                    None if overflow is None else overflow[i].data_ptr(), scratch.data_ptr(), nbytes, stream))
                eng.enforce_connectivity(labels[b0:b0 + c], K, thres)
    return FeatureSlic(labels, position, centroids, count)


def feature_slic(features, K, compactness, max_iter=10, subsample_stride=3, min_size_factor=0.25, init=None):
    """SLIC superpixels of float32 feature maps [B,C,H,W] (cuda) -> FeatureSlic(labels, position, features, count).

    Seeds lie on the grid of the uint8 path (step S = sqrt(H*W/K)) with the features of their pixel, or come from
    init = (position, features) of an earlier result (a video's previous frame; positions are clamped into the image).
    Pass t < max_iter assigns the rows i with i % subsample_stride == t % subsample_stride to the centre minimising
    sum_c (f_c - mu_c)^2 + (compactness / S)^2 * ((i - cy)^2 + (j - cx)^2) among the centres within S rows and columns,
    ties to the lower index, and moves every centre with members on those rows to their mean position and pooled mean
    features; one assign over every row follows, then connectivity enforcement (components smaller than
    round(S^2 * min_size_factor) pixels are absorbed), like iterate_batch.  compactness has no default: the feature
    distance has no fixed scale.  For statistics of the returned map use pooling.pool (per-superpixel means of any
    feature map) and geometry.region_properties (area, centroid, bounding box, moments).  Limits: 1 <= C <= 1024,
    1 <= K <= min(65534, H*W), H, W <= 32767, H*W <= 2^29, B*K <= 2^30, 1 <= subsample_stride <= 255."""
    return _run(features, K, compactness, max_iter, subsample_stride, min_size_factor, init)


def pass_tiles(H, W, max_iter, subsample_stride):
    """Tiles per image of every assign pass: max_iter strided passes, then the full one."""
    return slic_pass_tiles((H, W), (TILE_R, TILE_W), max_iter, subsample_stride)


def feature_slic_dispatch(features, K, compactness, max_iter=10, subsample_stride=3, min_size_factor=0.25, init=None):
    """feature_slic with a record of the assign kernels it ran (synchronises): (result, [(tiles, overflowed)] per
    pass), the tiles of the pass over the whole batch and how many of them overflowed the tile kernel's candidate
    list and went to the per-pixel kernel."""
    return slic_dispatch(lambda it, overflow: _run(features, K, compactness, it, subsample_stride, min_size_factor,
                                                   init, overflow), features, max_iter, subsample_stride,
                         (TILE_R, TILE_W))
