"""Supervoxels on the GPU (csrc/float_slic.cuh, csrc/sv_cca.cuh): SLIC over float32 volumes [B,C,D,H,W] -- CT, MRI,
microscopy stacks -- with a voxel spacing, and connectivity enforcement of label volumes in 6-connectivity::

    x = ct[:, None]                                                                        # [B,1,D,H,W] float32
    r = supervoxel_slic(x, K=16384, compactness=0.1, spacing=(2.5, 0.7, 0.7))
    K2 = r.position.shape[1]
    means = pool(x.view(B, 1, D * H, W), r.labels.view(B, D * H, W), K2)                    # per-supervoxel means

A new algorithm with its own contract, not a reference port (DESIGN.md section 4.22 gives every float32 operation and
its order, and the enforcement rules): the result is exact and deterministic -- the bits of volume b depend only on
volumes[b] and the arguments, not on the batch, the chunking, the stream or the run.  Cuda tensors only.  Work is
enqueued on the volumes' device on its current torch stream with no host synchronisation and no read-back, so a CUDA
graph can capture it; every argument is checked (ValueError) before any device work.  Not differentiable.
"""
import collections
import math

import numpy as np
import torch

from . import _lib
from ._labelmaps import FLOAT_SLIC_MAX_C as MAX_C
from ._labelmaps import FLOAT_SLIC_MAX_NODES as MAX_NODES
from ._labelmaps import FLOAT_SLIC_MAX_SIDE as MAX_SIDE
from ._labelmaps import FLOAT_SLIC_MAX_STRIDE as MAX_STRIDE
from ._labelmaps import MAX_K, MAX_PIXELS, check_int, check_number, chunk, slic_dispatch, slic_pass_tiles, tensor
# Device memory one launch takes for its scratch at most (about 20 bytes per voxel for the enforcement, more for the
# passes at large C): a batch that needs more runs in chunks of volumes, with identical results.
SUPERVOXEL_SCRATCH_CAP = 1 << 30
TILE_W, TILE_R, TILE_D = 16, 4, 4  # VolumeSlic::TILE_W, TILE_R, TILE_D of float_slic.cuh

Supervoxels = collections.namedtuple("Supervoxels", "labels position features count grid")
Supervoxels.__doc__ = """labels int16 [B,D,H,W] after connectivity enforcement (read them as uint16 when K' > 32767);
position float32 [B,K',3] (z, y, x), features float32 [B,K',C] and count int32 [B,K'] of the centres after the last
update (the seeds when max_iter == 0, count 0 then), which describe the labels before enforcement; grid (nd, nh, nw),
K' = nd * nh * nw."""


def _spacing(spacing):
    if not isinstance(spacing, (tuple, list)) or len(spacing) != 3:
        raise ValueError("spacing must be (z, y, x), got %r" % (spacing,))
    sp = tuple(check_number("spacing", v) for v in spacing)
    if not all(math.isfinite(v) and v > 0 for v in sp):
        raise ValueError("spacing must be finite and > 0, got %r" % (spacing,))
    return sp


def _sides(D, H, W):
    if not all(1 <= v <= MAX_SIDE for v in (D, H, W)) or D * H * W > MAX_PIXELS:
        raise ValueError("volumes must be 1 to %d voxels on each side and at most %d voxels, got %dx%dx%d" % (
            MAX_SIDE, MAX_PIXELS, D, H, W))


def volume_grid(D, H, W, K, spacing=(1.0, 1.0, 1.0)):
    """The seed grid (nd, nh, nw) of K supervoxels of a D x H x W volume: an int K gives n_a = clamp(floor(E_a / s0 +
    0.5), 1, L_a) on each axis, with the physical extents E_a = L_a * spacing_a and s0 = cbrt(E_z E_y E_x / K) (float64);
    an explicit (nd, nh, nw) is checked.  K' = nd * nh * nw is at most 65534."""
    D, H, W = (check_int(n, v, 1, MAX_SIDE) for n, v in (("D", D), ("H", H), ("W", W)))
    sp = _spacing(spacing)
    L = (D, H, W)
    if isinstance(K, (tuple, list)):
        if len(K) != 3:
            raise ValueError("K must be an int or (nd, nh, nw), got %r" % (K,))
        grid = tuple(check_int("K[%d]" % a, v, 1, L[a]) for a, v in enumerate(K))
    else:
        K = check_int("K", K, 1, 2 ** 31 - 1)
        E = [float(l) * s for l, s in zip(L, sp)]
        s0 = float(np.cbrt(E[0] * E[1] * E[2] / K))
        grid = tuple(min(max(int(math.floor(e / s0 + 0.5)), 1), l) for e, l in zip(E, L))
    if grid[0] * grid[1] * grid[2] > MAX_K:
        raise ValueError("the grid %s has %d cells, more than %d" % (grid, grid[0] * grid[1] * grid[2], MAX_K))
    return grid


def weights(D, H, W, grid, compactness, spacing):
    """float32 (w2z, w2y, w2x) = ((compactness * spacing_a / s)^2 rounded to float32, s = cbrt(prod E_a / n_a)."""
    sp = _spacing(spacing)
    E = [float(l) * s for l, s in zip((D, H, W), sp)]
    s = float(np.cbrt((E[0] / grid[0]) * (E[1] / grid[1]) * (E[2] / grid[2])))
    out = []
    with np.errstate(over="ignore"):  # an overflow to inf is the caller's to reject
        for a in range(3):
            q = compactness * sp[a] / s
            out.append(float(np.float32(q * q)))
    return tuple(out)


def min_size_threshold(D, H, W, grid, min_size_factor):
    """floor(float32(min_size_factor) * (D*H*W // K') + 0.5), at most 2^31 - 1 (more than any volume's voxels)."""
    x = float(np.float32(min_size_factor)) * ((D * H * W) // (grid[0] * grid[1] * grid[2]))
    return int(min(math.floor(x + 0.5), 2 ** 31 - 1))


def _check(volumes, K, compactness, spacing, max_iter, subsample_stride, min_size_factor):
    tensor("volumes", volumes, torch.float32, 5)
    B, C, D, H, W = (int(v) for v in volumes.shape)
    if not 1 <= C <= MAX_C:
        raise ValueError("volumes must have 1 to %d channels, got %d" % (MAX_C, C))
    _sides(D, H, W)
    sp = _spacing(spacing)
    grid = volume_grid(D, H, W, K, sp)
    Kp = grid[0] * grid[1] * grid[2]
    if B * Kp > MAX_NODES:
        raise ValueError("B*K' must be at most %d, got %d" % (MAX_NODES, B * Kp))
    compactness = check_number("compactness", compactness)
    if not (math.isfinite(compactness) and compactness > 0):
        raise ValueError("compactness must be finite and > 0, got %r" % compactness)
    w2 = weights(D, H, W, grid, compactness, sp)
    if not all(math.isfinite(w) for w in w2):
        raise ValueError("compactness * spacing / s overflows float32 when squared: %r" % (w2,))
    max_iter = check_int("max_iter", max_iter, 0, 2 ** 31 - 2)
    subsample_stride = check_int("subsample_stride", subsample_stride, 1, MAX_STRIDE)
    min_size_factor = check_number("min_size_factor", min_size_factor)
    if not (math.isfinite(min_size_factor) and min_size_factor >= 0):
        raise ValueError("min_size_factor must be finite and >= 0, got %r" % min_size_factor)
    if volumes.device.type != "cuda":
        raise ValueError("volumes is a %s tensor: pass cuda tensors (torch.from_numpy(...).cuda())" %
                         volumes.device.type)
    thres = min_size_threshold(D, H, W, grid, min_size_factor)
    return (B, C, D, H, W), grid, w2, max_iter, subsample_stride, thres


def _run(volumes, K, compactness, spacing, max_iter, subsample_stride, min_size_factor, overflow=None):
    (B, C, D, H, W), grid, w2, max_iter, stride, thres = _check(volumes, K, compactness, spacing, max_iter,
                                                                subsample_stride, min_size_factor)
    Kp = grid[0] * grid[1] * grid[2]
    dev = volumes.device
    L = _lib.lib()
    with torch.cuda.device(dev):
        labels = torch.empty((B, D, H, W), dtype=torch.int16, device=dev)
        position = torch.empty((B, Kp, 3), dtype=torch.float32, device=dev)
        centroids = torch.empty((B, Kp, C), dtype=torch.float32, device=dev)
        count = torch.empty((B, Kp), dtype=torch.int32, device=dev)
        if B == 0:
            return Supervoxels(labels, position, centroids, count, grid)
        x = volumes.contiguous()
        f = L.fslic_b200_sv_slic_scratch_bytes
        n = chunk(lambda c: f(c, D, H, W, C, *grid, stride, max_iter), SUPERVOXEL_SCRATCH_CAP, B, limit=65535)
        nbytes = int(f(n, D, H, W, C, *grid, stride, max_iter))
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        stream = torch.cuda.current_stream(dev).cuda_stream
        for i, b0 in enumerate(range(0, B, n)):
            c = min(n, B - b0)
            _lib.check(L.fslic_b200_sv_slic(
                dev.index, c, D, H, W, C, *grid, *w2, stride, max_iter, thres, x[b0].data_ptr(),
                labels[b0].data_ptr(), position[b0].data_ptr(), centroids[b0].data_ptr(), count[b0].data_ptr(),
                None if overflow is None else overflow[i].data_ptr(), scratch.data_ptr(), nbytes, stream))
    return Supervoxels(labels, position, centroids, count, grid)


def supervoxel_slic(volumes, K, compactness, spacing=(1.0, 1.0, 1.0), max_iter=10, subsample_stride=3,
                    min_size_factor=0.25):
    """SLIC supervoxels of float32 volumes [B,C,D,H,W] (cuda) -> Supervoxels(labels, position, features, count, grid).

    K is an int (the grid follows volume_grid with the voxel spacing (z, y, x)) or an explicit (nd, nh, nw).  Seeds sit
    at the centres of the grid's cells with the features of their voxel.  Pass t < max_iter assigns the voxels of the
    rows y % subsample_stride == t % subsample_stride of every slice to the centre minimising sum_c (f_c - mu_c)^2 +
    w2z dz^2 + w2y dy^2 + w2x dx^2, w2_a = (compactness * spacing_a / s)^2 with s the mean physical cell side, among
    the centres within R_a = ceil(L_a / n_a) voxels on every axis, ties to the lower index, and moves every centre with
    members to their mean position and pooled mean features; one assign over every voxel follows, then
    enforce_connectivity_3d with min_size = round(min_size_factor * D*H*W / K').  compactness has no default: the
    feature distance has no fixed scale.  At D = 1 this is not feature_slic: the seed grids and windows differ.
    Per-supervoxel statistics come from pooling.pool over the volume viewed as [B,C,D*H,W]; the supervoxel graph from
    region_graph.region_adjacency_3d and the shapes from geometry.region_properties_3d.  merge_regions, pool,
    class_histogram and the ASA / undersegmentation fields of segmentation_scores read labels per voxel and are correct
    on the [B,D*H,W] view; boundaries and the boundary-recall fields of segmentation_scores remain 2-D.  Limits:
    1 <= C <= 1024, D, H, W <= 32767, D*H*W <= 2^29, K' <= 65534, B*K' <= 2^30, 1 <= subsample_stride <= 255, spacing
    finite and > 0."""
    return _run(volumes, K, compactness, spacing, max_iter, subsample_stride, min_size_factor)


def enforce_connectivity_3d(labels, K, min_size):
    """Connectivity enforcement of label volumes int16 [B,D,H,W] (cuda) -> new int16 [B,D,H,W] with values in [0, K).

    Components are the 6-connected sets of equal labels (read as uint16), numbered in the raster order of their
    leaders (smallest voxel index).  Those with at least min_size voxels are candidates; of more than K, the K first
    by (area descending, leader ascending) are kept.  Kept components take 0, 1, .. in leader order, component 0 takes
    0 if not kept, and every other component takes the label of the component holding its leader's predecessor voxel
    (leader - 1 if x > 0, else leader - W if y > 0, else leader - H*W).  At D = 1 this is the 2-D enforcement of the
    uint8 path whenever at most K components reach min_size (or the K-th largest area is not tied).
    Limits: 1 <= K <= 65534, min_size >= 0, D, H, W <= 32767, D*H*W <= 2^29."""
    tensor("labels", labels, torch.int16, 4)
    B, D, H, W = (int(v) for v in labels.shape)
    _sides(D, H, W)
    K = check_int("K", K, 1, MAX_K)
    min_size = check_int("min_size", min_size, 0, 2 ** 31 - 1)
    if labels.device.type != "cuda":
        raise ValueError("labels is a %s tensor: pass cuda tensors (torch.from_numpy(...).cuda())" % labels.device.type)
    dev = labels.device
    L = _lib.lib()
    with torch.cuda.device(dev):
        out = torch.empty_like(labels, memory_format=torch.contiguous_format)
        if B == 0:
            return out
        x = labels.contiguous()
        f = L.fslic_b200_sv_enforce_scratch_bytes
        n = chunk(lambda c: f(c, D, H, W), SUPERVOXEL_SCRATCH_CAP, B, limit=65535)
        nbytes = int(f(n, D, H, W))
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        stream = torch.cuda.current_stream(dev).cuda_stream
        for b0 in range(0, B, n):
            c = min(n, B - b0)
            _lib.check(L.fslic_b200_sv_enforce(dev.index, c, D, H, W, K, min_size, x[b0].data_ptr(),
                                               out[b0].data_ptr(), scratch.data_ptr(), nbytes, stream))
    return out


def pass_tiles(D, H, W, max_iter, subsample_stride):
    """Tiles per volume of every assign pass: max_iter strided passes, then the full one."""
    return slic_pass_tiles((D, H, W), (TILE_D, TILE_R, TILE_W), max_iter, subsample_stride)


def supervoxel_dispatch(volumes, K, compactness, spacing=(1.0, 1.0, 1.0), max_iter=10, subsample_stride=3,
                        min_size_factor=0.25):
    """supervoxel_slic with a record of the assign kernels it ran (synchronises): (result, [(tiles, overflowed)] per
    pass), the tiles of the pass over the whole batch and how many of them overflowed the tile kernel's candidate list
    and went to the per-voxel kernel."""
    return slic_dispatch(lambda it, overflow: _run(volumes, K, compactness, spacing, it, subsample_stride,
                                                   min_size_factor, overflow), volumes, max_iter, subsample_stride,
                         (TILE_D, TILE_R, TILE_W))
