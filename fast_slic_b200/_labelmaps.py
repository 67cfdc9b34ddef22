"""What the batched label-map APIs (pooling, region_graph, groundtruth, geometry, merging, graph_batch) and SLIC over
float data (feature_slic, supervoxels) share: their argument checks, their limits and the search for how many images one
launch takes under a scratch cap."""
import operator

import torch

MAX_K = 65534
# Pixels per image: every count over one image fits int32
MAX_PIXELS = 1 << 29
# What a *_scratch_bytes entry point returns for arguments no single call takes
NO_SIZE = 2 ** 64 - 1
# SLIC over float data (csrc/capi_float_slic.cu): channels, side, B*K and subsample stride
FLOAT_SLIC_MAX_C = 1024
FLOAT_SLIC_MAX_SIDE = 32767
FLOAT_SLIC_MAX_NODES = 1 << 30
FLOAT_SLIC_MAX_STRIDE = 255


def tensor(name, x, dtype, ndim):
    if not isinstance(x, torch.Tensor):
        raise ValueError("%s must be a cuda tensor (got %s): use torch.from_numpy(...).cuda()" % (name, type(x).__name__))
    if x.dtype != dtype or x.dim() != ndim:
        raise ValueError("%s must be a %s tensor with %d dimensions, got %s %s" % (name, dtype, ndim, x.dtype,
                                                                                 tuple(x.shape)))


def check_int(name, v, lo, hi):
    try:
        v = operator.index(v)
    except TypeError:
        raise ValueError("%s must be an int, got %r" % (name, v)) from None
    if not lo <= v <= hi:
        raise ValueError("%s must be in [%d, %d], got %d" % (name, lo, hi, v))
    return v


def check_number(name, v):
    if isinstance(v, bool) or not isinstance(v, (int, float)) and not hasattr(v, "__float__"):
        raise ValueError("%s must be a number, got %r" % (name, v))
    return float(v)


def check_K(K):
    return check_int("K", K, 1, MAX_K)


def check_connectivity(connectivity):
    try:
        connectivity = operator.index(connectivity)
    except TypeError:
        raise ValueError("connectivity must be 4 or 8, got %r" % (connectivity,)) from None
    if connectivity not in (4, 8):
        raise ValueError("connectivity must be 4 or 8, got %r" % (connectivity,))
    return connectivity


def check_connectivity_3d(connectivity):
    try:
        connectivity = operator.index(connectivity)
    except TypeError:
        raise ValueError("connectivity must be 6, 18 or 26, got %r" % (connectivity,)) from None
    if connectivity not in (6, 18, 26):
        raise ValueError("connectivity must be 6, 18 or 26, got %r" % (connectivity,))
    return connectivity


def check_pixels(H, W, reason=""):
    """Images of at most MAX_PIXELS pixels; `reason` ends the message."""
    if H * W > MAX_PIXELS:
        raise ValueError("images of %dx%d pixels exceed %d pixels%s" % (H, W, MAX_PIXELS, reason))


def check_voxels(D, H, W, reason=""):
    """Volumes of at most MAX_PIXELS voxels; `reason` ends the message."""
    if D * H * W > MAX_PIXELS:
        raise ValueError("volumes of %dx%dx%d voxels exceed %d voxels%s" % (D, H, W, MAX_PIXELS, reason))


def check_features(labels, name, x, ndim):
    """labels int16 [B,H,W] and x float32 with ndim dimensions, same B (and H, W for ndim 4); returns (B, H, W, C)."""
    tensor("labels", labels, torch.int16, 3)
    tensor(name, x, torch.float32, ndim)
    B, H, W = (int(v) for v in labels.shape)
    if int(x.shape[0]) != B or (ndim == 4 and tuple(int(v) for v in x.shape[2:]) != (H, W)):
        raise ValueError("%s %s do not match labels %s" % (name, tuple(x.shape), (B, H, W)))
    C = int(x.shape[1])
    if C < 1:
        raise ValueError("%s needs at least one channel" % name)
    return B, H, W, C


def check_graph(graph, B, K):
    """graph.indptr of B*K + 1 entries and int64 graph.edge_index [2,E]; returns (edge_index, E)."""
    indptr, edge_index = graph.indptr, graph.edge_index
    if not isinstance(indptr, torch.Tensor) or indptr.numel() != B * K + 1:
        raise ValueError("graph.indptr must have B*K + 1 = %d entries, got %s" % (
            B * K + 1, indptr.numel() if isinstance(indptr, torch.Tensor) else type(indptr).__name__))
    tensor("graph.edge_index", edge_index, torch.int64, 2)
    if int(edge_index.shape[0]) != 2:
        raise ValueError("graph.edge_index must be int64 [2,E], got %s" % (tuple(edge_index.shape),))
    return edge_index, int(edge_index.shape[1])


def same_device(labels, *named):
    """Every (name, tensor) of named on the labels' device."""
    for name, x in named:
        if x.device != labels.device:
            raise ValueError("%s is on %s, labels on %s" % (name, x.device, labels.device))


def cuda_device(labels, *named):
    """Every (name, tensor) of named on the labels' device, which must be a cuda device; returns it."""
    same_device(labels, *named)
    if labels.device.type != "cuda":
        raise ValueError("labels is a %s tensor: pass cuda tensors (torch.from_numpy(...).cuda())" % labels.device.type)
    return labels.device


def chunk(size_of, cap, B, limit=None):
    """Images per launch: as many as size_of(images) bytes of scratch fit in cap, at most B and limit, at least one.
    A size of NO_SIZE (more images than one launch takes) halves the count."""
    c = max(1, min(B, B if limit is None else limit, cap // max(1, size_of(1))))
    while c > 1:
        nbytes = size_of(c)
        if nbytes == NO_SIZE:
            c //= 2
        elif nbytes <= cap:
            break
        else:
            c = max(1, min(c - 1, c * cap // nbytes))
    return c


def slic_pass_tiles(shape, tile, max_iter, subsample_stride):
    """Tiles per image of every assign pass of SLIC over float data: max_iter strided passes over the rows (the
    second-last axis of shape, (H, W) or (D, H, W)), then the full one, with tiles of the shape `tile` (same axes)."""
    rows = shape[-2]
    out = []
    for t in range(max_iter + 1):
        r, s = (t % subsample_stride, subsample_stride) if t < max_iter else (0, 1)
        npr = (rows - 1 - r) // s + 1 if r < rows else 0
        n = 1
        for a, (L, T) in enumerate(zip(shape, tile)):
            n *= -(-(npr if a == len(shape) - 2 else L) // T)
        out.append(n)
    return out


def slic_dispatch(run, x, max_iter, subsample_stride, tile):
    """run(max_iter, overflow) on x [B,C,*shape] with a record of the assign kernels it ran (synchronises): (result,
    [(tiles, overflowed)] per pass), the tiles of the pass over the whole batch and how many of them overflowed the
    tile kernel's candidate list and went to the per-pixel kernel."""
    B = int(x.shape[0]) if isinstance(x, torch.Tensor) else 0
    max_iter = operator.index(max_iter)
    overflow = torch.zeros((max(B, 1), max_iter + 1), dtype=torch.int32, device=x.device)
    r = run(max_iter, overflow)
    tiles = slic_pass_tiles(tuple(int(v) for v in x.shape[2:]), tile, max_iter, subsample_stride)
    return r, [(B * t, int(o)) for t, o in zip(tiles, overflow.sum(0).tolist())]
