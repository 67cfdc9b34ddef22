"""Differentiable soft SLIC on the GPU (csrc/soft_slic.cuh), the soft superpixels of Superpixel Sampling Networks
(Jampani et al., ECCV 2018): every pixel gets a softmax association over the 9 grid cells around it, every centroid is
the association-weighted mean of the pixels, and autograd runs through every iteration::

    feats = torch.cat([conv(images), yx_channels * scale], 1)        # [B,C,H,W] float32, requires grad
    r = soft_slic(feats, 1600, n_iter=5)
    recon = soft_unpool(soft_pool(onehot, r.assoc, r.grid), r.assoc, r.grid)
    loss = torch.nn.functional.cross_entropy(recon.clamp_min(1e-8).log(), target)
    loss.backward()                                                   # through the 5 iterations into conv

A new algorithm with its own contract, not a reference port (DESIGN.md section 4.20 gives every float32 operation and
its order, forward and backward): the results and gradients are exact and deterministic -- the bits of image b depend
only on image b's inputs, not on the batch, the stream or the run.  No float atomics.  Cuda float32 tensors only;
non-contiguous inputs are made contiguous once.  Work is enqueued on the inputs' device on its current torch stream
with no host synchronisation and no read-back, so a CUDA graph can capture it (soft_slic's connectivity enforcement
included); every argument is checked (ValueError) before any device work.  Each function is differentiable in both
tensor arguments (first-order: the backward is not itself differentiable).
"""
import collections
import math

import torch
from torch.autograd.function import once_differentiable

from . import _lib
from ._labelmaps import MAX_K, MAX_PIXELS, check_int, check_number, tensor
from .base_slic import _locked, get_cca_engine
from .feature_slic import min_size_threshold, superpixel_size
from .pooling import pool

MAX_NODES = 1 << 30
SLOTS = 9

SoftSlic = collections.namedtuple("SoftSlic", "labels assoc centroids grid")
SoftSlic.__doc__ = """labels int16 [B,H,W] (the cell of each pixel's largest association, after connectivity
enforcement unless min_size_factor is None); assoc float32 [B,9,H,W], the last iteration's associations; centroids
float32 [B,C,K], soft_pool of the features by assoc; grid (nh, nw), K = nh * nw."""


def cell_grid(H, W, num_cells):
    """(nh, nw) of a grid of num_cells cells over H x W images.  num_cells is (nh, nw), checked against
    1 <= nh <= H, 1 <= nw <= W (H, W taken as 1 when 0), nh * nw <= 65534; or an int K, which gives SSN's grid
    nw = int(sqrt(K * W / H)), nh = int(sqrt(K * H / W)) in float64, clamped to [1, W] and [1, H] ((1, 1) for an
    empty image), with the same limit on nh * nw.  Pixel (i, j) is in cell (i * nh // H, j * nw // W)."""
    H = check_int("H", H, 0, 2 ** 31 - 1)
    W = check_int("W", W, 0, 2 ** 31 - 1)
    if isinstance(num_cells, (tuple, list)):
        if len(num_cells) != 2:
            raise ValueError("num_cells must be an int or (nh, nw), got %r" % (num_cells,))
        nh = check_int("nh", num_cells[0], 1, max(H, 1))
        nw = check_int("nw", num_cells[1], 1, max(W, 1))
    else:
        K = check_int("num_cells", num_cells, 1, 2 ** 31 - 1)
        if H == 0 or W == 0:
            nh = nw = 1
        else:
            nw = min(max(int(math.sqrt(K * W / H)), 1), W)
            nh = min(max(int(math.sqrt(K * H / W)), 1), H)
    if nh * nw > MAX_K:
        raise ValueError("the grid has %d x %d = %d cells: at most %d" % (nh, nw, nh * nw, MAX_K))
    return nh, nw


def _grid(H, W, grid):
    if not isinstance(grid, (tuple, list)):
        raise ValueError("grid must be (nh, nw), as cell_grid returns it, got %r" % (grid,))
    return cell_grid(H, W, tuple(grid))


def _image(name, x):
    """A float32 [B,C,H,W] tensor with C >= 1 and at most MAX_PIXELS pixels per image; returns its shape."""
    tensor(name, x, torch.float32, 4)
    B, c, h, w = (int(v) for v in x.shape)
    if h * w > MAX_PIXELS:
        raise ValueError("%s: images of %dx%d pixels exceed %d pixels" % (name, h, w, MAX_PIXELS))
    if c < 1:
        raise ValueError("%s needs at least one channel" % name)
    return B, c, h, w


def _assoc(assoc, B, H, W):
    tensor("assoc", assoc, torch.float32, 4)
    if tuple(int(v) for v in assoc.shape) != (B, SLOTS, H, W):
        raise ValueError("assoc must be [B,9,H,W] = %s, got %s" % ((B, SLOTS, H, W), tuple(assoc.shape)))


def _cells(name, x, B, C, K):
    tensor(name, x, torch.float32, 3)
    if tuple(int(v) for v in x.shape) != (B, C, K):
        raise ValueError("%s must be [B,C,K] = %s, got %s" % (name, (B, C, K), tuple(x.shape)))


def _device(first, *named):
    """Every tensor of named on first's device, which must be a cuda device; returns it."""
    name0, x0 = first
    for name, x in named:
        if x.device != x0.device:
            raise ValueError("%s is on %s, %s on %s" % (name, x.device, name0, x0.device))
    if x0.device.type != "cuda":
        raise ValueError("%s is a %s tensor: pass cuda tensors (torch.from_numpy(...).cuda())" % (name0,
                                                                                               x0.device.type))
    return x0.device


def _nodes(B, K):
    if B * K > MAX_NODES:
        raise ValueError("B*K must be at most %d, got %d" % (MAX_NODES, B * K))


def _ptr(x):
    return None if x is None else x.data_ptr()


def _launch(name, dev, B, H, W, C, g, *ptrs):
    """fslic_b200_<name> over the whole batch on dev's current stream; nothing for an empty batch or image."""
    if B == 0 or H == 0 or W == 0:
        return
    with torch.cuda.device(dev):
        _lib.check(getattr(_lib.lib(), "fslic_b200_" + name)(
            dev.index, B, H, W, C, g[0], g[1], *[_ptr(p) for p in ptrs], torch.cuda.current_stream(dev).cuda_stream))


def _empty(B, *shape, dev, fill=None):
    if fill is not None:
        return torch.full((B,) + shape, fill, dtype=torch.float32, device=dev)
    return torch.empty((B,) + shape, dtype=torch.float32, device=dev)


class _SoftAssign(torch.autograd.Function):
    @staticmethod
    def forward(ctx, features, centroids, g):
        B, C, H, W = (int(v) for v in features.shape)
        dev = features.device
        q = _empty(B, SLOTS, H, W, dev=dev)
        _launch("soft_assign", dev, B, H, W, C, g, features, centroids, q)
        ctx.save_for_backward(features, centroids, q)
        ctx.g = g
        return q

    @staticmethod
    @once_differentiable
    def backward(ctx, grad):
        features, centroids, q = ctx.saved_tensors
        B, C, H, W = (int(v) for v in features.shape)
        dev = features.device
        need_f, need_mu = ctx.needs_input_grad[:2]
        gf = _empty(B, C, H, W, dev=dev) if need_f else None
        # an empty block sums to +0.0, and -2 * +0.0 is -0.0
        gmu = _empty(B, C, ctx.g[0] * ctx.g[1], dev=dev, fill=None if H and W else -0.0) if need_mu else None
        if need_f or need_mu:
            gd = torch.empty_like(q)
            _launch("soft_assign_backward", dev, B, H, W, C, ctx.g, features, centroids, q, grad.contiguous(), gd, gf,
                    gmu)
        return gf, gmu, None


class _SoftPool(torch.autograd.Function):
    @staticmethod
    def forward(ctx, values, assoc, g):
        B, C, H, W = (int(v) for v in values.shape)
        K = g[0] * g[1]
        dev = values.device
        means = _empty(B, C, K, dev=dev, fill=None if H and W else 0.0)
        weights = _empty(B, K, dev=dev, fill=None if H and W else 0.0)
        _launch("soft_pool", dev, B, H, W, C, g, values, assoc, means, weights)
        ctx.save_for_backward(values, assoc, means, weights)
        ctx.g = g
        return means

    @staticmethod
    @once_differentiable
    def backward(ctx, grad):
        values, assoc, means, weights = ctx.saved_tensors
        B, C, H, W = (int(v) for v in values.shape)
        dev = values.device
        need_v, need_q = ctx.needs_input_grad[:2]
        gv = _empty(B, C, H, W, dev=dev) if need_v else None
        gq = _empty(B, SLOTS, H, W, dev=dev) if need_q else None
        if need_v or need_q:
            gsum, gweight = torch.empty_like(means), torch.empty_like(weights)
            _launch("soft_pool_backward", dev, B, H, W, C, ctx.g, values, assoc, means, weights, grad.contiguous(), gsum,
                    gweight, gv, gq)
        return gv, gq, None


class _SoftUnpool(torch.autograd.Function):
    @staticmethod
    def forward(ctx, values, assoc, g):
        B, C, K = (int(v) for v in values.shape)
        H, W = int(assoc.shape[2]), int(assoc.shape[3])
        dev = values.device
        out = _empty(B, C, H, W, dev=dev)
        _launch("soft_unpool", dev, B, H, W, C, g, values, assoc, out)
        ctx.save_for_backward(values, assoc)
        ctx.g = g
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad):
        values, assoc = ctx.saved_tensors
        B, C, K = (int(v) for v in values.shape)
        H, W = int(assoc.shape[2]), int(assoc.shape[3])
        dev = values.device
        need_v, need_q = ctx.needs_input_grad[:2]
        gv = _empty(B, C, K, dev=dev, fill=None if H and W else 0.0) if need_v else None
        gq = _empty(B, SLOTS, H, W, dev=dev) if need_q else None
        if need_v or need_q:
            _launch("soft_unpool_backward", dev, B, H, W, C, ctx.g, values, assoc, grad.contiguous(), gv, gq)
        return gv, gq, None


def soft_assign(features, centroids, grid):
    """float32 features [B,C,H,W], centroids [B,C,K] and grid (nh, nw), K = nh * nw -> float32 assoc [B,9,H,W]: over
    the valid slots n of pixel p (slot n = (da+1)*3 + (db+1) is the cell (a+da, b+db) around the pixel's own cell
    (a, b); a slot outside the grid is invalid and gets +0.0), d_n = sum_c (f_pc - mu_{k(n)c})^2, m = min_n d_n (fminf),
    q_n = expf(m - d_n) / sum_n expf(m - d_n).  Differentiable in features and centroids."""
    B, C, H, W = _image("features", features)
    g = _grid(H, W, grid)
    _cells("centroids", centroids, B, C, g[0] * g[1])
    _nodes(B, g[0] * g[1])
    _device(("features", features), ("centroids", centroids))
    return _SoftAssign.apply(features.contiguous(), centroids.contiguous(), g)


def soft_pool(values, assoc, grid):
    """float32 values [B,C,H,W] and assoc [B,9,H,W] over grid (nh, nw) -> float32 [B,C,K]: per cell k,
    M_kc = sum q * v_c / sum q over the pixels that have k in a valid slot (q their association with k), 0 where
    sum q == 0.  With values = the features this is SSN's centroid update; with any per-pixel map (one-hot labels, say)
    it maps that map onto the superpixels.  Differentiable in values and assoc."""
    B, C, H, W = _image("values", values)
    g = _grid(H, W, grid)
    _assoc(assoc, B, H, W)
    _nodes(B, g[0] * g[1])
    _device(("values", values), ("assoc", assoc))
    return _SoftPool.apply(values.contiguous(), assoc.contiguous(), g)


def soft_unpool(values, assoc, grid):
    """float32 values [B,C,K] and assoc [B,9,H,W] over grid (nh, nw) -> float32 [B,C,H,W]:
    out_pc = sum over the valid slots n of q_pn * values_{k(n)c}.  Differentiable in values and assoc."""
    tensor("assoc", assoc, torch.float32, 4)
    B, S, H, W = (int(v) for v in assoc.shape)
    if S != SLOTS:
        raise ValueError("assoc must be [B,9,H,W], got %s" % (tuple(assoc.shape),))
    if H * W > MAX_PIXELS:
        raise ValueError("assoc: images of %dx%d pixels exceed %d pixels" % (H, W, MAX_PIXELS))
    g = _grid(H, W, grid)
    tensor("values", values, torch.float32, 3)
    C = int(values.shape[1])
    if C < 1:
        raise ValueError("values needs at least one channel")
    _cells("values", values, B, C, g[0] * g[1])
    _nodes(B, g[0] * g[1])
    _device(("values", values), ("assoc", assoc))
    return _SoftUnpool.apply(values.contiguous(), assoc.contiguous(), g)


def grid_labels(B, H, W, grid, device):
    """int16 [B,H,W]: the cell a * nw + b of every pixel (i, j), (a, b) = (i * nh // H, j * nw // W)."""
    nh, nw = grid
    rows = torch.arange(H, device=device, dtype=torch.int64) * nh // H
    cols = torch.arange(W, device=device, dtype=torch.int64) * nw // W
    return (rows[:, None] * nw + cols[None, :]).to(torch.int16).expand(B, H, W).contiguous()


def soft_slic(features, num_cells, n_iter=5, min_size_factor=0.25):
    """Soft SLIC of float32 features [B,C,H,W] (cuda) -> SoftSlic(labels, assoc, centroids, grid).

    The grid is cell_grid(H, W, num_cells).  The initial centroids are the cell means, pool(features, grid_labels, K);
    then n_iter >= 1 times assoc = soft_assign(features, centroids), centroids = soft_pool(features, assoc), SSN's loop.
    labels (int16, not differentiable) is the cell of each pixel's first largest association (a NaN counts as the
    largest), then connectivity enforcement absorbs components smaller than round(S^2 * min_size_factor) pixels,
    S = superpixel_size(H, W, K), as feature_slic does; min_size_factor=None returns the map without enforcement.
    Differentiable in features through assoc and centroids.  Autograd keeps one assoc per iteration, 36 bytes per
    pixel each (plus the features and B * K * (C + 1) floats per iteration), until the backward pass.  SSN gives the
    distance a spatial term by concatenating scaled (y, x) channels to the features; so does the caller here."""
    B, C, H, W = _image("features", features)
    g = cell_grid(H, W, num_cells)
    K = g[0] * g[1]
    _nodes(B, K)
    n_iter = check_int("n_iter", n_iter, 1, 2 ** 31 - 1)
    if min_size_factor is not None:
        min_size_factor = check_number("min_size_factor", min_size_factor)
        if not min_size_factor >= 0:
            raise ValueError("min_size_factor must be >= 0 or None, got %r" % min_size_factor)
    dev = _device(("features", features))
    with torch.cuda.device(dev):
        x = features.contiguous()
        mu = pool(x, grid_labels(B, H, W, g, dev), K)
        for _ in range(n_iter):
            q = soft_assign(x, mu, g)
            mu = soft_pool(x, q, g)
        labels = torch.empty((B, H, W), dtype=torch.int16, device=dev)
        if B and H and W:
            _lib.check(_lib.lib().fslic_b200_soft_labels(dev.index, B, H, W, g[0], g[1], q.data_ptr(), labels.data_ptr(),
                                                          torch.cuda.current_stream(dev).cuda_stream))
            if min_size_factor is not None:
                thres = min_size_threshold(superpixel_size(H, W, K), min_size_factor)
                with _locked(lambda: get_cca_engine(H, W, B, dev.index)) as eng:
                    eng.enforce_connectivity(labels, K, thres)
    return SoftSlic(labels, q, mu, g)


__all__ = ["SoftSlic", "cell_grid", "grid_labels", "soft_assign", "soft_pool", "soft_slic", "soft_unpool"]
