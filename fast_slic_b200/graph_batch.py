"""Batched consumers of label maps: the adjacency graph, mask density and density broadcast of every image of a batch
(csrc/graph.cuh), each image equal to what the reference's fast_slic_get_connectivity / fast_slic_get_mask_density /
fast_slic_cluster_density_to_mask give for it alone.  The reference has no batch API; SlicModel.get_connectivity /
get_mask_density / broadcast_density_to_mask, its single-image calls, are batches of one here.

Cuda tensors in give cuda tensors out on the same device, enqueued on that device's current stream with no
synchronisation (a CUDA graph can capture them); numpy arrays in give numpy arrays out.  Arguments are checked before
any device is touched.
"""
import numpy as np
import torch

from . import _lib
from ._labelmaps import chunk
from .engine import CLUSTER_DTYPE, require_cuda

# Device memory one get_connectivity_batch launch gives its pair tables at most (24 bytes per table slot, 32 slots or
# more per superpixel and image): a batch whose tables need more runs in chunks of images, with identical results.
GRAPH_SCRATCH_CAP = 1 << 30


def _check(name, x, np_dtype, torch_dtype, ndim):
    """True for a cuda tensor, False for a numpy array; ValueError for anything else."""
    if isinstance(x, torch.Tensor):
        if x.dtype != torch_dtype or x.dim() != ndim:
            raise ValueError("%s must be a %s tensor with %d dimensions, got %s %s" % (name, torch_dtype, ndim, x.dtype,
                                                                                     tuple(x.shape)))
        if x.device.type != "cuda":
            raise ValueError("%s is a %s tensor: pass a cuda tensor or a numpy array" % (name, x.device.type))
        return True
    if not isinstance(x, np.ndarray):
        raise ValueError("%s must be a numpy array or a cuda tensor" % name)
    if x.dtype != np_dtype or x.ndim != ndim:
        raise ValueError("%s must be a %s array with %d dimensions, got %s %s" % (name, np.dtype(np_dtype).name, ndim,
                                                                                x.dtype, x.shape))
    return False


def _same_kind(labels, is_tensor, name, x, x_is_tensor):
    if x_is_tensor != is_tensor:
        raise ValueError("%s and labels must both be cuda tensors or both numpy arrays" % name)
    if is_tensor and x.device != labels.device:
        raise ValueError("%s is on %s, labels on %s" % (name, x.device, labels.device))


def _check_labels(labels):
    is_tensor = _check("labels", labels, np.int16, torch.int16, 3)
    return (is_tensor,) + tuple(int(v) for v in labels.shape)


def _device(labels, is_tensor, device):
    return labels.device if is_tensor else torch.device("cuda", int(device))


def _upload(x, is_tensor, dev):
    return x.contiguous() if is_tensor else torch.from_numpy(np.ascontiguousarray(x)).to(dev)


def graph_chunk(K, B):
    """Images per get_connectivity_batch launch: as many as fit GRAPH_SCRATCH_CAP, at least one."""
    f = _lib.lib().fslic_b200_connectivity_batch_scratch_bytes
    return chunk(lambda c: f(K, c), GRAPH_SCRATCH_CAP, B)


def get_connectivity_batch(K, device, labels, return_replayed=False):
    """int16 labels [B,H,W] -> (counts int32[B,K], neighbors int32[B,K,12][, replayed int32[B]])."""
    is_tensor, B, H, W = _check_labels(labels)
    require_cuda()
    dev = _device(labels, is_tensor, device)
    L = _lib.lib()
    with torch.cuda.device(dev):
        lab = _upload(labels, is_tensor, dev)
        if B == 0 or H == 0 or W == 0:  # no pixel pair: empty lists
            counts = torch.zeros((B, K), dtype=torch.int32, device=dev)
            nb = torch.zeros((B, K, 12), dtype=torch.int32, device=dev)
            replayed = torch.zeros(B, dtype=torch.int32, device=dev)
        else:
            counts = torch.empty((B, K), dtype=torch.int32, device=dev)
            nb = torch.empty((B, K, 12), dtype=torch.int32, device=dev)
            replayed = torch.empty(B, dtype=torch.int32, device=dev)
            chunk = graph_chunk(K, B)
            nbytes = int(L.fslic_b200_connectivity_batch_scratch_bytes(K, chunk))
            scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            stream = torch.cuda.current_stream(dev).cuda_stream
            for b0 in range(0, B, chunk):
                c = min(chunk, B - b0)
                _lib.check(L.fslic_b200_get_connectivity_batch(
                    dev.index, c, H, W, K, lab[b0].data_ptr(), counts[b0].data_ptr(), nb[b0].data_ptr(),
                    replayed[b0].data_ptr(), scratch.data_ptr(), nbytes, stream))
        out = (counts, nb, replayed) if return_replayed else (counts, nb)
        if not is_tensor:
            out = tuple(t.cpu().numpy() for t in out)
    return out


def get_mask_density_batch(K, device, masks, labels, clusters):
    """uint8 masks [B,H,W], int16 labels [B,H,W], clusters [B,K] (structured array) or [B,K,32] (uint8 cuda tensor)
    -> uint8[B,K]: min(255, sum of the mask over label k / max(num_members, 1)) per image."""
    is_tensor, B, H, W = _check_labels(labels)
    _same_kind(labels, is_tensor, "masks", masks, _check("masks", masks, np.uint8, torch.uint8, 3))
    if tuple(masks.shape) != (B, H, W):
        raise ValueError("masks %s do not match labels %s" % (tuple(masks.shape), (B, H, W)))
    if isinstance(clusters, torch.Tensor):
        _same_kind(labels, is_tensor, "clusters", clusters, _check("clusters", clusters, np.uint8, torch.uint8, 3))
        if tuple(clusters.shape) != (B, K, 32):
            raise ValueError("clusters must be [B,K,32] = %s, got %s" % ((B, K, 32), tuple(clusters.shape)))
    else:
        if not isinstance(clusters, np.ndarray) or clusters.dtype != CLUSTER_DTYPE or clusters.ndim != 2:
            raise ValueError("clusters must be a [B,K] Cluster array or a [B,K,32] uint8 cuda tensor")
        _same_kind(labels, is_tensor, "clusters", clusters, False)
        if clusters.shape != (B, K):
            raise ValueError("clusters must be [B,K] = %s, got %s" % ((B, K), clusters.shape))
    require_cuda()
    dev = _device(labels, is_tensor, device)
    L = _lib.lib()
    with torch.cuda.device(dev):
        lab = _upload(labels, is_tensor, dev)
        msk = _upload(masks, is_tensor, dev)
        cl = clusters.contiguous() if is_tensor else \
            torch.from_numpy(np.ascontiguousarray(clusters).view(np.uint8).reshape(B, K, 32)).to(dev)
        if B == 0 or H == 0 or W == 0:
            dens = torch.zeros((B, K), dtype=torch.uint8, device=dev)
        else:
            dens = torch.empty((B, K), dtype=torch.uint8, device=dev)
            scratch = torch.empty((B, K), dtype=torch.int32, device=dev)
            _lib.check(L.fslic_b200_get_mask_density_batch(dev.index, B, H, W, K, cl.data_ptr(), lab.data_ptr(),
                                                           msk.data_ptr(), dens.data_ptr(), scratch.data_ptr(),
                                                           torch.cuda.current_stream(dev).cuda_stream))
        return dens if is_tensor else dens.cpu().numpy()


def broadcast_density_to_mask_batch(K, device, densities, labels):
    """uint8 densities [B,K], int16 labels [B,H,W] -> uint8[B,H,W]: each pixel's density (0 where its label is
    outside [0, K))."""
    is_tensor, B, H, W = _check_labels(labels)
    _same_kind(labels, is_tensor, "densities", densities, _check("densities", densities, np.uint8, torch.uint8, 2))
    if tuple(densities.shape) != (B, K):
        raise ValueError("densities must be [B,K] = %s, got %s" % ((B, K), tuple(densities.shape)))
    require_cuda()
    dev = _device(labels, is_tensor, device)
    L = _lib.lib()
    with torch.cuda.device(dev):
        lab = _upload(labels, is_tensor, dev)
        dens = _upload(densities, is_tensor, dev)
        out = torch.empty((B, H, W), dtype=torch.uint8, device=dev)
        if B and H and W:
            _lib.check(L.fslic_b200_cluster_density_to_mask_batch(dev.index, B, H, W, K, lab.data_ptr(), dens.data_ptr(),
                                                                  out.data_ptr(), torch.cuda.current_stream(dev).cuda_stream))
        return out if is_tensor else out.cpu().numpy()
