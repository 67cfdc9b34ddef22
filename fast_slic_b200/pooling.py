"""Superpixel pooling on the GPU (csrc/pool.cuh): per-superpixel sums and means of float feature maps, the gather of
per-superpixel values back to pixels, and the per-pixel class of a per-superpixel score table, for whole batches of the
int16 label maps iterate_batch returns.  These close the device loop of SimpleCRFGroup at both ends::

    labels, clusters = slic.iterate_batch(images, return_clusters=True)
    group.push_label_frames(labels, clusters)
    group.set_proba(pool(softmax, labels, K))          # [B,C,H,W] per pixel -> [B,C,K] per superpixel
    group.inference(n)
    classes = paint_argmax(group.get_inferred(out=q), labels)   # [B,C,K] -> int16 [B,H,W]

Cuda tensors only.  Work is enqueued on the labels' device, on its current torch stream, with no host synchronisation
(a CUDA graph can capture it); every argument is checked (ValueError) before any device work.  A label outside [0, K)
(-1 included) belongs to no superpixel.  The sums use no float atomics: the bits of image b's result depend only on
labels[b] and features[b] -- not on the batch, the image's place in it, the chunking, the stream or the run
(DESIGN.md section 4.12 gives the summation order).  pool and unpool are differentiable in features / values.
"""
import torch
from torch.autograd.function import once_differentiable

from . import _lib
from ._labelmaps import MAX_K, NO_SIZE, check_features, check_K, chunk, cuda_device

# Device memory one pool launch takes for its sort at most (about 16 bytes per pixel plus 8 per superpixel): a batch
# that needs more runs in chunks of images, with identical results.
POOL_SCRATCH_CAP = 1 << 30


def pool_chunk(B, H, W, K):
    """Images per pool launch: as many as fit POOL_SCRATCH_CAP, at least one."""
    f = _lib.lib().fslic_b200_pool_batch_scratch_bytes
    if f(1, H, W, K) == NO_SIZE:
        raise ValueError("an image of %dx%d pixels is too large to pool" % (H, W))
    return chunk(lambda c: f(c, H, W, K), POOL_SCRATCH_CAP, B, limit=65536)


def _pool(features, labels, K, mean):
    """(out f32[B,C,K], counts int32[B,K]) of checked, contiguous cuda tensors."""
    B, C, H, W = (int(v) for v in features.shape)
    dev = labels.device
    L = _lib.lib()
    with torch.cuda.device(dev):
        if B == 0 or H == 0 or W == 0:
            return (torch.zeros((B, C, K), dtype=torch.float32, device=dev),
                    torch.zeros((B, K), dtype=torch.int32, device=dev))
        out = torch.empty((B, C, K), dtype=torch.float32, device=dev)
        counts = torch.empty((B, K), dtype=torch.int32, device=dev)
        chunk = pool_chunk(B, H, W, K)
        nbytes = int(L.fslic_b200_pool_batch_scratch_bytes(chunk, H, W, K))
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        stream = torch.cuda.current_stream(dev).cuda_stream
        for b0 in range(0, B, chunk):
            c = min(chunk, B - b0)
            _lib.check(L.fslic_b200_pool_batch(dev.index, c, H, W, C, K, labels[b0].data_ptr(), features[b0].data_ptr(),
                                               int(mean), out[b0].data_ptr(), counts[b0].data_ptr(), scratch.data_ptr(),
                                               nbytes, stream))
    return out, counts


def _unpool(values, labels, divisor=None):
    """f32[B,C,H,W] of checked, contiguous cuda tensors; divisor: int32[B,K] counts or None."""
    B, C, K = (int(v) for v in values.shape)
    H, W = int(labels.shape[1]), int(labels.shape[2])
    dev = labels.device
    with torch.cuda.device(dev):
        if B == 0 or H == 0 or W == 0:
            return torch.zeros((B, C, H, W), dtype=torch.float32, device=dev)
        out = torch.empty((B, C, H, W), dtype=torch.float32, device=dev)
        _lib.check(_lib.lib().fslic_b200_pool_unpool_batch(
            dev.index, B, H, W, C, K, labels.data_ptr(), values.data_ptr(),
            None if divisor is None else divisor.data_ptr(), out.data_ptr(), torch.cuda.current_stream(dev).cuda_stream))
    return out


class _Pool(torch.autograd.Function):
    @staticmethod
    def forward(ctx, features, labels, K, mean):
        out, counts = _pool(features, labels, K, mean)
        ctx.save_for_backward(labels, counts)
        ctx.mean = mean
        ctx.mark_non_differentiable(counts)
        return out, counts

    @staticmethod
    @once_differentiable
    def backward(ctx, grad, _grad_counts):
        labels, counts = ctx.saved_tensors
        return _unpool(grad.contiguous(), labels, counts if ctx.mean else None), None, None, None


class _Unpool(torch.autograd.Function):
    @staticmethod
    def forward(ctx, values, labels):
        ctx.save_for_backward(labels)
        ctx.K = int(values.shape[2])
        return _unpool(values, labels)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad):
        labels, = ctx.saved_tensors
        return _pool(grad.contiguous(), labels, ctx.K, False)[0], None


def pool(features, labels, K, reduce="mean", return_counts=False):
    """float32 features [B,C,H,W], int16 labels [B,H,W] (read as uint16) -> float32 [B,C,K]: per superpixel k of image
    b, the sum (reduce="sum") or mean (reduce="mean") of features[b, c] over the pixels labelled k.  The mean is
    sum / (float)count, one correctly rounded division; an empty superpixel gives 0.0.  NaN and inf stay in their own
    superpixel.  With return_counts, also int32 counts [B,K]: the pixel count of each label in the label map -- not
    Cluster.num_members, which is the member count of the last subsampled update and is what get_mask_density divides
    by.  1 <= K <= 65534.  Differentiable in features: the gradient of the mean is unpool(grad) / count, that of the sum
    unpool(grad), 0 at pixels of no superpixel."""
    if reduce not in ("mean", "sum"):
        raise ValueError("reduce must be 'mean' or 'sum', got %r" % (reduce,))
    check_features(labels, "features", features, 4)
    K = check_K(K)
    cuda_device(labels, ("features", features))
    out, counts = _Pool.apply(features.contiguous(), labels.contiguous(), K, reduce == "mean")
    return (out, counts) if return_counts else out


def unpool(values, labels):
    """float32 values [B,C,K], int16 labels [B,H,W] -> float32 [B,C,H,W]: out[b,c,p] = values[b,c,label(p)], 0.0 where
    the label is outside [0, K).  Differentiable in values: the gradient is pool(grad, labels, K, reduce="sum")."""
    check_features(labels, "values", values, 3)
    check_K(int(values.shape[2]))
    cuda_device(labels, ("values", values))
    return _Unpool.apply(values.contiguous(), labels.contiguous())


def paint_argmax(q, labels):
    """float32 q [B,C,K] (e.g. SimpleCRFGroup.get_inferred), int16 labels [B,H,W] -> int16 [B,H,W]: the class of each
    pixel's superpixel, the first index of the maximum of q[b, :, label] (a NaN counts as the maximum, as in
    torch.argmax); -1 where the label is outside [0, K).  C <= 32767.  Not differentiable."""
    B, H, W, C = check_features(labels, "q", q, 3)
    K = check_K(int(q.shape[2]))
    if C > 32767:
        raise ValueError("paint_argmax gives int16 classes: C must be at most 32767, got %d" % C)
    dev = cuda_device(labels, ("q", q))
    with torch.cuda.device(dev):
        out = torch.empty((B, H, W), dtype=torch.int16, device=dev)
        if B and H and W:
            qc, lab = q.detach().contiguous(), labels.contiguous()
            node = torch.empty((B, K), dtype=torch.int32, device=dev)
            _lib.check(_lib.lib().fslic_b200_pool_paint_argmax_batch(
                dev.index, B, H, W, C, K, lab.data_ptr(), qc.data_ptr(), node.data_ptr(), out.data_ptr(),
                torch.cuda.current_stream(dev).cuda_stream))
    return out
