"""Superpixels against ground truth on the GPU (csrc/groundtruth.cuh), for whole batches of the int16 label maps
iterate_batch returns: per-superpixel class histograms (the node targets of a superpixel classifier or GNN), the
standard superpixel quality scores (achievable segmentation accuracy, undersegmentation error, boundary recall and
precision within a pixel tolerance) and the boundary map of a label map.  With pooling.pool and
region_graph.region_adjacency it gives a superpixel GNN its targets::

    x = pool(features, labels, K)                                           # [B,C,K] node features
    g = region_adjacency(labels, K)                                         # their graph
    h = class_histogram(seg, labels, K, num_classes)                        # seg: [B,H,W] class map -> int32 [B,K,C]
    y = torch.where(h.sum(-1) > 0, h.argmax(-1), -100).reshape(-1)          # [B*K] targets; -100: CrossEntropyLoss's
                                                                            # ignore_index for empty superpixels

(argmax picks the lowest class on ties.)  No counterpart in the reference.  Cuda tensors only: labels int16 [B,H,W],
read as uint16, and a class / gt map of the same shape, uint8, int16, int32 or int64.  Every argument is checked
(ValueError) before any device work.  Work runs on the labels' device, on its current stream, and nothing is read back
to the host, so a CUDA graph can capture every call.  All arithmetic is integer: image b's result depends only on
labels[b] and gt[b] -- not on the batch, its place in it, the chunking, the stream or the run.  segmentation_scores_3d
and boundaries_3d are the same for label volumes [B,D,H,W], with 3-D boundaries and a box tolerance window that can
differ per axis.  DESIGN.md sections 4.14 and 4.24 describe the kernels.
"""
import collections

import torch

from . import _lib
from ._labelmaps import NO_SIZE, check_int, check_K, check_pixels, check_voxels, chunk, cuda_device, tensor

# Device memory one scores launch takes at most (about 20.4 bytes per pixel, 20.6 per voxel, and 16 per superpixel,
# plus the sort's storage): a batch that needs more runs in chunks of images or volumes, with identical results.
GT_SCRATCH_CAP = 1 << 30
MAX_CLASSES = 65536
MAX_TOLERANCE = 32
_MAX_CHUNK = 1 << 17  # the image bits of an overlap key
_INT64 = (-2 ** 63, 2 ** 63 - 1)
# the FSLIC_GT_* codes of include/fslic_b200.h: the element size
_DTYPES = {torch.uint8: 1, torch.int16: 2, torch.int32: 4, torch.int64: 8}

SegmentationScores = collections.namedtuple("SegmentationScores", [
    "pixels", "asa_pixels", "ue_pixels", "gt_boundary", "gt_boundary_hits", "sp_boundary", "sp_boundary_hits",
    "asa", "undersegmentation", "boundary_recall", "boundary_precision"])


def _check(name, gt, labels, ndim=3):
    """labels: int16 [B,H,W] (ndim 3) or [B,D,H,W] (ndim 4); gt: a map of the same shape and a _DTYPES dtype; images
    or volumes of at most MAX_PIXELS pixels.  Returns the shape."""
    tensor("labels", labels, torch.int16, ndim)
    if not isinstance(gt, torch.Tensor):
        raise ValueError("%s must be a cuda tensor (got %s): use torch.from_numpy(...).cuda()" % (name, type(gt).__name__))
    if gt.dtype not in _DTYPES:
        raise ValueError("%s must be a uint8, int16, int32 or int64 tensor, got %s" % (name, gt.dtype))
    if tuple(gt.shape) != tuple(labels.shape):
        raise ValueError("%s %s does not match labels %s" % (name, tuple(gt.shape), tuple(labels.shape)))
    shape = tuple(int(v) for v in labels.shape)
    if ndim == 4:
        check_voxels(*shape[1:], ": a count could overflow int32")
    else:
        check_pixels(*shape[1:], ": a count could overflow int32")
    return shape


def class_histogram(classes, labels, K, num_classes):
    """Class map classes [B,H,W] (uint8, int16, int32 or int64), int16 labels [B,H,W] (read as uint16) -> int32
    [B, K, num_classes]: out[b, k, c] is the number of pixels of image b with label k and class c.  A pixel whose label
    is outside [0, K) (-1 included) or whose class is outside [0, num_classes) (such as the ignore values 255 or -1) is
    not counted.  1 <= K <= 65534, 1 <= num_classes <= 65536.

    The majority class of each superpixel, as node targets (argmax picks the lowest class on ties; -100 is
    CrossEntropyLoss's ignore_index, for superpixels with no counted pixel)::

        h = class_histogram(seg, labels, K, C)
        y = torch.where(h.sum(-1) > 0, h.argmax(-1), -100).reshape(-1)     # [B*K]
    """
    B, H, W = _check("classes", classes, labels)
    K = check_K(K)
    C = check_int("num_classes", num_classes, 1, MAX_CLASSES)
    dev = cuda_device(labels, ("classes", classes))
    with torch.cuda.device(dev):
        out = torch.empty((B, K, C), dtype=torch.int32, device=dev)
        if B == 0 or H == 0 or W == 0:
            return out.zero_()
        cls, lab = classes.contiguous(), labels.contiguous()
        _lib.check(_lib.lib().fslic_b200_gt_histogram_batch(
            dev.index, B, H, W, K, C, _DTYPES[cls.dtype], cls.data_ptr(), lab.data_ptr(), out.data_ptr(),
            torch.cuda.current_stream(dev).cuda_stream))
    return out


def gt_chunk(B, H, W, K):
    """Images per scores launch: as many as fit GT_SCRATCH_CAP, at least one."""
    f = _lib.lib().fslic_b200_gt_scores_scratch_bytes
    if f(1, H, W, K) == NO_SIZE:
        raise ValueError("an image of %dx%d pixels is too large to score" % (H, W))
    return chunk(lambda c: f(c, H, W, K), GT_SCRATCH_CAP, B, limit=_MAX_CHUNK)


def _ratio(num, den):
    return torch.where(den > 0, num.double() / den.double(), torch.full_like(num, float("nan"), dtype=torch.float64))


def segmentation_scores(labels, gt, K, tolerance=2, ignore_index=None):
    """Scores of int16 superpixel labels [B,H,W] (read as uint16) against a ground-truth segmentation gt [B,H,W]
    (uint8, int16, int32 or int64) -> SegmentationScores, every field a [B] tensor on the labels' device.

    A gt pixel is valid when 0 <= gt <= 2^31 - 1 and gt != ignore_index; a pixel is counted when it is valid and its
    label is in [0, K).  n_kg is the number of counted pixels of an image with label k and gt value g, n_k = sum_g n_kg.
    Integer fields (int64), exact, so that dataset totals can be summed over images before dividing:
    - pixels: the counted pixels N;
    - asa_pixels: sum_k max_g n_kg;
    - ue_pixels: the sum over the pairs with n_kg > 0 of min(n_kg, n_k - n_kg) (Neubert and Protzel's corrected
      undersegmentation error);
    - gt_boundary: the gt boundary pixels, valid pixels whose right or lower neighbour is valid and has another gt value;
    - gt_boundary_hits: those with a superpixel boundary pixel (see boundaries) in their window;
    - sp_boundary: the superpixel boundary pixels that are valid in gt;
    - sp_boundary_hits: those with a gt boundary pixel in their window.
    The window of a pixel is the square |di|, |dj| <= tolerance (an int in [0, 32]) clipped to the image.  This is the
    common fast form of boundary recall, not the BSDS bipartite matching of boundary pixels.
    Ratios (float64, NaN where the denominator is 0): asa = asa_pixels / pixels, undersegmentation = ue_pixels /
    pixels, boundary_recall = gt_boundary_hits / gt_boundary, boundary_precision = sp_boundary_hits / sp_boundary.

    For several annotations per image, as in BSDS, stack them along B and repeat the labels to match
    (labels.repeat_interleave(A, 0) for A annotations per image)."""
    B, H, W = _check("gt", gt, labels)
    K = check_K(K)
    r = check_int("tolerance", tolerance, 0, MAX_TOLERANCE)
    ignore = None if ignore_index is None else check_int("ignore_index", ignore_index, *_INT64)
    dev = cuda_device(labels, ("gt", gt))
    with torch.cuda.device(dev):
        out = torch.zeros((B, 7), dtype=torch.int64, device=dev)
        if B and H and W:
            g, lab = gt.contiguous(), labels.contiguous()
            L = _lib.lib()
            chunk = gt_chunk(B, H, W, K)
            nbytes = int(L.fslic_b200_gt_scores_scratch_bytes(chunk, H, W, K))
            scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            stream = torch.cuda.current_stream(dev).cuda_stream
            for b0 in range(0, B, chunk):
                c = min(chunk, B - b0)
                _lib.check(L.fslic_b200_gt_scores_batch(
                    dev.index, c, H, W, K, r, _DTYPES[g.dtype], g[b0].data_ptr(), lab[b0].data_ptr(),
                    int(ignore is not None), 0 if ignore is None else ignore, out[b0].data_ptr(), scratch.data_ptr(),
                    nbytes, stream))
        f = out.t().contiguous().unbind(0)
        return SegmentationScores(*f, _ratio(f[1], f[0]), _ratio(f[2], f[0]), _ratio(f[4], f[3]), _ratio(f[6], f[5]))


def boundaries(labels):
    """int16 labels [B,H,W] -> bool [B,H,W]: True at superpixel boundary pixels, those whose right or lower neighbour
    exists and carries another raw label -- a one-sided, 1-pixel-wide outline (what skimage's mark_boundaries draws),
    the same predicate segmentation_scores uses."""
    tensor("labels", labels, torch.int16, 3)
    B, H, W = (int(v) for v in labels.shape)
    check_pixels(H, W)
    dev = cuda_device(labels)
    with torch.cuda.device(dev):
        out = torch.empty((B, H, W), dtype=torch.bool, device=dev)
        if B and H and W:
            lab = labels.contiguous()
            _lib.check(_lib.lib().fslic_b200_gt_boundaries_batch(dev.index, B, H, W, lab.data_ptr(), out.data_ptr(),
                                                                 torch.cuda.current_stream(dev).cuda_stream))
    return out


def gt3d_chunk(B, D, H, W, K):
    """Volumes per scores launch of segmentation_scores_3d: as many as fit GT_SCRATCH_CAP, at least one."""
    f = _lib.lib().fslic_b200_gt_scores3d_scratch_bytes
    if f(1, D, H, W, K) == NO_SIZE:
        raise ValueError("a volume of %dx%dx%d voxels is too large to score" % (D, H, W))
    return chunk(lambda c: f(c, D, H, W, K), GT_SCRATCH_CAP, B, limit=_MAX_CHUNK)


def check_tolerance_3d(tolerance):
    """An int r in [0, 32] -> (r, r, r); a tuple or list (rz, ry, rx) of such ints -> itself as a tuple."""
    if isinstance(tolerance, (tuple, list)):
        if len(tolerance) != 3:
            raise ValueError("tolerance must be an int or a (rz, ry, rx) tuple, got %r" % (tolerance,))
        return tuple(check_int("tolerance", r, 0, MAX_TOLERANCE) for r in tolerance)
    r = check_int("tolerance", tolerance, 0, MAX_TOLERANCE)
    return r, r, r


def segmentation_scores_3d(labels, gt, K, tolerance=2, ignore_index=None):
    """Scores of int16 supervoxel labels [B,D,H,W] (read as uint16) against a ground-truth segmentation gt [B,D,H,W]
    (uint8, int16, int32 or int64) -> SegmentationScores, every field a [B] tensor: segmentation_scores for volumes.
    - pixels, asa_pixels, ue_pixels and their ratios count voxels and equal segmentation_scores on the [B, D*H, W]
      views of labels and gt (the overlap table does not depend on the layout).
    - The boundaries are 3-D and one-sided: a supervoxel boundary voxel is one of boundaries_3d, a gt boundary voxel
      is valid and has a valid +x, +y or +z neighbour with another value; sp_boundary counts the supervoxel boundary
      voxels valid in gt.
    - The window of a voxel is the box |dz| <= rz, |dy| <= ry, |dx| <= rx clipped to the volume.  tolerance is an int
      r in [0, 32] (rz = ry = rx = r) or a tuple (rz, ry, rx) of such ints, for anisotropic voxels such as CT's thick
      slices.
    At D = 1 every field equals segmentation_scores on labels[:, 0] with the tolerance ry = rx.  The call reads nothing
    back, so a CUDA graph can capture it; volumes run in chunks under GT_SCRATCH_CAP with identical results."""
    B, D, H, W = _check("gt", gt, labels, 4)
    K = check_K(K)
    rz, ry, rx = check_tolerance_3d(tolerance)
    ignore = None if ignore_index is None else check_int("ignore_index", ignore_index, *_INT64)
    dev = cuda_device(labels, ("gt", gt))
    with torch.cuda.device(dev):
        out = torch.zeros((B, 7), dtype=torch.int64, device=dev)
        if B and D and H and W:
            g, lab = gt.contiguous(), labels.contiguous()
            L = _lib.lib()
            chunk = gt3d_chunk(B, D, H, W, K)
            nbytes = int(L.fslic_b200_gt_scores3d_scratch_bytes(chunk, D, H, W, K))
            scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            stream = torch.cuda.current_stream(dev).cuda_stream
            for b0 in range(0, B, chunk):
                c = min(chunk, B - b0)
                _lib.check(L.fslic_b200_gt_scores3d_batch(
                    dev.index, c, D, H, W, K, rz, ry, rx, _DTYPES[g.dtype], g[b0].data_ptr(), lab[b0].data_ptr(),
                    int(ignore is not None), 0 if ignore is None else ignore, out[b0].data_ptr(), scratch.data_ptr(),
                    nbytes, stream))
        f = out.t().contiguous().unbind(0)
        return SegmentationScores(*f, _ratio(f[1], f[0]), _ratio(f[2], f[0]), _ratio(f[4], f[3]), _ratio(f[6], f[5]))


def boundaries_3d(labels):
    """int16 labels [B,D,H,W] -> bool [B,D,H,W]: True at supervoxel boundary voxels, those whose +x, +y or +z neighbour
    exists and carries another raw label -- a one-sided, 1-voxel-wide outline, the predicate segmentation_scores_3d
    uses.  No scratch and no read-back: a CUDA graph can capture it."""
    tensor("labels", labels, torch.int16, 4)
    B, D, H, W = (int(v) for v in labels.shape)
    check_voxels(D, H, W)
    dev = cuda_device(labels)
    with torch.cuda.device(dev):
        out = torch.empty((B, D, H, W), dtype=torch.bool, device=dev)
        if B and D and H and W:
            lab = labels.contiguous()
            _lib.check(_lib.lib().fslic_b200_gt_boundaries3d_batch(dev.index, B, D, H, W, lab.data_ptr(), out.data_ptr(),
                                                                   torch.cuda.current_stream(dev).cuda_stream))
    return out
