"""Superpixels merged into regions on the GPU (csrc/merge.cuh): single-linkage cuts of a region adjacency graph, at a
weight threshold (skimage's cut_threshold) or down to a number of regions per image, for whole batches of the int16
label maps iterate_batch returns.  The result is a label map of the same kind, so pool, region_adjacency,
region_properties and groundtruth take it unchanged, with the same K::

    g = region_adjacency(labels, K)
    x = pool(features, labels, K).transpose(1, 2).reshape(-1, C)          # [B*K, C]
    w = (x[g.edge_index[0]] - x[g.edge_index[1]]).norm(dim=1)              # float32 [E]
    m = merge_regions(labels, K, g, w, num_regions=200)                    # or threshold=0.15
    xm = pool(features, m.labels, K)                                       # region features [B,C,K]

No counterpart in the reference.  DESIGN.md section 4.16 describes the kernels.
"""
import collections
import math
import numbers
import operator

import torch

from . import _lib
from ._labelmaps import NO_SIZE, check_graph, check_K, cuda_device, same_device, tensor

MERGE_THRESHOLD, MERGE_NUM_REGIONS = 0, 1  # FSLIC_MERGE_THRESHOLD, FSLIC_MERGE_NUM_REGIONS
MAX_NODES = 1 << 30  # B * K: node ids are int32 on the device

MergeResult = collections.namedtuple("MergeResult", ["labels", "region", "num_regions"])


def _check_cut(threshold, num_regions):
    """(mode, threshold as a float, num_regions as an int) of exactly one given cut."""
    if (threshold is None) == (num_regions is None):
        raise ValueError("give exactly one of threshold and num_regions")
    if num_regions is not None:
        if isinstance(num_regions, bool):
            raise ValueError("num_regions must be an int, got %r" % (num_regions,))
        try:
            num_regions = operator.index(num_regions)
        except TypeError:
            raise ValueError("num_regions must be an int, got %r" % (num_regions,)) from None
        if num_regions < 1:
            raise ValueError("num_regions must be at least 1, got %d" % num_regions)
        return MERGE_NUM_REGIONS, 0.0, num_regions
    if isinstance(threshold, bool) or not isinstance(threshold, numbers.Real):
        raise ValueError("threshold must be a real number, got %r" % (threshold,))
    threshold = float(threshold)
    if math.isnan(threshold):
        raise ValueError("threshold must not be NaN")
    return MERGE_THRESHOLD, threshold, 0


def merge_regions(labels, K, graph, weights, threshold=None, num_regions=None):
    """Single-linkage merging of the superpixels of int16 labels [B,H,W] (read as uint16) over a region adjacency graph
    -> MergeResult(labels, region, num_regions):
    - labels      int16 [B,H,W]: each pixel's region id (read as uint16, like every label map here), -1 where the label
      is outside [0, K);
    - region      int32 [B,K]: the region of superpixel k of image b, -1 for a label no pixel carries;
    - num_regions int32 [B].
    Region ids are below K, numbered 0, 1, ... in each image in ascending order of their smallest member label.

    Node n = b*K + k is label k of image b; it is present when a pixel of labels[b] carries k.  graph is a RegionGraph
    (region_adjacency(labels, K), or any object with indptr of B*K + 1 entries and int64 edge_index [2,E]); weights is
    float32 [E].  Only entries with source < target are read, and the weight of the undirected edge {u, v} is weights[e]
    at that entry: the reverse direction is never read.  An entry is ignored when an endpoint is outside [0, B*K), the
    endpoints lie in different images, an endpoint is not present or its weight is NaN; such graphs never raise.

    Edges are ordered by (weight, lower local id, higher local id), -0.0 equal to +0.0, a total order in each image;
    single linkage is Kruskal over that order.
    - threshold=t: two nodes share a region exactly when a path of edges with weight < t joins them, compared in double
      precision ((double)w < t, skimage's strict <).
    - num_regions=R (an int >= 1): Kruskal stops after P_b - R merges or when it runs out of edges, P_b being the present
      nodes of image b.  That leaves max(R, c_b) regions, c_b the connected components among present nodes over non-NaN
      edges; R >= P_b merges nothing.

    Exactly one of threshold and num_regions is given.  ValueError, before any device work, for: labels that are not a
    cuda int16 [B,H,W] tensor, K outside [1, 65534], B*K > 2^30, indptr without B*K + 1 entries, edge_index that is not
    int64 [2,E], weights that are not float32 [E], tensors on different devices, both or neither cut, num_regions that is
    not an int >= 1, threshold that is NaN or not a real number.  B, H or W = 0 and E = 0 are fine.

    Runs on the labels' current stream.  Output shapes depend on B, H, W and K only and nothing is read back to the host,
    so a CUDA graph can capture the call.  Scratch comes from torch, sized from B and K.  Once weights are keys all
    arithmetic is integer: the result depends only on the inputs, not on the run, the stream, the batch order or
    splitting the batch."""
    tensor("labels", labels, torch.int16, 3)
    K = check_K(K)
    B, H, W = (int(v) for v in labels.shape)
    if B * K > MAX_NODES:
        raise ValueError("%d images of K = %d are %d nodes, more than %d: split the batch" % (B, K, B * K, MAX_NODES))
    edge_index, E = check_graph(graph, B, K)
    tensor("weights", weights, torch.float32, 1)
    if int(weights.shape[0]) != E:
        raise ValueError("weights must be float32 [E] with E = %d, got %s" % (E, tuple(weights.shape)))
    same_device(labels, ("graph.indptr", graph.indptr), ("graph.edge_index", edge_index), ("weights", weights))
    mode, t, R = _check_cut(threshold, num_regions)
    dev = cuda_device(labels)
    with torch.cuda.device(dev):
        out = MergeResult(torch.empty((B, H, W), dtype=torch.int16, device=dev),
                          torch.empty((B, K), dtype=torch.int32, device=dev),
                          torch.empty(B, dtype=torch.int32, device=dev))
        if B == 0:
            return out
        L = _lib.lib()
        nbytes = int(L.fslic_b200_merge_scratch_bytes(B, K))
        if nbytes == NO_SIZE:
            raise ValueError("no merge of %d images of K = %d" % (B, K))
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        lab = labels.contiguous()
        ei = edge_index.contiguous()
        w = weights.detach().contiguous()
        _lib.check(L.fslic_b200_merge_batch(dev.index, B, H, W, K, lab.data_ptr(), E, ei[0].data_ptr(),
                                            ei[1].data_ptr(), w.data_ptr(), mode, t, min(R, K), out.region.data_ptr(),
                                            out.num_regions.data_ptr(), out.labels.data_ptr(), scratch.data_ptr(),
                                            nbytes, torch.cuda.current_stream(dev).cuda_stream))
    return out
