"""Region adjacency graphs of superpixel label maps on the GPU (csrc/rag.cuh): for a batch of the int16 label maps
iterate_batch returns, every pair of superpixels that touch, weighted by the length of their shared boundary, in the
CSR / COO layout graph libraries take.  With pooling.pool it gives a superpixel GNN its node features and its graph::

    x = pool(features, labels, K)                        # [B,C,K] node features
    g = region_adjacency(labels, K)                      # the B*K nodes' graph, one block per image
    A = torch.sparse_csr_tensor(g.indptr, g.edge_index[1], g.boundary.float(), (B * K, B * K))

boundary_stats gives each edge the mean, min and max of pixel maps along its shared boundary (PyG's edge_attr), such
as the strength of an edge map between two superpixels, which merging.merge_regions takes as its weights::

    s = boundary_stats(labels, K, g, edge_map[:, None])  # [E,1] mean / min / max, [E] pair counts
    m = merge_regions(labels, K, g, s.mean[:, 0], threshold=t)

knn_graph gives the other standard graph over superpixel nodes: each joined to its k nearest superpixels in feature
space (the MNIST / CIFAR10 superpixel GNN benchmarks use k = 8 over position and mean colour), exact, with ties broken
by the lower index, in the same node numbering and CSR layout::

    kg = knn_graph(x, 8, present=p.area > 0, symmetric=True)  # x: [B,K,D] node features, p region_properties
    A = torch.sparse_csr_tensor(kg.indptr, kg.edge_index[1], torch.exp(-kg.distance), (B * K, B * K))

No counterpart in the reference: its get_connectivity keeps at most 12 neighbours per superpixel, in scan order, and
is kept for parity with it; its get_knn_connectivity has no defined result and raises NotImplementedError here.
region_adjacency_3d is the graph of supervoxel label volumes [B,D,H,W], in 6-, 18- or 26-connectivity, and
boundary_stats_3d the statistics of voxel maps along its faces.  DESIGN.md sections 4.13, 4.17, 4.18, 4.23 and 4.24
describe the kernels.
"""
import collections

import numpy as np
import torch

from . import _lib
from ._labelmaps import (MAX_PIXELS, NO_SIZE, check_connectivity, check_connectivity_3d, check_features, check_graph,
                         check_int, check_K, check_pixels, check_voxels, chunk, cuda_device, tensor)

# Device memory the pair tables of one count launch take at most (8 bytes per slot, a power of two >= max(4096, 32 K)
# slots per image): a batch that needs more runs in chunks of images, with identical results.
RAG_SCRATCH_CAP = 1 << 30
# Device memory the boundary pair selection of one launch takes at most (4 bytes per pixel pair, 2 or 4 per pixel),
# sized before the pair count is known: a batch that needs more runs in chunks of images, with identical results.  A
# chunk whose boundary pairs need more than this for their sort is split again (only maps that are not superpixel maps,
# such as noise, have that many).
# boundary_stats_3d takes the same cap for its selection, which takes 6 bytes per voxel (so a 256x512x512 volume fits
# at any connectivity), and halves a chunk in the same way.
BOUNDARY_SCRATCH_CAP = 1 << 30
# Device memory one kNN launch takes at most (about 17 + 4 D + 8 k bytes per node, 72 k more for a symmetric graph):
# a batch that needs more runs in chunks of images, with identical results.
KNN_SCRATCH_CAP = 1 << 30
_INT_MAX = 2 ** 31 - 1
KNN_MAX_D = 64
KNN_MAX_NEIGHBORS = 32
KNN_MAX_NODES = 1 << 30  # B * K

# The forward half of the 3x3x3 neighbourhood, (dz, dy, dx) with the first non-zero component positive: the voxel
# pairs of region_adjacency_3d are each voxel with these neighbours (connectivity 6: the first 3, 18: 9, 26: 13)
RAG3D_OFFSETS = ((0, 0, 1), (0, 1, 0), (1, 0, 0), (0, 1, 1), (0, 1, -1), (1, 1, 0), (1, -1, 0), (1, 0, 1), (1, 0, -1),
                 (1, 1, 1), (1, 1, -1), (1, -1, 1), (1, -1, -1))

RegionGraph = collections.namedtuple("RegionGraph", ["indptr", "edge_index", "boundary"])
BoundaryStats = collections.namedtuple("BoundaryStats", ["mean", "min", "max", "count"])
KnnGraph = collections.namedtuple("KnnGraph", ["indptr", "edge_index", "distance"])


def rag_chunk(B, H, W, K, connectivity):
    """Images per count launch: as many as fit RAG_SCRATCH_CAP, at least one."""
    f = _lib.lib().fslic_b200_rag_batch_scratch_bytes
    if f(1, H, W, K, connectivity, 0) == NO_SIZE:
        raise ValueError("an image of %dx%d pixels is too large for a region adjacency graph" % (H, W))
    return chunk(lambda c: f(c, H, W, K, connectivity, 0), RAG_SCRATCH_CAP, B)


def _split(b0, flags):
    """The images of a count whose tables overflowed, each on its own with an exact table, and the runs between them
    with the usual one: (first image, images, exact) in batch order."""
    runs, start = [], 0
    for i, flag in enumerate(flags + [1]):
        if flag:
            if i > start:
                runs.append((b0 + start, i - start, 0))
            if i < len(flags):
                runs.append((b0 + i, 1, 1))
            start = i + 1
    return runs


def region_adjacency(labels, K, connectivity=4):
    """Region adjacency graph of int16 labels [B,H,W] (read as uint16) -> RegionGraph(indptr, edge_index, boundary).

    Node n = b*K + k is label k of image b; no edge joins two images (the block-diagonal batch graph of PyG's Batch).
    - indptr     int64 [B*K + 1]: CSR row offsets; node n's edges are indptr[n]:indptr[n+1].
    - edge_index int64 [2, E]: (source, target) of both directions of every edge, sorted by source then target, so
      edge_index[1] is the CSR column array.
    - boundary   int32 [E]: the number of adjacent pixel pairs whose labels are the edge's two nodes.
    Pixel pairs are the horizontally and vertically adjacent pixels (connectivity=4), plus both diagonals
    (connectivity=8), each unordered pair once, the last row and column included.  A label outside [0, K) (-1 included)
    belongs to no node and its pairs are ignored; a pair with equal labels is no edge.  1 <= K <= 65534 and
    H * W <= 2^29; anything else, a tensor that is not a cuda int16 [B,H,W] tensor, or a connectivity other than 4 or 8
    raises ValueError before any device work.  B, H or W = 0 gives zero rows and no edges.

    Work runs on the labels' device, on its current stream.  The edge count is data-dependent, so, like torch.unique,
    this call waits for the device: it reads (images + 1) int64 words back once per chunk of images (the edge total
    and which images' pair tables overflowed; such images are counted again with an exact table, one read more per
    run of images recounted -- only label maps that are not superpixel maps, such as noise, need that).  It cannot be
    captured in a CUDA graph and raises RuntimeError under capture, before any device work.  All arithmetic is
    integer: the result is exact and the same across runs, batch order, chunking and streams."""
    tensor("labels", labels, torch.int16, 3)
    connectivity = check_connectivity(connectivity)
    K = check_K(K)
    B, H, W = (int(v) for v in labels.shape)
    check_pixels(H, W, ": a boundary count could overflow int32")
    dev = cuda_device(labels)
    with torch.cuda.device(dev):
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError("region_adjacency reads its edge count back to the host and cannot be captured in a "
                               "CUDA graph")
        if B == 0 or H == 0 or W == 0:
            return RegionGraph(torch.zeros(B * K + 1, dtype=torch.int64, device=dev),
                               torch.empty((2, 0), dtype=torch.int64, device=dev),
                               torch.empty(0, dtype=torch.int32, device=dev))
        L = _lib.lib()
        return _rag(labels.contiguous(), B, K, rag_chunk(B, H, W, K, connectivity), (H, W, K, connectivity), "image",
                    L.fslic_b200_rag_batch_scratch_bytes, L.fslic_b200_rag_batch_count, L.fslic_b200_rag_batch_fill)


def _rag(lab, B, K, first_chunk, dims, what, scratch_bytes, count, fill):
    """The count / read / fill loop of region_adjacency and region_adjacency_3d over B contiguous images or volumes
    lab on the current device: chunks of first_chunk, overflowed ones split by _split and recounted, those of more
    than 2^31 - 1 edges halved.  dims are the entry points' arguments between the batch and `exact`."""
    dev = lab.device
    L = _lib.lib()
    stream = torch.cuda.current_stream(dev).cuda_stream
    indptr = torch.empty(B * K + 1, dtype=torch.int64, device=dev)
    work = [(b0, min(first_chunk, B - b0), 0) for b0 in range(0, B, first_chunk)][::-1]
    pieces, edges = [], 0
    while work:
        b0, c, exact = work.pop()
        nbytes = int(scratch_bytes(c, *dims, exact))
        if nbytes == NO_SIZE:
            raise MemoryError("%s %d has too many distinct adjacent label pairs for an exact pair table" % (what, b0))
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        info = torch.empty(c + 1, dtype=torch.int64, device=dev)
        _lib.check(count(dev.index, c, *dims, exact, lab[b0].data_ptr(), edges, indptr[b0 * K:].data_ptr(),
                         info.data_ptr(), scratch.data_ptr(), nbytes, stream))
        info = info.tolist()  # the host wait: overflow flags and the edge total
        flags, total = info[:c], info[c]
        if any(flags):
            work.extend(_split(b0, flags)[::-1])
            continue
        if total > _INT_MAX:  # one segmented sort per fill
            if c == 1:
                raise MemoryError("%s %d has %d directed edges, more than one fill takes" % (what, b0, total))
            work.extend([(b0 + c // 2, c - c // 2, exact), (b0, c // 2, exact)])
            continue
        edge_index = torch.empty((2, total), dtype=torch.int64, device=dev)
        boundary = torch.empty(total, dtype=torch.int32, device=dev)
        if total:
            fbytes = int(L.fslic_b200_rag_fill_scratch_bytes(c, K, total))
            fill_scratch = torch.empty(fbytes, dtype=torch.uint8, device=dev)
            _lib.check(fill(dev.index, c, *dims, exact, b0 * K, total, scratch.data_ptr(), nbytes,
                            fill_scratch.data_ptr(), fbytes, edge_index[0].data_ptr(), edge_index[1].data_ptr(),
                            boundary.data_ptr(), stream))
        pieces.append((edge_index, boundary))
        edges += total
    if len(pieces) == 1:
        edge_index, boundary = pieces[0]
    else:
        edge_index = torch.cat([p[0] for p in pieces], dim=1)
        boundary = torch.cat([p[1] for p in pieces])
    return RegionGraph(indptr, edge_index, boundary)


def voxel_pairs(D, H, W, connectivity):
    """Voxel pairs of one D x H x W volume at connectivity 6, 18 or 26: sum over the forward offsets (dz, dy, dx) with
    at most 1, 2 or 3 non-zero components of (D - |dz|)(H - |dy|)(W - |dx|)."""
    if D * H * W == 0:
        return 0
    most = {6: 1, 18: 2, 26: 3}[connectivity]
    return sum((D - abs(dz)) * (H - abs(dy)) * (W - abs(dx)) for dz, dy, dx in RAG3D_OFFSETS
               if (dz != 0) + (dy != 0) + (dx != 0) <= most)


def rag3d_chunk(B, D, H, W, K, connectivity):
    """Volumes per count launch of region_adjacency_3d: as many as fit RAG_SCRATCH_CAP, at least one."""
    f = _lib.lib().fslic_b200_rag3d_batch_scratch_bytes
    if f(1, D, H, W, K, connectivity, 0) == NO_SIZE:
        raise ValueError("a volume of %dx%dx%d voxels is too large for a region adjacency graph" % (D, H, W))
    return chunk(lambda c: f(c, D, H, W, K, connectivity, 0), RAG_SCRATCH_CAP, B)


def region_adjacency_3d(labels, K, connectivity=6):
    """Region adjacency graph of int16 label volumes [B,D,H,W] (read as uint16) -> RegionGraph(indptr, edge_index,
    boundary), the volume form of region_adjacency with the same node numbering n = b*K + k, dtypes and CSR / COO
    layout, so every consumer of region_adjacency's graph (merge_regions, knn_graph's users, message_passing) takes it.
    - boundary int32 [E]: the number of adjacent voxel pairs whose labels are the edge's two nodes.
    Voxel pairs are the forward half of the 3x3x3 neighbourhood, each unordered pair once, the last slice, row and
    column included: the 3 face neighbours (connectivity=6), plus the 6 edge neighbours (18), plus the 4 corner
    neighbours (26).  A label outside [0, K) (-1 included) belongs to no node and its pairs are ignored; a pair with
    equal labels is no edge.  1 <= K <= 65534, D * H * W <= 2^29 and the volume's voxel pair count (voxel_pairs) at
    most 2^31 - 1 (so every boundary count fits int32: a 512^3 volume fits at 26-connectivity; 2^29 voxels at 18 or
    26 do not); anything else, a tensor that is not a cuda int16 [B,D,H,W] tensor, or a connectivity other than 6, 18
    or 26 raises ValueError before any device work.  B, D, H or W = 0 gives zero rows and no edges.

    Host behaviour is region_adjacency's: one read of (volumes + 1) int64 words per chunk of volumes
    (RAG_SCRATCH_CAP), volumes whose pair table overflowed counted again alone with an exact table, RuntimeError under
    CUDA graph capture before any device work.  All arithmetic is integer: the result is exact and the same across
    runs, batch order, chunking and streams."""
    tensor("labels", labels, torch.int16, 4)
    connectivity = check_connectivity_3d(connectivity)
    K = check_K(K)
    B, D, H, W = (int(v) for v in labels.shape)
    if D * H * W > MAX_PIXELS:
        raise ValueError("volumes of %dx%dx%d voxels exceed %d voxels" % (D, H, W, MAX_PIXELS))
    P = voxel_pairs(D, H, W, connectivity)
    if P > _INT_MAX:
        raise ValueError("volumes of %dx%dx%d voxels have %d voxel pairs at connectivity %d, more than %d: a "
                         "boundary count could overflow int32" % (D, H, W, P, connectivity, _INT_MAX))
    dev = cuda_device(labels)
    with torch.cuda.device(dev):
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError("region_adjacency_3d reads its edge count back to the host and cannot be captured in a "
                               "CUDA graph")
        if B == 0 or D == 0 or H == 0 or W == 0:
            return RegionGraph(torch.zeros(B * K + 1, dtype=torch.int64, device=dev),
                               torch.empty((2, 0), dtype=torch.int64, device=dev),
                               torch.empty(0, dtype=torch.int32, device=dev))
        L = _lib.lib()
        return _rag(labels.contiguous(), B, K, rag3d_chunk(B, D, H, W, K, connectivity), (D, H, W, K, connectivity),
                    "volume", L.fslic_b200_rag3d_batch_scratch_bytes, L.fslic_b200_rag3d_batch_count,
                    L.fslic_b200_rag3d_batch_fill)


def boundary_chunk(B, H, W, K, connectivity):
    """Images per boundary pair selection: as many as fit BOUNDARY_SCRATCH_CAP, at least one."""
    f = _lib.lib().fslic_b200_boundary_select_scratch_bytes
    if f(1, H, W, K, connectivity) == NO_SIZE:
        raise ValueError("an image of %dx%d pixels is too large for boundary statistics" % (H, W))
    return chunk(lambda c: f(c, H, W, K, connectivity), BOUNDARY_SCRATCH_CAP, B)


def boundary_stats(labels, K, graph, values, connectivity=4):
    """Statistics of pixel maps along the shared boundary of every entry of a region adjacency graph
    -> BoundaryStats(mean, min, max, count), detached:
    - mean, min, max float32 [E, C]: one row per entry of graph.edge_index, in its order (PyG's edge_attr layout);
    - count          int32 [E]: the number of boundary pixel pairs of the entry.
    labels is a cuda int16 [B,H,W] tensor (read as uint16), values float32 [B,C,H,W] (C >= 1, pool's layout) on the same
    device.  graph is a RegionGraph (region_adjacency(labels, K, ...)) or any object with indptr of B*K + 1 entries and
    int64 edge_index [2,E]; only edge_index is read.

    Pixel pairs are region_adjacency's: each pixel (the anchor) with its right and down neighbour, with connectivity 8
    also the down-right and down-left one.  A pair is a boundary pair when both labels are in [0, K) and differ; its
    ordinal is anchor_index * D + d, d the direction in that order and D = 2 or 4.  Entry e = (u, v) gets the boundary
    pairs of image b whose labels are {u % K, v % K} when 0 <= u, v < B*K, u // K == v // K == b and u != v, and none
    otherwise: both directions of an edge and duplicate entries get identical rows, and entries across images, out of
    range or with equal endpoints never fault or raise.  The result does not depend on indptr or on the entries' order.
    - The 2n values of an entry with n pairs, per channel, are values[b, c, anchor] then values[b, c, other] of each
      pair in increasing ordinal.  count is n: for a graph from region_adjacency with the same labels and connectivity
      it equals graph.boundary.
    - mean is their sum in pool's order (dealt to 32 lanes left to right from +0.0, five butterfly steps, lane 0's
      value) divided by (float)(2n), one correctly rounded division.
    - min / max follow the total order of non-NaN floats with -0.0 < +0.0; any NaN value makes them NaN (torch.amin /
      amax).
    - An entry with no pairs gets count 0 and NaN in mean, min and max, which merge_regions ignores.
    Each row depends only on labels[b], values[b] and the entry: not on the batch, the chunking, the stream or the run.

    ValueError, before any device work, for: labels that are not a cuda int16 [B,H,W] tensor, values that are not
    float32 [B,C,H,W] with the labels' B, H, W and C >= 1, K outside [1, 65534], images over 2^29 pixels, connectivity
    other than 4 or 8, indptr without B*K + 1 entries, edge_index that is not int64 [2,E] (E < 2^31), tensors on
    different devices.  B, H or W = 0 and E = 0 launch nothing.

    Work runs on the labels' device, on its current stream.  The boundary pair count is data-dependent, so, like
    region_adjacency, this call reads one int32 back per chunk of images (BOUNDARY_SCRATCH_CAP; a chunk whose pairs need
    more than the cap to sort is halved and read again, which only maps that are not superpixel maps come near): it
    cannot be captured in a CUDA graph and raises RuntimeError under capture, before any device work."""
    B, H, W, C = check_features(labels, "values", values, 4)
    connectivity = check_connectivity(connectivity)
    K = check_K(K)
    check_pixels(H, W, ": a boundary count could overflow int32")
    edge_index, E = check_graph(graph, B, K)
    if E > _INT_MAX:
        raise ValueError("graph.edge_index has %d entries, more than %d: split the graph" % (E, _INT_MAX))
    dev = cuda_device(labels, ("values", values), ("graph.indptr", graph.indptr), ("graph.edge_index", edge_index))
    with torch.cuda.device(dev):
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError("boundary_stats reads its boundary pair count back to the host and cannot be captured in "
                               "a CUDA graph")
        if B == 0 or H == 0 or W == 0 or E == 0:  # no pixel pair: every row is absent
            nan = float("nan")
            return BoundaryStats(torch.full((E, C), nan, dtype=torch.float32, device=dev),
                                 torch.full((E, C), nan, dtype=torch.float32, device=dev),
                                 torch.full((E, C), nan, dtype=torch.float32, device=dev),
                                 torch.zeros(E, dtype=torch.int32, device=dev))
        out = BoundaryStats(*(torch.empty((E, C), dtype=torch.float32, device=dev) for _ in range(3)),
                            torch.empty(E, dtype=torch.int32, device=dev))
        lab = labels.contiguous()
        val = values.detach().contiguous()
        ei = edge_index.contiguous()
        L = _lib.lib()
        stream = torch.cuda.current_stream(dev).cuda_stream
        chunk = boundary_chunk(B, H, W, K, connectivity)
        work = [(b0, min(chunk, B - b0)) for b0 in range(0, B, chunk)][::-1]
        first = 1
        while work:
            b0, c = work.pop()
            nbytes = int(L.fslic_b200_boundary_select_scratch_bytes(c, H, W, K, connectivity))
            select = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            npairs = torch.empty(1, dtype=torch.int32, device=dev)
            _lib.check(L.fslic_b200_boundary_select_batch(dev.index, c, H, W, K, connectivity, lab[b0].data_ptr(),
                                                          npairs.data_ptr(), select.data_ptr(), nbytes, stream))
            pairs = int(npairs.item())  # the host wait: the boundary pair count
            sbytes = int(L.fslic_b200_boundary_stats_scratch_bytes(pairs, E))
            if sbytes > BOUNDARY_SCRATCH_CAP and c > 1:  # too many pairs to sort at once: halve the chunk
                work.extend([(b0 + c // 2, c - c // 2), (b0, c // 2)])
                continue
            scratch = torch.empty(sbytes, dtype=torch.uint8, device=dev)
            _lib.check(L.fslic_b200_boundary_stats_batch(
                dev.index, c, H, W, K, C, connectivity, lab[b0].data_ptr(), val[b0].data_ptr(), pairs,
                select.data_ptr(), nbytes, b0, B * K, E, ei[0].data_ptr(), ei[1].data_ptr(), first,
                out.mean.data_ptr(), out.min.data_ptr(), out.max.data_ptr(), out.count.data_ptr(), scratch.data_ptr(),
                sbytes, stream))
            first = 0
    return out


def boundary3d_chunk(B, D, H, W, K, connectivity):
    """Volumes per boundary voxel selection of boundary_stats_3d: as many as fit BOUNDARY_SCRATCH_CAP, at least one."""
    f = _lib.lib().fslic_b200_boundary3d_select_scratch_bytes
    if f(1, D, H, W, K, connectivity) == NO_SIZE:
        raise ValueError("a volume of %dx%dx%d voxels is too large for boundary statistics" % (D, H, W))
    return chunk(lambda c: f(c, D, H, W, K, connectivity), BOUNDARY_SCRATCH_CAP, B)


def boundary_stats_3d(labels, K, graph, values, connectivity=6):
    """Statistics of voxel maps along the shared boundary of every entry of a region adjacency graph of label volumes
    -> BoundaryStats(mean, min, max, count), detached: boundary_stats for volumes, with the same outputs, float32
    [E, C] and int32 [E], and the same rules.  labels is a cuda int16 [B,D,H,W] tensor (read as uint16), values float32
    [B,C,D,H,W] (C >= 1) on the same device.  graph is a RegionGraph (region_adjacency_3d(labels, K, connectivity)) or
    any object with indptr of B*K + 1 entries and int64 edge_index [2,E]; only edge_index is read.

    Voxel pairs are region_adjacency_3d's: each voxel (the anchor) with its forward neighbours RAG3D_OFFSETS[:3]
    (connectivity 6), [:9] (18) or [:13] (26); a pair's ordinal is anchor_index * Ndir + d, d its index in
    RAG3D_OFFSETS.  A boundary pair has both labels in [0, K) and different.  Entry e = (u, v) of volume b gets the
    boundary pairs whose labels are {u % K, v % K}; the 2n values of an entry, per channel, are values[b, c, anchor]
    then values[b, c, other] of each pair in increasing ordinal; mean is their sum in pool's lane order divided by
    (float)(2n); min / max follow the total order of non-NaN floats with -0.0 < +0.0, NaN when any value is NaN.  An
    entry with no pairs, across volumes, out of range or with equal endpoints gets NaN and count 0 and never faults.
    For a graph from region_adjacency_3d with the same labels and connectivity, count equals graph.boundary.  At D = 1
    the result equals boundary_stats on labels[:, 0] with connectivity 4 (for 6) or 8 (for 18 and 26).

    ValueError, before any device work, for: labels that are not a cuda int16 [B,D,H,W] tensor, values that are not
    float32 [B,C,D,H,W] with the labels' B, D, H, W and C >= 1, K outside [1, 65534], volumes over 2^29 voxels or with
    more than 2^31 - 1 voxel pairs (voxel_pairs), connectivity other than 6, 18 or 26, indptr without B*K + 1 entries,
    edge_index that is not int64 [2,E] (E < 2^31), tensors on different devices.  B, D, H, W = 0 and E = 0 launch
    nothing.

    Host behaviour is boundary_stats': one read of two int64 (the boundary voxel and pair counts) per chunk of volumes
    (BOUNDARY_SCRATCH_CAP, a chunk whose pairs need more than the cap to sort halved and read again), RuntimeError under
    CUDA graph capture before any device work.  Each row depends only on labels[b], values[b] and the entry."""
    tensor("labels", labels, torch.int16, 4)
    tensor("values", values, torch.float32, 5)
    B, D, H, W = (int(v) for v in labels.shape)
    if int(values.shape[0]) != B or tuple(int(v) for v in values.shape[2:]) != (D, H, W):
        raise ValueError("values %s do not match labels %s" % (tuple(values.shape), (B, D, H, W)))
    C = int(values.shape[1])
    if C < 1:
        raise ValueError("values needs at least one channel")
    connectivity = check_connectivity_3d(connectivity)
    K = check_K(K)
    check_voxels(D, H, W, ": a boundary count could overflow int32")
    P = voxel_pairs(D, H, W, connectivity)
    if P > _INT_MAX:
        raise ValueError("volumes of %dx%dx%d voxels have %d voxel pairs at connectivity %d, more than %d: a "
                         "boundary count could overflow int32" % (D, H, W, P, connectivity, _INT_MAX))
    edge_index, E = check_graph(graph, B, K)
    if E > _INT_MAX:
        raise ValueError("graph.edge_index has %d entries, more than %d: split the graph" % (E, _INT_MAX))
    dev = cuda_device(labels, ("values", values), ("graph.indptr", graph.indptr), ("graph.edge_index", edge_index))
    with torch.cuda.device(dev):
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError("boundary_stats_3d reads its boundary pair count back to the host and cannot be captured "
                               "in a CUDA graph")
        if B == 0 or D == 0 or H == 0 or W == 0 or E == 0:  # no voxel pair: every row is absent
            nan = float("nan")
            return BoundaryStats(torch.full((E, C), nan, dtype=torch.float32, device=dev),
                                 torch.full((E, C), nan, dtype=torch.float32, device=dev),
                                 torch.full((E, C), nan, dtype=torch.float32, device=dev),
                                 torch.zeros(E, dtype=torch.int32, device=dev))
        out = BoundaryStats(*(torch.empty((E, C), dtype=torch.float32, device=dev) for _ in range(3)),
                            torch.empty(E, dtype=torch.int32, device=dev))
        lab = labels.contiguous()
        val = values.detach().contiguous()
        ei = edge_index.contiguous()
        L = _lib.lib()
        stream = torch.cuda.current_stream(dev).cuda_stream
        chunk = boundary3d_chunk(B, D, H, W, K, connectivity)
        work = [(b0, min(chunk, B - b0)) for b0 in range(0, B, chunk)][::-1]
        first = 1
        while work:
            b0, c = work.pop()
            nbytes = int(L.fslic_b200_boundary3d_select_scratch_bytes(c, D, H, W, K, connectivity))
            select = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            counts = torch.empty(2, dtype=torch.int64, device=dev)
            _lib.check(L.fslic_b200_boundary3d_select_batch(dev.index, c, D, H, W, K, connectivity, lab[b0].data_ptr(),
                                                            counts.data_ptr(), select.data_ptr(), nbytes, stream))
            voxels, pairs = counts.tolist()  # the host wait: the boundary voxel and pair counts
            sbytes = int(L.fslic_b200_boundary3d_stats_scratch_bytes(voxels, pairs, E))
            if sbytes > BOUNDARY_SCRATCH_CAP and c > 1:  # too many pairs to sort at once: halve the chunk
                work.extend([(b0 + c // 2, c - c // 2), (b0, c // 2)])
                continue
            scratch = torch.empty(sbytes, dtype=torch.uint8, device=dev)
            _lib.check(L.fslic_b200_boundary3d_stats_batch(
                dev.index, c, D, H, W, K, C, connectivity, lab[b0].data_ptr(), val[b0].data_ptr(), voxels, pairs,
                select.data_ptr(), nbytes, b0, B * K, E, ei[0].data_ptr(), ei[1].data_ptr(), first,
                out.mean.data_ptr(), out.min.data_ptr(), out.max.data_ptr(), out.count.data_ptr(), scratch.data_ptr(),
                sbytes, stream))
            first = 0
    return out


def knn_chunk(B, K, D, k, symmetric):
    """Images per kNN launch: as many as fit KNN_SCRATCH_CAP, at least one."""
    f = _lib.lib().fslic_b200_knn_scratch_bytes
    return chunk(lambda c: f(c, K, D, k, int(symmetric)), KNN_SCRATCH_CAP, B)


def knn_graph(points, k, present=None, symmetric=False):
    """k-nearest-neighbour graph of feature points -> KnnGraph(indptr, edge_index, distance).

    points is a cuda float32 [B,K,D] tensor (read detached; a non-contiguous one is made contiguous once); node
    n = b*K + i is row i of image b and each image is a graph of its own (the block-diagonal numbering of
    region_adjacency).  present is an optional cuda bool [B,K] on the same device (such as region_properties(...).area
    > 0); None means every node.  A node is a candidate when it is present and all D coordinates are finite: a node with
    NaN or +-inf coordinates gets no edges and is no one's neighbour, without raising.
    - s(i, j), the squared Euclidean distance in float32: t_c = p_i[c] - p_j[c], s = +0.0, s = s + t_c * t_c for
      c = 0 .. D-1, each operation rounded to nearest on its own (no FMA).  s(i, j) and s(j, i) are the same bits, s is
      never NaN or -0.0 and is +inf where coordinates are huge; numpy float32 operations in that order give the same.
    - Node i's neighbours are the first min(k, P_b - 1) other candidates of its image in the order of (s, j), j the
      local index (ties go to the lower index), P_b being the image's candidate count.  No self loops.
    - symmetric=False: the directed edges (i -> j), j among i's neighbours.  symmetric=True: those and their reverses,
      each (source, target) once, which is what PyG's to_undirected makes of the directed graph.
    Output:
    - indptr     int64 [B*K + 1]: CSR row offsets; rows of non-candidates are empty.
    - edge_index int64 [2, E]: (source, target) in global node ids, sorted by source then target, so edge_index[1] is
      the CSR column array, as in RegionGraph.  Source i -> target j means j is among i's nearest: for PyG's
      flow="source_to_target" message passing (messages from neighbours to i), pass edge_index.flip(0).
    - distance   float32 [E]: s of each edge.
    No edge crosses images.  1 <= K <= 65534, 1 <= D <= 64, 1 <= k <= 32 (an int, not a bool) and B*K <= 2^30;
    anything else, or points / present of the wrong type, dtype, shape or device, raises ValueError before any device
    work.  B = 0 gives zero indptr and E = 0.

    Work runs on the points' device, on its current stream.  E is data-dependent, so, like region_adjacency, the call
    reads the edge total back once per chunk of images (KNN_SCRATCH_CAP); it cannot be captured in a CUDA graph and
    raises RuntimeError under capture, before any device work.  The result is exact and the same across runs, batch
    order, chunking and streams: image b's rows depend only on points[b] and present[b]."""
    tensor("points", points, torch.float32, 3)
    B, K, D = (int(v) for v in points.shape)
    K = check_K(K)
    check_int("D", D, 1, KNN_MAX_D)
    if B * K > KNN_MAX_NODES:
        raise ValueError("%d images of K = %d are %d nodes, more than %d: split the batch" % (B, K, B * K, KNN_MAX_NODES))
    if isinstance(k, (bool, np.bool_)):
        raise ValueError("k must be an int, got %r" % (k,))
    k = check_int("k", k, 1, KNN_MAX_NEIGHBORS)
    symmetric = bool(symmetric)
    named = []
    if present is not None:
        tensor("present", present, torch.bool, 2)
        if tuple(int(v) for v in present.shape) != (B, K):
            raise ValueError("present %s do not match points %s" % (tuple(present.shape), (B, K, D)))
        named.append(("present", present))
    for name, x in named:
        if x.device != points.device:
            raise ValueError("%s is on %s, points on %s" % (name, x.device, points.device))
    if points.device.type != "cuda":
        raise ValueError("points is a %s tensor: pass cuda tensors (torch.from_numpy(...).cuda())" % points.device.type)
    dev = points.device
    with torch.cuda.device(dev):
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError("knn_graph reads its edge count back to the host and cannot be captured in a CUDA graph")
        indptr = torch.zeros(B * K + 1, dtype=torch.int64, device=dev)
        if B == 0:
            return KnnGraph(indptr, torch.empty((2, 0), dtype=torch.int64, device=dev),
                            torch.empty(0, dtype=torch.float32, device=dev))
        pts = points.detach().contiguous()
        pres = present.detach().contiguous().view(torch.uint8) if present is not None else None
        L = _lib.lib()
        stream = torch.cuda.current_stream(dev).cuda_stream
        c = knn_chunk(B, K, D, k, symmetric)
        nbytes = int(L.fslic_b200_knn_scratch_bytes(c, K, D, k, int(symmetric)))
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        total = torch.empty(1, dtype=torch.int64, device=dev)
        pieces, edges = [], 0
        for b0 in range(0, B, c):
            n = min(c, B - b0)
            _lib.check(L.fslic_b200_knn_count(dev.index, n, K, D, k, int(symmetric), pts[b0].data_ptr(),
                                              None if pres is None else pres[b0].data_ptr(), edges,
                                              indptr[b0 * K:].data_ptr(), total.data_ptr(), scratch.data_ptr(), nbytes,
                                              stream))
            e = int(total.item())  # the host wait: the chunk's edge total
            edge_index = torch.empty((2, e), dtype=torch.int64, device=dev)
            distance = torch.empty(e, dtype=torch.float32, device=dev)
            _lib.check(L.fslic_b200_knn_fill(dev.index, n, K, D, k, int(symmetric), b0 * K, e, scratch.data_ptr(),
                                             nbytes, edge_index[0].data_ptr(), edge_index[1].data_ptr(),
                                             distance.data_ptr(), stream))
            pieces.append((edge_index, distance))
            edges += e
        if len(pieces) == 1:
            edge_index, distance = pieces[0]
        else:
            edge_index = torch.cat([p[0] for p in pieces], dim=1)
            distance = torch.cat([p[1] for p in pieces])
    return KnnGraph(indptr, edge_index, distance)
