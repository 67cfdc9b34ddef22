"""Message passing over superpixel graphs on the GPU (csrc/message_passing.cuh): the building blocks of the standard
superpixel GNN layers -- GCN and GraphSAGE (sum / mean / max aggregation), GIN, GAT (edge softmax) and GatedGCN
(per-channel edge gates) -- over the graphs region_adjacency and knn_graph build::

    g = region_adjacency(labels, K)                         # or knn_graph(...): any indptr / edge_index pair
    h = x @ W                                               # [N,C] node features, N = B*K
    s = edge_gather(h @ a_src, g, "source") + edge_gather(h @ a_dst, g, "target")   # [E,H] GAT scores
    alpha = edge_softmax(torch.nn.functional.leaky_relu(s, 0.2), g)                  # over each node's entries
    out = aggregate(h, g, alpha, reduce="sum")              # [N,C]: sum over entries of alpha[e,h] * h[t_e]

A graph is any object with indptr int64 [N+1] (CSR offsets) and edge_index int64 [2,E]: the row of entry e is the node
n with indptr[n] <= e < indptr[n+1], its target t_e = edge_index[1, e]; edge_index[0] is not read.  indptr must be a
CSR offset array, as the builders return it; for any other the results are unspecified, but every device read stays in
bounds.  An entry whose target is outside [0, N) is no edge: it takes part in no sum, maximum or softmax and receives no
gradient.

The results and gradients are exact and deterministic (DESIGN.md section 4.21 gives every float32 operation and its
order): sums over a node's entries, or over the entries that target it, run in increasing entry order; no float
atomics.  So with graphs whose images are blocks of nodes, as the builders make them, image b's bits depend only on
image b's graph and rows.  Cuda float32 tensors only; non-contiguous inputs are made contiguous once.  Work runs on the
inputs' device on its current torch stream with no host synchronisation and no read-back, so a CUDA graph can capture
it; every argument is checked (ValueError) before any device work.  Each function is a first-order autograd Function.
"""
import torch
from torch.autograd.function import once_differentiable

from . import _lib
from ._labelmaps import tensor

MAX_ITEMS = 2 ** 31 - 1  # N and E
ENDS = ("target", "source")
REDUCES = ("sum", "mean", "max")


def _graph(graph, N=None):
    """(indptr, edge_index, N, E) of a graph object: indptr int64 [N+1] (N + 1 = x's rows + 1 when N is given),
    edge_index int64 [2,E], N and E at most 2^31 - 1."""
    indptr, edge_index = getattr(graph, "indptr", None), getattr(graph, "edge_index", None)
    tensor("graph.indptr", indptr, torch.int64, 1)
    tensor("graph.edge_index", edge_index, torch.int64, 2)
    if int(edge_index.shape[0]) != 2:
        raise ValueError("graph.edge_index must be int64 [2,E], got %s" % (tuple(edge_index.shape),))
    n = int(indptr.numel()) - 1
    if n < 0:
        raise ValueError("graph.indptr needs N + 1 >= 1 entries")
    if N is not None and n != N:
        raise ValueError("graph.indptr must have N + 1 = %d entries (x has N = %d rows), got %d" % (N + 1, N, n + 1))
    E = int(edge_index.shape[1])
    if n > MAX_ITEMS or E > MAX_ITEMS:
        raise ValueError("N and E must be below 2^31, got N = %d, E = %d" % (n, E))
    return indptr, edge_index, n, E


def _device(first, *named):
    """Every (name, tensor) of named on first's device, which must be a cuda device; returns it."""
    name0, x0 = first
    for name, x in named:
        if x is not None and x.device != x0.device:
            raise ValueError("%s is on %s, %s on %s" % (name, x.device, name0, x0.device))
    if x0.device.type != "cuda":
        raise ValueError("%s is a %s tensor: pass cuda tensors (torch.from_numpy(...).cuda())" % (name0, x0.device.type))
    return x0.device


def _heads(name, w, E):
    """float32 w [E] or [E,H] -> H."""
    if not isinstance(w, torch.Tensor) or w.dtype != torch.float32 or w.dim() not in (1, 2):
        raise ValueError("%s must be a float32 tensor [E] or [E,H], got %s" % (
            name, "%s %s" % (w.dtype, tuple(w.shape)) if isinstance(w, torch.Tensor) else type(w).__name__))
    if int(w.shape[0]) != E or (w.dim() == 2 and int(w.shape[1]) < 1):
        raise ValueError("%s must be [E] or [E,H] with E = %d and H >= 1, got %s" % (name, E, tuple(w.shape)))
    return 1 if w.dim() == 1 else int(w.shape[1])


def _nodes(x):
    tensor("x", x, torch.float32, 2)
    N, C = (int(v) for v in x.shape)
    if C < 1:
        raise ValueError("x needs at least one channel")
    return N, C


def _ptr(x):
    return None if x is None else x.data_ptr()


def _call(name, dev, *args):
    with torch.cuda.device(dev):
        _lib.check(getattr(_lib.lib(), "fslic_b200_" + name)(
            dev.index, *[a.data_ptr() if isinstance(a, torch.Tensor) else a for a in args],
            torch.cuda.current_stream(dev).cuda_stream))


def _scratch(nbytes, dev):
    return torch.empty(int(nbytes), dtype=torch.uint8, device=dev)


class _EdgeGather(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, indptr, targets, end):
        N, C = (int(v) for v in x.shape)
        E = int(targets.numel())
        out = torch.empty((E, C), dtype=torch.float32, device=x.device)
        _call("mp_gather", x.device, N, E, C, end, indptr, targets, x, out)
        ctx.save_for_backward(indptr, targets)
        ctx.N, ctx.end = N, end
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad):
        indptr, targets = ctx.saved_tensors
        N, E, C, dev = ctx.N, int(targets.numel()), int(grad.shape[1]), grad.device
        gx = torch.empty((N, C), dtype=torch.float32, device=dev)
        # the transposed order ("target") needs scratch; the row sums ("source") do not
        nbytes = _lib.lib().fslic_b200_mp_gather_backward_scratch_bytes(N, E) if ctx.end == 0 else 0
        _call("mp_gather_backward", dev, N, E, C, ctx.end, indptr, targets, grad.contiguous(), gx,
              _scratch(nbytes, dev) if nbytes else None, nbytes)
        return gx, None, None, None


class _EdgeSoftmax(torch.autograd.Function):
    @staticmethod
    def forward(ctx, scores, indptr, targets, N):
        E, H = int(scores.shape[0]), 1 if scores.dim() == 1 else int(scores.shape[1])
        out = torch.empty_like(scores)
        _call("mp_softmax", scores.device, N, E, H, indptr, targets, scores, out)
        ctx.save_for_backward(indptr, targets, out)
        ctx.N, ctx.H = N, H
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad):
        indptr, targets, out = ctx.saved_tensors
        gs = torch.empty_like(out)
        _call("mp_softmax_backward", out.device, ctx.N, int(out.shape[0]), ctx.H, indptr, targets, out,
              grad.contiguous(), gs)
        return gs, None, None, None


class _Aggregate(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, indptr, targets, reduce):
        N, C = (int(v) for v in x.shape)
        E = int(targets.numel())
        H = 1 if weight is None or weight.dim() == 1 else int(weight.shape[1])
        dev = x.device
        out = torch.empty((N, C), dtype=torch.float32, device=dev)
        deg = torch.empty(N, dtype=torch.int32, device=dev) if reduce == 1 else None
        amax = torch.empty((N, C), dtype=torch.int32, device=dev) if reduce == 2 else None
        _call("mp_aggregate", dev, N, E, C, H, reduce, indptr, targets, x, _ptr(weight), out, _ptr(deg), _ptr(amax))
        ctx.save_for_backward(x, weight, indptr, targets, deg, amax)
        ctx.reduce, ctx.H = reduce, H
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad):
        x, weight, indptr, targets, deg, amax = ctx.saved_tensors
        N, C = (int(v) for v in x.shape)
        E = int(targets.numel())
        dev = x.device
        need_x, need_w = ctx.needs_input_grad[:2]
        need_w = need_w and weight is not None
        gx = torch.empty((N, C), dtype=torch.float32, device=dev) if need_x else None
        gw = torch.empty_like(weight) if need_w else None
        if need_x or need_w:
            nbytes = _lib.lib().fslic_b200_mp_aggregate_backward_scratch_bytes(N, E, C, ctx.reduce)
            scratch = _scratch(nbytes, dev)
            _call("mp_aggregate_backward", dev, N, E, C, ctx.H, ctx.reduce, indptr, targets, x, _ptr(weight),
                  _ptr(deg), _ptr(amax), grad.contiguous(), _ptr(gx), _ptr(gw), scratch, nbytes)
        return gx, gw, None, None, None


def edge_gather(x, graph, end="target"):
    """float32 x [N,C] -> float32 [E,C]: row e is x[t_e] (end="target") or x[row(e)] (end="source"), +0.0 for an entry
    whose target is outside [0, N).  Differentiable in x: the gradient of node n sums grad rows in increasing e over
    the entries that target n ("target") or over n's own entries ("source")."""
    if end not in ENDS:
        raise ValueError("end must be 'target' or 'source', got %r" % (end,))
    N, C = _nodes(x)
    indptr, edge_index, N, E = _graph(graph, N)
    dev = _device(("x", x), ("graph.indptr", indptr), ("graph.edge_index", edge_index))
    with torch.cuda.device(dev):
        targets = edge_index.contiguous()[1]
        return _EdgeGather.apply(x.contiguous(), indptr.contiguous(), targets, ENDS.index(end))


def edge_softmax(scores, graph):
    """float32 scores [E] or [E,H] -> the same shape: per node and head, the softmax over the node's entries.
    m = the maximum (a NaN wins; otherwise -0.0 < +0.0), y_e = expf(s_e - m) (glibc's), Z = the sum of y_e in increasing
    e from +0.0, out_e = y_e / Z; a row that is all -inf gives NaN, as torch.softmax does; +0.0 for an entry whose
    target is outside [0, N).  Differentiable in scores: grad_e = out_e * (g_e - sum_e' out_e' * g_e')."""
    indptr, edge_index, N, E = _graph(graph)
    _heads("scores", scores, E)
    dev = _device(("scores", scores), ("graph.indptr", indptr), ("graph.edge_index", edge_index))
    with torch.cuda.device(dev):
        targets = edge_index.contiguous()[1]
        return _EdgeSoftmax.apply(scores.contiguous(), indptr.contiguous(), targets, N)


def aggregate(x, graph, weight=None, reduce="sum"):
    """float32 x [N,C] -> float32 [N,C]: per node n and channel c, the reduction over n's entries e of the terms
    weight[e,h] * x[t_e, c] (one rounded product; x[t_e, c] itself without a weight), h = c // (C / H) for a weight
    [E] or [E,H] (H divides C; H = C gives per-channel gates).  reduce="sum": the terms added in increasing e from +0.0;
    "mean": that sum / (float)deg, deg the number of n's entries with a valid target; "max": the first maximal term
    (a NaN wins; otherwise -0.0 < +0.0).  A node without entries gives +0.0.  Differentiable in x and weight."""
    if reduce not in REDUCES:
        raise ValueError("reduce must be 'sum', 'mean' or 'max', got %r" % (reduce,))
    N, C = _nodes(x)
    indptr, edge_index, N, E = _graph(graph, N)
    if weight is not None:
        H = _heads("weight", weight, E)
        if C % H:
            raise ValueError("weight has H = %d heads, which does not divide C = %d" % (H, C))
    dev = _device(("x", x), ("graph.indptr", indptr), ("graph.edge_index", edge_index), ("weight", weight))
    with torch.cuda.device(dev):
        targets = edge_index.contiguous()[1]
        return _Aggregate.apply(x.contiguous(), None if weight is None else weight.contiguous(), indptr.contiguous(),
                                targets, REDUCES.index(reduce))


__all__ = ["aggregate", "edge_gather", "edge_softmax"]
