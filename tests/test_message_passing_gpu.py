"""Message passing over superpixel graphs on the GPU (fast_slic_b200.message_passing) against the numpy restatement
(message_passing_cases.py): every output and every gradient bit for bit (NaN as a class) on region adjacency graphs
and kNN graphs of SLIC label maps and on hand-made graphs (empty rows, self loops, duplicate entries, invalid targets,
a node with more than 5000 entries), C from 1 to 300 and H from 1 to C with NaN, +-inf and -0.0 inputs; per-image,
run, stream and CUDA graph invariance; and a two-step GAT training loop that is bit-reproducible across runs, with
node gradients bit-identical across batch splits."""
import numpy as np
import pytest
import torch

from cases import make_image
from message_passing_cases import F32, Graph, make_graph, nan_class_equal, special_values

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _needs_cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _np(x):
    return x.detach().cpu().numpy()


def _cuda(x, grad=False):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda().requires_grad_(grad)


def _bits(a, b):
    return len(a) == len(b) and all(torch.equal(x.view(torch.int32), y.view(torch.int32)) for x, y in zip(a, b))


class _G:
    def __init__(self, indptr, edge_index):
        self.indptr, self.edge_index = indptr, edge_index


def _dev_graph(indptr, t):
    t = np.asarray(t, np.int64)
    return _G(_cuda(np.asarray(indptr, np.int64)), _cuda(np.stack([np.zeros_like(t), t])))


def _run_all(dg, x, s, w, reduce, rng):
    """Every function and its gradients on the GPU -> dict of numpy arrays."""
    from fast_slic_b200.message_passing import aggregate, edge_gather, edge_softmax
    E, C = int(dg.edge_index.shape[1]), x.shape[1]
    gE, gN = rng.randn(E, C).astype(F32), rng.randn(x.shape[0], C).astype(F32)
    gS = rng.randn(*s.shape).astype(F32)
    r = {}
    for end in ("target", "source"):
        X = _cuda(x, True)
        y = edge_gather(X, dg, end)
        r["gather_" + end], = (_np(y),)
        r["ggather_" + end] = _np(torch.autograd.grad(y, X, _cuda(gE))[0])
    S = _cuda(s, True)
    y = edge_softmax(S, dg)
    r["softmax"], r["gsoftmax"] = _np(y), _np(torch.autograd.grad(y, S, _cuda(gS))[0])
    X, W = _cuda(x, True), None if w is None else _cuda(w, True)
    y = aggregate(X, dg, W, reduce)
    r["agg"] = _np(y)
    grads = torch.autograd.grad(y, (X,) if W is None else (X, W), _cuda(gN))
    r["gagg_x"] = _np(grads[0])
    if W is not None:
        r["gagg_w"] = _np(grads[1])
    return r, (gE, gN, gS)


def _check_graph(indptr, t, x, s, w, reduce, seed):
    """The GPU against the restatement for one graph and one set of inputs."""
    rng = np.random.RandomState(seed)
    got, (gE, gN, gS) = _run_all(_dev_graph(indptr, t), x, s, w, reduce, rng)
    g = Graph(indptr, t)
    s2 = s if s.ndim == 2 else s[:, None]
    for end in ("target", "source"):
        assert nan_class_equal(got["gather_" + end], g.gather(x, end)), end
        assert nan_class_equal(got["ggather_" + end], g.gather_backward(gE, end)), end
    sm = g.softmax(s2)
    assert nan_class_equal(got["softmax"].reshape(s2.shape), sm)
    assert nan_class_equal(got["gsoftmax"].reshape(s2.shape), g.softmax_backward(sm, gS.reshape(s2.shape)))
    w2 = None if w is None else (w if w.ndim == 2 else w[:, None])
    out, _, amax = g.aggregate(x, w2, reduce)
    assert nan_class_equal(got["agg"], out), reduce
    gx, gw = g.aggregate_backward(x, w2, gN, reduce, amax)
    assert nan_class_equal(got["gagg_x"], gx), reduce
    if w is not None:
        assert nan_class_equal(got["gagg_w"].reshape(w2.shape), gw), reduce
    return sm


# (seed, N, max_deg, invalid, self_loops, duplicates, big, C, H, weight rank, special values)
HAND = [
    (1, 50, 8, 0.1, 0.1, 0.1, None, 1, 1, 1, False),
    (2, 40, 12, 0.2, 0.2, 0.3, None, 7, 7, 2, True),        # per-channel gates
    (3, 30, 6, 0.0, 0.0, 0.0, None, 32, 4, 2, True),
    (4, 60, 16, 0.1, 0.1, 0.1, None, 129, 3, 2, True),      # more than one 128-channel pass, D = 43
    (5, 20, 4, 0.3, 0.0, 0.5, None, 300, 300, 2, False),
    (6, 25, 5, 0.1, 0.1, 0.1, None, 300, 1, 1, True),
    (7, 70, 8, 0.05, 0.05, 0.05, (3, 5200), 48, 16, 2, True),  # one node with 5200 entries
    (8, 40, 10, 0.1, 0.3, 0.1, (0, 40), 20, 5, 2, True),     # D = 4: 8 heads per warp pass
    (9, 1, 3, 0.5, 0.0, 0.0, None, 5, 1, 0, True),           # one node, no weight
    (10, 35, 9, 0.0, 0.1, 0.1, None, 64, 2, 0, False),
]


@pytest.mark.parametrize("case", HAND, ids=lambda c: "seed%d" % c[0])
def test_hand_made_graphs(case):
    seed, N, md, inv, sl, dup, big, C, H, wr, special = case
    indptr, t = make_graph(seed, N, md, inv, sl, dup, 0.15, big)
    rng = np.random.RandomState(seed)
    E = t.size
    mk = (lambda *sh: special_values(rng, sh)) if special else (lambda *sh: rng.randn(*sh).astype(F32))
    x = mk(N, C)
    s = mk(E, H) if H > 1 or wr == 2 else mk(E)
    w = None if wr == 0 else (mk(E, H) if wr == 2 else mk(E))
    for reduce in ("sum", "mean", "max"):
        _check_graph(indptr, t, x, s, w, reduce, seed)
    if big is not None:
        assert np.diff(indptr).max() > 5000 or big[1] < 5000


def test_channel_and_head_sweep():
    rng = np.random.RandomState(20)
    indptr, t = make_graph(20, 30, 9, 0.1, 0.1, 0.1)
    for C in (1, 2, 3, 16, 17, 31, 33, 100, 128, 257, 300):
        for H in sorted({1, 2, 3, C} & {h for h in range(1, C + 1) if C % h == 0}):
            x, w = special_values(rng, (30, C)), special_values(rng, (t.size, H))
            reduce = ("sum", "mean", "max")[(C + H) % 3]
            _check_graph(indptr, t, x, w, w, reduce, C * 1000 + H)


def test_softmax_special_rows():
    """All -inf rows give NaN as torch.softmax does; +inf and NaN scores; -0.0 and +0.0 ties; empty rows."""
    indptr = np.array([0, 3, 6, 6, 9, 11, 13], np.int64)
    t = np.array([0, 1, 2, 3, 4, 5, 0, 0, 1, 2, 9, 3, 4], np.int64)
    s = np.array([-np.inf, -np.inf, -np.inf, np.inf, 1, 2, -0.0, 0.0, -0.0, np.nan, 5, 1, 1], F32)
    sm = _check_graph(indptr, t, np.ones((6, 2), F32), s, s, "max", 30)
    assert np.isnan(sm[0:3]).all() and np.isnan(sm[3:6]).any()
    assert not np.isnan(sm[6:9]).any() and np.isnan(sm[9]) and sm[10] == 0
    from fast_slic_b200.message_passing import edge_softmax
    got = _np(edge_softmax(_cuda(s), _dev_graph(indptr, t)))
    want = torch.softmax(torch.from_numpy(s[:3]), 0).numpy()
    assert np.isnan(got[:3]).all() and np.isnan(want).all()


@pytest.fixture(scope="module")
def slic_graphs():
    """4 SLIC maps of 240x320 at K = 300: node features, RAGs at connectivity 4 and 8, directed and symmetric 8-NN
    graphs with absent nodes."""
    from fast_slic_b200 import Slic
    from fast_slic_b200.geometry import region_properties
    from fast_slic_b200.pooling import pool
    from fast_slic_b200.region_graph import knn_graph, region_adjacency
    B, H, W = 4, 240, 320
    imgs = torch.from_numpy(np.stack([make_image("syn", H, W, seed=90 + b) for b in range(B)])).cuda()
    labels, clusters = Slic(num_components=300).iterate_batch(imgs, return_clusters=True)
    K = int(clusters.shape[1])
    feats = pool(imgs.permute(0, 3, 1, 2).float().contiguous() / 255, labels, K).transpose(1, 2).contiguous()
    p = region_properties(labels, K)
    present = p.area > 0
    present[:, ::7] = False
    graphs = {"rag4": region_adjacency(labels, K, 4), "rag8": region_adjacency(labels, K, 8),
              "knn": knn_graph(feats, 8, present), "knn_sym": knn_graph(feats, 8, present, symmetric=True)}
    assert not bool(present.all())
    return B, K, feats, graphs


@pytest.mark.parametrize("name", ["rag4", "rag8", "knn", "knn_sym"])
def test_superpixel_graphs(slic_graphs, name):
    B, K, feats, graphs = slic_graphs
    g = graphs[name]
    indptr, t = _np(g.indptr), _np(g.edge_index[1])
    rng = np.random.RandomState(40)
    x = np.concatenate([_np(feats).reshape(B * K, -1), rng.randn(B * K, 5).astype(F32)], 1)  # C = 8
    s = rng.randn(t.size, 2).astype(F32)
    for reduce in ("sum", "mean", "max"):
        _check_graph(indptr, t, x, s, s, reduce, 41)
        _check_graph(indptr, t, x, s[:, 0], None, reduce, 42)


def _subgraph(g, b, K):
    """Image b's block of a batched graph, its nodes renumbered from 0."""
    lo, hi = int(g.indptr[b * K]), int(g.indptr[(b + 1) * K])
    ei = g.edge_index[:, lo:hi] - b * K
    return _G((g.indptr[b * K:(b + 1) * K + 1] - lo).contiguous(), ei.contiguous()), lo, hi


def _layer(x, g, p, reduce="sum"):
    """One GAT-style layer with per-channel attention (H = C) built from the three functions and elementwise torch
    only, so every node's bits depend on nothing but its graph block: [N,C] -> [N,C]."""
    from fast_slic_b200.message_passing import aggregate, edge_gather, edge_softmax
    h = x * p["w"] + p["b"]
    sc = edge_gather(h, g, "source") * p["a_s"] + edge_gather(h, g, "target") * p["a_t"]
    alpha = edge_softmax(torch.nn.functional.leaky_relu(sc, 0.2), g)
    return torch.relu(aggregate(h, g, alpha, reduce)) + aggregate(h, g, reduce="max")


def _params(C, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    return {k: (torch.randn(C, device="cuda", generator=gen) * 0.5).requires_grad_(True)
            for k in ("w", "b", "a_s", "a_t")}


def test_per_image_run_stream_and_graph_invariance(slic_graphs):
    B, K, feats, graphs = slic_graphs
    p = _params(feats.shape[2], 0)

    def run(x, g, grad=True):
        x = x.detach().clone().requires_grad_(grad)
        outs = [_layer(x, g, p, reduce) for reduce in ("sum", "mean", "max")]
        if grad:
            # the gradient of a sum of squares is 2 * out, elementwise: x.grad is per node too
            x.grad, = torch.autograd.grad([o.square().sum() for o in outs], x)
        return [o.detach() for o in outs] + ([x.grad] if grad else [])

    x = feats.reshape(B * K, -1).contiguous()
    for name in ("rag8", "knn_sym"):
        g = graphs[name]
        a = run(x, g)
        assert _bits(a, run(x, g))
        for b in range(B):
            sg, lo, hi = _subgraph(g, b, K)
            one = run(x[b * K:(b + 1) * K], sg)
            assert _bits([v[b * K:(b + 1) * K] for v in a], one), (name, b)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            c = run(x, g)
        s.synchronize()
        assert _bits(a, c)
        # the forward under CUDA graph capture
        xs = torch.zeros_like(x)
        torch.cuda.synchronize()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            run(xs, g, grad=False)
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            got = run(xs, g, grad=False)
        xs.copy_(x)
        graph.replay()
        torch.cuda.synchronize()
        assert _bits(a[:3], got), name


def test_backward_under_graph_capture(slic_graphs):
    """The backward passes (transposed sort included) captured in a CUDA graph and replayed."""
    B, K, feats, graphs = slic_graphs
    g = graphs["knn"]
    p = _params(feats.shape[2], 1)
    x = feats.reshape(B * K, -1).contiguous()

    def run(xx):
        xx = xx.detach().requires_grad_(True)
        outs = [_layer(xx, g, p, reduce) for reduce in ("sum", "mean", "max")]
        return torch.autograd.grad([o.square().sum() for o in outs], [xx] + list(p.values()))

    want = run(x)
    xs = torch.zeros_like(x)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        run(xs)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        got = run(xs)
    xs.copy_(x)
    graph.replay()
    torch.cuda.synchronize()
    assert _bits(want[:1], got[:1])
    for u, v in zip(want[1:], got[1:]):
        torch.testing.assert_close(u, v, rtol=0, atol=0)


def test_gat_training_is_reproducible_across_runs_and_batch_splits(slic_graphs):
    """Two SGD steps of a two-layer GAT over the batch, whole and split into per-image graphs and into halves.  Every
    gradient is bit-identical across two runs of the same split.  Across splits the node features' gradient of the
    first step is bit-identical per node (the layers are per node).  The parameter gradients are not compared across
    splits: they sum over the nodes with torch's reductions and over the parts with autograd's accumulation, whose
    orders depend on the split."""
    B, K, feats, graphs = slic_graphs
    x0 = feats.reshape(B * K, -1).contiguous()
    C = x0.shape[1]
    target = (torch.arange(B * K, device="cuda") % 3)
    head = torch.randn(C, 3, device="cuda", generator=torch.Generator(device="cuda").manual_seed(7))

    def train(parts):
        p1, p2 = _params(C, 2), _params(C, 3)
        params = list(p1.values()) + list(p2.values())
        opt = torch.optim.SGD(params, lr=0.05)
        grads, xgrad = [], None
        for step in range(2):
            opt.zero_grad()
            xg = []
            for g, lo, hi in parts:
                x = x0[lo:hi].clone().requires_grad_(True)
                h = _layer(_layer(x, g, p1), g, p2, "mean")
                logits = torch.cat([(h * head[:, k]).sum(1, keepdim=True) for k in range(3)], 1)
                loss = torch.nn.functional.cross_entropy(logits, target[lo:hi], reduction="sum")
                loss.backward()
                xg.append(x.grad)
            if step == 0:
                xgrad = torch.cat(xg)
            grads += [q.grad.clone() for q in params]
            opt.step()
        return grads, xgrad

    for name in ("rag4", "knn_sym"):
        g = graphs[name]
        a, xa = train([(g, 0, B * K)])
        b, xb = train([(g, 0, B * K)])
        assert _bits(a, b) and _bits([xa], [xb]), name
        assert all(torch.isfinite(t).all() and t.abs().sum() > 0 for t in a)
        halves = []
        for b0, b1 in ((0, B // 2), (B // 2, B)):
            lo, hi = int(g.indptr[b0 * K]), int(g.indptr[b1 * K])
            halves.append((_G((g.indptr[b0 * K:b1 * K + 1] - lo).contiguous(),
                              (g.edge_index[:, lo:hi] - b0 * K).contiguous()), b0 * K, b1 * K))
        singles = [(_subgraph(g, b, K)[0], b * K, (b + 1) * K) for b in range(B)]
        for parts in (halves, singles):
            u, xu = train(parts)
            v, xv = train(parts)
            assert _bits(u, v) and _bits([xu], [xv]), name
            assert _bits([xa], [xu]), name


def test_empty_inputs():
    from fast_slic_b200.message_passing import aggregate, edge_gather, edge_softmax
    g = _G(torch.zeros(4, dtype=torch.int64, device="cuda"), torch.zeros((2, 0), dtype=torch.int64, device="cuda"))
    x = torch.randn(3, 5, device="cuda", requires_grad=True)
    assert tuple(edge_gather(x, g).shape) == (0, 5)
    assert tuple(edge_softmax(torch.zeros(0, 2, device="cuda"), g).shape) == (0, 2)
    for reduce in ("sum", "mean", "max"):
        y = aggregate(x, g, reduce=reduce)
        assert not y.any() and not y.signbit().any()
        gx, = torch.autograd.grad(y.sum(), x)
        assert not gx.any()
    g0 = _G(torch.zeros(1, dtype=torch.int64, device="cuda"), torch.zeros((2, 0), dtype=torch.int64, device="cuda"))
    assert tuple(aggregate(torch.zeros(0, 4, device="cuda"), g0).shape) == (0, 4)
