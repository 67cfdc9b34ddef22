"""Superpixel merging on the GPU (fast_slic_b200.merging) against the numpy restatement (merge_cases.py), exactly, with
dtype, shape and device: 720p SLIC maps at K = 1600 and B = 32 with pooled-colour weights, boundary-length weights
with heavy ties, all-equal weights, NaN / inf / -0.0 weights, garbage in the reverse entries, noise at K = 65534, a
2160p image, K = 1, absent and foreign labels, empty shapes and hand-built graphs; invariance to batch order, batch
splitting, streams and runs, non-contiguous inputs, CUDA graph capture, and composition with pool."""
import types

import numpy as np
import pytest
import torch

from cases import make_image
from merge_cases import ref_forest, ref_merge, ref_present

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _needs_cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _np(x):
    return x.detach().cpu().numpy()


def _cuda(x):
    return x if isinstance(x, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _same(a, b):
    return all(torch.equal(x, y) for x, y in zip(a, b))


class Case:
    """A label batch, its graph and weights, and the restatement's forest (computed once per case)."""

    def __init__(self, labels, K, graph, weights):
        self.labels, self.K, self.graph, self.weights = _cuda(labels), K, graph, _cuda(weights)
        self.lab_np = _np(self.labels)
        ei = graph.edge_index
        self.src, self.dst, self.w = _np(ei[0]), _np(ei[1]), _np(self.weights)
        self.present = ref_present(self.lab_np, K)
        self.forest = ref_forest(self.present, self.src, self.dst, self.w)

    def check(self, **cut):
        """merge_regions against the restatement, exactly; returns the device result."""
        from fast_slic_b200.merging import merge_regions
        m = merge_regions(self.labels, self.K, self.graph, self.weights, **cut)
        want = ref_merge(self.lab_np, self.K, self.src, self.dst, self.w, forest=self.forest, **cut)
        B, H, W = self.labels.shape
        for x, dtype, shape, ref, name in zip(m, (torch.int16, torch.int32, torch.int32),
                                              ((B, H, W), (B, self.K), (B,)), want, m._fields):
            assert x.dtype == dtype and tuple(x.shape) == shape and x.device == self.labels.device, name
            got = _np(x)
            assert np.array_equal(got, ref), (name, cut, np.argwhere(got != ref)[:5])
        return m


def _graph(labels, K):
    from fast_slic_b200.region_graph import region_adjacency
    return region_adjacency(labels, K)


def _colour_weights(features, labels, K, g):
    from fast_slic_b200.pooling import pool
    C = features.shape[1]
    x = pool(features, labels, K).transpose(1, 2).reshape(-1, C)
    return (x[g.edge_index[0]] - x[g.edge_index[1]]).norm(dim=1)


@pytest.fixture(scope="module")
def slic32():
    from fast_slic_b200 import Slic
    imgs = np.stack([make_image("syn", 720, 1280, seed=40 + b) for b in range(32)])
    images = torch.from_numpy(imgs).cuda()
    labels, clusters = Slic(num_components=1600, min_size_factor=0.25).iterate_batch(images, return_clusters=True)
    K = int(clusters.shape[1])
    features = images.permute(0, 3, 1, 2).float().contiguous()
    g = _graph(labels, K)
    return types.SimpleNamespace(labels=labels, K=K, features=features, graph=g,
                                 case=Case(labels, K, g, _colour_weights(features, labels, K, g)))


def test_slic_maps_threshold(slic32):
    c = slic32.case
    q = np.quantile(c.w, [0.1, 0.5, 0.9]).tolist()
    for t in [-1.0, 0.0, float(c.w.min()), *q, float(np.nextafter(np.float32(q[1]), np.float32(np.inf))), 1e30,
              float("inf")]:
        c.check(threshold=t)


def test_slic_maps_num_regions(slic32):
    c = slic32.case
    for R in (1, 2, 200, c.K - 1, c.K, c.K + 1, 10 ** 9):
        m = c.check(num_regions=R)
        if R == 200:
            assert (m.num_regions == 200).all()  # every SLIC map is one connected component


def test_composition(slic32):
    from fast_slic_b200.pooling import pool
    c = slic32.case
    m = c.check(num_regions=200)
    for b in range(0, 32, 7):
        vals = torch.unique(m.labels[b].long())
        assert int((vals >= 0).sum()) == int(m.num_regions[b])
    ones = torch.ones((32, 1) + tuple(c.labels.shape[1:]), dtype=torch.float32, device="cuda")
    _, counts = pool(ones, c.labels, c.K, return_counts=True)
    _, merged = pool(ones, m.labels, c.K, return_counts=True)
    want = torch.zeros_like(counts).scatter_add_(1, m.region.clamp(min=0).long(), counts * (m.region >= 0))
    assert torch.equal(merged, want)
    # the merged map feeds region_adjacency: a coarse graph with at most num_regions nodes per image
    g2 = _graph(m.labels, c.K)
    assert int(g2.edge_index.max()) < 32 * c.K
    assert bool(((g2.edge_index[0] % c.K) < int(m.num_regions.max())).all())


def test_boundary_weights_with_ties(slic32):
    labels = slic32.labels[:8]
    g = _graph(labels, slic32.K)
    c = Case(labels, slic32.K, g, g.boundary.float())
    for kw in ({"threshold": 3.0}, {"threshold": 20.0}, {"num_regions": 1}, {"num_regions": 50}, {"num_regions": 400}):
        c.check(**kw)
    c = Case(labels, slic32.K, g, torch.ones(g.edge_index.shape[1], device="cuda"))  # all equal
    for kw in ({"threshold": 1.0}, {"threshold": 1.5}, {"num_regions": 3}, {"num_regions": 800}):
        c.check(**kw)


def test_special_weights(slic32):
    labels = slic32.labels[:6]
    g = _graph(labels, slic32.K)
    rng = np.random.RandomState(7)
    vals = np.array([np.nan, np.inf, -np.inf, -0.0, 0.0, 1.0, -1.0, 2.5], np.float32)
    c = Case(labels, slic32.K, g, vals[rng.randint(0, len(vals), g.edge_index.shape[1])])
    for kw in ({"threshold": 0.0}, {"threshold": 1e-45}, {"threshold": 2.0}, {"threshold": float("inf")},
               {"threshold": -float("inf")}, {"num_regions": 1}, {"num_regions": 100}, {"num_regions": 1000}):
        c.check(**kw)


def test_reverse_entries_are_never_read(slic32):
    from fast_slic_b200.merging import merge_regions
    c = slic32.case
    ei = c.graph.edge_index
    garbage = c.weights.clone()
    rev = ei[0] > ei[1]
    rng = torch.Generator(device="cuda").manual_seed(3)
    noise = torch.randn(int(rev.sum()), device="cuda", generator=rng) * 1e6
    noise[::5] = float("nan")
    garbage[rev] = noise
    for kw in ({"threshold": float(np.median(c.w))}, {"num_regions": 200}):
        assert _same(merge_regions(c.labels, c.K, c.graph, garbage, **kw),
                     merge_regions(c.labels, c.K, c.graph, c.weights, **kw))


def test_noise_at_max_K():
    rng = np.random.RandomState(6)
    labels = rng.randint(0, 65536, (2, 192, 256)).astype(np.uint16).view(np.int16)  # 65534, 65535: no node
    K = 65534
    g = _graph(_cuda(labels), K)
    c = Case(labels, K, g, rng.rand(g.edge_index.shape[1]).astype(np.float32))
    for kw in ({"threshold": 0.3}, {"threshold": 2.0}, {"num_regions": 1}, {"num_regions": 30000}):
        c.check(**kw)


def test_2160p_image():
    H, W = 2160, 3840
    yy, xx = np.mgrid[:H, :W]
    labels = ((yy // 45) * 86 + (xx + yy // 3) // 45 % 86).astype(np.int16)[None]
    labels[:, :40, ::3] = -1
    K = 48 * 86
    lab = _cuda(labels)
    g = _graph(lab, K)
    img = torch.from_numpy(make_image("tiled", H, W, seed=5)).cuda().permute(2, 0, 1)[None].float().contiguous()
    c = Case(labels, K, g, _colour_weights(img, lab, K, g))
    for kw in ({"threshold": float(np.median(c.w))}, {"num_regions": 1}, {"num_regions": 300}):
        c.check(**kw)


def test_small_and_foreign_labels():
    rng = np.random.RandomState(11)
    # K = 1
    lab = rng.randint(-1, 3, (3, 5, 6)).astype(np.int16)
    c = Case(lab, 1, _graph(_cuda(lab), 1), np.zeros(0, np.float32))
    c.check(threshold=1.0)
    c.check(num_regions=1)
    # absent labels, -1 and labels >= K
    for K in (7, 20, 300):
        lab = rng.randint(-1, K + 3, (4, 17, 23)).astype(np.int16)
        lab[lab == 3] = 4
        lab[2] = -1  # an image with no superpixel pixel
        g = _graph(_cuda(lab), K)
        c = Case(lab, K, g, rng.rand(g.edge_index.shape[1]).astype(np.float32))
        for kw in ({"threshold": 0.5}, {"num_regions": 1}, {"num_regions": 3}, {"num_regions": K}):
            c.check(**kw)


def test_empty_shapes():
    from fast_slic_b200.merging import merge_regions
    for B, H, W in ((0, 5, 6), (2, 0, 6), (2, 5, 0)):
        lab = torch.zeros((B, H, W), dtype=torch.int16, device="cuda")
        g = _graph(lab, 7)
        for kw in ({"threshold": 1.0}, {"num_regions": 2}):
            m = merge_regions(lab, 7, g, torch.zeros(0, device="cuda"), **kw)
            assert tuple(m.labels.shape) == (B, H, W) and m.labels.dtype == torch.int16
            assert tuple(m.region.shape) == (B, 7) and bool((m.region == -1).all())
            assert tuple(m.num_regions.shape) == (B,) and not m.num_regions.any()
    # E = 0: every present label its own region
    lab = np.array([[[0, 4, 4], [2, 2, 9]]], np.int16)
    g = types.SimpleNamespace(indptr=torch.zeros(6, dtype=torch.int64, device="cuda"),
                              edge_index=torch.zeros((2, 0), dtype=torch.int64, device="cuda"))
    c = Case(lab, 5, g, np.zeros(0, np.float32))
    m = c.check(num_regions=1)
    assert m.region.tolist() == [[0, -1, 1, -1, 2]] and m.num_regions.tolist() == [3]
    c.check(threshold=float("inf"))


def test_hand_built_graph():
    rng = np.random.RandomState(13)
    B, K = 5, 40
    lab = rng.randint(0, K, (B, 12, 14)).astype(np.int16)
    lab[lab == 7] = 8
    E = 4000
    src = rng.randint(-10, B * K + 10, E).astype(np.int64)
    dst = src + rng.randint(-60, 60, E)
    src[:5] = [-(2 ** 62), 2 ** 62, 0, B * K - 1, 39]
    dst[:5] = [3, 2 ** 62 + 1, B * K, B * K, 40]  # out of range, out of range, dst = B*K, cross-image
    w = rng.rand(E).astype(np.float32)
    w[rng.rand(E) < 0.05] = np.nan
    g = types.SimpleNamespace(indptr=torch.zeros(B * K + 1, dtype=torch.int64, device="cuda"),
                              edge_index=torch.from_numpy(np.stack([src, dst])).cuda())
    c = Case(lab, K, g, w)
    for kw in ({"threshold": 0.2}, {"threshold": 0.9}, {"num_regions": 1}, {"num_regions": 5}, {"num_regions": 30}):
        c.check(**kw)


def test_batch_stream_and_run_invariance(slic32):
    from fast_slic_b200.merging import merge_regions
    labels, K, feat = slic32.labels[:6], slic32.K, slic32.features[:6]

    def run(idx, **kw):
        lab = labels[idx]
        g = _graph(lab, K)
        return merge_regions(lab, K, g, _colour_weights(feat[idx], lab, K, g), **kw)

    for kw in ({"threshold": 12.0}, {"num_regions": 150}):
        everything = torch.arange(6, device="cuda")
        full = run(everything, **kw)
        assert _same(run(everything, **kw), full)  # a second run
        idx = torch.tensor([4, 1, 5, 0, 3, 2], device="cuda")
        perm = run(idx, **kw)
        assert _same(perm, [x[idx] for x in full])
        for part in (torch.arange(0, 2, device="cuda"), torch.arange(2, 6, device="cuda")):
            assert _same(run(part, **kw), [x[part] for x in full])
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            on_s = run(everything, **kw)
        s.synchronize()
        assert _same(on_s, full)


def test_non_contiguous_inputs(slic32):
    from fast_slic_b200.merging import merge_regions
    labels, K = slic32.labels[:3], slic32.K
    lab_t = labels.transpose(1, 2)
    assert not lab_t.is_contiguous()
    g = _graph(lab_t, K)
    w = _colour_weights(slic32.features[:3].transpose(2, 3), lab_t, K, g)
    ei_nc = g.edge_index.t().contiguous().t()
    w_nc = torch.stack([w, -w], 1)[:, 0]
    assert not ei_nc.is_contiguous() and not w_nc.is_contiguous()
    g_nc = types.SimpleNamespace(indptr=g.indptr, edge_index=ei_nc)
    for kw in ({"threshold": 10.0}, {"num_regions": 100}):
        want = merge_regions(lab_t.contiguous(), K, g, w, **kw)
        assert _same(merge_regions(lab_t, K, g_nc, w_nc, **kw), want)
    Case(lab_t, K, g, w).check(num_regions=100)


def test_cuda_graph_capture(slic32):
    from fast_slic_b200.merging import merge_regions
    c = slic32.case
    lab, w = c.labels.clone(), c.weights.clone()
    for kw in ({"threshold": float(np.median(c.w))}, {"num_regions": 200}):
        want = merge_regions(lab, c.K, c.graph, w, **kw)
        torch.cuda.synchronize()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            merge_regions(lab, c.K, c.graph, w, **kw)  # warm-up on the capture stream
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            got = merge_regions(lab, c.K, c.graph, w, **kw)
        graph.replay()
        torch.cuda.synchronize()
        assert _same(got, want)
        w.copy_(torch.flip(c.weights, [0]))  # new weights in place, one more replay
        graph.replay()
        torch.cuda.synchronize()
        assert _same(got, merge_regions(lab, c.K, c.graph, w, **kw))
        w.copy_(c.weights)
