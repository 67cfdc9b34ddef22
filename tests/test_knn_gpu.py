"""kNN graphs on the GPU (fast_slic_b200.region_graph.knn_graph) against the numpy restatement (knn_cases.py):
indptr and edge_index equal, distance the same bytes.  The 720p superpixel workload, ties, shape limits, odd values,
the present mask, invariance under batch order, chunking, streams, repeats and strides, empty batches, the refusal
under CUDA graph capture, and merging over the symmetric graph."""
import numpy as np
import pytest
import torch

from cases import make_image
from knn_cases import ref_knn, union
from merge_cases import ref_merge

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _needs_cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _np(x):
    return x.detach().cpu().numpy()


def _same(a, b):
    return (torch.equal(a.indptr, b.indptr) and torch.equal(a.edge_index, b.edge_index) and
            torch.equal(a.distance.view(torch.int32), b.distance.view(torch.int32)))


def _check(points, k, present=None, symmetric=False, ref=None):
    """knn_graph against the restatement (or a given one); returns the device result."""
    from fast_slic_b200.region_graph import knn_graph
    if not isinstance(points, torch.Tensor):
        points = torch.from_numpy(np.ascontiguousarray(points, np.float32)).cuda()
    if present is not None and not isinstance(present, torch.Tensor):
        present = torch.from_numpy(np.asarray(present, bool)).cuda()
    g = knn_graph(points, k, present, symmetric)
    B, K = int(points.shape[0]), int(points.shape[1])
    assert g.indptr.dtype == torch.int64 and tuple(g.indptr.shape) == (B * K + 1,)
    assert g.edge_index.dtype == torch.int64 and g.edge_index.shape[0] == 2
    assert g.distance.dtype == torch.float32 and g.distance.shape[0] == g.edge_index.shape[1]
    assert g.indptr.device == points.device and not g.distance.requires_grad
    if ref is None:
        ref = ref_knn(_np(points), k, None if present is None else _np(present), symmetric)
    assert np.array_equal(_np(g.indptr), ref[0])
    assert np.array_equal(_np(g.edge_index), ref[1])
    assert np.array_equal(_np(g.distance).view(np.uint32), ref[2].view(np.uint32))
    return g


@pytest.fixture(scope="module")
def hd_points():
    """README's node features of 32 1280x720 SLIC maps at K = 1600: pooled RGB means, normalised centroids and
    compactness, with present = area > 0."""
    from fast_slic_b200 import Slic
    from fast_slic_b200.geometry import region_properties
    from fast_slic_b200.pooling import pool
    B, H, W = 32, 720, 1280
    imgs = torch.from_numpy(np.stack([make_image("syn", H, W, seed=70 + b) for b in range(B)])).cuda()
    labels, clusters = Slic(num_components=1600).iterate_batch(imgs, return_clusters=True)
    K = int(clusters.shape[1])
    features = imgs.permute(0, 3, 1, 2).float().contiguous() / 255
    p = region_properties(labels, K)
    hw = torch.tensor([H, W], dtype=torch.float64, device="cuda")
    x = torch.cat([pool(features, labels, K).transpose(1, 2), (p.centroid / hw).float(),
                   (p.perimeter / p.area.clamp(min=1)).float()[..., None]], -1)
    return x.contiguous(), p.area > 0


@pytest.mark.parametrize("k", [1, 8, 32])
def test_hd_workload(hd_points, k):
    x, present = hd_points
    ref = ref_knn(_np(x), k, _np(present))
    _check(x, k, present, ref=ref)
    _check(x, k, present, True, ref=union(ref))


def test_ties_on_an_integer_grid():
    g = np.stack(np.meshgrid(np.arange(20), np.arange(30), indexing="ij"), -1).reshape(1, -1, 2).astype(np.float32)
    pts = np.concatenate([g, g[:, ::-1] * 2, np.round(g / 3)])  # several images, each with mass ties and duplicates
    for k in (1, 4, 8, 13, 32):
        for sym in (False, True):
            _check(pts, k, symmetric=sym)


@pytest.mark.parametrize("D", [1, 2, 3, 5, 8, 9, 17, 33, 64])
def test_dimensions(D):
    rng = np.random.RandomState(D)
    pts = rng.randn(3, 500, D).astype(np.float32)
    pts[1] = np.round(pts[1] * 2)  # ties
    for k in (1, 8, 9, 32):
        _check(pts, k, symmetric=k == 9)


def test_one_node_per_image_and_tiny_images():
    _check(np.zeros((4, 1, 3), np.float32), 8)
    _check(np.zeros((4, 1, 3), np.float32), 8, symmetric=True)
    rng = np.random.RandomState(1)
    for K in (2, 3, 31, 129, 130):
        pts = rng.rand(5, K, 2).astype(np.float32)
        _check(pts, 32)
        _check(pts, 5, symmetric=True)


def test_sparse_present_at_the_largest_K():
    rng = np.random.RandomState(2)
    K = 65534
    pts = rng.rand(2, K, 5).astype(np.float32)
    present = np.zeros((2, K), bool)
    present[0, rng.choice(K, 300, replace=False)] = True
    present[1, rng.choice(K, 17, replace=False)] = True
    present[1, [0, K - 1]] = True
    for k, sym in ((8, False), (32, True)):
        _check(pts, k, present, sym)


def test_one_large_image():
    rng = np.random.RandomState(4)
    pts = rng.rand(1, 8192, 3).astype(np.float32)
    ref = ref_knn(pts, 8)
    _check(pts, 8, ref=ref)
    _check(pts, 8, symmetric=True, ref=union(ref))


def test_non_finite_coordinates_and_infinite_distances():
    rng = np.random.RandomState(5)
    pts = rng.randn(3, 400, 4).astype(np.float32)
    pick = rng.rand(3, 400, 4)
    pts[pick < 0.01] = np.nan
    pts[(pick >= 0.01) & (pick < 0.02)] = np.inf
    pts[(pick >= 0.02) & (pick < 0.03)] = -np.inf
    pts[2, ::3] *= np.float32(2e38)  # differences overflow: +inf distances and ties among them
    pts[2, 1::3] *= np.float32(-2e38)
    for k in (1, 8, 32):
        for sym in (False, True):
            g = _check(pts, k, symmetric=sym)
    assert torch.isinf(g.distance).any()


def test_present_none_equals_all_true():
    from fast_slic_b200.region_graph import knn_graph
    x = torch.from_numpy(np.random.RandomState(6).rand(4, 300, 6).astype(np.float32)).cuda()
    for sym in (False, True):
        assert _same(knn_graph(x, 8, None, sym), knn_graph(x, 8, torch.ones(4, 300, dtype=torch.bool, device="cuda"),
                                                           sym))


def test_batch_order_chunks_streams_repeats_and_strides(hd_points, monkeypatch):
    from fast_slic_b200 import region_graph
    from fast_slic_b200.region_graph import knn_graph
    x, present = hd_points
    B, K, D = (int(v) for v in x.shape)
    for sym in (False, True):
        full = knn_graph(x, 8, present, sym)
        assert _same(knn_graph(x, 8, present, sym), full)  # a repeated run
        # reversed batch: image b's rows move to B - 1 - b, unchanged
        rev = knn_graph(x.flip(0), 8, present.flip(0), sym)
        for b in (0, 5, B - 1):
            lo, hi = int(full.indptr[b * K]), int(full.indptr[(b + 1) * K])
            r = B - 1 - b
            rlo, rhi = int(rev.indptr[r * K]), int(rev.indptr[(r + 1) * K])
            assert torch.equal(rev.edge_index[:, rlo:rhi] - r * K, full.edge_index[:, lo:hi] - b * K)
            assert torch.equal(rev.distance[rlo:rhi].view(torch.int32), full.distance[lo:hi].view(torch.int32))
            assert torch.equal(rev.indptr[r * K:(r + 1) * K + 1] - rlo, full.indptr[b * K:(b + 1) * K + 1] - lo)
        # chunks of 3 images
        with monkeypatch.context() as m:
            m.setattr(region_graph, "KNN_SCRATCH_CAP", 3 * region_graph._lib.lib().fslic_b200_knn_scratch_bytes(
                1, K, D, 8, int(sym)))
            assert region_graph.knn_chunk(B, K, D, 8, sym) == 3
            assert _same(knn_graph(x, 8, present, sym), full)
        # another stream
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            on_s = knn_graph(x, 8, present, sym)
        s.synchronize()
        assert _same(on_s, full)
        # a non-contiguous view of the points
        wide = torch.full((B, K, 2 * D), float("nan"), device="cuda")
        wide[:, :, ::2] = x
        assert _same(knn_graph(wide[:, :, ::2], 8, present, sym), full)
        assert _same(knn_graph(x.transpose(0, 1).contiguous().transpose(0, 1), 8, present, sym), full)


def test_empty_batch_and_capture():
    from fast_slic_b200.region_graph import knn_graph
    g = knn_graph(torch.zeros((0, 7, 3), device="cuda"), 4)
    assert g.indptr.tolist() == [0] and tuple(g.edge_index.shape) == (2, 0) and g.distance.shape == (0,)
    x = torch.rand(2, 50, 3, device="cuda")
    y = torch.zeros(4, device="cuda")
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y.add_(1)
        with pytest.raises(RuntimeError, match="CUDA graph"):
            knn_graph(x, 4)
    graph.replay()
    torch.cuda.synchronize()
    assert y.tolist() == [1.0] * 4
    _check(x, 4)  # the device is fine afterwards


def test_merging_over_the_symmetric_graph():
    """merge_regions with the kNN distances as weights, against the restatements of both."""
    from fast_slic_b200 import Slic
    from fast_slic_b200.geometry import region_properties
    from fast_slic_b200.merging import merge_regions
    from fast_slic_b200.pooling import pool
    B, H, W = 3, 240, 320
    imgs = torch.from_numpy(np.stack([make_image("syn", H, W, seed=90 + b) for b in range(B)])).cuda()
    labels, clusters = Slic(num_components=200).iterate_batch(imgs, return_clusters=True)
    K = int(clusters.shape[1])
    p = region_properties(labels, K)
    x = torch.cat([pool(imgs.permute(0, 3, 1, 2).float().contiguous() / 255, labels, K).transpose(1, 2),
                   (p.centroid / torch.tensor([H, W], dtype=torch.float64, device="cuda")).float()], -1)
    g = _check(x, 6, p.area > 0, True)
    ei, w = _np(g.edge_index), _np(g.distance)
    for kw in ({"threshold": float(np.median(w))}, {"num_regions": 20}):
        m = merge_regions(labels, K, g, g.distance, **kw)
        ref = ref_merge(_np(labels), K, ei[0], ei[1], w, **kw)
        for got, exp in zip(m, ref):
            assert np.array_equal(_np(got), exp), kw
