"""Boundary statistics on the GPU (fast_slic_b200.region_graph.boundary_stats) against the numpy restatement
(boundary_cases.py): mean, min and max bit for bit (any NaN equal to any NaN), count exactly, on SLIC maps, adversarial
maps and values, hand-built graphs; batch, chunk and stream invariance; the host reads of one call; the refusal under
CUDA graph capture; and boundary-strength merging end to end."""
import json
import os
import tempfile

import numpy as np
import pytest
import torch

from boundary_cases import ref_boundary
from cases import make_image
from merge_cases import ref_merge
from pool_cases import nan_class_equal

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _needs_cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _np(x):
    return x.detach().cpu().numpy()


def _slic(H, W, K, B, msf, seed):
    from fast_slic_b200 import Slic
    imgs = torch.from_numpy(np.stack([make_image("syn", H, W, seed=seed + b) for b in range(B)])).cuda()
    labels, clusters = Slic(num_components=K, min_size_factor=msf).iterate_batch(imgs, return_clusters=True)
    return labels, int(clusters.shape[1])


def _values(shape, seed, special=False):
    rng = np.random.RandomState(seed)
    v = rng.randn(*shape).astype(np.float32)
    if special:
        pick = rng.rand(*shape)
        v[pick < 0.02] = np.nan
        v[(pick >= 0.02) & (pick < 0.04)] = np.inf
        v[(pick >= 0.04) & (pick < 0.06)] = -np.inf
        v[(pick >= 0.06) & (pick < 0.1)] = 0.0
        v[(pick >= 0.1) & (pick < 0.14)] = -0.0
    return v


def _graph(labels, K, connectivity):
    from fast_slic_b200.region_graph import region_adjacency
    return region_adjacency(labels, K, connectivity)


def _check(labels, K, graph, values, connectivity):
    """boundary_stats against the restatement; returns the device result."""
    from fast_slic_b200.region_graph import boundary_stats
    if not isinstance(labels, torch.Tensor):
        labels = torch.from_numpy(labels).cuda()
    if not isinstance(values, torch.Tensor):
        values = torch.from_numpy(values).cuda()
    s = boundary_stats(labels, K, graph, values, connectivity)
    E, C = int(graph.edge_index.shape[1]), int(values.shape[1])
    for x in s[:3]:
        assert x.dtype == torch.float32 and tuple(x.shape) == (E, C) and x.device == labels.device
        assert not x.requires_grad
    assert s.count.dtype == torch.int32 and tuple(s.count.shape) == (E,)
    ei = _np(graph.edge_index)
    want = ref_boundary(_np(labels), K, ei[0], ei[1], _np(values), connectivity)
    for name, got, ref in zip(("mean", "min", "max"), s[:3], want[:3]):
        assert nan_class_equal(_np(got), ref), name
    assert np.array_equal(_np(s.count), want[3])
    return s


def _same(a, b):
    return all(nan_class_equal(_np(x), _np(y)) for x, y in zip(a, b))


@pytest.fixture(scope="module", params=[0.0, 0.25], ids=["msf0", "msf.25"])
def slic_maps(request):
    return _slic(240, 320, 300, 6, request.param, seed=41)


@pytest.mark.parametrize("connectivity", [4, 8])
def test_slic_maps(slic_maps, connectivity):
    labels, K = slic_maps
    g = _graph(labels, K, connectivity)
    for C in (1, 3, 4, 5, 16):
        s = _check(labels, K, g, _values((labels.shape[0], C, 240, 320), C), connectivity)
        assert torch.equal(s.count, g.boundary)
        assert not torch.isnan(s.mean).any()


@pytest.mark.parametrize("connectivity", [4, 8])
def test_hd_slic_maps(connectivity):
    labels, K = _slic(720, 1280, 1600, 3, 0.25, seed=73)
    g = _graph(labels, K, connectivity)
    for C in (1, 5):
        s = _check(labels, K, g, _values((3, C, 720, 1280), 7 + C), connectivity)
        assert torch.equal(s.count, g.boundary)


def _adversarial():
    rng = np.random.RandomState(17)
    yield "noise K=65534", rng.randint(0, 65534, (2, 40, 53)).astype(np.uint16).view(np.int16), 65534
    mixed = rng.randint(0, 30, (3, 37, 45)).astype(np.int16)
    mixed[rng.rand(*mixed.shape) < 0.2] = -1
    big = rng.rand(*mixed.shape) < 0.1
    mixed[big] = 30 + rng.randint(0, 30000, int(big.sum()))
    yield "-1 and labels >= K", mixed, 30
    yield "H=1", rng.randint(0, 9, (3, 1, 300)).astype(np.int16), 9
    yield "W=1", rng.randint(0, 9, (3, 300, 1)).astype(np.int16), 9
    yield "H*W<32", rng.randint(-1, 6, (7, 3, 5)).astype(np.int16), 6
    yield "2x2", rng.randint(0, 4, (11, 2, 2)).astype(np.int16), 4
    yy, xx = np.mgrid[:64, :96]
    yield "stripes", np.stack([(xx // 5 % 2), (yy // 3 % 3)]).astype(np.int16), 3


@pytest.mark.parametrize("connectivity", [4, 8])
def test_adversarial_maps_and_values(connectivity):
    for name, labels, K in _adversarial():
        B, H, W = labels.shape
        g = _graph(torch.from_numpy(labels).cuda(), K, connectivity)
        for C, special in ((1, False), (5, True), (4, True)):
            s = _check(labels, K, g, _values((B, C, H, W), B + C, special), connectivity)
            assert torch.equal(s.count, g.boundary), name


def test_diagonal_edges_read_with_connectivity_4(slic_maps):
    labels, K = slic_maps
    g8 = _graph(labels, K, 8)
    s = _check(labels, K, g8, _values((labels.shape[0], 2, 240, 320), 3), 4)
    g4 = _graph(labels, K, 4)
    n = labels.shape[0] * K
    in4 = torch.isin(g8.edge_index[0] * n + g8.edge_index[1], g4.edge_index[0] * n + g4.edge_index[1])
    assert (~in4).any()  # some edges touch only diagonally
    assert (s.count[~in4] == 0).all() and torch.isnan(s.mean[~in4]).all() and torch.isnan(s.min[~in4]).all()
    assert (s.count[in4] > 0).all()


def test_hand_built_entries(slic_maps):
    import types
    labels, K = slic_maps
    B = labels.shape[0]
    g = _graph(labels, K, 4)
    ei = g.edge_index
    rng = np.random.RandomState(2)
    pick = torch.from_numpy(rng.randint(0, ei.shape[1], 50)).cuda()
    fwd = ei[:, pick]
    extra = torch.tensor([[0, K, -1, B * K, 5, 2 * K + 3, 7, B * K - 1],
                          [K, 0, 3, 1, 5, 2 * K + 3, B * K + 7, B * K - 2]], dtype=torch.int64, device="cuda")
    rev_only = ei[:, ei[0] > ei[1]][:, :20]
    entries = torch.cat([fwd, fwd.flip(0), fwd, extra, rev_only], dim=1)
    hand = types.SimpleNamespace(indptr=g.indptr, edge_index=entries.contiguous())
    s = _check(labels, K, hand, _values((B, 3, 240, 320), 9), 4)
    # both directions and duplicates: identical rows; cross-image, out of range and self loops: none
    assert _same([x[:50] for x in s], [x[50:100] for x in s]) and _same([x[:50] for x in s], [x[100:150] for x in s])
    bad = s.count[150:156]
    assert (bad == 0).all() and torch.isnan(s.mean[150:156]).all()


def test_batch_chunk_and_stream_invariance(slic_maps, monkeypatch):
    from fast_slic_b200 import _lib, region_graph
    from fast_slic_b200.region_graph import boundary_stats
    labels, K = slic_maps
    B = labels.shape[0]
    values = torch.from_numpy(_values((B, 4, 240, 320), 5, special=True)).cuda()
    for conn in (4, 8):
        g = _graph(labels, K, conn)
        full = boundary_stats(labels, K, g, values, conn)
        assert _same(boundary_stats(labels, K, g, values, conn), full)  # a second run
        for b in (0, 3):
            gb = _graph(labels[b:b + 1], K, conn)
            lo, hi = int(g.indptr[b * K]), int(g.indptr[(b + 1) * K])
            alone = boundary_stats(labels[b:b + 1], K, gb, values[b:b + 1], conn)
            assert _same(alone, [x[lo:hi] for x in full])
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            on_s = boundary_stats(labels, K, g, values, conn)
        s.synchronize()
        assert _same(on_s, full)
        with monkeypatch.context() as m:
            m.setattr(region_graph, "BOUNDARY_SCRATCH_CAP",
                      2 * _lib.lib().fslic_b200_boundary_select_scratch_bytes(1, 240, 320, K, conn))
            assert region_graph.boundary_chunk(B, 240, 320, K, conn) == 2
            assert _same(boundary_stats(labels, K, g, values, conn), full)
        # a non-contiguous view of the values gives the same bits
        wide = torch.zeros((B, 8, 240, 320), dtype=torch.float32, device="cuda")
        wide[:, ::2] = values
        assert _same(boundary_stats(labels, K, g, wide[:, ::2], conn), full)


def _dtoh_copies(fn):
    """The device-to-host copies a profiler trace of fn() records.  In a long-running process the profiler at times
    loses the device record of a copy; such an incomplete trace is taken again."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(5):
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        with tempfile.TemporaryDirectory() as d:
            path = os.path.join(d, "trace.json")
            prof.export_chrome_trace(path)
            events = json.load(open(path))["traceEvents"]
        calls = [e for e in events if e.get("cat") == "cuda_runtime" and "Memcpy" in e.get("name", "")]
        copies = [e for e in events if e.get("cat") == "gpu_memcpy" and "DtoH" in e["name"]]
        if len(copies) == len(calls):
            break
    return [e.get("args", {}).get("bytes") for e in copies]


def test_one_readback_per_chunk(slic_maps, monkeypatch):
    """One int32 read per selection.  With a cap of a few images, the batch is selected in chunks; a chunk whose
    boundary pairs need more than the cap for their sort is halved and each half selected again, down to single
    images.  The selections (a spy on the entry point) follow that rule, each is read back once, and the result is the
    same bits as with the default cap."""
    from fast_slic_b200 import _lib, region_graph
    from fast_slic_b200.region_graph import boundary_stats
    labels, K = slic_maps
    B = labels.shape[0]
    values = torch.from_numpy(_values((B, 3, 240, 320), 1)).cuda()
    L = _lib.lib()
    selections = []
    select = L.fslic_b200_boundary_select_batch

    def spy(*args):
        selections.append(args[1])
        return select(*args)

    monkeypatch.setattr(L, "fslic_b200_boundary_select_batch", spy)
    for conn, per in ((4, 3), (8, 2)):
        g = _graph(labels, K, conn)
        E = int(g.edge_index.shape[1])
        image = (g.edge_index[0] // K).cpu()
        boundary = g.boundary.cpu().long()
        cap = per * L.fslic_b200_boundary_select_scratch_bytes(1, 240, 320, K, conn)

        def expect(b0, c):
            pairs = int(boundary[(image >= b0) & (image < b0 + c)].sum()) // 2
            if c == 1 or L.fslic_b200_boundary_stats_scratch_bytes(pairs, E) <= cap:
                return [c]
            return [c] + expect(b0, c // 2) + expect(b0 + c // 2, c - c // 2)

        full = boundary_stats(labels, K, g, values, conn)
        monkeypatch.setattr(region_graph, "BOUNDARY_SCRATCH_CAP", cap)
        assert region_graph.boundary_chunk(B, 240, 320, K, conn) == per
        want = [n for b0 in range(0, B, per) for n in expect(b0, min(per, B - b0))]
        torch.cuda.synchronize()
        selections.clear()
        copies = _dtoh_copies(lambda: boundary_stats(labels, K, g, values, conn))
        assert selections == want and copies == [4] * len(want), (selections, want, copies)
        assert _same(boundary_stats(labels, K, g, values, conn), full)
        monkeypatch.setattr(region_graph, "BOUNDARY_SCRATCH_CAP", 1 << 30)
        selections.clear()
        assert _dtoh_copies(lambda: boundary_stats(labels, K, g, values, conn)) == [4] and selections == [B]


def test_refused_under_graph_capture(slic_maps):
    from fast_slic_b200.region_graph import boundary_stats
    labels, K = slic_maps
    g = _graph(labels, K, 4)
    values = torch.zeros((labels.shape[0], 1, 240, 320), device="cuda")
    x = torch.zeros(4, device="cuda")
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        x.add_(1)
        with pytest.raises(RuntimeError, match="CUDA graph"):
            boundary_stats(labels, K, g, values)
    graph.replay()
    torch.cuda.synchronize()
    assert x.tolist() == [1.0] * 4
    _check(labels, K, g, values, 4)  # the device is fine afterwards


def test_empty_shapes_and_no_entries(slic_maps):
    import types
    from fast_slic_b200.region_graph import boundary_stats
    for B, H, W in ((0, 5, 6), (2, 0, 6), (2, 5, 0)):
        lab = torch.zeros((B, H, W), dtype=torch.int16, device="cuda")
        val = torch.zeros((B, 3, H, W), dtype=torch.float32, device="cuda")
        for E in (0, 4):
            g = types.SimpleNamespace(indptr=torch.zeros(B * 7 + 1, dtype=torch.int64, device="cuda"),
                                      edge_index=torch.ones((2, E), dtype=torch.int64, device="cuda"))
            s = boundary_stats(lab, 7, g, val)
            assert all(tuple(x.shape) == (E, 3) and torch.isnan(x).all() for x in s[:3])
            assert tuple(s.count.shape) == (E,) and not s.count.any()
    labels, K = slic_maps
    g = types.SimpleNamespace(indptr=torch.zeros(labels.shape[0] * K + 1, dtype=torch.int64, device="cuda"),
                              edge_index=torch.empty((2, 0), dtype=torch.int64, device="cuda"))
    s = boundary_stats(labels, K, g, torch.zeros((labels.shape[0], 2, 240, 320), device="cuda"))
    assert all(tuple(x.shape) == (0, 2) for x in s[:3]) and tuple(s.count.shape) == (0,)


def test_boundary_strength_merging(slic_maps):
    """merge_regions over the mean of an edge map along each boundary, against the restatements of both."""
    from fast_slic_b200.merging import merge_regions
    from fast_slic_b200.region_graph import boundary_stats
    labels, K = slic_maps
    B = labels.shape[0]
    imgs = np.stack([make_image("syn", 240, 320, seed=41 + b) for b in range(B)]).astype(np.float32)
    gray = imgs.mean(axis=3)
    edge = np.zeros_like(gray)
    edge[:, 1:-1, 1:-1] = np.hypot(gray[:, 1:-1, 2:] - gray[:, 1:-1, :-2], gray[:, 2:, 1:-1] - gray[:, :-2, 1:-1])
    edge_map = torch.from_numpy(edge.astype(np.float32)).cuda()
    g = _graph(labels, K, 4)
    s = boundary_stats(labels, K, g, edge_map[:, None])
    ei = _np(g.edge_index)
    want = ref_boundary(_np(labels), K, ei[0], ei[1], edge[:, None].astype(np.float32), 4)
    assert nan_class_equal(_np(s.mean), want[0])
    w = want[0][:, 0]
    for kw in ({"threshold": float(np.median(w))}, {"threshold": float(np.quantile(w, 0.2))}, {"num_regions": 40}):
        m = merge_regions(labels, K, g, s.mean[:, 0], **kw)
        ref = ref_merge(_np(labels), K, ei[0], ei[1], w, **kw)
        for got, exp in zip(m, ref):
            assert np.array_equal(_np(got), exp), kw
