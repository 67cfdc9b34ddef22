"""Region adjacency graphs on the GPU (fast_slic_b200.region_graph) against the numpy restatement (rag_cases.py),
exactly, all three tensors with dtype and shape: SLIC maps, adversarial maps (the overflow re-run included), batch /
chunk / stream invariance, cross-checks against torch and the reference's adjacency lists, the host copies of one
call, and the refusal under CUDA graph capture."""
import json
import os
import tempfile

import numpy as np
import pytest
import torch

from cases import make_image
from rag_cases import ref_rag

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


@pytest.fixture(scope="module", params=[0.0, 0.25], ids=["msf0", "msf.25"])
def slic_maps(request):
    return _slic(240, 320, 300, 8, request.param, seed=31)


def _check(labels, K, connectivity):
    """region_adjacency against the restatement, exactly; returns the device result."""
    from fast_slic_b200.region_graph import region_adjacency
    if not isinstance(labels, torch.Tensor):
        labels = torch.from_numpy(labels).cuda()
    g = region_adjacency(labels, K, connectivity)
    indptr, edge_index, boundary = ref_rag(_np(labels), K, connectivity)
    assert g.indptr.dtype == torch.int64 and g.edge_index.dtype == torch.int64 and g.boundary.dtype == torch.int32
    assert g.indptr.device == g.edge_index.device == g.boundary.device == labels.device
    assert tuple(g.indptr.shape) == indptr.shape and tuple(g.edge_index.shape) == edge_index.shape
    assert tuple(g.boundary.shape) == boundary.shape
    assert np.array_equal(_np(g.indptr), indptr)
    assert np.array_equal(_np(g.edge_index), edge_index)
    assert np.array_equal(_np(g.boundary), boundary)
    return g


def _same(a, b):
    return all(torch.equal(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize("connectivity", [4, 8])
def test_slic_maps(slic_maps, connectivity):
    labels, K = slic_maps
    g = _check(labels, K, connectivity)
    assert int(g.indptr[-1]) > 4 * labels.shape[0] * K  # a superpixel has several neighbours


@pytest.mark.parametrize("connectivity", [4, 8])
def test_hd_slic_maps(connectivity):
    labels, K = _slic(720, 1280, 1600, 4, 0.25, seed=70)
    _check(labels, K, connectivity)


def _blocky(B, H, W, bh, bw):
    yy, xx = np.mgrid[:H, :W]
    lab = (yy // bh * ((W + bw - 1) // bw) + xx // bw).astype(np.int16)
    return np.stack([np.roll(lab, 3 * b, axis=1) for b in range(B)])


def _adversarial():
    rng = np.random.RandomState(9)
    yield "one label", np.zeros((2, 50, 70), np.int16), 1
    yield "one label K=5", np.full((2, 33, 40), 3, np.int16), 5
    yield "all -1", np.full((3, 20, 30), -1, np.int16), 7
    mixed = rng.randint(0, 40, (3, 45, 67)).astype(np.int16)
    mixed[rng.rand(*mixed.shape) < 0.2] = -1
    big = rng.rand(*mixed.shape) < 0.1
    mixed[big] = 40 + rng.randint(0, 30000, int(big.sum()))
    yield "labels >= K", mixed, 40
    yield "only labels >= K", rng.randint(50, 32000, (2, 20, 20)).astype(np.int16), 50
    yield "K=1", rng.randint(-1, 2, (2, 33, 65)).astype(np.int16), 1
    yield "H=1", rng.randint(0, 9, (3, 1, 300)).astype(np.int16), 9
    yield "W=1", rng.randint(0, 9, (3, 300, 1)).astype(np.int16), 9
    yield "1x1", np.array([[[0]], [[-1]], [[2]]], np.int16), 3
    yield "H*W<32, B>1", rng.randint(-1, 6, (7, 3, 5)).astype(np.int16), 6
    yield "H*W<32, B>1, 2x2", rng.randint(0, 4, (11, 2, 2)).astype(np.int16), 4
    yy, xx = np.mgrid[:512, :384]
    yield "checkerboard 2", np.stack([((yy + xx) % 2), ((yy + xx + 1) % 2)]).astype(np.int16), 2
    yield "checkerboard 4", (((yy % 2) * 2 + xx % 2)[None]).astype(np.int16), 4
    yield "noise K=5000", rng.randint(0, 5000, (2, 61, 77)).astype(np.int16), 5000
    few = rng.choice(np.array([0, 17, 30000, 65533, 65535], np.uint16), (2, 40, 50)).view(np.int16)
    yield "K=65534 few labels", few, 65534
    yield "blocky", _blocky(3, 97, 131, 7, 9), 15 * 14


@pytest.mark.parametrize("connectivity", [4, 8])
def test_adversarial_maps(connectivity):
    for name, labels, K in _adversarial():
        g = _check(labels, K, connectivity)
        if name.startswith(("one label", "all -1", "only labels", "K=1", "1x1")):
            assert g.edge_index.shape == (2, 0), name


@pytest.mark.parametrize("connectivity", [4, 8])
def test_overflow_rerun(monkeypatch, connectivity):
    """Uniform noise at K = 65534 on 1100x1000 has about 2.2M (4.4M) distinct pairs: more than its 2^21-slot table
    holds, so that image alone is counted again with an exact table; the ordinary maps around it are not."""
    from fast_slic_b200 import region_graph
    calls = []
    split = region_graph._split

    def spy(b0, flags):
        calls.append((b0, list(flags)))
        return split(b0, flags)

    monkeypatch.setattr(region_graph, "_split", spy)
    rng = np.random.RandomState(4)
    labels = _blocky(4, 1100, 1000, 23, 31).astype(np.int16)
    labels[2] = rng.randint(0, 65534, (1100, 1000)).astype(np.uint16).view(np.int16)
    _check(labels, 65534, connectivity)
    assert calls and all(flags == [0, 0, 1, 0] for _, flags in calls), calls


@pytest.mark.parametrize("connectivity", [4, 8])
def test_star(connectivity):
    """Label 0 touches all 65533 others: a CSR row of 65533 targets."""
    W = 65533
    row = np.arange(1, W + 1, dtype=np.int64).astype(np.uint16).view(np.int16)
    star = np.stack([row, np.zeros(W, np.int16)])
    labels = np.stack([star, star[::-1, ::-1]])
    g = _check(np.ascontiguousarray(labels), 65534, connectivity)
    assert int(g.indptr[1] - g.indptr[0]) == 65533


def test_empty_shapes():
    from fast_slic_b200.region_graph import region_adjacency
    for B, H, W in ((0, 5, 6), (2, 0, 6), (2, 5, 0)):
        for conn in (4, 8):
            g = region_adjacency(torch.zeros((B, H, W), dtype=torch.int16, device="cuda"), 7, conn)
            assert g.indptr.dtype == torch.int64 and tuple(g.indptr.shape) == (B * 7 + 1,) and not g.indptr.any()
            assert tuple(g.edge_index.shape) == (2, 0) and g.edge_index.dtype == torch.int64
            assert tuple(g.boundary.shape) == (0,) and g.boundary.dtype == torch.int32


def test_large_map():
    H, W = 4100, 4200
    labels = _blocky(1, H, W, 97, 101)  # 43 x 42 blocks
    labels[0, :40, ::3] = -1
    labels[0, -50:, -60:] = 30000
    g = _check(labels, 43 * 42, 4)
    assert int(g.boundary.max()) >= 97


def _image_block(g, b, K):
    """Image b's rows of a batch graph, renumbered to local node ids."""
    lo, hi = int(g.indptr[b * K]), int(g.indptr[(b + 1) * K])
    return (g.indptr[b * K:(b + 1) * K + 1] - lo, g.edge_index[:, lo:hi] - b * K, g.boundary[lo:hi])


def test_batch_chunk_and_stream_invariance(slic_maps, monkeypatch):
    from fast_slic_b200 import _lib, region_graph
    from fast_slic_b200.region_graph import region_adjacency
    labels, K = slic_maps
    B = labels.shape[0]
    for conn in (4, 8):
        full = region_adjacency(labels, K, conn)
        assert _same(region_adjacency(labels, K, conn), full)  # a second run
        perm = [5, 2, 7, 0, 3, 1, 6, 4]
        permuted = region_adjacency(labels[torch.tensor(perm, device="cuda")], K, conn)
        for i, b in enumerate(perm):
            assert _same(_image_block(permuted, i, K), _image_block(full, b, K))
        assert _same(_image_block(region_adjacency(labels[3:4], K, conn), 0, K), _image_block(full, 3, K))
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            on_s = region_adjacency(labels, K, conn)
        s.synchronize()
        assert _same(on_s, full)
        with monkeypatch.context() as m:
            m.setattr(region_graph, "RAG_SCRATCH_CAP",
                      3 * _lib.lib().fslic_b200_rag_batch_scratch_bytes(1, 240, 320, K, conn, 0))
            assert region_graph.rag_chunk(B, 240, 320, K, conn) < B
            assert _same(region_adjacency(labels, K, conn), full)


def test_cross_checks(slic_maps):
    from fast_slic_b200.graph_batch import get_connectivity_batch
    from fast_slic_b200.region_graph import region_adjacency
    labels, K = slic_maps
    B = labels.shape[0]
    lab = labels.long() & 0xFFFF
    pairs = [(lab[:, :, :-1], lab[:, :, 1:]), (lab[:, :-1, :], lab[:, 1:, :])]
    diag = [(lab[:, :-1, :-1], lab[:, 1:, 1:]), (lab[:, :-1, 1:], lab[:, 1:, :-1])]
    graphs = {}
    for conn, ends in ((4, pairs), (8, pairs + diag)):
        g = region_adjacency(labels, K, conn)
        graphs[conn] = g
        # symmetric: the reversed edges, sorted, are the edges
        n = B * K
        fwd = g.edge_index[0] * n + g.edge_index[1]
        rev = g.edge_index[1] * n + g.edge_index[0]
        order = torch.argsort(rev)
        assert torch.equal(rev[order], fwd) and torch.equal(g.boundary[order], g.boundary)
        assert torch.equal(torch.diff(g.indptr) >= 0, torch.ones(n, dtype=torch.bool, device="cuda"))
        # every differing valid pixel pair, counted by torch, in both directions
        total = sum(int(((a < K) & (c < K) & (a != c)).sum()) for a, c in ends)
        assert int(g.boundary.long().sum()) == 2 * total
    # every pair the reference's 12-neighbour lists hold is an edge of the connectivity-8 graph
    counts, nb = get_connectivity_batch(K, 0, labels)
    edges = set((_np(graphs[8].edge_index[0]) * (B * K) + _np(graphs[8].edge_index[1])).tolist())
    counts, nb = _np(counts), _np(nb)
    listed = 0
    for b in range(B):
        for k in range(K):
            for v in nb[b, k, :counts[b, k]].tolist():
                assert (b * K + k) * (B * K) + b * K + v in edges, (b, k, v)
                listed += 1
    assert listed > B * K


def test_one_readback_per_chunk_complete_trace(slic_maps, monkeypatch):
    """A profiler trace of one call over three chunks: three memcpy calls on the host, and three device-to-host copies,
    of (images + 1) int64 words.  In a long-running process the profiler at times loses the device record of a copy
    whose host call it did record; such an incomplete trace is taken again."""
    from torch.profiler import ProfilerActivity, profile
    from fast_slic_b200 import _lib, region_graph
    from fast_slic_b200.region_graph import region_adjacency
    labels, K = slic_maps
    monkeypatch.setattr(region_graph, "RAG_SCRATCH_CAP", 3 * _lib.lib().fslic_b200_rag_batch_scratch_bytes(1, 240, 320, K, 8, 0))
    assert region_graph.rag_chunk(8, 240, 320, K, 8) == 3
    region_adjacency(labels, K, 8)
    torch.cuda.synchronize()
    for _ in range(5):
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            region_adjacency(labels, K, 8)
            torch.cuda.synchronize()
        with tempfile.TemporaryDirectory() as d:
            path = os.path.join(d, "trace.json")
            prof.export_chrome_trace(path)
            events = json.load(open(path))["traceEvents"]
        calls = [e["name"] for e in events if e.get("cat") == "cuda_runtime" and "Memcpy" in e.get("name", "")]
        copies = [e for e in events if e.get("cat") == "gpu_memcpy" and "DtoH" in e["name"]]
        assert len(calls) == 3, calls
        if len(copies) == len(calls):
            break
    assert sorted(e.get("args", {}).get("bytes") for e in copies) == [24, 32, 32], copies


def test_refused_under_graph_capture(slic_maps):
    from fast_slic_b200.region_graph import region_adjacency
    labels, K = slic_maps
    x = torch.zeros(4, device="cuda")
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        x.add_(1)
        with pytest.raises(RuntimeError, match="CUDA graph"):
            region_adjacency(labels, K)
    graph.replay()
    torch.cuda.synchronize()
    assert x.tolist() == [1.0] * 4
    _check(labels, K, 4)  # the device is fine afterwards
