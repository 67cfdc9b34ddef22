"""Region adjacency graphs (region_adjacency_3d) and shapes (region_properties_3d) of label volumes on the GPU against
the numpy restatement (volume_graph_cases.py), exactly, every tensor with dtype and shape: supervoxel maps at every
connectivity (labels above 32767 included), adversarial volumes, the overflow re-run, batch / chunk / stream / repeat
invariance, equality with the 2-D calls at D = 1, CUDA graph capture, empty shapes, and the supervoxel pipeline of the
README through merge_regions."""
import numpy as np
import pytest
import torch

from geometry_cases import ref_properties
from merge_cases import ref_merge
from supervoxel_cases import make_volumes
from volume_graph_cases import FIELDS_3D, ref_properties_3d, ref_rag3d

pytestmark = pytest.mark.gpu
CONNS = (6, 18, 26)


@pytest.fixture(scope="module", autouse=True)
def _needs_cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _np(x):
    return x.detach().cpu().numpy()


def _same(a, b):
    return all(torch.equal(x.view(torch.int64) if x.dtype == torch.float64 else x,
                           y.view(torch.int64) if y.dtype == torch.float64 else y) for x, y in zip(a, b))


def _cuda(labels):
    return labels if isinstance(labels, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(labels)).cuda()


def _check_graph(labels, K, connectivity):
    """region_adjacency_3d against the restatement, exactly; returns the device result."""
    from fast_slic_b200.region_graph import region_adjacency_3d
    labels = _cuda(labels)
    g = region_adjacency_3d(labels, K, connectivity)
    want = ref_rag3d(_np(labels), K, connectivity)
    for got, w, dt in zip(g, want, (torch.int64, torch.int64, torch.int32)):
        assert got.dtype == dt and got.device == labels.device and tuple(got.shape) == w.shape
        assert np.array_equal(_np(got), w)
    return g


def _check_props(labels, K):
    """region_properties_3d against the restatement, bit for bit; returns the device result."""
    from fast_slic_b200.geometry import region_properties_3d
    labels = _cuda(labels)
    p = region_properties_3d(labels, K)
    want = ref_properties_3d(_np(labels), K)
    assert p._fields == FIELDS_3D
    for f in FIELDS_3D:
        got, w = _np(getattr(p, f)), want[f]
        assert got.dtype == w.dtype and got.shape == w.shape, f
        if w.dtype == np.float64:
            assert np.array_equal(got.view(np.int64), w.view(np.int64)), f
        else:
            assert np.array_equal(got, w), f
    return p


def _supervoxels(seed, B, D, H, W, K, compactness=1.0):
    from fast_slic_b200.supervoxels import supervoxel_slic
    x = torch.from_numpy(make_volumes(seed, B, 1, D, H, W)).cuda()
    r = supervoxel_slic(x, K, compactness)
    return r.labels, int(r.position.shape[1]), x


@pytest.fixture(scope="module")
def sv_maps():
    return _supervoxels(3, 4, 48, 128, 128, 600)[:2]


@pytest.fixture()
def no_recount(monkeypatch):
    """Fails the test if any volume's pair table overflows and is counted again."""
    from fast_slic_b200 import region_graph
    calls = []
    split = region_graph._split

    def spy(b0, flags):
        calls.append((b0, list(flags)))
        return split(b0, flags)

    monkeypatch.setattr(region_graph, "_split", spy)
    yield
    assert not calls, calls


@pytest.mark.parametrize("connectivity", CONNS)
def test_supervoxel_maps(sv_maps, connectivity, no_recount):
    labels, K = sv_maps
    g = _check_graph(labels, K, connectivity)
    assert int(g.indptr[-1]) > 6 * labels.shape[0] * K  # a supervoxel has many neighbours


def test_supervoxel_properties(sv_maps):
    labels, K = sv_maps
    p = _check_props(labels, K)
    assert int((p.area > 0).sum()) > labels.shape[0] * K // 2


@pytest.mark.parametrize("connectivity", CONNS)
def test_supervoxel_maps_above_32767(connectivity, no_recount):
    """K' = 40000 on a 40x200x200 volume: labels above 32767 are negative as int16 and read as uint16."""
    labels, K, _ = _supervoxels(4, 1, 40, 200, 200, 40000)
    assert K > 32767 and int((labels < 0).sum()) > 0
    _check_graph(labels, K, connectivity)
    if connectivity == 6:
        _check_props(labels, K)


def _blocky(B, D, H, W, bz, by, bx):
    zz, yy, xx = np.mgrid[:D, :H, :W]
    nx, ny = -(-W // bx), -(-H // by)
    lab = (zz // bz * ny * nx + yy // by * nx + xx // bx).astype(np.int16)
    return np.stack([np.roll(lab, 3 * b, axis=2) for b in range(B)])


def _adversarial():
    rng = np.random.RandomState(9)
    yield "one label", np.zeros((2, 10, 20, 30), np.int16), 1
    yield "one label K=5", np.full((2, 7, 9, 40), 3, np.int16), 5
    yield "all -1", np.full((3, 4, 20, 30), -1, np.int16), 7
    mixed = rng.randint(0, 40, (3, 9, 25, 37)).astype(np.int16)
    mixed[rng.rand(*mixed.shape) < 0.2] = -1
    big = rng.rand(*mixed.shape) < 0.1
    mixed[big] = 40 + rng.randint(0, 30000, int(big.sum()))
    yield "labels >= K", mixed, 40
    yield "only labels >= K", rng.randint(50, 32000, (2, 5, 10, 10)).astype(np.int16), 50
    yield "D=1", rng.randint(0, 9, (2, 1, 40, 70)).astype(np.int16), 9
    yield "H=1", rng.randint(0, 9, (2, 30, 1, 70)).astype(np.int16), 9
    yield "W=1", rng.randint(0, 9, (2, 30, 70, 1)).astype(np.int16), 9
    yield "1x1x1", np.array([[[[0]]], [[[-1]]], [[[2]]]], np.int16), 3
    yield "DHW<32, B>1", rng.randint(-1, 6, (7, 2, 3, 4)).astype(np.int16), 6
    yield "DHW<32, B>1, 2x2x2", rng.randint(0, 4, (11, 2, 2, 2)).astype(np.int16), 4
    zz, yy, xx = np.mgrid[:24, :64, :96]
    yield "checkerboard", np.stack([(zz + yy + xx) % 2, (zz + yy + xx + 1) % 2]).astype(np.int16), 2
    yield "checkerboard 8", (((zz % 2) * 4 + (yy % 2) * 2 + xx % 2)[None]).astype(np.int16), 8
    yield "noise K=5000", rng.randint(0, 5000, (2, 20, 41, 53)).astype(np.int16), 5000
    few = rng.choice(np.array([0, 17, 30000, 65533, 65535], np.uint16), (2, 6, 30, 40)).view(np.int16)
    yield "K=65534 few labels", few, 65534
    yield "blocky", _blocky(3, 33, 70, 90, 5, 7, 9), 7 * 10 * 10


@pytest.mark.parametrize("connectivity", CONNS)
def test_adversarial_volumes(connectivity):
    for name, labels, K in _adversarial():
        g = _check_graph(labels, K, connectivity)
        if name.startswith(("one label", "all -1", "only labels", "1x1x1")):
            assert g.edge_index.shape == (2, 0), name
        if connectivity == 6:
            _check_props(labels, K)


@pytest.mark.parametrize("connectivity", CONNS)
def test_star(connectivity):
    """Label 0 touches all 65533 others: a CSR row of 65533 targets."""
    W = 65533
    row = np.arange(1, W + 1, dtype=np.int64).astype(np.uint16).view(np.int16)
    star = np.stack([row, np.zeros(W, np.int16)])[None]          # [1,2,W]: slice 0 rows (labels, zeros)
    vol = np.stack([star, star[::-1, ::-1, ::-1]])                # [2,1,2,W] and its mirror
    g = _check_graph(np.ascontiguousarray(vol), 65534, connectivity)
    assert int(g.indptr[1] - g.indptr[0]) == 65533


@pytest.mark.parametrize("connectivity", [6, 26])
def test_overflow_rerun(monkeypatch, connectivity):
    """Uniform noise at K = 65534 on 64x128x128 has about 3.1M (13M) distinct pairs: more than its 2^21-slot table
    holds, so that volume alone is counted again with an exact table; the ordinary volumes around it are not."""
    from fast_slic_b200 import region_graph
    calls = []
    split = region_graph._split

    def spy(b0, flags):
        calls.append((b0, list(flags)))
        return split(b0, flags)

    monkeypatch.setattr(region_graph, "_split", spy)
    rng = np.random.RandomState(4)
    labels = _blocky(4, 64, 128, 128, 5, 9, 11)
    labels[2] = rng.randint(0, 65534, (64, 128, 128)).astype(np.uint16).view(np.int16)
    _check_graph(labels, 65534, connectivity)
    assert calls and all(flags == [0, 0, 1, 0] for _, flags in calls), calls
    if connectivity == 6:
        _check_props(labels, 65534)  # the shared tables overflow to global memory everywhere in the noise


def _block(g, b, K):
    """Volume b's rows of a batch graph, renumbered to local node ids."""
    lo, hi = int(g.indptr[b * K]), int(g.indptr[(b + 1) * K])
    return (g.indptr[b * K:(b + 1) * K + 1] - lo, g.edge_index[:, lo:hi] - b * K, g.boundary[lo:hi])


def test_batch_chunk_stream_and_repeat_invariance(sv_maps, monkeypatch):
    from fast_slic_b200 import _lib, region_graph
    from fast_slic_b200.geometry import region_properties_3d
    from fast_slic_b200.region_graph import region_adjacency_3d
    labels, K = sv_maps
    B, D, H, W = labels.shape
    perm = [2, 0, 3, 1]
    props = region_properties_3d(labels, K)
    assert _same(region_properties_3d(labels, K), props)
    permuted = region_properties_3d(labels[torch.tensor(perm, device="cuda")], K)
    assert _same(permuted, [f[perm] for f in props])
    for conn in CONNS:
        full = region_adjacency_3d(labels, K, conn)
        assert _same(region_adjacency_3d(labels, K, conn), full)  # a second run
        permuted = region_adjacency_3d(labels[torch.tensor(perm, device="cuda")], K, conn)
        for i, b in enumerate(perm):
            assert _same(_block(permuted, i, K), _block(full, b, K))
        assert _same(_block(region_adjacency_3d(labels[1:2], K, conn), 0, K), _block(full, 1, K))
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            on_s = region_adjacency_3d(labels, K, conn)
            props_s = region_properties_3d(labels, K)
        s.synchronize()
        assert _same(on_s, full) and _same(props_s, props)
        with monkeypatch.context() as m:
            m.setattr(region_graph, "RAG_SCRATCH_CAP",
                      2 * _lib.lib().fslic_b200_rag3d_batch_scratch_bytes(1, D, H, W, K, conn, 0))
            assert region_graph.rag3d_chunk(B, D, H, W, K, conn) == 2
            assert _same(region_adjacency_3d(labels, K, conn), full)


def test_one_slice_equals_the_2d_calls():
    """At D = 1: region_adjacency_3d(l[:, None], K, 6) == region_adjacency(l, K, 4), 18 and 26 == 8, and the shape
    identities of the restatement tests hold on the device results."""
    from fast_slic_b200.geometry import region_properties, region_properties_3d
    from fast_slic_b200.region_graph import region_adjacency, region_adjacency_3d
    rng = np.random.RandomState(8)
    lab = np.kron(rng.randint(-1, 300, (3, 30, 40)), np.ones((1, 7, 9), np.int64)).astype(np.int16)
    lab[rng.rand(*lab.shape) < 0.01] = 1000
    l2 = torch.from_numpy(lab).cuda()
    l3 = l2[:, None]
    for c3, c2 in ((6, 4), (18, 8), (26, 8)):
        assert _same(region_adjacency_3d(l3, 300, c3), region_adjacency(l2, 300, c2))
    p3, p2 = region_properties_3d(l3, 300), region_properties(l2, 300)
    some = p2.area > 0
    assert torch.equal(p3.area, p2.area)
    assert torch.equal(p3.bbox[..., [1, 2, 4, 5]], p2.bbox)
    assert torch.equal(p3.bbox[..., 0], torch.zeros_like(p2.area)) and torch.equal(p3.bbox[..., 3], some.int())
    assert not p3.moments[..., [0, 3, 4, 5]].any() and torch.equal(p3.moments[..., [1, 2, 6, 7, 8]], p2.moments)
    assert torch.equal(p3.surface, p2.perimeter.long() + 2 * p2.area.long())
    assert torch.equal(p3.border, p2.border + 2 * p2.area)
    assert not p3.centroid[..., 0].any() and torch.equal(p3.centroid[..., 1:], p2.centroid)
    assert not p3.covariance[..., :3].any() and torch.equal(p3.covariance[..., 3:], p2.covariance)
    want = ref_properties(lab, 300)
    assert np.array_equal(_np(p3.surface), want["perimeter"] + 2 * want["area"].astype(np.int64))


def test_capture(sv_maps):
    """region_adjacency_3d refuses capture before any device work; region_properties_3d captures and replays."""
    from fast_slic_b200.geometry import region_properties_3d
    from fast_slic_b200.region_graph import region_adjacency_3d
    labels, K = sv_maps
    lab = labels[:2].clone()
    want = region_properties_3d(lab, K)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        region_properties_3d(lab, K)  # warm-up on the capture stream
    s.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        got = region_properties_3d(lab, K)
    graph.replay()
    torch.cuda.synchronize()
    assert _same(got, want)
    lab.copy_(labels[2:4])
    graph.replay()
    torch.cuda.synchronize()
    assert _same(got, region_properties_3d(labels[2:4], K))
    g2 = torch.cuda.CUDAGraph()
    with pytest.raises(RuntimeError, match="CUDA graph"):
        with torch.cuda.graph(g2, stream=s):
            region_adjacency_3d(lab, K)
    torch.cuda.synchronize()
    _check_graph(lab, K, 6)  # the device is fine afterwards


def test_empty_shapes():
    from fast_slic_b200.geometry import region_properties_3d
    from fast_slic_b200.region_graph import region_adjacency_3d
    for shape in ((0, 3, 5, 6), (2, 0, 5, 6), (2, 3, 0, 6), (2, 3, 5, 0)):
        lab = torch.zeros(shape, dtype=torch.int16, device="cuda")
        B = shape[0]
        for conn in CONNS:
            g = region_adjacency_3d(lab, 7, conn)
            assert g.indptr.dtype == torch.int64 and tuple(g.indptr.shape) == (B * 7 + 1,) and not g.indptr.any()
            assert tuple(g.edge_index.shape) == (2, 0) and g.edge_index.dtype == torch.int64
            assert tuple(g.boundary.shape) == (0,) and g.boundary.dtype == torch.int32
        _check_props(lab, 7)


def test_readme_pipeline():
    """Supervoxels -> 3-D graph -> pooled features -> edge weights -> merge_regions on the [B, D*H, W] view, against
    merge_cases.ref_merge given the restated graph and the same weights."""
    from fast_slic_b200.geometry import region_properties_3d
    from fast_slic_b200.merging import merge_regions
    from fast_slic_b200.pooling import pool
    from fast_slic_b200.region_graph import region_adjacency_3d
    labels, K2, x = _supervoxels(6, 2, 32, 96, 96, 500)
    B, C, D, H, W = x.shape
    g = region_adjacency_3d(labels, K2)
    p = region_properties_3d(labels, K2)
    assert tuple(p.centroid.shape) == (B, K2, 3)
    feat = pool(x.view(B, C, D * H, W), labels.view(B, D * H, W), K2).transpose(1, 2).reshape(-1, C)
    w = (feat[g.edge_index[0]] - feat[g.edge_index[1]]).norm(dim=1)
    m = merge_regions(labels.view(B, D * H, W), K2, g, w, num_regions=64)
    _, edge_index, _ = ref_rag3d(_np(labels), K2, 6)
    assert np.array_equal(_np(g.edge_index), edge_index)
    want_labels, want_region, want_count = ref_merge(_np(labels.view(B, D * H, W)), K2, edge_index[0], edge_index[1],
                                                     _np(w), num_regions=64)
    assert np.array_equal(_np(m.labels), want_labels) and np.array_equal(_np(m.region), want_region)
    assert np.array_equal(_np(m.num_regions), want_count) and (want_count == 64).all()
