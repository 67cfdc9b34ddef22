"""Boundary statistics (boundary_stats_3d), outlines (boundaries_3d) and segmentation scores (segmentation_scores_3d)
of label volumes on the GPU against the numpy restatement (volume_boundary_cases.py), exactly, with dtypes and shapes:
supervoxel maps at every connectivity (labels above 32767 included), adversarial volumes, non-finite values, graph
entries across volumes or out of range, count == region_adjacency_3d's boundary, chunk / stream / repeat invariance,
bit-for-bit equality with the 2-D calls at D = 1, anisotropic tolerances, CUDA graph capture, and the agglomeration
pipeline of the README."""
import numpy as np
import pytest
import torch

from pool_cases import nan_class_equal
from supervoxel_cases import make_volumes
from volume_boundary_cases import ref_boundaries_3d, ref_boundary3d, ref_scores_3d

pytestmark = pytest.mark.gpu
CONNS = (6, 18, 26)
GT_FIELDS = ("pixels", "asa_pixels", "ue_pixels", "gt_boundary", "gt_boundary_hits", "sp_boundary", "sp_boundary_hits",
             "asa", "undersegmentation", "boundary_recall", "boundary_precision")


@pytest.fixture(scope="module", autouse=True)
def _needs_cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _np(x):
    return x.detach().cpu().numpy()


def _cuda(x):
    return x if isinstance(x, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _bits(x):
    return x.view(torch.int32) if x.dtype == torch.float32 else (x.view(torch.int64) if x.dtype == torch.float64 else x)


def _same(a, b):
    return all(torch.equal(_bits(x), _bits(y)) for x, y in zip(a, b))


def _check_stats(labels, K, graph, values, connectivity):
    """boundary_stats_3d against the restatement, bit for bit; returns the device result."""
    from fast_slic_b200.region_graph import boundary_stats_3d
    labels, values = _cuda(labels), _cuda(values)
    s = boundary_stats_3d(labels, K, graph, values, connectivity)
    ei = _np(graph.edge_index)
    want = ref_boundary3d(_np(labels), K, ei[0], ei[1], _np(values), connectivity)
    E, C = ei.shape[1], values.shape[1]
    for got, w, dt, shape in zip(s, want, (torch.float32,) * 3 + (torch.int32,), ((E, C),) * 3 + ((E,),)):
        assert got.dtype == dt and tuple(got.shape) == shape and got.device == labels.device
        assert nan_class_equal(_np(got), w)
    return s


def _check_scores(labels, gt, K, tolerance=2, ignore_index=None):
    from fast_slic_b200.groundtruth import segmentation_scores_3d
    labels, gt = _cuda(labels), _cuda(gt)
    s = segmentation_scores_3d(labels, gt, K, tolerance, ignore_index)
    want = ref_scores_3d(_np(labels), _np(gt), K, tolerance, ignore_index)
    assert s._fields == GT_FIELDS
    for f in GT_FIELDS:
        got = getattr(s, f)
        assert got.dtype == (torch.int64 if f in GT_FIELDS[:7] else torch.float64), f
        assert np.array_equal(_np(got), want[f], equal_nan=True), f
    return s


def _check_outline(labels):
    from fast_slic_b200.groundtruth import boundaries_3d
    labels = _cuda(labels)
    out = boundaries_3d(labels)
    assert out.dtype == torch.bool and out.shape == labels.shape
    assert np.array_equal(_np(out), ref_boundaries_3d(_np(labels)))
    return out


def _values(seed, B, C, shape, nonfinite=True):
    rng = np.random.RandomState(seed)
    v = rng.randn(B, C, *shape).astype(np.float32)
    if nonfinite:
        for val, p in ((np.nan, 0.002), (np.inf, 0.002), (-np.inf, 0.002), (-0.0, 0.05), (0.0, 0.05)):
            v[rng.rand(*v.shape) < p] = np.float32(val)
    return torch.from_numpy(v).cuda()


def _supervoxels(seed, B, D, H, W, K, compactness=1.0):
    from fast_slic_b200.supervoxels import supervoxel_slic
    x = torch.from_numpy(make_volumes(seed, B, 1, D, H, W)).cuda()
    r = supervoxel_slic(x, K, compactness)
    return r.labels, int(r.position.shape[1]), x


@pytest.fixture(scope="module")
def sv_maps():
    return _supervoxels(3, 3, 24, 64, 64, 300)[:2]


@pytest.mark.parametrize("connectivity", CONNS)
def test_supervoxel_maps(sv_maps, connectivity):
    from fast_slic_b200.region_graph import region_adjacency_3d
    labels, K = sv_maps
    g = region_adjacency_3d(labels, K, connectivity)
    for C, nonfinite in ((1, False), (5, True)):
        s = _check_stats(labels, K, g, _values(connectivity + C, labels.shape[0], C, labels.shape[1:], nonfinite),
                         connectivity)
        assert torch.equal(s.count, g.boundary)
    gt = torch.from_numpy(np.kron(np.random.RandomState(1).randint(0, 9, (3, 4, 4, 4)),
                                  np.ones((1, 6, 16, 16), np.int64))).cuda()
    _check_scores(labels, gt, K, (1, 2, 3))
    _check_outline(labels)


@pytest.mark.parametrize("connectivity", CONNS)
def test_supervoxel_maps_above_32767(connectivity):
    from fast_slic_b200.region_graph import region_adjacency_3d
    labels, K, _ = _supervoxels(4, 1, 32, 160, 160, 40000)
    assert K > 32767 and int((labels < 0).sum()) > 0
    g = region_adjacency_3d(labels, K, connectivity)
    s = _check_stats(labels, K, g, _values(7, 1, 2, labels.shape[1:]), connectivity)
    assert torch.equal(s.count, g.boundary)
    if connectivity == 6:
        _check_scores(labels, labels.int() % 7, K, 2)
        _check_scores(labels, labels, K, (0, 1, 1))


def _adversarial():
    rng = np.random.RandomState(9)
    yield "one label", np.zeros((2, 10, 20, 30), np.int16), 1
    yield "all -1", np.full((3, 4, 20, 30), -1, np.int16), 7
    mixed = rng.randint(0, 40, (3, 9, 25, 37)).astype(np.int16)
    mixed[rng.rand(*mixed.shape) < 0.2] = -1
    big = rng.rand(*mixed.shape) < 0.1
    mixed[big] = 40 + rng.randint(0, 30000, int(big.sum()))
    yield "labels >= K", mixed, 40
    yield "D=1", rng.randint(0, 9, (2, 1, 40, 70)).astype(np.int16), 9
    yield "H=1", rng.randint(0, 9, (2, 30, 1, 70)).astype(np.int16), 9
    yield "W=1", rng.randint(0, 9, (2, 30, 70, 1)).astype(np.int16), 9
    yield "1x1x1", np.array([[[[0]]], [[[-1]]], [[[2]]]], np.int16), 3
    zz, yy, xx = np.mgrid[:12, :20, :35]  # one or two long runs: the restatement sums them 32 values at a time
    yield "slabs z", np.stack([zz % 2, zz % 3]).astype(np.int16), 3
    yield "slabs x", (xx % 2)[None].astype(np.int16), 2
    yield "checkerboard", np.stack([(zz + yy + xx) % 2, (zz + yy + xx + 1) % 2]).astype(np.int16), 2
    yield "noise K=3000", rng.randint(0, 3000, (2, 20, 41, 53)).astype(np.int16), 3000
    few = rng.choice(np.array([0, 17, 30000, 65533, 65535], np.uint16), (2, 6, 30, 40)).view(np.int16)
    yield "K=65534 few labels", few, 65534


@pytest.mark.parametrize("connectivity", CONNS)
def test_adversarial_volumes(connectivity):
    from fast_slic_b200.region_graph import region_adjacency_3d
    rng = np.random.RandomState(connectivity)
    for name, labels, K in _adversarial():
        lab = _cuda(labels)
        g = region_adjacency_3d(lab, K, connectivity)
        s = _check_stats(lab, K, g, _values(connectivity, labels.shape[0], 3, labels.shape[1:]), connectivity)
        assert torch.equal(s.count, g.boundary), name
        if connectivity == 6:
            _check_outline(lab)
            gt = rng.randint(-1, 4, labels.shape).astype(np.int16)
            for tol, ignore in ((0, None), ((2, 0, 1), 3), ((1, 5, 0), None)):
                _check_scores(lab, gt, K, tol, ignore)


def test_entries_across_volumes_out_of_range_and_duplicates(sv_maps):
    from fast_slic_b200.region_graph import RegionGraph, region_adjacency_3d
    labels, K = sv_maps
    B = labels.shape[0]
    g = region_adjacency_3d(labels, K, 18)
    ei = g.edge_index
    rng = np.random.RandomState(2)
    n = 3000
    extra = torch.from_numpy(np.stack([rng.randint(-5, B * K + 5, n), rng.randint(-5, B * K + 5, n)])).cuda()
    extra[1, :100] = extra[0, :100]                                   # self loops
    extra[1, 100:200] = (extra[0, 100:200] + K) % (B * K)             # the same label in another volume
    mixed = torch.cat([ei[:, ::3], extra, ei[:, :500], ei.flip(0)[:, ::7]], dim=1)  # duplicates, both directions
    graph = RegionGraph(g.indptr, mixed, None)
    s = _check_stats(labels, K, graph, _values(5, B, 2, labels.shape[1:]), 18)
    assert torch.equal(s.count[:ei[:, ::3].shape[1]], g.boundary[::3])


class _StatsSpy:
    """The library, recording the volumes of each boundary_stats_3d stats call."""

    def __init__(self, L, batches):
        self._L, self._batches = L, batches

    def __getattr__(self, name):
        f = getattr(self._L, name)
        if name != "fslic_b200_boundary3d_stats_batch":
            return f

        def call(*args):
            self._batches.append(args[1])
            return f(*args)
        return call


def _select_counts(labels, K, connectivity):
    """(boundary voxels, boundary pairs) of a whole batch from the select entry point alone."""
    from fast_slic_b200 import _lib
    L = _lib.lib()
    B, D, H, W = labels.shape
    nbytes = L.fslic_b200_boundary3d_select_scratch_bytes(B, D, H, W, K, connectivity)
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=labels.device)
    counts = torch.empty(2, dtype=torch.int64, device=labels.device)
    _lib.check(L.fslic_b200_boundary3d_select_batch(labels.device.index, B, D, H, W, K, connectivity,
                                                    labels.data_ptr(), counts.data_ptr(), scratch.data_ptr(), nbytes,
                                                    torch.cuda.current_stream().cuda_stream))
    return tuple(counts.tolist())


def test_chunk_stream_and_repeat_invariance(sv_maps, monkeypatch):
    from fast_slic_b200 import _lib, groundtruth, region_graph
    from fast_slic_b200.groundtruth import boundaries_3d, segmentation_scores_3d
    from fast_slic_b200.region_graph import boundary_stats_3d, region_adjacency_3d
    labels, K = sv_maps
    B, D, H, W = labels.shape
    L = _lib.lib()
    values = _values(11, B, 3, (D, H, W))
    gt = (labels.int() * 7919 % 13).to(torch.uint8)
    for conn in CONNS:
        g = region_adjacency_3d(labels, K, conn)
        full = boundary_stats_3d(labels, K, g, values, conn)
        assert _same(boundary_stats_3d(labels, K, g, values, conn), full)  # a second run
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            on_s = boundary_stats_3d(labels, K, g, values, conn)
        s.synchronize()
        assert _same(on_s, full)
        with monkeypatch.context() as m:  # one volume per select
            m.setattr(region_graph, "BOUNDARY_SCRATCH_CAP", L.fslic_b200_boundary3d_select_scratch_bytes(1, D, H, W, K,
                                                                                                         conn))
            assert region_graph.boundary3d_chunk(B, D, H, W, K, conn) == 1
            assert _same(boundary_stats_3d(labels, K, g, values, conn), full)
        with monkeypatch.context() as m:  # the select takes all volumes, their pairs are too many to sort at once
            # chunk() sizes from one volume's scratch, so a cap of B of them takes the whole batch
            cap = B * L.fslic_b200_boundary3d_select_scratch_bytes(1, D, H, W, K, conn)
            m.setattr(region_graph, "BOUNDARY_SCRATCH_CAP", cap)
            assert region_graph.boundary3d_chunk(B, D, H, W, K, conn) == B
            voxels, pairs = _select_counts(labels, K, conn)
            assert L.fslic_b200_boundary3d_stats_scratch_bytes(voxels, pairs, g.edge_index.shape[1]) > cap
            batches = []
            m.setattr(_lib, "lib", lambda: _StatsSpy(L, batches))
            assert _same(boundary_stats_3d(labels, K, g, values, conn), full)
            assert sum(batches) == B and len(batches) > 1, batches  # the chunk was halved and read again
    scores = segmentation_scores_3d(labels, gt, K, (1, 3, 2), 5)
    assert _same(segmentation_scores_3d(labels, gt, K, (1, 3, 2), 5), scores)
    with monkeypatch.context() as m:
        m.setattr(groundtruth, "GT_SCRATCH_CAP", L.fslic_b200_gt_scores3d_scratch_bytes(1, D, H, W, K))
        assert groundtruth.gt3d_chunk(B, D, H, W, K) == 1
        assert _same(segmentation_scores_3d(labels, gt, K, (1, 3, 2), 5), scores)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        on_s = segmentation_scores_3d(labels, gt, K, (1, 3, 2), 5)
        outline = boundaries_3d(labels)
    s.synchronize()
    assert _same(on_s, scores) and torch.equal(outline, boundaries_3d(labels))
    perm = [2, 0, 1]
    permuted = segmentation_scores_3d(labels[perm], gt[perm], K, (1, 3, 2), 5)
    assert _same(permuted, [f[perm] for f in scores])


def test_one_slice_equals_the_2d_calls():
    """At D = 1: boundary_stats_3d at 6 == boundary_stats at 4, at 18 and 26 == at 8; boundaries_3d == boundaries;
    segmentation_scores_3d with an int tolerance == segmentation_scores, bit for bit."""
    from fast_slic_b200.groundtruth import boundaries, boundaries_3d, segmentation_scores, segmentation_scores_3d
    from fast_slic_b200.region_graph import boundary_stats, boundary_stats_3d, region_adjacency, region_adjacency_3d
    rng = np.random.RandomState(8)
    lab = np.kron(rng.randint(-1, 300, (3, 30, 40)), np.ones((1, 7, 9), np.int64)).astype(np.int16)
    lab[rng.rand(*lab.shape) < 0.01] = 1000
    l2 = torch.from_numpy(lab).cuda()
    l3 = l2[:, None]
    v2 = _values(3, 3, 6, lab.shape[1:])
    for c3, c2 in ((6, 4), (18, 8), (26, 8)):
        g = region_adjacency(l2, 300, c2)
        assert _same(boundary_stats_3d(l3, 300, g, v2[:, :, None], c3), boundary_stats(l2, 300, g, v2, c2))
        assert _same(boundary_stats_3d(l3, 300, region_adjacency_3d(l3, 300, c3), v2[:, :, None], c3),
                     boundary_stats(l2, 300, g, v2, c2))
    assert torch.equal(boundaries_3d(l3)[:, 0], boundaries(l2))
    gt = torch.from_numpy(np.kron(rng.randint(0, 20, (3, 15, 20)), np.ones((1, 14, 18), np.int64))).cuda()
    for r in (0, 2, 32):
        for ignore in (None, 3):
            assert _same(segmentation_scores_3d(l3, gt[:, None], 300, r, ignore),
                         segmentation_scores(l2, gt, 300, r, ignore))


def test_overlap_fields_equal_the_2d_view(sv_maps):
    from fast_slic_b200.groundtruth import segmentation_scores, segmentation_scores_3d
    labels, K = sv_maps
    B, D, H, W = labels.shape
    for gt in ((labels.long() * 31 % 11) - 1, (labels.int() % 4).to(torch.int16)):
        a = segmentation_scores_3d(labels, gt, K, 1, 2)
        b = segmentation_scores(labels.view(B, D * H, W), gt.view(B, D * H, W), K, 1, 2)
        for f in ("pixels", "asa_pixels", "ue_pixels", "asa", "undersegmentation"):
            assert torch.equal(_bits(getattr(a, f)), _bits(getattr(b, f))), f


def test_anisotropic_tolerances(sv_maps):
    labels, K = sv_maps
    rng = np.random.RandomState(4)
    gt = np.kron(rng.randint(0, 30, (3, 6, 8, 8)), np.ones((1, 4, 8, 8), np.int64)).astype(np.int32)
    for tol in ((0, 0, 0), (0, 4, 4), (3, 1, 0), (1, 32, 32), (32, 0, 7), (5, 5, 5)):
        _check_scores(labels, gt, K, tol)
    for dt in (np.uint8, np.int16, np.int64):
        _check_scores(labels, gt.astype(dt), K, (2, 1, 1), 4)


def test_capture(sv_maps):
    """segmentation_scores_3d and boundaries_3d capture and replay; boundary_stats_3d refuses capture before any
    device work."""
    from fast_slic_b200.groundtruth import boundaries_3d, segmentation_scores_3d
    from fast_slic_b200.region_graph import boundary_stats_3d, region_adjacency_3d
    labels, K = sv_maps
    lab = labels[:2].clone()
    gt = (labels.int() % 5)[:2].clone()
    want = (segmentation_scores_3d(lab, gt, K, (1, 2, 3)), boundaries_3d(lab))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        segmentation_scores_3d(lab, gt, K, (1, 2, 3))  # warm-up on the capture stream
        boundaries_3d(lab)
    s.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        got = (segmentation_scores_3d(lab, gt, K, (1, 2, 3)), boundaries_3d(lab))
    graph.replay()
    torch.cuda.synchronize()
    assert _same(got[0], want[0]) and torch.equal(got[1], want[1])
    lab.copy_(labels[1:3])
    gt.copy_(labels[1:3].int() % 5)
    graph.replay()
    torch.cuda.synchronize()
    assert _same(got[0], segmentation_scores_3d(labels[1:3], labels[1:3].int() % 5, K, (1, 2, 3)))
    assert torch.equal(got[1], boundaries_3d(labels[1:3]))
    g = region_adjacency_3d(lab, K)
    values = _values(1, 2, 1, lab.shape[1:])
    g2 = torch.cuda.CUDAGraph()
    with pytest.raises(RuntimeError, match="CUDA graph"):
        with torch.cuda.graph(g2, stream=s):
            boundary_stats_3d(lab, K, g, values)
    torch.cuda.synchronize()
    _check_stats(lab, K, g, values, 6)  # the device is fine afterwards


def test_empty_shapes():
    from fast_slic_b200.groundtruth import boundaries_3d, segmentation_scores_3d
    from fast_slic_b200.region_graph import boundary_stats_3d, region_adjacency_3d
    for shape in ((0, 3, 5, 6), (2, 0, 5, 6), (2, 3, 0, 6), (2, 3, 5, 0)):
        lab = torch.zeros(shape, dtype=torch.int16, device="cuda")
        B = shape[0]
        for conn in CONNS:
            g = region_adjacency_3d(lab, 7, conn)
            s = boundary_stats_3d(lab, 7, g, torch.zeros((B, 2) + shape[1:], device="cuda"), conn)
            assert tuple(s.mean.shape) == (0, 2) and tuple(s.count.shape) == (0,)
        sc = segmentation_scores_3d(lab, lab, 7)
        assert all(tuple(f.shape) == (B,) for f in sc) and not sc.pixels.any()
        assert tuple(boundaries_3d(lab).shape) == shape


def test_readme_agglomeration():
    """The README's CT / EM snippet: supervoxels -> region_adjacency_3d -> boundary_stats_3d of a membrane map ->
    merge_regions(threshold=), against merge_cases.ref_merge given the restated mean boundary strengths."""
    from merge_cases import ref_merge

    from fast_slic_b200.merging import merge_regions
    from fast_slic_b200.region_graph import boundary_stats_3d, region_adjacency_3d
    labels, K, x = _supervoxels(6, 2, 32, 96, 96, 500)
    B, C, D, H, W = x.shape
    membrane = torch.sigmoid(x[:, :1])  # a boundary probability per voxel, [B,1,D,H,W]
    g = region_adjacency_3d(labels, K, 6)
    s = boundary_stats_3d(labels, K, g, membrane)
    m = merge_regions(labels.view(B, D * H, W), K, g, s.mean[:, 0], threshold=0.5)
    ei = _np(g.edge_index)
    want_mean = ref_boundary3d(_np(labels), K, ei[0], ei[1], _np(membrane), 6)[0][:, 0]
    assert np.array_equal(_np(s.mean[:, 0]).view(np.int32), want_mean.view(np.int32))
    want_labels, want_region, want_count = ref_merge(_np(labels.view(B, D * H, W)), K, ei[0], ei[1], want_mean,
                                                     threshold=0.5)
    assert np.array_equal(_np(m.labels), want_labels) and np.array_equal(_np(m.region), want_region)
    assert np.array_equal(_np(m.num_regions), want_count)
    present = [np.unique(v).size for v in _np(labels).reshape(B, -1)]
    assert all(0 < c < p for c, p in zip(want_count.tolist(), present))  # the cut merges some supervoxels
