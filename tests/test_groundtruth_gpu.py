"""Ground-truth scores on the GPU (fast_slic_b200.groundtruth) against the numpy restatement (groundtruth_cases.py),
exactly, with dtype and shape: SLIC maps against gt from image colour regions and a 21-class map, every gt dtype with
ignore_index, noise at K = 65534, tiny, thin and large images, tolerances 0, 2 and 32; batch / chunk / stream / run
invariance, non-contiguous inputs, empty batches, CUDA graph capture, and one superpixel GNN step end to end."""
import numpy as np
import pytest
import torch

from cases import make_image
from groundtruth_cases import FIELDS, ref_boundaries, ref_class_histogram, ref_scores

pytestmark = pytest.mark.gpu

RATIOS = ("asa", "undersegmentation", "boundary_recall", "boundary_precision")


@pytest.fixture(scope="module", autouse=True)
def _needs_cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _np(x):
    return x.detach().cpu().numpy()


def _cuda(x):
    return x if isinstance(x, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _check_scores(labels, gt, K, tolerance=2, ignore_index=None):
    """segmentation_scores against the restatement, exactly; returns the device result."""
    from fast_slic_b200.groundtruth import segmentation_scores
    labels, gt = _cuda(labels), _cuda(gt)
    s = segmentation_scores(labels, gt, K, tolerance, ignore_index)
    want = ref_scores(_np(labels), _np(gt), K, tolerance, ignore_index)
    B = labels.shape[0]
    for f in FIELDS:
        x = getattr(s, f)
        assert x.dtype == torch.int64 and tuple(x.shape) == (B,) and x.device == labels.device, f
        assert np.array_equal(_np(x), want[f]), (f, _np(x), want[f])
    for f in RATIOS:
        x = getattr(s, f)
        assert x.dtype == torch.float64 and tuple(x.shape) == (B,), f
        assert np.array_equal(_np(x), want[f], equal_nan=True), (f, _np(x), want[f])
    return s


def _check_hist(classes, labels, K, C):
    from fast_slic_b200.groundtruth import class_histogram
    labels, classes = _cuda(labels), _cuda(classes)
    h = class_histogram(classes, labels, K, C)
    assert h.dtype == torch.int32 and tuple(h.shape) == (labels.shape[0], K, C) and h.device == labels.device
    assert np.array_equal(_np(h), ref_class_histogram(_np(classes), _np(labels), K, C))
    return h


def _check_boundaries(labels):
    from fast_slic_b200.groundtruth import boundaries
    labels = _cuda(labels)
    out = boundaries(labels)
    assert out.dtype == torch.bool and out.shape == labels.shape
    assert np.array_equal(_np(out), ref_boundaries(_np(labels)))
    return out


def _check_all(labels, gt, K, C, tolerances=(0, 2, 32), ignore_index=None):
    for r in tolerances:
        _check_scores(labels, gt, K, r, ignore_index)
    _check_hist(gt, labels, K, C)
    _check_boundaries(labels)


def _blocks(B, H, W, seed):
    """Images of 8x8 colour patches and their colour region ids (uint8 in [0, 64))."""
    imgs = np.stack([make_image("blocks", H, W, seed=seed + b) for b in range(B)])
    q = imgs.astype(np.int64) // 60
    return imgs, (q[..., 0] * 16 + q[..., 1] * 4 + q[..., 2]).astype(np.uint8)


def _classes21(B, H, W, seed):
    rng = np.random.RandomState(seed)
    small = rng.randint(0, 21, (B, H // 24 + 1, W // 24 + 1))
    return np.ascontiguousarray(np.kron(small, np.ones((1, 24, 24), np.int64))[:, :H, :W]).astype(np.int64)


@pytest.fixture(scope="module", params=[0.0, 0.25], ids=["msf0", "msf.25"])
def slic_case(request):
    from fast_slic_b200 import Slic
    imgs, regions = _blocks(6, 240, 320, seed=41)
    labels, clusters = Slic(num_components=300, min_size_factor=request.param).iterate_batch(
        torch.from_numpy(imgs).cuda(), return_clusters=True)
    return labels, int(clusters.shape[1]), regions, _classes21(6, 240, 320, seed=42)


def test_slic_maps_against_colour_regions(slic_case):
    labels, K, regions, _ = slic_case
    _check_all(labels, regions, K, 64)


def test_slic_maps_against_21_classes(slic_case):
    labels, K, _, classes = slic_case
    _check_all(labels, classes, K, 21)
    _check_hist(classes.astype(np.uint8), labels, K, 21)
    _check_hist(classes, labels, K, 5)  # classes >= num_classes are not counted


def test_every_gt_dtype_with_ignore_index(slic_case):
    labels, K, regions, _ = slic_case
    rng = np.random.RandomState(3)
    holes = rng.rand(*regions.shape) < 0.05
    for dtype, ignore, extra in ((np.uint8, 255, []), (np.int16, -1, [-5, 32767]), (np.int32, -1, [2 ** 31 - 1, -9]),
                                 (np.int64, 7, [2 ** 31, -1, 2 ** 31 - 1, -2 ** 62])):
        gt = regions.astype(dtype)
        gt[holes] = ignore
        if extra:
            odd = rng.rand(*regions.shape) < 0.02
            gt[odd] = rng.choice(np.array(extra, dtype), int(odd.sum()))
        for r in (0, 2, 32):
            _check_scores(labels, gt, K, r, ignore)
            _check_scores(labels, gt, K, r)  # ignore_index=None: the ignore value is a class
        _check_hist(gt, labels, K, 64)


def test_noise_labels_at_max_K():
    rng = np.random.RandomState(6)
    labels = rng.randint(0, 65536, (2, 300, 400)).astype(np.uint16).view(np.int16)  # 65534 and 65535 are not counted
    gt = rng.randint(0, 3000, (2, 300, 400)).astype(np.int16)
    for r in (0, 2, 32):
        _check_scores(labels, gt, 65534, r)
    _check_boundaries(labels)
    _check_hist(gt % 7, labels, 65534, 7)


def test_tiny_and_thin_images():
    rng = np.random.RandomState(10)
    cases = [
        (rng.randint(-1, 6, (9, 3, 5)).astype(np.int16), rng.randint(0, 4, (9, 3, 5)).astype(np.uint8), 6),  # warps straddle
        (rng.randint(0, 4, (13, 2, 2)).astype(np.int16), rng.randint(-1, 3, (13, 2, 2)).astype(np.int32), 4),
        (np.array([[[0]], [[-1]], [[2]]], np.int16), np.array([[[1]], [[0]], [[255]]], np.uint8), 3),
        (rng.randint(0, 9, (3, 1, 700)).astype(np.int16), rng.randint(0, 3, (3, 1, 700)).astype(np.int16), 9),
        (rng.randint(0, 9, (3, 700, 1)).astype(np.int16), rng.randint(0, 3, (3, 700, 1)).astype(np.int64), 9),
        (rng.randint(0, 9, (2, 33, 65)).astype(np.int16), rng.randint(0, 3, (2, 33, 65)).astype(np.uint8), 9),
    ]
    for labels, gt, K in cases:
        _check_all(labels, gt, K, 4, tolerances=(0, 1, 2, 32))
        _check_all(labels, gt, K, 4, tolerances=(2,), ignore_index=0)


def test_large_image():
    H, W = 4100, 4200
    yy, xx = np.mgrid[:H, :W]
    labels = (yy // 97 * 44 + xx // 101).astype(np.int16)
    labels[:40, ::3] = -1
    gt = ((yy + 30) // 150 * 30 + (xx + 20) // 170).astype(np.int32)
    gt[-50:, -60:] = -1
    _check_all(labels[None], gt[None], 43 * 44, 30 * 30, tolerances=(0, 2, 32), ignore_index=-1)


def test_empty_batches():
    from fast_slic_b200.groundtruth import boundaries, class_histogram, segmentation_scores
    for B, H, W in ((0, 5, 6), (2, 0, 6), (2, 5, 0)):
        lab = torch.zeros((B, H, W), dtype=torch.int16, device="cuda")
        gt = torch.zeros((B, H, W), dtype=torch.uint8, device="cuda")
        h = class_histogram(gt, lab, 7, 3)
        assert h.dtype == torch.int32 and tuple(h.shape) == (B, 7, 3) and not h.any()
        s = segmentation_scores(lab, gt, 7)
        for f in FIELDS:
            assert getattr(s, f).dtype == torch.int64 and tuple(getattr(s, f).shape) == (B,)
            assert not getattr(s, f).any()
        for f in RATIOS:
            assert getattr(s, f).dtype == torch.float64 and bool(torch.isnan(getattr(s, f)).all())
        b = boundaries(lab)
        assert b.dtype == torch.bool and tuple(b.shape) == (B, H, W)


def _all(labels, gt, K, C, r=2, ignore=None):
    from fast_slic_b200.groundtruth import boundaries, class_histogram, segmentation_scores
    return (class_histogram(gt, labels, K, C), torch.stack(list(segmentation_scores(labels, gt, K, r, ignore)[:7])),
            boundaries(labels))


def _same(a, b):
    return all(torch.equal(x, y) for x, y in zip(a, b))


def test_batch_chunk_stream_and_run_invariance(slic_case, monkeypatch):
    from fast_slic_b200 import _lib, groundtruth
    labels, K, regions, _ = slic_case
    gt = torch.from_numpy(regions).cuda()
    B = labels.shape[0]
    full = _all(labels, gt, K, 64)
    assert _same(_all(labels, gt, K, 64), full)  # a second run
    perm = [4, 1, 5, 0, 3, 2]
    idx = torch.tensor(perm, device="cuda")
    permuted = _all(labels[idx], gt[idx], K, 64)
    assert _same(permuted, (full[0][idx], full[1][:, idx], full[2][idx]))
    one = _all(labels[3:4], gt[3:4], K, 64)
    assert _same(one, (full[0][3:4], full[1][:, 3:4], full[2][3:4]))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        on_s = _all(labels, gt, K, 64)
    s.synchronize()
    assert _same(on_s, full)
    monkeypatch.setattr(groundtruth, "GT_SCRATCH_CAP", 2 * _lib.lib().fslic_b200_gt_scores_scratch_bytes(1, 240, 320, K))
    assert 1 < groundtruth.gt_chunk(B, 240, 320, K) < B
    assert _same(_all(labels, gt, K, 64), full)


def test_non_contiguous_inputs(slic_case):
    labels, K, regions, classes = slic_case
    lab_t = labels.transpose(1, 2)           # [B,W,H] views
    gt_t = torch.from_numpy(regions).cuda().transpose(1, 2)
    assert not lab_t.is_contiguous() and not gt_t.is_contiguous()
    got = _all(lab_t, gt_t, K, 64)
    want = _all(lab_t.contiguous(), gt_t.contiguous(), K, 64)
    assert _same(got, want)
    _check_scores(lab_t, gt_t, K, 2)
    step = torch.from_numpy(classes).cuda()[:, ::2, 1::3]
    _check_hist(step, labels[:, ::2, 1::3], K, 21)


def test_cuda_graph_capture(slic_case):
    labels, K, regions, _ = slic_case
    gt = torch.from_numpy(regions).cuda()
    want = _all(labels, gt, K, 64, 2, 63)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _all(labels, gt, K, 64, 2, 63)  # warm-up on the capture stream
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        got = _all(labels, gt, K, 64, 2, 63)
    graph.replay()
    torch.cuda.synchronize()
    assert _same(got, want)
    gt.copy_(torch.flip(gt, [2]))  # new inputs in place, one more replay
    graph.replay()
    torch.cuda.synchronize()
    assert _same(got, _all(labels, gt, K, 64, 2, 63))


def test_superpixel_gnn_step():
    """iterate_batch -> pool -> region_adjacency -> class_histogram: node features, graph and targets that fit."""
    from fast_slic_b200 import Slic
    from fast_slic_b200.groundtruth import class_histogram
    from fast_slic_b200.pooling import pool
    from fast_slic_b200.region_graph import region_adjacency
    imgs, regions = _blocks(4, 180, 240, seed=77)
    frames = torch.from_numpy(imgs).cuda()
    labels, clusters = Slic(num_components=200, min_size_factor=0.25).iterate_batch(frames, return_clusters=True)
    K = int(clusters.shape[1])
    B, C = 4, 3
    features = frames.permute(0, 3, 1, 2).float().contiguous() / 255
    x, counts = pool(features, labels, K, return_counts=True)
    x = x.transpose(1, 2).reshape(-1, C)
    g = region_adjacency(labels, K)
    h = class_histogram(torch.from_numpy(regions).cuda(), labels, K, 64)
    y = torch.where(h.sum(-1) > 0, h.argmax(-1), -100).reshape(-1)
    assert x.shape == (B * K, C) and y.shape == (B * K,) and y.dtype == torch.int64
    assert g.indptr.shape == (B * K + 1,) and int(g.edge_index.max()) < B * K
    counts = counts.reshape(-1)
    assert torch.equal(h.sum(-1).reshape(-1), counts)  # every pixel of a superpixel has a region
    assert torch.equal(y >= 0, counts > 0)
    ref = ref_class_histogram(regions, _np(labels), K, 64)
    assert np.array_equal(_np(h), ref)
    loss = torch.nn.functional.cross_entropy(torch.nn.Linear(C, 64).cuda()(x), y)
    assert torch.isfinite(loss)
