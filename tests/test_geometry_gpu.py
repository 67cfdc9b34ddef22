"""Superpixel shapes on the GPU (fast_slic_b200.geometry) against the numpy restatement (geometry_cases.py), exactly,
with dtype, shape and device: SLIC maps at 720p, maps with -1 and labels >= K, noise at K = 65534 (the shared table
overflows), 1x1, 1xW and Hx1 images, batches of images under 32 pixels, more than 65535 images, one 2160p image;
batch / stream / run invariance, non-contiguous inputs, empty batches, CUDA graph capture, and agreement with pool's
counts."""
import numpy as np
import pytest
import torch

from cases import make_image
from geometry_cases import FIELDS, ref_properties

pytestmark = pytest.mark.gpu

DTYPES = {"area": torch.int32, "bbox": torch.int32, "moments": torch.int64, "perimeter": torch.int32,
          "border": torch.int32, "centroid": torch.float64, "covariance": torch.float64}
TAIL = {"area": (), "bbox": (4,), "moments": (5,), "perimeter": (), "border": (), "centroid": (2,), "covariance": (3,)}


@pytest.fixture(scope="module", autouse=True)
def _needs_cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _np(x):
    return x.detach().cpu().numpy()


def _cuda(x):
    return x if isinstance(x, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _check(labels, K):
    """region_properties against the restatement, exactly; returns the device result."""
    from fast_slic_b200.geometry import region_properties
    labels = _cuda(labels)
    p = region_properties(labels, K)
    want = ref_properties(_np(labels), K)
    B = labels.shape[0]
    for f in FIELDS:
        x = getattr(p, f)
        assert x.dtype == DTYPES[f] and tuple(x.shape) == (B, K) + TAIL[f] and x.device == labels.device, f
        got = _np(x)
        assert np.array_equal(got, want[f]), (f, np.argwhere(got != want[f])[:5])
    assert not torch.isnan(p.centroid).any() and not torch.isnan(p.covariance).any()
    return p


def _same(a, b):
    return all(torch.equal(x, y) for x, y in zip(a, b))


@pytest.fixture(scope="module", params=[0.0, 0.25], ids=["msf0", "msf.25"])
def slic_case(request):
    from fast_slic_b200 import Slic
    imgs = np.stack([make_image("syn", 720, 1280, seed=21 + b) for b in range(3)])
    labels, clusters = Slic(num_components=1600, min_size_factor=request.param).iterate_batch(
        torch.from_numpy(imgs).cuda(), return_clusters=True)
    return labels, int(clusters.shape[1])


def test_slic_maps(slic_case):
    labels, K = slic_case
    p = _check(labels, K)
    lab = labels.long() & 0xFFFF
    if bool((lab < K).all()):
        assert torch.equal(p.area.sum(1), torch.full((labels.shape[0],), 720 * 1280, dtype=torch.int64, device="cuda"))


def test_area_equals_pool_counts(slic_case):
    from fast_slic_b200.geometry import region_properties
    from fast_slic_b200.pooling import pool
    labels, K = slic_case
    features = torch.ones((labels.shape[0], 1) + tuple(labels.shape[1:]), dtype=torch.float32, device="cuda")
    _, counts = pool(features, labels, K, return_counts=True)
    assert torch.equal(region_properties(labels, K).area, counts)


def test_foreign_labels(slic_case):
    labels, K = slic_case
    rng = np.random.RandomState(3)
    lab = _np(labels).copy()
    holes = rng.rand(*lab.shape) < 0.03
    lab[holes] = rng.choice(np.array([-1, K, K + 7, 32767], np.int16), int(holes.sum()))
    lab[:, 100:140, 200:260] = -1
    _check(lab, K)
    _check(lab, K // 2)  # half the superpixels' labels are now >= K


def test_noise_labels_at_max_K():
    rng = np.random.RandomState(6)
    labels = rng.randint(0, 65536, (2, 300, 400)).astype(np.uint16).view(np.int16)  # 65534 and 65535 are not counted
    _check(labels, 65534)
    _check(rng.randint(0, 600, (2, 300, 400)).astype(np.int16), 65534)  # about 200 labels per table: mixed paths


def test_tiny_and_thin_images():
    rng = np.random.RandomState(10)
    for shape, K in (((1, 1, 1), 1), ((3, 1, 1), 4), ((2, 1, 700), 9), ((2, 1, 65535), 9), ((2, 700, 1), 9),
                     ((2, 65535, 1), 9), ((9, 3, 5), 6), ((13, 2, 2), 4), ((5, 1, 31), 5), ((4, 31, 1), 5),
                     ((3, 33, 65), 9), ((2, 70, 257), 40)):
        _check(rng.randint(-1, K + 2, shape).astype(np.int16), K)
        runs = np.repeat(rng.randint(0, K, shape[:2] + (shape[2] // 7 + 1,)), 7, axis=2)[:, :, :shape[2]]
        _check(runs.astype(np.int16), K)


def test_more_than_65535_images():
    rng = np.random.RandomState(12)
    _check(rng.randint(-1, 4, (65537 + 9, 2, 3)).astype(np.int16), 3)


def test_2160p_image():
    H, W = 2160, 3840
    yy, xx = np.mgrid[:H, :W]
    labels = ((yy // 45) * 86 + (xx + yy // 3) // 45 % 86).astype(np.int16)
    labels[:40, ::3] = -1
    _check(labels[None], 48 * 86)


def test_empty_batches():
    from fast_slic_b200.geometry import region_properties
    for B, H, W in ((0, 5, 6), (2, 0, 6), (2, 5, 0)):
        p = region_properties(torch.zeros((B, H, W), dtype=torch.int16, device="cuda"), 7)
        for f in FIELDS:
            x = getattr(p, f)
            assert x.dtype == DTYPES[f] and tuple(x.shape) == (B, 7) + TAIL[f] and not x.any(), f


def test_batch_stream_and_run_invariance(slic_case):
    from fast_slic_b200.geometry import region_properties
    labels, K = slic_case
    full = region_properties(labels, K)
    assert _same(region_properties(labels, K), full)  # a second run
    idx = torch.tensor([2, 0, 1], device="cuda")
    assert _same(region_properties(labels[idx], K), [f[idx] for f in full])
    assert _same(region_properties(labels[1:2], K), [f[1:2] for f in full])
    assert _same(region_properties(torch.cat([labels[2:], labels[:2]]), K), [torch.cat([f[2:], f[:2]]) for f in full])
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        on_s = region_properties(labels, K)
    s.synchronize()
    assert _same(on_s, full)


def test_non_contiguous_inputs(slic_case):
    from fast_slic_b200.geometry import region_properties
    labels, K = slic_case
    lab_t = labels.transpose(1, 2)  # [B,W,H] views
    assert not lab_t.is_contiguous()
    assert _same(region_properties(lab_t, K), region_properties(lab_t.contiguous(), K))
    _check(lab_t, K)
    _check(labels[:, ::2, 1::3], K)


def test_cuda_graph_capture(slic_case):
    from fast_slic_b200.geometry import region_properties
    labels, K = slic_case
    lab = labels.clone()
    want = region_properties(lab, K)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        region_properties(lab, K)  # warm-up on the capture stream
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        got = region_properties(lab, K)
    graph.replay()
    torch.cuda.synchronize()
    assert _same(got, want)
    lab.copy_(torch.flip(lab, [2]))  # new inputs in place, one more replay
    graph.replay()
    torch.cuda.synchronize()
    assert _same(got, region_properties(lab, K))
    _check(lab, K)
