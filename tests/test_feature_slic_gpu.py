"""SLIC over float feature maps on the GPU (fast_slic_b200.feature_slic) against the numpy restatement
(feature_slic_cases.py): labels, positions, centroid features and counts bit for bit (NaN as a class) over a seeded
sweep of channel counts, K, S, image shapes, strides, iteration counts, compactness, ties, non-finite pixels and warm
starts; the centroid features against pool on the GPU; both assign kernels; batch splits, chunking, streams and
CUDA graph capture."""
import numpy as np
import pytest
import torch

from feature_slic_cases import make_features, nan_class_equal, ref_feature_slic, ref_feature_slic_image

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _needs_cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _np(x):
    return x.detach().cpu().numpy()


def _same(a, b):
    return all(torch.equal(x.view(torch.int32) if x.dtype == torch.float32 else x,
                           y.view(torch.int32) if y.dtype == torch.float32 else y) for x, y in zip(a, b))


def _check(f, K, compactness, max_iter, stride, min_size_factor=0.25, init=None):
    """feature_slic against the restatement; returns (result, [(tiles, overflowed)] per pass)."""
    from fast_slic_b200.feature_slic import feature_slic_dispatch
    x = torch.from_numpy(f).cuda()
    dinit = None if init is None else tuple(torch.from_numpy(v).cuda() for v in init)
    r, disp = feature_slic_dispatch(x, K, compactness, max_iter, stride, min_size_factor, dinit)
    final, pre, pos, mu, cnt = ref_feature_slic(f, K, compactness, max_iter, stride, min_size_factor, init)
    assert r.labels.dtype == torch.int16 and r.count.dtype == torch.int32
    assert np.array_equal(_np(r.count), cnt)
    assert nan_class_equal(_np(r.position), pos)
    assert nan_class_equal(_np(r.features), mu)
    assert np.array_equal(_np(r.labels), final)
    return r, disp


# (seed, B, C, H, W, K, compactness, max_iter, stride, kind)
SWEEP = [
    (1, 2, 1, 60, 80, 50, 1.0, 10, 3, "smooth"),
    (2, 1, 3, 120, 100, 1, 1.0, 4, 3, "smooth"),          # K = 1, S = 109
    (3, 1, 4, 20, 20, 400, 1.0, 3, 1, "smooth"),          # K = H*W, S = 1
    (4, 2, 5, 1, 200, 20, 2.0, 10, 3, "smooth"),          # one row: passes without rows
    (5, 1, 16, 300, 1, 30, 2.0, 10, 5, "smooth"),         # one column
    (6, 1, 33, 64, 64, 100, 1.0, 10, 255, "smooth"),
    (7, 1, 64, 100, 120, 5000, 1.0, 2, 3, "smooth"),      # K > 4096, S = 1
    (8, 1, 300, 40, 50, 40, 1e3, 3, 3, "smooth"),         # C over several shared-memory chunks
    (9, 1, 3, 64, 48, 30, 1.0, 5, 3, "constant"),         # everything ties
    (10, 2, 4, 50, 60, 40, 1.0, 5, 2, "nonfinite"),       # NaN, +inf, -inf pixels and a NaN row
    (11, 1, 3, 60, 60, 36, 1e-3, 10, 3, "smooth"),
    (12, 1, 3, 30, 40, 12, 1e3, 10, 3, "smooth"),
    (13, 1, 4, 45, 50, 20, 1.0, 0, 3, "smooth"),          # seeds only
    (14, 1, 4, 45, 50, 20, 1.0, 1, 3, "smooth"),
    (15, 1, 2, 30, 30, 200, 1.0, 10, 2, "smooth"),        # S = 2
    (16, 1, 2, 33, 35, 120, 1.0, 10, 3, "smooth"),        # S = 3
]


def test_exact_sweep_and_both_assign_kernels():
    tile_only = overflowed = mixed = False
    for seed, B, C, H, W, K, comp, it, stride, kind in SWEEP:
        f = make_features(seed, B, C, H, W, kind)
        r, disp = _check(f, K, comp, it, stride)
        tiles = sum(t for t, _ in disp)
        ovf = sum(o for _, o in disp)
        assert 0 <= ovf <= tiles
        tile_only |= tiles > 0 and ovf == 0
        overflowed |= ovf > 0
        mixed |= 0 < ovf < tiles
    assert tile_only and overflowed and mixed


def test_warm_start_from_an_earlier_result():
    from fast_slic_b200.feature_slic import feature_slic
    f = make_features(30, 2, 6, 70, 90, "smooth")
    g = make_features(31, 2, 6, 70, 90, "smooth")
    a = feature_slic(torch.from_numpy(f).cuda(), 60, 2.0, 5, 3)
    init = (_np(a.position), _np(a.features))
    _check(g, 60, 2.0, 4, 3, init=init)
    # out-of-image and NaN positions are clamped, features taken as given (NaN included)
    init[0][0, :3] = [[-5, 1e6], [np.nan, 3.5], [np.inf, -np.inf]]
    init[1][1, 4, 2] = np.nan
    _check(g, 60, 2.0, 2, 2, init=init)
    _check(g, 60, 2.0, 0, 2, init=init)


def test_centroids_are_pool_over_the_last_pass():
    from fast_slic_b200.feature_slic import feature_slic
    from fast_slic_b200.pooling import pool
    f = make_features(40, 1, 7, 90, 110, "smooth")
    K, it, stride = 80, 5, 3
    r = feature_slic(torch.from_numpy(f).cuda(), K, 1.0, it, stride)
    pass_labels = ref_feature_slic_image(f[0], K, 1.0, it, stride, with_pass_labels=True)[4]
    means, counts = pool(torch.from_numpy(f).cuda(), torch.from_numpy(pass_labels.view(np.int16)[None]).cuda(), K,
                         return_counts=True)
    assert torch.equal(counts, r.count)
    live = r.count[0] > 0
    assert live.any()
    assert torch.equal(means[0].T[live].view(torch.int32), r.features[0][live].view(torch.int32))


def test_enforcement_matches_the_gpu_enforcer():
    from fast_slic_b200.base_slic import get_cca_engine
    from fast_slic_b200.feature_slic import feature_slic, min_size_threshold, superpixel_size
    f = make_features(50, 2, 3, 80, 100, "smooth")
    K, msf = 60, 0.7
    r = feature_slic(torch.from_numpy(f).cuda(), K, 1.0, 6, 3, msf)
    _, pre, _, _, _ = ref_feature_slic(f, K, 1.0, 6, 3, msf)
    thres = min_size_threshold(superpixel_size(80, 100, K), msf)
    want = torch.from_numpy(pre.view(np.int16)).cuda()
    get_cca_engine(80, 100, 2, 0).enforce_connectivity(want, K, thres)
    assert torch.equal(r.labels, want)


def test_batch_splits_chunks_streams_and_repeats(monkeypatch):
    from fast_slic_b200 import feature_slic as fs
    f = torch.from_numpy(make_features(60, 7, 5, 48, 64, "smooth")).cuda()
    args = (40, 1.5, 6, 3)
    a = fs.feature_slic(f, *args)
    assert _same(a, fs.feature_slic(f, *args))
    singles = [fs.feature_slic(f[b:b + 1], *args) for b in range(7)]
    assert _same(a, [torch.cat([s[i] for s in singles]) for i in range(4)])
    one = fs._lib.lib().fslic_b200_feature_slic_scratch_bytes(3, 48, 64, 5, 40, 3, 6)
    with monkeypatch.context() as m:
        m.setattr(fs, "FEATURE_SLIC_SCRATCH_CAP", one)  # chunks of 3 images: 3 + 3 + 1
        assert _same(a, fs.feature_slic(f, *args))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        b = fs.feature_slic(f, *args)
    s.synchronize()
    assert _same(a, b)
    # the same seeds for a permuted batch give the permuted result
    perm = torch.tensor([3, 0, 6, 1, 5, 2, 4], device="cuda")
    assert _same([x[perm] for x in a], fs.feature_slic(f[perm].contiguous(), *args))


def test_graph_capture_replays_the_eager_result():
    from fast_slic_b200.feature_slic import feature_slic
    f = torch.from_numpy(make_features(70, 3, 4, 40, 56, "smooth")).cuda()
    want = feature_slic(f, 30, 1.0, 5, 3)
    x = torch.zeros_like(f)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        feature_slic(x, 30, 1.0, 5, 3)  # warm-up on the capture stream
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        got = feature_slic(x, 30, 1.0, 5, 3)
    x.copy_(f)
    graph.replay()
    torch.cuda.synchronize()
    assert _same(got, want)


def test_empty_batch():
    from fast_slic_b200.feature_slic import feature_slic
    r = feature_slic(torch.zeros((0, 3, 10, 12), device="cuda"), 5, 1.0)
    assert tuple(r.labels.shape) == (0, 10, 12) and tuple(r.position.shape) == (0, 5, 2)
    assert tuple(r.features.shape) == (0, 5, 3) and tuple(r.count.shape) == (0, 5)
