"""Supervoxels on the GPU (fast_slic_b200.supervoxels) against the numpy restatement (supervoxel_cases.py): labels,
positions, centroid features and counts bit for bit (NaN as a class) over a seeded sweep of channel counts, grids,
shapes, spacings, strides, compactness, ties and non-finite voxels; both assign kernels; the 3-D enforcement on its
own, and at D = 1 against the 2-D GPU enforcer; one volume at a real size; batch splits, chunking, streams, CUDA graph
capture and repeats."""
import numpy as np
import pytest
import torch

from supervoxel_cases import (block_labels, components, make_volumes, nan_class_equal, ref_enforce,
                              ref_supervoxel_slic)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _needs_cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _np(x):
    return x.detach().cpu().numpy()


def _same(a, b):
    return all(torch.equal(x.view(torch.int32) if x.dtype == torch.float32 else x,
                           y.view(torch.int32) if y.dtype == torch.float32 else y) for x, y in zip(a[:4], b[:4]))


def _check(f, K, compactness, spacing, max_iter, stride, min_size_factor=0.25):
    """supervoxel_slic against the restatement; returns (result, [(tiles, overflowed)] per pass)."""
    from fast_slic_b200.supervoxels import supervoxel_dispatch
    x = torch.from_numpy(f).cuda()
    r, disp = supervoxel_dispatch(x, K, compactness, spacing, max_iter, stride, min_size_factor)
    final, pre, pos, mu, cnt, grid = ref_supervoxel_slic(f, K, compactness, spacing, max_iter, stride,
                                                         min_size_factor)
    assert r.grid == grid
    assert r.labels.dtype == torch.int16 and r.count.dtype == torch.int32
    assert np.array_equal(_np(r.count), cnt)
    assert nan_class_equal(_np(r.position), pos)
    assert nan_class_equal(_np(r.features), mu)
    assert np.array_equal(_np(r.labels), final)
    return r, disp


ISO, ANISO = (1.0, 1.0, 1.0), (4.0, 0.5, 0.8)
# (seed, B, C, D, H, W, K, compactness, spacing, max_iter, stride, kind)
SWEEP = [
    (1, 2, 1, 24, 24, 24, 8, 1.0, ISO, 6, 3, "smooth"),            # R = 12: the tile kernel alone
    (2, 1, 3, 20, 30, 40, 1, 1.0, ISO, 3, 3, "smooth"),            # K' = 1
    (3, 1, 2, 4, 8, 40, 1280, 1.0, ISO, 3, 1, "smooth"),           # K' = D*H*W, one-voxel cells: the fallback alone
    (4, 1, 1, 24, 40, 40, 40000, 1.0, ISO, 2, 3, "smooth"),        # K' = 38400 > 32767: labels read as uint16
    (5, 2, 4, 1, 40, 60, 30, 2.0, ISO, 6, 3, "smooth"),            # D = 1
    (6, 1, 2, 40, 1, 50, 20, 2.0, ISO, 6, 2, "smooth"),            # H = 1: passes without rows
    (7, 1, 2, 30, 40, 1, 20, 2.0, ISO, 6, 4, "smooth"),            # W = 1
    (8, 1, 3, 1, 1, 1, 1, 1.0, ISO, 3, 1, "smooth"),               # one voxel
    (9, 1, 5, 16, 48, 48, 60, 1.0, ANISO, 6, 3, "smooth"),         # strongly anisotropic spacing
    (10, 1, 33, 20, 24, 28, 40, 1.0, ISO, 5, 255, "smooth"),
    (11, 1, 300, 10, 20, 24, 12, 1e3, ISO, 3, 3, "smooth"),        # C over several shared-memory chunks
    (12, 1, 64, 12, 30, 30, 100, 1e-3, (1.0, 2.0, 1.0), 4, 2, "smooth"),
    (13, 1, 3, 16, 32, 32, 20, 1.0, ISO, 5, 3, "constant"),        # everything ties
    (14, 2, 4, 12, 30, 36, 30, 1.0, ISO, 5, 2, "nonfinite"),       # NaN, +inf, -inf voxels and a NaN row
    (15, 1, 2, 24, 40, 40, 800, 1.0, ISO, 4, 3, "smooth"),         # R = 4: tiles of both kinds
    (16, 1, 2, 40, 96, 96, 300, 1.0, (2.0, 1.0, 1.0), 4, 3, "smooth"),
    (17, 1, 4, 20, 30, 40, 24, 1.0, ISO, 0, 3, "smooth"),          # seeds only
    (18, 1, 2, 30, 30, 30, (3, 5, 2), 1.0, ISO, 5, 1, "smooth"),   # an explicit grid, stride 1
]


def test_exact_sweep_and_both_assign_kernels():
    tile_only = overflowed = mixed = False
    for seed, B, C, D, H, W, K, comp, sp, it, stride, kind in SWEEP:
        f = make_volumes(seed, B, C, D, H, W, kind)
        r, disp = _check(f, K, comp, sp, it, stride)
        tiles = sum(t for t, _ in disp)
        ovf = sum(o for _, o in disp)
        assert 0 <= ovf <= tiles
        tile_only |= tiles > 0 and ovf == 0
        overflowed |= ovf > 0 and ovf == tiles
        mixed |= 0 < ovf < tiles
    assert tile_only and overflowed and mixed


def test_min_size_factor_zero_and_large():
    f = make_volumes(20, 1, 2, 20, 24, 24, "smooth")
    _check(f, 50, 1.0, ISO, 4, 3, min_size_factor=0.0)
    _check(f, 50, 1.0, ISO, 4, 3, min_size_factor=3.0)


def _enforce(lab, K, min_size):
    from fast_slic_b200.supervoxels import enforce_connectivity_3d
    got = enforce_connectivity_3d(torch.from_numpy(lab.view(np.int16)).cuda(), K, min_size)
    assert got.dtype == torch.int16
    return _np(got)


def test_enforcement_on_block_volumes():
    for seed, shape, nlab, block, K, min_size in [(1, (20, 30, 40), 4, (1, 2, 3), 65534, 4),
                                                  (2, (16, 40, 33), 3, (2, 2, 2), 200, 8),
                                                  (3, (9, 17, 70), 5, (1, 1, 1), 50, 2),      # the cap binds
                                                  (4, (30, 30, 30), 2, (3, 3, 3), 65534, 0)]:
        lab = np.stack([block_labels(seed + 10 * b, *shape, nlab, block) for b in range(3)])
        want = np.stack([ref_enforce(v, K, min_size) for v in lab])
        assert np.array_equal(_enforce(lab, K, min_size), want)


def test_enforcement_of_checkerboards_and_labels_above_32767():
    D, H, W = 16, 40, 64  # 40960 voxels, every one its own component
    z, y, x = np.mgrid[0:D, 0:H, 0:W]
    lab = ((z + y + x) % 2).astype(np.uint16)[None]
    got = _enforce(lab, 65534, 1)
    assert np.array_equal(got.view(np.uint16)[0].ravel(), np.arange(D * H * W))
    for K, min_size in [(1000, 1), (7, 1), (65534, 2)]:
        assert np.array_equal(_enforce(lab, K, min_size)[0], ref_enforce(lab[0], K, min_size))


def test_enforcement_with_the_cap_binding_on_tied_areas():
    # 2 x 2 x 2 blocks of random labels: many components of area 8 tie at the K-th place
    lab = block_labels(7, 12, 20, 24, 6, (2, 2, 2))[None]
    comp, _ = components(lab[0])
    area = np.bincount(comp)
    for K in (40, 200):
        assert (area >= 8).sum() > K and (np.sort(area)[::-1][K - 1] == np.sort(area)[::-1][K])
        assert np.array_equal(_enforce(lab, K, 8)[0], ref_enforce(lab[0], K, 8))


def test_enforcement_along_long_predecessor_chains():
    # alternating labels along x, z and y: every component is one voxel and its predecessor is the previous one
    x = (np.arange(30000) % 2).astype(np.uint16).reshape(1, 1, 30000)
    z = (np.arange(5000) % 2).astype(np.uint16).reshape(5000, 1, 1)
    y = (np.arange(3000) % 2).astype(np.uint16).reshape(1, 3000, 1)
    for lab in (x, z, y):
        for K, min_size in [(10, 2), (10, 1), (65534, 1)]:
            assert np.array_equal(_enforce(lab[None], K, min_size)[0], ref_enforce(lab, K, min_size))
    # a staircase: each run's leader sits under the run before
    st = np.zeros((3, 64, 64), np.uint16)
    for i in range(64):
        st[:, i, i:] = i % 3 + 1
    assert np.array_equal(_enforce(st[None], 20, 100)[0], ref_enforce(st, 20, 100))


def test_enforcement_at_one_slice_is_the_2d_enforcer():
    from fast_slic_b200.base_slic import get_cca_engine
    for seed, H, W, nlab, K, thres in [(1, 60, 80, 6, 2000, 4), (2, 90, 70, 3, 500, 9), (3, 33, 129, 12, 4000, 2)]:
        lab = np.stack([block_labels(seed + b, 1, H, W, nlab, (1, 2, 2))[0] for b in range(2)])
        for b in range(2):
            comp, _ = components(lab[b][None])
            assert (np.bincount(comp) >= thres).sum() <= K  # the cap does not bind
        want = torch.from_numpy(lab.view(np.int16)).cuda()
        get_cca_engine(H, W, 2, 0).enforce_connectivity(want, K, thres)
        assert np.array_equal(_enforce(lab[:, None], K, thres)[:, 0], _np(want))


def test_a_volume_at_a_real_size():
    f = make_volumes(90, 1, 2, 160, 256, 256, "smooth")
    r, disp = _check(f, 4000, 1.0, ISO, 4, 3)
    assert r.grid[0] * r.grid[1] * r.grid[2] > 4000 and sum(o for _, o in disp) < sum(t for t, _ in disp)


def test_batch_splits_chunks_streams_and_repeats(monkeypatch):
    from fast_slic_b200 import supervoxels as sv
    f = torch.from_numpy(make_volumes(60, 7, 3, 12, 20, 24, "smooth")).cuda()
    args = (30, 1.5, (1.5, 1.0, 1.0), 5, 3)
    a = sv.supervoxel_slic(f, *args)
    assert _same(a, sv.supervoxel_slic(f, *args))
    singles = [sv.supervoxel_slic(f[b:b + 1], *args) for b in range(7)]
    assert _same(a, [torch.cat([s[i] for s in singles]) for i in range(4)])
    one = sv._lib.lib().fslic_b200_sv_slic_scratch_bytes(3, 12, 20, 24, 3, *a.grid, 3, 5)
    with monkeypatch.context() as m:
        m.setattr(sv, "SUPERVOXEL_SCRATCH_CAP", one)  # chunks of 3 volumes: 3 + 3 + 1
        assert _same(a, sv.supervoxel_slic(f, *args))
        lab = a.labels.clone()
        e = sv.enforce_connectivity_3d(lab, 10, 50)
        assert torch.equal(e, torch.cat([sv.enforce_connectivity_3d(lab[b:b + 1], 10, 50) for b in range(7)]))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        b = sv.supervoxel_slic(f, *args)
    s.synchronize()
    assert _same(a, b)
    perm = torch.tensor([3, 0, 6, 1, 5, 2, 4], device="cuda")
    assert _same([x[perm] for x in a[:4]], sv.supervoxel_slic(f[perm].contiguous(), *args))


def test_graph_capture_replays_the_eager_result():
    from fast_slic_b200.supervoxels import enforce_connectivity_3d, supervoxel_slic
    f = torch.from_numpy(make_volumes(70, 3, 2, 10, 24, 28, "smooth")).cuda()
    want = supervoxel_slic(f, 30, 1.0, (1.0, 1.0, 1.0), 5, 3)
    want_e = enforce_connectivity_3d(want.labels, 12, 40)
    x = torch.zeros_like(f)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        enforce_connectivity_3d(supervoxel_slic(x, 30, 1.0, (1.0, 1.0, 1.0), 5, 3).labels, 12, 40)  # warm-up
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        got = supervoxel_slic(x, 30, 1.0, (1.0, 1.0, 1.0), 5, 3)
        got_e = enforce_connectivity_3d(got.labels, 12, 40)
    x.copy_(f)
    graph.replay()
    torch.cuda.synchronize()
    assert _same(got, want) and torch.equal(got_e, want_e)


def test_empty_batch():
    from fast_slic_b200.supervoxels import enforce_connectivity_3d, supervoxel_slic
    r = supervoxel_slic(torch.zeros((0, 3, 4, 10, 12), device="cuda"), 8, 1.0)
    assert tuple(r.labels.shape) == (0, 4, 10, 12) and tuple(r.position.shape[::2]) == (0, 3)
    assert tuple(r.features.shape)[::2] == (0, 3) and r.count.shape[0] == 0
    assert enforce_connectivity_3d(torch.zeros((0, 2, 3, 4), dtype=torch.int16, device="cuda"), 4, 1).shape[0] == 0
