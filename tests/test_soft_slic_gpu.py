"""Differentiable soft SLIC on the GPU (fast_slic_b200.soft_slic) against the numpy restatement (soft_slic_cases.py):
the forwards of soft_assign, soft_pool, soft_unpool and soft_slic and every backward bit for bit (NaN as a class) over
a seeded sweep of channel counts, grids, image shapes, iteration counts, ties, non-finite pixels, underflowing
associations and zero-weight cells; soft_slic's gradients through 5 iterations against float64 autograd; the labels
against the connectivity enforcer; batch, stream and CUDA graph invariance; and a small SSN-style training loop."""
import numpy as np
import pytest
import torch

from soft_slic_cases import (F32, Image, dense_torch, grid_labels, make_features, nan_class_equal,
                             ref_soft_slic_image)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _needs_cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _np(x):
    return x.detach().cpu().numpy()


def _cuda(x, grad=False):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda().requires_grad_(grad)


def _bits(a, b):
    return all(torch.equal(x.view(torch.int32) if x.dtype == torch.float32 else x,
                           y.view(torch.int32) if y.dtype == torch.float32 else y) for x, y in zip(a, b))


# (seed, B, C, H, W, grid, kind, scale, n_iter)
SWEEP = [
    (1, 2, 1, 37, 53, (5, 7), "smooth", 1.0, 3),       # cells that do not divide the image
    (2, 1, 300, 20, 24, (3, 4), "smooth", 0.3, 2),     # C over many channel groups
    (3, 1, 33, 30, 40, (1, 1), "smooth", 1.0, 1),      # one cell
    (4, 2, 3, 1, 80, (1, 10), "smooth", 1.0, 5),       # one row, a 1 x W grid
    (5, 1, 3, 60, 1, (7, 1), "smooth", 1.0, 4),        # one column, an H x 1 grid
    (6, 1, 2, 12, 10, (12, 10), "smooth", 1.0, 10),    # a cell per pixel
    (7, 1, 9, 70, 90, (6, 8), "smooth", 1.0, 5),       # blocks wider than a warp
    (8, 1, 3, 20, 30, (4, 5), "constant", 1.0, 3),     # everything ties
    (9, 2, 4, 25, 33, (4, 5), "nonfinite", 1.0, 2),
    (10, 1, 3, 30, 30, (5, 5), "smooth", 30.0, 2),     # expf underflows most q to exactly 0
]


def _per_function(f, grid, seed):
    """Every function's forward and backward on the GPU against the restatement, image by image, at random centroids
    (one far away from everything, so its q underflow to 0 and its Z is 0), values and output gradients."""
    from fast_slic_b200.soft_slic import soft_assign, soft_pool, soft_unpool
    B, C, H, W = f.shape
    K = grid[0] * grid[1]
    rng = np.random.RandomState(seed)
    mu = (rng.randn(B, C, K) * f[np.isfinite(f)].std()).astype(F32)
    mu[:, :, K // 2] = 1e4
    v, M = rng.randn(B, C, H, W).astype(F32), rng.randn(B, C, K).astype(F32)
    g9, gK, gP = rng.randn(B, 9, H, W).astype(F32), rng.randn(B, C, K).astype(F32), rng.randn(B, C, H, W).astype(F32)

    F, m = _cuda(f, True), _cuda(mu, True)
    q = soft_assign(F, m, grid)
    gF, gm = torch.autograd.grad(q, (F, m), _cuda(g9))
    qc = _cuda(_np(q), True)
    V = _cuda(v, True)
    Mp = soft_pool(V, qc, grid)
    gV, gQp = torch.autograd.grad(Mp, (V, qc), _cuda(gK))
    Mc = _cuda(M, True)
    up = soft_unpool(Mc, qc, grid)
    gMu, gQu = torch.autograd.grad(up, (Mc, qc), _cuda(gP))
    zero_cell = False
    for b in range(B):
        im = Image(H, W, *grid)
        rq = im.assign(f[b], mu[b])
        assert nan_class_equal(_np(q[b]), rq)
        gd, rgF, rgm = im.assign_backward(f[b], mu[b], rq, g9[b])
        assert nan_class_equal(_np(gF[b]), rgF) and nan_class_equal(_np(gm[b]), rgm)
        rM, Z = im.pool(v[b], rq)
        assert nan_class_equal(_np(Mp[b]), rM)
        zero_cell |= bool((Z == 0).any())
        rgV, rgQ = im.pool_backward(v[b], rq, rM, Z, gK[b])
        assert nan_class_equal(_np(gV[b]), rgV) and nan_class_equal(_np(gQp[b]), rgQ)
        assert nan_class_equal(_np(up[b]), im.unpool(M[b], rq))
        rgM, rgQ = im.unpool_backward(M[b], rq, gP[b])
        assert nan_class_equal(_np(gMu[b]), rgM) and nan_class_equal(_np(gQu[b]), rgQ)
    return zero_cell


def test_exact_sweep():
    from fast_slic_b200.soft_slic import soft_slic
    zero_cell = underflow = False
    for seed, B, C, H, W, grid, kind, scale, n_iter in SWEEP:
        f = make_features(seed, B, C, H, W, kind, scale)
        zero_cell |= _per_function(f, grid, seed)
        r = soft_slic(_cuda(f), grid, n_iter, min_size_factor=None)
        assert r.grid == grid and r.labels.dtype == torch.int16
        for b in range(B):
            lab, q, mu = ref_soft_slic_image(f[b], grid, n_iter)
            assert nan_class_equal(_np(r.assoc[b]), q), (seed, b)
            assert nan_class_equal(_np(r.centroids[b]), mu), (seed, b)
            assert np.array_equal(_np(r.labels[b]).astype(np.int64), lab), (seed, b)
            underflow |= bool((q[Image(H, W, *grid).valid] == 0).any())
    assert zero_cell and underflow


def test_labels_are_the_enforced_argmax_map():
    from fast_slic_b200.base_slic import get_cca_engine
    from fast_slic_b200.feature_slic import min_size_threshold, superpixel_size
    from fast_slic_b200.soft_slic import soft_slic
    f = make_features(20, 2, 4, 64, 80, "smooth", 2.0)
    grid, msf = (8, 10), 0.5
    r = soft_slic(_cuda(f), grid, 4, msf)
    want = torch.from_numpy(np.stack([ref_soft_slic_image(f[b], grid, 4)[0] for b in range(2)]).astype(np.int16)).cuda()
    raw = want.clone()
    get_cca_engine(64, 80, 2, 0).enforce_connectivity(want, 80, min_size_threshold(superpixel_size(64, 80, 80), msf))
    assert torch.equal(r.labels, want)
    assert not torch.equal(raw, want)  # the argmax map had fragments to absorb


def test_end_to_end_gradients_against_float64_autograd():
    """soft_slic's feature gradient through the initial cell means and 5 iterations against float64 autograd of
    dense_torch.  Each float32 operation is off by at most half an ulp; through 5 softmax iterations these errors grow
    to a few 1e-5 of the gradient's scale at these feature scales, so rtol 1e-3 with an absolute term of 1e-3 times
    the largest magnitude has a margin and still fails any wrong term, which is O(1)."""
    from fast_slic_b200.soft_slic import soft_slic
    grid, n_iter = (3, 4), 5
    f = make_features(30, 1, 3, 24, 30, "smooth", 0.5)
    rng = np.random.RandomState(31)
    g9, gK = rng.randn(1, 9, 24, 30).astype(F32), rng.randn(1, 3, 12).astype(F32)
    x = _cuda(f, True)
    r = soft_slic(x, grid, n_iter, min_size_factor=None)
    ((r.assoc * _cuda(g9)).sum() + (r.centroids * _cuda(gK)).sum()).backward()

    assign, pool, unpool = dense_torch(24, 30, grid)
    F = torch.tensor(f[0], dtype=torch.float64, requires_grad=True)
    lab = torch.from_numpy(grid_labels(24, 30, *grid).ravel())
    cnt = torch.bincount(lab, minlength=12).to(torch.float64)
    mu = torch.zeros(3, 12, dtype=torch.float64).index_add(1, lab, F.reshape(3, -1)) / cnt
    for _ in range(n_iter):
        q = assign(F, mu)
        mu = pool(F, q)
    ((q * torch.tensor(g9[0], dtype=torch.float64).reshape(9, -1)).sum() +
     (mu * torch.tensor(gK[0], dtype=torch.float64)).sum()).backward()
    want = F.grad.numpy()
    np.testing.assert_allclose(_np(r.assoc[0]).reshape(9, -1), q.detach().numpy(), rtol=1e-3, atol=1e-5)
    np.testing.assert_allclose(_np(x.grad[0]), want, rtol=1e-3, atol=1e-3 * np.abs(want).max())


def test_batch_stream_and_graph_invariance():
    from fast_slic_b200.soft_slic import soft_pool, soft_slic, soft_unpool

    def run(x, grad=True):
        x = x.detach().clone().requires_grad_(grad)
        r = soft_slic(x, (6, 7), 3)
        loss = soft_unpool(soft_pool(x, r.assoc, r.grid), r.assoc, r.grid).square().sum() + r.centroids.sum()
        if grad:
            loss.backward()
        return [r.labels, r.assoc.detach(), r.centroids.detach()] + ([x.grad] if grad else [])

    f = _cuda(make_features(40, 5, 6, 48, 64, "smooth"))
    a = run(f)
    assert _bits(a, run(f))
    singles = [run(f[b:b + 1]) for b in range(5)]
    assert _bits(a, [torch.cat([s[i] for s in singles]) for i in range(4)])
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        b = run(f)
    s.synchronize()
    assert _bits(a, b)
    # forward under CUDA graph capture, connectivity enforcement included
    x = torch.zeros_like(f)
    torch.cuda.synchronize()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        run(x, grad=False)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        got = run(x, grad=False)
    x.copy_(f)
    graph.replay()
    torch.cuda.synchronize()
    assert _bits(a[:3], got)


def test_ssn_training_steps_are_finite_and_reproducible():
    from fast_slic_b200.soft_slic import soft_pool, soft_slic, soft_unpool
    img = _cuda(make_features(50, 2, 3, 40, 48, "smooth"))
    target = (torch.arange(40, device="cuda")[:, None] // 10 * 4 + torch.arange(48, device="cuda")[None] // 12) % 5
    onehot = torch.nn.functional.one_hot(target, 5).permute(2, 0, 1)[None].expand(2, 5, 40, 48).float().contiguous()
    yx = torch.stack(torch.meshgrid(torch.arange(40.), torch.arange(48.), indexing="ij")).cuda()[None].expand(2, 2, 40, 48)

    def train():
        torch.manual_seed(0)
        conv = torch.nn.Conv2d(3, 6, 3, padding=1).cuda()
        opt = torch.optim.SGD(conv.parameters(), lr=0.1)
        grads = []
        for _ in range(2):
            opt.zero_grad()
            feats = torch.cat([conv(img), yx * 0.1], 1)
            r = soft_slic(feats, 30, 5)
            recon = soft_unpool(soft_pool(onehot, r.assoc, r.grid), r.assoc, r.grid)
            loss = (recon - onehot).square().mean()
            loss.backward()
            grads.append(conv.weight.grad.clone())
            opt.step()
        return grads

    flags = torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    try:
        a, b = train(), train()
    finally:
        torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = flags
    assert all(torch.isfinite(g).all() and g.abs().sum() > 0 for g in a)
    assert _bits(a, b)


def test_empty_inputs():
    from fast_slic_b200.soft_slic import soft_slic
    r = soft_slic(torch.zeros((0, 3, 10, 12), device="cuda"), (2, 3))
    assert tuple(r.labels.shape) == (0, 10, 12) and tuple(r.assoc.shape) == (0, 9, 10, 12)
    assert tuple(r.centroids.shape) == (0, 3, 6)
