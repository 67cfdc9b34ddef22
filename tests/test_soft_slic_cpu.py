"""soft_slic without a GPU: the numpy restatement (soft_slic_cases.py) against a plain per-pixel, per-cell loop, its
backward formulas against float64 autograd of an independent dense implementation, the grid rule, the argument checks
(they come before any device work) and the ABI."""
import os
import re

import numpy as np
import pytest
import torch

from soft_slic_cases import F32, Image, dense_torch, expf, make_features, nan_class_equal, ref_soft_slic_image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cell(i, j, H, W, nh, nw):
    return i * nh // H, j * nw // W


def _slots(i, j, H, W, nh, nw):
    """[(n, k)] of the valid slots of pixel (i, j), in n order."""
    a, b = _cell(i, j, H, W, nh, nw)
    return [(n, (a + n // 3 - 1) * nw + b + n % 3 - 1) for n in range(9)
            if 0 <= a + n // 3 - 1 < nh and 0 <= b + n % 3 - 1 < nw]


def _block(k, H, W, nh, nw):
    """[(i, j, n)] of cell k's block in raster order, n the slot through which (i, j) sees k."""
    out = []
    for i in range(H):
        for j in range(W):
            for n, kk in _slots(i, j, H, W, nh, nw):
                if kk == k:
                    out.append((i, j, n))
    return out


def _lanes(values):
    lanes = [F32(0)] * 32
    for m, v in enumerate(values):
        lanes[m % 32] = F32(lanes[m % 32] + v)
    for off in (16, 8, 4, 2, 1):
        lanes = [F32(lanes[l] + lanes[l ^ off]) for l in range(32)]
    return lanes[0]


def loop_assign(f, mu, grid):
    C, H, W = f.shape
    q = np.zeros((9, H, W), F32)
    for i in range(H):
        for j in range(W):
            sl = _slots(i, j, H, W, *grid)
            d = {}
            for n, k in sl:
                acc = F32(0)
                for c in range(C):
                    t = F32(f[c, i, j] - mu[c, k])
                    acc = F32(acc + F32(t * t))
                d[n] = acc
            m = None
            for n, _ in sl:
                m = d[n] if m is None else np.fmin(m, d[n])
            e = {n: expf(np.array([F32(m - d[n])]))[0] for n, _ in sl}
            s = F32(0)
            for n, _ in sl:
                s = F32(s + e[n])
            for n, _ in sl:
                q[n, i, j] = F32(e[n] / s)
    return q


def loop_block_sum(term, K, H, W, grid):
    """[K] sums over every cell's block of term(k, i, j, n)."""
    return np.array([_lanes([term(k, i, j, n) for i, j, n in _block(k, H, W, *grid)]) for k in range(K)], F32)


def loop_slot_sum(term, i, j, H, W, grid):
    acc = F32(0)
    for n, k in _slots(i, j, H, W, *grid):
        acc = F32(acc + term(n, k))
    return acc


def loop_all(f, mu, v, M, g9, gK, gP, grid):
    """Every forward and backward of the contract, one scalar at a time."""
    C, H, W = f.shape
    K = grid[0] * grid[1]
    q = loop_assign(f, mu, grid)
    A = np.stack([loop_block_sum(lambda k, i, j, n: F32(q[n, i, j] * v[c, i, j]), K, H, W, grid) for c in range(C)])
    Z = loop_block_sum(lambda k, i, j, n: q[n, i, j], K, H, W, grid)
    Mp = np.where(Z != 0, A / Z, F32(0)).astype(F32)
    up = np.zeros((C, H, W), F32)
    gd = np.zeros((9, H, W), F32)
    gF = np.zeros((C, H, W), F32)
    for i in range(H):
        for j in range(W):
            for c in range(C):
                up[c, i, j] = loop_slot_sum(lambda n, k: F32(q[n, i, j] * M[c, k]), i, j, H, W, grid)
            t = loop_slot_sum(lambda n, k: F32(q[n, i, j] * g9[n, i, j]), i, j, H, W, grid)
            for n, k in _slots(i, j, H, W, *grid):
                gd[n, i, j] = F32(q[n, i, j] * F32(t - g9[n, i, j]))
            for c in range(C):
                gF[c, i, j] = F32(2) * loop_slot_sum(
                    lambda n, k: F32(gd[n, i, j] * F32(f[c, i, j] - mu[c, k])), i, j, H, W, grid)
    gmu = np.stack([F32(-2) * loop_block_sum(lambda k, i, j, n: F32(gd[n, i, j] * F32(f[c, i, j] - mu[c, k])),
                                             K, H, W, grid) for c in range(C)])
    # soft_pool backward at gK
    gA = np.zeros((C, K), F32)
    gZ = np.zeros(K, F32)
    for k in range(K):
        if Z[k] != 0:
            acc = F32(0)
            for c in range(C):
                gA[c, k] = F32(gK[c, k] / Z[k])
                acc = F32(acc + F32(gA[c, k] * Mp[c, k]))
            gZ[k] = -acc
    gV = np.zeros((C, H, W), F32)
    gQp = np.zeros((9, H, W), F32)
    gQu = np.zeros((9, H, W), F32)
    for i in range(H):
        for j in range(W):
            for c in range(C):
                gV[c, i, j] = loop_slot_sum(lambda n, k: F32(q[n, i, j] * gA[c, k]), i, j, H, W, grid)
            for n, k in _slots(i, j, H, W, *grid):
                acc, accu = F32(0), F32(0)
                for c in range(C):
                    acc = F32(acc + F32(gA[c, k] * v[c, i, j]))
                    accu = F32(accu + F32(gP[c, i, j] * M[c, k]))
                gQp[n, i, j] = F32(acc + gZ[k])
                gQu[n, i, j] = accu
    gMu = np.stack([loop_block_sum(lambda k, i, j, n: F32(q[n, i, j] * gP[c, i, j]), K, H, W, grid)
                    for c in range(C)])
    return dict(q=q, M=Mp, Z=Z, up=up, gd=gd, gF=gF, gmu=gmu, gV=gV, gQp=gQp, gMu=gMu, gQu=gQu)


def restated_all(f, mu, v, M, g9, gK, gP, grid):
    im = Image(f.shape[1], f.shape[2], *grid)
    q = im.assign(f, mu)
    Mp, Z = im.pool(v, q)
    gd, gF, gmu = im.assign_backward(f, mu, q, g9)
    gV, gQp = im.pool_backward(v, q, Mp, Z, gK)
    gMu, gQu = im.unpool_backward(M, q, gP)
    return dict(q=q, M=Mp, Z=Z, up=im.unpool(M, q), gd=gd, gF=gF, gmu=gmu, gV=gV, gQp=gQp, gMu=gMu, gQu=gQu)


def _inputs(seed, C, H, W, grid, kind="smooth", scale=1.0):
    rng = np.random.RandomState(seed + 1000)
    K = grid[0] * grid[1]
    f = make_features(seed, 1, C, H, W, kind, scale)[0]
    mu = (rng.randn(C, K) * scale).astype(F32)
    v = rng.randn(C, H, W).astype(F32)
    M = rng.randn(C, K).astype(F32)
    g9, gK, gP = rng.randn(9, H, W).astype(F32), rng.randn(C, K).astype(F32), rng.randn(C, H, W).astype(F32)
    return f, mu, v, M, g9, gK, gP


@pytest.mark.parametrize("seed,C,H,W,grid,kind,scale", [
    (1, 2, 7, 9, (2, 3), "smooth", 1.0),
    (2, 3, 11, 13, (3, 4), "smooth", 1.0),       # cells that do not divide the image
    (3, 1, 1, 10, (1, 4), "smooth", 1.0),        # one row
    (4, 2, 9, 1, (3, 1), "smooth", 1.0),         # one column
    (5, 2, 6, 6, (1, 1), "smooth", 1.0),         # one cell: every other slot invalid
    (6, 1, 5, 6, (5, 6), "smooth", 1.0),         # a cell per pixel
    (7, 2, 6, 7, (2, 2), "constant", 1.0),       # everything ties
    (8, 2, 8, 9, (2, 3), "nonfinite", 1.0),
    (9, 2, 8, 9, (3, 3), "smooth", 30.0),        # expf underflows some q to 0
])
def test_restatement_against_a_pixel_loop(seed, C, H, W, grid, kind, scale):
    args = _inputs(seed, C, H, W, grid, kind, scale)
    want, got = loop_all(*args, grid), restated_all(*args, grid)
    for name in want:
        assert nan_class_equal(got[name], want[name]), name
    if scale > 1:
        assert (got["q"][Image(H, W, *grid).valid] == 0).any()


def test_zero_weight_cells_pool_to_zero():
    f, mu, v, M, g9, gK, gP = _inputs(1, 2, 6, 6, (2, 2))
    im = Image(6, 6, 2, 2)
    q = np.zeros((9, 6, 6), F32)
    Mp, Z = im.pool(v, q)
    assert not Z.any() and not Mp.any() and not np.signbit(Mp).any()
    gV, gQ = im.pool_backward(v, q, Mp, Z, gK)
    assert not gV.any() and not gQ.any() and not np.signbit(gQ).any()


def test_backward_formulas_against_float64_autograd():
    """The restated gradients of each function against float64 autograd of dense_torch at the same float32 inputs.
    The restatement rounds every operation to float32 (relative error about 6e-8 each) and sums up to a few hundred
    terms, which gives relative differences up to about 1e-5 of the gradient's scale: rtol 1e-4 with an absolute
    term of 1e-4 times the largest gradient magnitude leaves a margin without hiding a wrong formula, which would differ
    by O(1)."""
    grid, C, H, W = (3, 4), 3, 12, 14
    f, mu, v, M, g9, gK, gP = _inputs(3, C, H, W, grid)
    assign, pool, unpool = dense_torch(H, W, grid)
    got = restated_all(f, mu, v, M, g9, gK, gP, grid)

    def check(restated, want):
        want = want.detach().numpy().astype(np.float64)
        np.testing.assert_allclose(restated, want, rtol=1e-4, atol=1e-4 * np.abs(want).max())

    F = torch.tensor(f, dtype=torch.float64, requires_grad=True)
    m = torch.tensor(mu, dtype=torch.float64, requires_grad=True)
    q = assign(F, m)
    check(got["q"].reshape(9, -1), q)
    (q * torch.tensor(g9, dtype=torch.float64).reshape(9, -1)).sum().backward()
    check(got["gF"], F.grad)
    check(got["gmu"], m.grad)

    qd = torch.tensor(got["q"], dtype=torch.float64).reshape(9, -1).requires_grad_(True)
    V = torch.tensor(v, dtype=torch.float64, requires_grad=True)
    (pool(V, qd) * torch.tensor(gK, dtype=torch.float64)).sum().backward()
    check(got["gV"], V.grad)
    check(got["gQp"].reshape(9, -1), qd.grad)

    qd.grad = None
    Md = torch.tensor(M, dtype=torch.float64, requires_grad=True)
    (unpool(Md, qd) * torch.tensor(gP, dtype=torch.float64)).sum().backward()
    check(got["gMu"], Md.grad)
    check(got["gQu"].reshape(9, -1), qd.grad)


def test_soft_slic_loop_and_argmax():
    f = make_features(5, 1, 3, 20, 24)[0]
    lab, q, mu, hist = ref_soft_slic_image(f, (3, 4), 3, with_history=True)
    im = Image(20, 24, 3, 4)
    assert len(hist) == 3 and nan_class_equal(hist[1][0], hist[0][2]) and nan_class_equal(mu, hist[2][2])
    assert nan_class_equal(q, hist[2][1])
    # the first largest association among the valid slots; a NaN wins
    qq = np.where(im.valid, np.float32(0.1), np.float32(0))
    qq[5, 3, 3], qq[7, 3, 3] = 0.5, 0.5
    qq[2, 10, 10], qq[6, 10, 10] = np.nan, 0.9
    got = im.argmax(qq)
    assert not im.valid[:3, 3, 3].any() and got[3, 3] == im.k[5, 3, 3]  # ties: the first valid slot
    assert im.valid[:, 10, 10].all() and got[10, 10] == im.k[2, 10, 10]
    assert got[15, 15] == im.k[0, 15, 15]


def test_cell_grid():
    from fast_slic_b200.soft_slic import cell_grid
    from soft_slic_cases import cell_grid as ref_grid
    assert cell_grid(720, 1280, 1600) == (30, 53) == ref_grid(720, 1280, 1600)
    assert cell_grid(37, 53, (5, 7)) == (5, 7) and cell_grid(37, 53, [5, 7]) == (5, 7)
    assert cell_grid(1, 100, 10) == (1, 31) and cell_grid(100, 1, 10) == (31, 1)
    assert cell_grid(5, 5, 1000) == (5, 5) and cell_grid(50, 50, 1) == (1, 1)
    assert cell_grid(3, 4, (3, 4)) == (3, 4) and cell_grid(0, 4, 7) == (1, 1)
    assert cell_grid(300, 300, 65534) == (255, 255) == ref_grid(300, 300, 65534)  # 65025 cells
    for H, W, K in [(720, 1280, 1600), (37, 53, 35), (480, 640, 1000), (7, 3000, 200)]:
        assert cell_grid(H, W, K) == ref_grid(H, W, K)
    for args, msg in [((5, 5, 0), "num_cells"), ((5, 5, 1.5), "num_cells"), ((5, 5, (0, 1)), "nh"),
                      ((5, 5, (6, 1)), "nh"), ((5, 5, (1, 6)), "nw"), ((5, 5, (1, 2, 3)), "num_cells"),
                      ((300, 300, (256, 256)), "cells"), ((1000, 1000, 100000), "cells"), ((-1, 5, 3), "H")]:
        with pytest.raises(ValueError, match=msg):
            cell_grid(*args)


def test_argument_errors():
    from fast_slic_b200.soft_slic import soft_assign, soft_pool, soft_slic, soft_unpool
    x = torch.zeros((2, 3, 8, 9))
    mu, q = torch.zeros((2, 3, 6)), torch.zeros((2, 9, 8, 9))
    g = (2, 3)
    for fn, args, kw, msg in [
        (soft_slic, (x.numpy(), 6), {}, "torch.from_numpy"), (soft_slic, (x.double(), 6), {}, "float32"),
        (soft_slic, (x[0], 6), {}, "dimensions"), (soft_slic, (x[:, :0], 6), {}, "channel"),
        (soft_slic, (torch.zeros(1, 1, 1, 1).expand(1, 1, 32768, 32768), 6), {}, "pixels"),
        (soft_slic, (x, 0), {}, "num_cells"), (soft_slic, (x, (9, 1)), {}, "nh"), (soft_slic, (x, (1, 10)), {}, "nw"),
        (soft_slic, (x, 6), {"n_iter": 0}, "n_iter"), (soft_slic, (x, 6), {"n_iter": 1.0}, "n_iter"),
        (soft_slic, (x, 6), {"min_size_factor": -1}, "min_size_factor"),
        (soft_slic, (x, 6), {"min_size_factor": "a"}, "min_size_factor"),
        (soft_slic, (torch.zeros(1, 1, 1, 1).expand(2 ** 15 + 1, 1, 256, 256), (128, 256)), {}, "B\\*K"),
        (soft_slic, (x, 6), {}, "cuda"),
        (soft_assign, (x, mu, 6), {}, "grid must be"), (soft_assign, (x, mu, (3, 3)), {}, "centroids must be"),
        (soft_assign, (x, mu[..., :5], g), {}, "centroids must be"), (soft_assign, (x, mu.double(), g), {}, "float32"),
        (soft_assign, (x, mu, (9, 1)), {}, "nh"), (soft_assign, (x, mu, g), {}, "cuda"),
        (soft_pool, (x, q[:, :8], g), {}, "assoc must be"), (soft_pool, (x, q[:1], g), {}, "assoc must be"),
        (soft_pool, (x, q.half(), g), {}, "float32"), (soft_pool, (x, q, (1, 10)), {}, "nw"),
        (soft_pool, (x, q, g), {}, "cuda"),
        (soft_unpool, (mu, q[:, :, :, :2], g), {}, "nw"), (soft_unpool, (mu, q[:, :8], g), {}, "assoc must be"),
        (soft_unpool, (mu[:1], q, g), {}, "values must be"), (soft_unpool, (mu[:, :0], q, g), {}, "channel"),
        (soft_unpool, (mu, q, g), {}, "cuda"),
    ]:
        with pytest.raises(ValueError, match=msg):
            fn(*args, **kw)
    # the limits themselves pass every check but the device one
    for fn, args, kw in [(soft_slic, (torch.zeros(1, 1, 1, 1).expand(2 ** 14, 1, 256, 258), (254, 258)), {}),
                         (soft_slic, (x, (8, 9)), {"min_size_factor": None}), (soft_slic, (x[:0], 6), {}),
                         (soft_slic, (torch.zeros(2, 1, 0, 5), (1, 1)), {}),
                         (soft_assign, (x[:, :1], mu[:, :1, :1], (1, 1)), {})]:
        with pytest.raises(ValueError, match="cuda"):
            fn(*args, **kw)


def test_abi_declares_and_binds_the_entry_points():
    from fast_slic_b200 import _lib
    L = _lib.lib()
    header = open(os.path.join(ROOT, "include", "fslic_b200.h")).read()
    declared = set(re.findall(r"\b(fslic_b200_\w+)\s*\(", header))
    for name, nargs in (("fslic_b200_soft_assign", 11), ("fslic_b200_soft_assign_backward", 15),
                        ("fslic_b200_soft_pool", 12), ("fslic_b200_soft_pool_backward", 17),
                        ("fslic_b200_soft_unpool", 11), ("fslic_b200_soft_unpool_backward", 13),
                        ("fslic_b200_soft_labels", 9)):
        assert name in declared and name in _lib.EXPORTED_SYMBOLS
        assert len(getattr(L, name).argtypes) == nargs
    # bad shapes are refused before any device work; an empty batch does nothing
    f = L.fslic_b200_soft_assign
    for args in [(0, -1, 8, 8, 3, 2, 2), (0, 1, 0, 8, 3, 1, 1), (0, 1, 8, 8, 0, 2, 2), (0, 1, 8, 8, 3, 9, 2),
                 (0, 1, 8, 8, 3, 2, 0), (0, 1, 300, 300, 3, 256, 256), (0, 1 << 15, 256, 256, 1, 128, 257)]:
        assert f(*args, None, None, None, None) == -1, args
    assert f(0, 0, 8, 8, 3, 2, 2, None, None, None, None) == 0
