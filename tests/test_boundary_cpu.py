"""Boundary statistics without a GPU: the ABI declarations, the argument checks (they come before any device work), the
numpy restatement against independent computations (region adjacency's boundary counts, a brute-force loop over pixel
pairs, float64 means), and hand-computed answers."""
import os
import re
import types

import numpy as np
import pytest
import torch

from boundary_cases import entry_keys, ref_boundary
from pool_cases import nan_class_equal
from rag_cases import ref_rag

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NO_SIZE = 2 ** 64 - 1
nan = np.float32("nan")


def test_abi_declares_and_binds_the_boundary_entry_points():
    from fast_slic_b200 import _lib
    L = _lib.lib()
    header = open(os.path.join(ROOT, "include", "fslic_b200.h")).read()
    declared = set(re.findall(r"\b(fslic_b200_\w+)\s*\(", header))
    for name, nargs in (("fslic_b200_boundary_select_scratch_bytes", 5), ("fslic_b200_boundary_select_batch", 11),
                        ("fslic_b200_boundary_stats_scratch_bytes", 2), ("fslic_b200_boundary_stats_batch", 25)):
        assert name in declared and name in _lib.EXPORTED_SYMBOLS
        assert len(getattr(L, name).argtypes) == nargs
    f = L.fslic_b200_boundary_select_scratch_bytes
    assert int(f(1, 10, 10, 0, 4)) == NO_SIZE and int(f(1, 10, 10, 65535, 4)) == NO_SIZE
    assert int(f(1, 10, 10, 5, 6)) == NO_SIZE and int(f(-1, 10, 10, 5, 4)) == NO_SIZE
    assert int(f(1, 2 ** 15, 2 ** 14 + 1, 5, 4)) == NO_SIZE  # over 2^29 pixels
    assert int(f(600, 1024, 1024, 5, 8)) == NO_SIZE  # more than 2^31 - 1 pixel pairs
    assert int(f(0, 10, 10, 5, 4)) == 256
    assert 4 * 2 * 720 * 1280 <= int(f(1, 720, 1280, 1600, 4)) < 4 * 2 * 720 * 1280 + (1 << 24)
    assert int(f(1, 720, 1280, 1600, 8)) >= 4 * 4 * 720 * 1280
    g = L.fslic_b200_boundary_stats_scratch_bytes
    assert int(g(-1, 0)) == NO_SIZE and int(g(0, -1)) == NO_SIZE
    assert int(g(2 ** 31, 0)) == NO_SIZE and int(g(0, 2 ** 31)) == NO_SIZE
    assert 25 * 1000 + 24 * 500 <= int(g(1000, 500)) < NO_SIZE


def _graph(n_nodes, E=3, dtype=torch.int64):
    return types.SimpleNamespace(indptr=torch.zeros(1, dtype=torch.int64).expand(n_nodes + 1),
                                 edge_index=torch.zeros((2, E), dtype=dtype))


def test_argument_errors():
    from fast_slic_b200.region_graph import boundary_stats
    B, K, H, W = 2, 10, 5, 7
    lab = torch.zeros((B, H, W), dtype=torch.int16)
    val = torch.zeros((B, 3, H, W), dtype=torch.float32)
    g = _graph(B * K)
    for args, msg in [
        ((lab.numpy(), K, g, val), "torch.from_numpy"),
        ((lab.int(), K, g, val), "int16"), ((lab[0], K, g, val), "dimensions"),
        ((lab, K, g, val.numpy()), "values must be a cuda tensor"),
        ((lab, K, g, val.double()), "values"), ((lab, K, g, val[0]), "values"),
        ((lab, K, g, val[:1]), "do not match"), ((lab, K, g, val[:, :, :4]), "do not match"),
        ((lab, K, g, val[:, :, :, :6]), "do not match"), ((lab, K, g, val[:, :0]), "at least one channel"),
        ((lab, 0, g, val), "K must be"), ((lab, 65535, g, val), "K must be"), ((lab, 2.0, g, val), "K must be"),
        ((torch.zeros((1, 2 ** 15, 2 ** 14 + 1), dtype=torch.int16).expand(1, -1, -1), K, _graph(K),
          torch.zeros(1, 1, 1, 1).expand(1, 1, 2 ** 15, 2 ** 14 + 1)), "exceed"),
        ((lab, K, _graph(B * K - 1), val), "indptr"), ((lab, K, _graph(B * K + 1), val), "indptr"),
        ((lab, K, types.SimpleNamespace(indptr=[0] * (B * K + 1), edge_index=g.edge_index), val), "indptr"),
        ((lab, K, _graph(B * K, dtype=torch.int32), val), "edge_index"),
        ((lab, K, types.SimpleNamespace(indptr=g.indptr, edge_index=torch.zeros((3, 3), dtype=torch.int64)), val),
         "edge_index"),
        ((lab, K, types.SimpleNamespace(indptr=g.indptr, edge_index=torch.zeros(3, dtype=torch.int64)), val),
         "edge_index"),
        ((lab, K, g, val), "cuda"),  # cpu tensors, every other check passed
    ]:
        with pytest.raises(ValueError, match=msg):
            boundary_stats(*args)
    for conn in (0, 6, 4.0, "4", None):
        with pytest.raises(ValueError, match="connectivity"):
            boundary_stats(lab, K, g, val, conn)
    if torch.cuda.is_available():
        gc = types.SimpleNamespace(indptr=g.indptr.cuda(), edge_index=g.edge_index.cuda())
        for graph, v, name in ((gc, val, "values"),
                               (types.SimpleNamespace(indptr=g.indptr, edge_index=gc.edge_index), val.cuda(),
                                "graph.indptr"),
                               (types.SimpleNamespace(indptr=gc.indptr, edge_index=g.edge_index), val.cuda(),
                                "graph.edge_index")):
            with pytest.raises(ValueError, match=name + " is on"):
                boundary_stats(lab.cuda(), K, graph, v)
    # the limits themselves pass every check but the device one
    for args in [(lab, 1, _graph(B), val), (lab, 65534, _graph(B * 65534), val), (lab, K, g, val, 8),
                 (lab[:0], K, _graph(0, 0), val[:0]), (lab[:, :0], K, g, val[:, :, :0])]:
        with pytest.raises(ValueError, match="cuda"):
            boundary_stats(*args)


def _brute(labels, K, src, dst, values, connectivity):
    """count, min, max and the float64 mean of each entry by a Python loop over every pixel pair."""
    lab = np.asarray(labels).view(np.uint16).astype(np.int64)
    B, H, W = lab.shape
    C = values.shape[1]
    dirs = [(0, 1), (1, 0)] + ([(1, 1), (1, -1)] if connectivity == 8 else [])
    acc = {}
    for b in range(B):
        for i in range(H):
            for j in range(W):
                for di, dj in dirs:
                    i2, j2 = i + di, j + dj
                    if i2 >= H or not 0 <= j2 < W:
                        continue
                    a, o = lab[b, i, j], lab[b, i2, j2]
                    if a < K and o < K and a != o:
                        acc.setdefault((b, min(a, o), max(a, o)), []).append(
                            np.concatenate([values[b, :, i, j], values[b, :, i2, j2]]).reshape(2, C))
    E = len(src)
    out = (np.zeros(E, np.int64), np.full((E, C), np.nan), np.full((E, C), np.nan), np.full((E, C), np.nan))
    for e, (u, v) in enumerate(zip(src, dst)):
        if not (0 <= u < B * K and 0 <= v < B * K and u != v and u // K == v // K):
            continue
        b = u // K
        vals = acc.get((b, min(u, v) - b * K, max(u, v) - b * K))
        if vals is None:
            continue
        x = np.concatenate(vals)  # [2n, C]
        out[0][e] = len(vals)
        out[1][e] = x.astype(np.float64).mean(axis=0)
        for c in range(C):
            col = x[:, c]
            if np.isnan(col).any():
                out[2][e, c] = out[3][e, c] = np.nan
            else:  # -0.0 before +0.0
                order = sorted(col.tolist(), key=lambda x: (x, not np.signbit(x)))
                out[2][e, c], out[3][e, c] = order[0], order[-1]
    return out


def _random_case(rng, B, H, W, K, C, with_foreign):
    labels = rng.randint(0, K, (B, H, W)).astype(np.int16)
    blocks = (np.arange(H)[:, None] // 3 * 5 + np.arange(W)[None, :] // 4) % K  # some longer boundaries
    labels[0] = np.where(rng.rand(H, W) < 0.3, labels[0], blocks)
    if with_foreign:
        labels[rng.rand(B, H, W) < 0.1] = -1
        labels[rng.rand(B, H, W) < 0.05] = K + 7
    values = rng.randn(B, C, H, W).astype(np.float32)
    return labels, values


@pytest.mark.parametrize("connectivity", [4, 8])
def test_restatement_against_independent_computations(connectivity):
    rng = np.random.RandomState(11 + connectivity)
    for B, H, W, K, C, foreign in ((2, 9, 11, 6, 3, False), (3, 7, 13, 9, 1, True), (1, 1, 17, 4, 2, True),
                                   (2, 12, 1, 5, 5, False), (2, 16, 16, 40, 4, True)):
        labels, values = _random_case(rng, B, H, W, K, C, foreign)
        _, edge_index, boundary = ref_rag(labels, K, connectivity)
        src, dst = edge_index
        # extra entries: cross-image, out of range, self loops, duplicates, never adjacent
        extra_src = np.array([0, -1, B * K, 3, src[0] if len(src) else 0, 1], np.int64)
        extra_dst = np.array([K + 1, 2, 0, 3, dst[0] if len(dst) else 1, 2], np.int64)
        s_all, d_all = np.concatenate([src, extra_src]), np.concatenate([dst, extra_dst])
        mean, mn, mx, count = ref_boundary(labels, K, s_all, d_all, values, connectivity)
        assert mean.dtype == mn.dtype == mx.dtype == np.float32 and count.dtype == np.int32
        assert np.array_equal(count[:len(src)], boundary)
        bc, bmean, bmin, bmax = _brute(labels, K, s_all, d_all, values, connectivity)
        assert np.array_equal(count, bc)
        assert nan_class_equal(mn, bmin.astype(np.float32)) and nan_class_equal(mx, bmax.astype(np.float32))
        has = count > 0
        assert np.isnan(mean[~has]).all() and np.isnan(mn[~has]).all() and np.isnan(mx[~has]).all()
        assert np.allclose(mean[has], bmean[has], rtol=1e-6, atol=1e-6)


def test_hand_computed_2x3():
    # labels    values (one channel)
    # 0 0 1      1   -0.0  +0.0
    # 2 1 1      4    NaN   2
    labels = np.array([[[0, 0, 1], [2, 1, 1]]], np.int16)
    values = np.array([[[[1, -0.0, 0.0], [4, nan, 2]]]], np.float32)
    K = 3
    src = np.array([0, 1, 0, 2, 1, 2, 1], np.int64)
    dst = np.array([1, 0, 2, 0, 2, 1, 1], np.int64)
    mean, mn, mx, count = ref_boundary(labels, K, src, dst, values, 4)
    # {0,1}: (0,1)-(0,2) right, (0,1)-(1,1) down -> -0.0, +0.0, -0.0, NaN
    # {0,2}: (0,0)-(1,0) down -> 1, 4
    # {1,2}: (1,0)-(1,1) right -> 4, NaN
    assert count.tolist() == [2, 2, 1, 1, 1, 1, 0]
    assert np.isnan(mean[0, 0]) and np.isnan(mn[0, 0]) and np.isnan(mx[0, 0])
    assert nan_class_equal(mean[:2], mean[[1, 0]]) and nan_class_equal(mn[:2], mn[[1, 0]])
    assert mean[2, 0] == 2.5 and mn[2, 0] == 1 and mx[2, 0] == 4
    assert np.isnan(mean[4, 0]) and np.isnan(mn[4, 0]) and np.isnan(mx[5, 0])
    assert np.isnan(mean[6]).all() and count[6] == 0  # self loop
    # connectivity 8 adds the down-right pairs (0,0)-(1,1) and (0,1)-(1,2) to {0,1} and the down-left pair (0,1)-(1,0)
    # to {0,2}: its values 1, 4 (down, ordinal 1), then -0.0, 4 (down-left, ordinal 7); (0,2)-(1,1) has equal labels
    mean8, mn8, mx8, count8 = ref_boundary(labels, K, src, dst, values, 8)
    assert count8.tolist() == [4, 4, 2, 2, 1, 1, 0]
    assert mean8[2, 0] == np.float32(2.25) and mx8[2, 0] == 4
    assert mn8[2, 0].tobytes() == np.float32(-0.0).tobytes()


def test_hand_computed_3x3_signed_zeros():
    # labels      values, two channels
    # 0 1 2       c0: -0  +0  -0     c1: 1  2  3
    # 0 1 2           +0  -0  -0         4  5  6
    # 5 5 5           -0  -0  -0         7  8  9     (label 5 >= K: no pairs)
    labels = np.array([[[0, 1, 2], [0, 1, 2], [5, 5, 5]]], np.int16)
    c0 = np.array([[-0.0, 0.0, -0.0], [0.0, -0.0, -0.0], [-0.0, -0.0, -0.0]], np.float32)
    c1 = np.arange(1, 10, dtype=np.float32).reshape(3, 3)
    values = np.stack([c0, c1])[None]
    K = 5
    src = np.array([0, 1, 0, 3], np.int64)
    dst = np.array([1, 2, 2, 4], np.int64)
    mean, mn, mx, count = ref_boundary(labels, K, src, dst, values, 4)
    assert count.tolist() == [2, 2, 0, 0]
    # {0,1}: (0,0)-(0,1): -0, +0; (1,0)-(1,1): +0, -0
    assert mn[0, 0].tobytes() == np.float32(-0.0).tobytes() and mx[0, 0].tobytes() == np.float32(0.0).tobytes()
    assert mean[0, 0].tobytes() == np.float32(0.0).tobytes()
    assert mean[0, 1] == np.float32(1 + 2 + 4 + 5) / 4 and mn[0, 1] == 1 and mx[0, 1] == 5
    # {1,2}: +0, -0, -0, -0 -> max +0, min -0; mean +0 (lanes start from +0.0)
    assert mn[1, 0].tobytes() == np.float32(-0.0).tobytes() and mx[1, 0].tobytes() == np.float32(0.0).tobytes()
    assert mean[1, 0].tobytes() == np.float32(0.0).tobytes()
    assert np.isnan(mean[2:]).all() and np.isnan(mn[2:]).all() and np.isnan(mx[2:]).all()


def test_long_runs_take_several_lanes_rows():
    """A boundary of 200 pairs: 400 values over 13 lane rows, summed in the lane order, not left to right."""
    W = 200
    labels = np.stack([np.zeros(W, np.int16), np.ones(W, np.int16)])[None]
    rng = np.random.RandomState(5)
    values = (rng.randn(1, 1, 2, W) * 1e4).astype(np.float32)
    mean, mn, mx, count = ref_boundary(labels, 2, [0], [1], values, 4)
    assert count[0] == 200
    x = np.empty(400, np.float32)
    x[0::2], x[1::2] = values[0, 0, 0], values[0, 0, 1]
    lanes = np.zeros(32, np.float32)
    for j, v in enumerate(x):
        lanes[j % 32] = np.float32(lanes[j % 32] + v)
    for off in (16, 8, 4, 2, 1):
        lanes = (lanes + lanes[np.arange(32) ^ off]).astype(np.float32)
    assert mean[0, 0] == np.float32(lanes[0] / np.float32(400))
    assert mn[0, 0] == x.min() and mx[0, 0] == x.max()


def test_entry_keys():
    # B = 2, K = 6: (0,1) and (9,7) are valid; cross-image, self loop, out of range and negative entries are not
    b, key, valid = entry_keys([0, 5, 3, -1, 12, 9], [1, 6, 3, 0, 5, 7], 2, 6)
    assert valid.tolist() == [True, False, False, False, False, True]
    assert (b[0], key[0]) == (0, 1) and (b[5], key[5]) == (1, 1 * 65536 + 3)
