"""kNN graphs without a GPU: the ABI declarations, the argument checks (they come before any device work), the numpy
restatement against scipy's kd-tree, and hand-worked small cases."""
import os
import re

import numpy as np
import pytest
import torch

from knn_cases import ref_knn, sqdist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NO_SIZE = 2 ** 64 - 1


def test_abi_declares_and_binds_the_knn_entry_points():
    from fast_slic_b200 import _lib
    L = _lib.lib()
    header = open(os.path.join(ROOT, "include", "fslic_b200.h")).read()
    declared = set(re.findall(r"\b(fslic_b200_\w+)\s*\(", header))
    for name, nargs in (("fslic_b200_knn_scratch_bytes", 5), ("fslic_b200_knn_count", 14),
                        ("fslic_b200_knn_fill", 14)):
        assert name in declared and name in _lib.EXPORTED_SYMBOLS
        assert len(getattr(L, name).argtypes) == nargs
    f = L.fslic_b200_knn_scratch_bytes
    for args in [(-1, 10, 3, 8, 0), (1, 0, 3, 8, 0), (1, 65535, 3, 8, 0), (1, 10, 0, 8, 0), (1, 10, 65, 8, 0),
                 (1, 10, 3, 0, 0), (1, 10, 3, 33, 1), (2 ** 15, 2 ** 15 + 1, 1, 1, 0),  # B*K > 2^30
                 (2 ** 14, 65534, 3, 2, 1)]:  # more edge slots than one sort takes
        assert int(f(*args)) == NO_SIZE, args
    assert int(f(0, 10, 3, 8, 0)) < NO_SIZE
    n = 32 * 1600
    directed, symmetric = int(f(32, 1600, 6, 8, 0)), int(f(32, 1600, 6, 8, 1))
    assert n * (9 + 4 * 8 + 8 * 8) <= directed < symmetric < NO_SIZE
    assert symmetric - directed >= n * 2 * 8 * 36
    assert int(f(1, 65534, 64, 32, 1)) < 1 << 30


def test_argument_errors():
    from fast_slic_b200.region_graph import knn_graph
    B, K, D = 2, 10, 3
    p = torch.zeros((B, K, D), dtype=torch.float32)
    m = torch.ones((B, K), dtype=torch.bool)
    for args, kw, msg in [
        ((p.numpy(), 4), {}, "torch.from_numpy"), ((p.double(), 4), {}, "float32"), ((p[0], 4), {}, "dimensions"),
        ((p[:, :0], 4), {}, "K must be"), ((torch.zeros(1, 65535, 1), 4), {}, "K must be"),
        ((p[:, :, :0], 4), {}, "D must be"), ((torch.zeros(1, 2, 65), 4), {}, "D must be"),
        ((torch.zeros(1, 1, 1).expand(2 ** 15, 2 ** 15 + 1, 1), 4), {}, "nodes"),
        ((p, 0), {}, "k must be"), ((p, 33), {}, "k must be"), ((p, 2.0), {}, "k must be"), ((p, "8"), {}, "k must be"),
        ((p, True), {}, "k must be an int"), ((p, np.bool_(True)), {}, "k must be an int"),
        ((p, 4), {"present": m.numpy()}, "present must be a cuda tensor"),
        ((p, 4), {"present": m.int()}, "bool"), ((p, 4), {"present": m[0]}, "dimensions"),
        ((p, 4), {"present": m[:1]}, "do not match"), ((p, 4), {"present": m[:, :5]}, "do not match"),
        ((p, 4), {}, "cuda"),  # cpu tensors, every other check passed
        ((p, 4), {"present": m}, "cuda"),
    ]:
        with pytest.raises(ValueError, match=msg):
            knn_graph(*args, **kw)
    if torch.cuda.is_available():
        with pytest.raises(ValueError, match="present is on"):
            knn_graph(p.cuda(), 4, present=m)
    # the limits themselves pass every check but the device one
    for args in [(torch.zeros(1, 65534, 1), 32), (torch.zeros(1, 1, 64), 1), (p[:0], 1),
                 (torch.zeros(1, 1, 1).expand(2 ** 14, 65534, 1), 1)]:
        with pytest.raises(ValueError, match="cuda"):
            knn_graph(*args)


def test_restatement_against_kd_tree():
    from scipy.spatial import cKDTree
    rng = np.random.RandomState(3)
    for K, D, k in ((300, 2, 8), (200, 5, 1), (150, 16, 32), (40, 64, 8)):
        pts = rng.rand(2, K, D).astype(np.float32)
        indptr, ei, dist = ref_knn(pts, k)
        assert np.array_equal(indptr, np.arange(2 * K + 1) * k)
        for b in range(2):
            p64 = pts[b].astype(np.float64)
            d, nb = cKDTree(p64).query(p64, k + 1)
            for i in range(K):
                row = slice(indptr[b * K + i], indptr[b * K + i + 1])
                assert np.all(ei[0, row] == b * K + i)
                got = ei[1, row] - b * K
                assert np.all(np.diff(got) > 0)
                want = nb[i][nb[i] != i][:k]
                assert set(got) == set(want)
                exact = ((p64[got] - p64[i]) ** 2).sum(1)
                assert np.allclose(dist[row], exact, rtol=4e-7 * (D + 2), atol=0)


def test_distance_rounding_order():
    a = np.array([[1e8, 1.0, 3.0]], np.float32)
    b = np.array([[0.0, 0.0, 0.0]], np.float32)
    s = np.float32(0)
    for c in range(3):
        t = np.float32(a[0, c] - b[0, c])
        s = np.float32(s + np.float32(t * t))
    assert sqdist(a, b)[0, 0] == s == np.float32(1e16)  # 1 + 9 vanish next to 1e16, in this order
    assert sqdist(a, b)[0, 0].view(np.uint32) == sqdist(b, a)[0, 0].view(np.uint32)


def _edges(ref):
    indptr, ei, dist = ref
    return indptr.tolist(), [(int(u), int(v), float(w)) for u, v, w in zip(ei[0], ei[1], dist)]


def test_ties_go_to_the_lower_index():
    p = np.array([[[0], [1], [2], [3]]], np.float32)
    assert _edges(ref_knn(p, 1)) == ([0, 1, 2, 3, 4], [(0, 1, 1.0), (1, 0, 1.0), (2, 1, 1.0), (3, 2, 1.0)])
    assert _edges(ref_knn(p, 1, symmetric=True)) == (
        [0, 1, 3, 5, 6], [(0, 1, 1.0), (1, 0, 1.0), (1, 2, 1.0), (2, 1, 1.0), (2, 3, 1.0), (3, 2, 1.0)])
    # a grid: node 4 of a 3x3 grid has four neighbours at 1 and four at 2
    g = np.array([[[y, x] for y in range(3) for x in range(3)]], np.float32)
    indptr, ei, dist = ref_knn(g, 5)
    assert ei[1, indptr[4]:indptr[5]].tolist() == [0, 1, 3, 5, 7] and dist[indptr[4]:indptr[5]].tolist() == [2, 1, 1,
                                                                                                          1, 1]


def test_fewer_candidates_than_k():
    p = np.array([[[0], [1], [5]], [[0], [0], [0]]], np.float32)
    indptr, ei, dist = ref_knn(p, 5)
    assert indptr.tolist() == [0, 2, 4, 6, 8, 10, 12]
    assert ei[1].tolist() == [1, 2, 0, 2, 0, 1, 4, 5, 3, 5, 3, 4]
    assert dist.tolist() == [1, 25, 1, 16, 25, 16, 0, 0, 0, 0, 0, 0]
    # one candidate: no edge; none: nothing
    assert ref_knn(p[:, :1], 3)[1].shape == (2, 0)


def test_absent_and_non_finite_nodes():
    nan, inf = np.nan, np.inf
    p = np.array([[[0, 0], [nan, 0], [1, 0], [0, inf], [3, 0], [2, 0]]], np.float32)
    present = np.array([[True, True, True, True, True, False]])
    indptr, ei, dist = ref_knn(p, 2, present)
    assert indptr.tolist() == [0, 2, 2, 4, 4, 6, 6]
    assert ei[1].tolist() == [2, 4, 0, 4, 0, 2]
    assert dist.tolist() == [1, 9, 1, 4, 9, 4]
    assert ref_knn(p, 2, present, symmetric=True)[0].tolist() == [0, 2, 2, 4, 4, 6, 6]


def test_infinite_distances():
    p = np.array([[[0], [3e38], [-3e38]]], np.float32)
    indptr, ei, dist = ref_knn(p, 1)
    assert ei[1].tolist() == [1, 0, 0] and np.all(np.isposinf(dist))
    indptr, ei, dist = ref_knn(p, 1, symmetric=True)
    assert ei.T.tolist() == [[0, 1], [0, 2], [1, 0], [2, 0]]
    # a huge coordinate difference overflows to +inf even when others are finite
    q = np.array([[[0, 0], [0, 1], [3e38, 0]]], np.float32)
    indptr, ei, dist = ref_knn(q, 2)
    assert ei[1].tolist() == [1, 2, 0, 2, 0, 1] and dist.tolist() == [1, np.inf, 1, np.inf, np.inf, np.inf]


def test_symmetric_union_of_an_asymmetric_relation():
    p = np.array([[[0], [1], [3], [7]]], np.float32)
    assert _edges(ref_knn(p, 1)) == ([0, 1, 2, 3, 4], [(0, 1, 1.0), (1, 0, 1.0), (2, 1, 4.0), (3, 2, 16.0)])
    assert _edges(ref_knn(p, 1, symmetric=True)) == (
        [0, 1, 3, 5, 6], [(0, 1, 1.0), (1, 0, 1.0), (1, 2, 4.0), (2, 1, 4.0), (2, 3, 16.0), (3, 2, 16.0)])
    # the union is what to_undirected makes of the directed edges: every pair in both directions, once
    rng = np.random.RandomState(0)
    q = rng.rand(3, 50, 3).astype(np.float32)
    d = ref_knn(q, 4)
    s = ref_knn(q, 4, symmetric=True)
    pairs = {(u, v) for u, v in d[1].T.tolist()}
    want = sorted(pairs | {(v, u) for u, v in pairs})
    assert [tuple(e) for e in s[1].T.tolist()] == want
    assert s[0][-1] == len(want) and np.all(s[1][0] // 50 == s[1][1] // 50)
