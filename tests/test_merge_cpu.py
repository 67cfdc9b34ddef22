"""Superpixel merging without a GPU: the ABI declarations, the argument checks (they come before any device work), the
numpy restatement's threshold cut against scipy's connected components, its region-count cut against a brute-force
loop, and hand-computed answers."""
import os
import re
import types

import numpy as np
import pytest
import torch
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components

from merge_cases import ref_edges, ref_forest, ref_merge, ref_present, wkey

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_abi_declares_and_binds_the_merge_entry_points():
    from fast_slic_b200 import _lib
    L = _lib.lib()
    header = open(os.path.join(ROOT, "include", "fslic_b200.h")).read()
    declared = set(re.findall(r"\b(fslic_b200_\w+)\s*\(", header))
    for name, nargs in (("fslic_b200_merge_scratch_bytes", 2), ("fslic_b200_merge_batch", 19),
                        ("fslic_b200_pool_paint_batch", 9)):
        assert name in declared and name in _lib.EXPORTED_SYMBOLS
        assert len(getattr(L, name).argtypes) == nargs
    assert int(L.fslic_b200_merge_scratch_bytes(1, 65535)) == 2 ** 64 - 1
    assert int(L.fslic_b200_merge_scratch_bytes(1, 0)) == 2 ** 64 - 1
    assert int(L.fslic_b200_merge_scratch_bytes(2 ** 14 + 1, 65536 - 2)) == 2 ** 64 - 1  # B*K past 2^30
    assert 40 * 1600 * 32 <= int(L.fslic_b200_merge_scratch_bytes(32, 1600)) < 2 ** 64 - 1


def _graph(n_nodes, E=3, dtype=torch.int64):
    return types.SimpleNamespace(indptr=torch.zeros(1, dtype=torch.int64).expand(n_nodes + 1),
                                 edge_index=torch.zeros((2, E), dtype=dtype))


def test_argument_errors():
    from fast_slic_b200.merging import merge_regions
    B, K = 2, 10
    lab = torch.zeros((B, 5, 7), dtype=torch.int16)
    g, w = _graph(B * K), torch.zeros(3, dtype=torch.float32)
    cut = {"threshold": 0.5}
    for args, kw, msg in [
        ((lab.numpy(), K, g, w), cut, "torch.from_numpy"),                     # numpy labels
        ((lab.int(), K, g, w), cut, "int16"),
        ((lab[0], K, g, w), cut, "dimensions"),
        ((lab, 0, g, w), cut, "K must be"), ((lab, 65535, g, w), cut, "K must be"), ((lab, 2.0, g, w), cut, "K must be"),
        ((torch.zeros((2 ** 14 + 1, 1, 1), dtype=torch.int16), 65534, _graph(0), w), cut, "split the batch"),
        ((lab, K, _graph(B * K - 1), w), cut, "indptr"), ((lab, K, _graph(B * K + 1), w), cut, "indptr"),
        ((lab, K, _graph(B * K, dtype=torch.int32), w), cut, "edge_index"),
        ((lab, K, types.SimpleNamespace(indptr=g.indptr, edge_index=torch.zeros((3, 3), dtype=torch.int64)), w), cut,
         "edge_index"),
        ((lab, K, types.SimpleNamespace(indptr=g.indptr, edge_index=torch.zeros(3, dtype=torch.int64)), w), cut,
         "edge_index"),
        ((lab, K, g, w.double()), cut, "weights"), ((lab, K, g, w[:2]), cut, "weights"),
        ((lab, K, g, torch.zeros(4)), cut, "weights"), ((lab, K, g, w[None]), cut, "weights"),
        ((lab, K, g, w), {}, "exactly one"), ((lab, K, g, w), {"threshold": 0.5, "num_regions": 3}, "exactly one"),
        ((lab, K, g, w), {"num_regions": 0}, "at least 1"), ((lab, K, g, w), {"num_regions": -5}, "at least 1"),
        ((lab, K, g, w), {"num_regions": 2.0}, "must be an int"), ((lab, K, g, w), {"num_regions": "3"}, "must be an int"),
        ((lab, K, g, w), {"num_regions": True}, "must be an int"),
        ((lab, K, g, w), {"threshold": float("nan")}, "NaN"), ((lab, K, g, w), {"threshold": np.float32("nan")}, "NaN"),
        ((lab, K, g, w), {"threshold": "0.5"}, "real number"), ((lab, K, g, w), {"threshold": 1j}, "real number"),
        ((lab, K, g, w), {"threshold": torch.tensor(0.5)}, "real number"),
        ((lab, K, g, w), {"threshold": None, "num_regions": None}, "exactly one"),
        ((lab, K, g, w), cut, "cuda"),                                          # cpu tensors, every other check passed
    ]:
        with pytest.raises(ValueError, match=msg):
            merge_regions(*args, **kw)
    if torch.cuda.is_available():
        with pytest.raises(ValueError, match="weights is on"):
            merge_regions(lab.cuda(), K, types.SimpleNamespace(indptr=g.indptr.cuda(), edge_index=g.edge_index.cuda()),
                          w, **cut)
    # the limits themselves pass every check but the device one
    for args, kw in [((lab, 1, _graph(B), w), cut), ((lab, 65534, _graph(B * 65534), w), cut),
                     ((torch.zeros((2 ** 14, 1, 1), dtype=torch.int16), 65534, _graph(2 ** 14 * 65534), w), cut),
                     ((lab, K, g, w), {"num_regions": 1}), ((lab, K, g, w), {"num_regions": 10 ** 30}),
                     ((lab, K, g, w), {"num_regions": np.int64(4)}),
                     ((lab, K, g, w), {"threshold": float("inf")}), ((lab, K, g, w), {"threshold": -float("inf")}),
                     ((lab, K, g, w), {"threshold": 3}), ((lab, K, g, w), {"threshold": np.float32(0.25)}),
                     ((lab[:0], K, _graph(0, 0), w[:0]), cut)]:
        with pytest.raises(ValueError, match="cuda"):
            merge_regions(*args, **kw)


def test_wkey_is_order_preserving():
    v = np.array([-np.inf, -3.4e38, -1.0, -1e-45, -0.0, 0.0, 1e-45, 1.0, 3.4e38, np.inf], np.float32)
    k = wkey(v)
    assert (np.diff(k.astype(np.int64)) >= 0).all() and k[4] == k[5] and len(set(k.tolist())) == len(v) - 1


def _random_graph(rng, B, K, p, with_absent=True):
    """Labels of B images over K labels (some absent), and both directions of random edges with random weights."""
    labels = rng.randint(0, K, (B, 6, 9)).astype(np.int16)
    if with_absent:
        labels[labels == K - 1] = 0
    src, dst = [], []
    for b in range(B):
        a = rng.rand(K, K) < p
        u, v = np.nonzero(np.triu(a, 1))
        src += list(b * K + u) + list(b * K + v)
        dst += list(b * K + v) + list(b * K + u)
    src, dst = np.array(src, np.int64), np.array(dst, np.int64)
    w = rng.randint(0, 6, len(src)).astype(np.float32) / 4  # ties
    return labels, src, dst, w


def test_threshold_cut_matches_connected_components():
    rng = np.random.RandomState(3)
    for trial in range(30):
        B, K = rng.randint(1, 4), rng.randint(1, 30)
        labels, src, dst, w = _random_graph(rng, B, K, rng.rand() * 0.3)
        present = ref_present(labels, K)
        forest = ref_forest(present, src, dst, w)
        for t in (-1.0, 0.0, 0.25, 0.5, 0.6, 1.0, 2.0, np.inf):
            _, region, count = ref_merge(labels, K, src, dst, w, threshold=t, forest=forest)
            b, lo, hi, ww = ref_edges(src, dst, w, present)
            sel = ww.astype(np.float64) < t
            n = B * K
            A = coo_matrix((np.ones(int(sel.sum())), (b[sel] * K + lo[sel], b[sel] * K + hi[sel])), shape=(n, n))
            _, comp = connected_components(A, directed=False)
            comp = comp.reshape(B, K)
            for i in range(B):
                nodes = np.nonzero(present[i])[0]
                # same partition of the present nodes
                pairs_cc = comp[i][nodes][:, None] == comp[i][nodes][None, :]
                pairs_ref = region[i][nodes][:, None] == region[i][nodes][None, :]
                assert np.array_equal(pairs_cc, pairs_ref), (trial, t, i)
                assert count[i] == len(np.unique(comp[i][nodes]))
                assert (region[i][~present[i]] == -1).all()


def _brute_count(present_b, edges, R):
    """Merge the globally smallest remaining inter-region edge, scanning every edge, until R regions or none left."""
    K = len(present_b)
    comp = list(range(K))
    regions = int(present_b.sum())
    while regions > R:
        best = None
        for key, u, v in edges:
            if comp[u] != comp[v] and (best is None or (key, u, v) < best):
                best = (key, u, v)
        if best is None:
            break
        _, u, v = best
        old, new = max(comp[u], comp[v]), min(comp[u], comp[v])
        comp = [new if c == old else c for c in comp]
        regions -= 1
    return np.array(comp)


def test_count_cut_matches_brute_force():
    rng = np.random.RandomState(5)
    for trial in range(25):
        B, K = rng.randint(1, 3), rng.randint(1, 16)
        labels, src, dst, w = _random_graph(rng, B, K, rng.rand() * 0.5)
        w[rng.rand(len(w)) < 0.1] = np.nan
        present = ref_present(labels, K)
        forest = ref_forest(present, src, dst, w)
        b, lo, hi, ww = ref_edges(src, dst, w, present)
        keys = wkey(ww).tolist()
        for R in range(1, K + 2):
            _, region, count = ref_merge(labels, K, src, dst, w, num_regions=R, forest=forest)
            for i in range(B):
                sel = b == i
                comp = _brute_count(present[i], list(zip([keys[j] for j in np.nonzero(sel)[0]], lo[sel].tolist(),
                                                          hi[sel].tolist())), R)
                nodes = np.nonzero(present[i])[0]
                assert np.array_equal(comp[nodes][:, None] == comp[nodes][None, :],
                                      region[i][nodes][:, None] == region[i][nodes][None, :]), (trial, R, i)
                assert count[i] == len(np.unique(comp[nodes]))


def _both(u, v):
    """Both directions of the undirected edges (u[i], v[i])."""
    return np.concatenate([u, v]).astype(np.int64), np.concatenate([v, u]).astype(np.int64)


def test_known_answers():
    lab = np.arange(4, dtype=np.int16).reshape(1, 2, 2)  # labels 0..3 all present
    # a path 0-1-2-3 with equal weights: ties go by (lo, hi), so one merge joins 0 and 1
    src, dst = _both(np.array([2, 0, 1]), np.array([3, 1, 2]))
    w = np.ones(6, np.float32)
    _, region, count = ref_merge(lab, 4, src, dst, w, num_regions=3)
    assert region.tolist() == [[0, 0, 1, 2]] and count.tolist() == [3]
    _, region, _ = ref_merge(lab, 4, src, dst, w, num_regions=2)
    assert region.tolist() == [[0, 0, 0, 1]]
    # -0.0 equals +0.0: the tie is decided by the ids, and threshold 0 merges neither
    w = np.array([0.0, -0.0, 5.0] * 2, np.float32)  # edges {2,3}: +0, {0,1}: -0, {1,2}: 5
    _, region, _ = ref_merge(lab, 4, src, dst, w, num_regions=3)
    assert region.tolist() == [[0, 0, 1, 2]]
    w = np.array([-0.0, 0.0, 5.0] * 2, np.float32)
    _, region, _ = ref_merge(lab, 4, src, dst, w, num_regions=3)
    assert region.tolist() == [[0, 0, 1, 2]]
    _, region, count = ref_merge(lab, 4, src, dst, w, threshold=0.0)
    assert region.tolist() == [[0, 1, 2, 3]] and count.tolist() == [4]
    _, region, _ = ref_merge(lab, 4, src, dst, w, threshold=1e-45)
    assert region.tolist() == [[0, 0, 1, 1]]
    # NaN never merges; +inf merges only under num_regions
    w = np.array([np.nan, np.inf, 1.0] * 2, np.float32)
    _, region, count = ref_merge(lab, 4, src, dst, w, num_regions=1)
    assert region.tolist() == [[0, 0, 0, 1]] and count.tolist() == [2]                  # c_b = 2 > R
    _, region, _ = ref_merge(lab, 4, src, dst, w, threshold=np.inf)
    assert region.tolist() == [[0, 1, 1, 2]]
    _, region, _ = ref_merge(lab, 4, src, dst, w, threshold=1.5)
    assert region.tolist() == [[0, 1, 1, 2]]
    # R >= P_b leaves every region alone
    w = np.ones(6, np.float32)
    for R in (4, 5, 100):
        _, region, count = ref_merge(lab, 4, src, dst, w, num_regions=R)
        assert region.tolist() == [[0, 1, 2, 3]] and count.tolist() == [4]
    # the reverse direction is never read
    w2 = np.concatenate([w[:3], [np.nan, -7.0, 1e9]]).astype(np.float32)
    for kw in ({"num_regions": 2}, {"threshold": 1.5}):
        assert all(np.array_equal(a, b) for a, b in zip(ref_merge(lab, 4, src, dst, w2, **kw),
                                                        ref_merge(lab, 4, src, dst, w, **kw)))
    # absent labels get -1, pixels with labels >= K or -1 get -1, numbering by smallest member
    lab = np.array([[[5, 5, 2], [-1, 7, 2]]], np.int16)                                # K = 6: 0, 1, 3, 4 absent
    src, dst = _both(np.array([2, 0, 3]), np.array([5, 2, 4]))
    w = np.zeros(6, np.float32)
    out, region, count = ref_merge(lab, 6, src, dst, w, threshold=1.0)
    assert region.tolist() == [[-1, -1, 0, -1, -1, 0]] and count.tolist() == [1]
    assert out.tolist() == [[[0, 0, 0], [-1, -1, 0]]]
    out, region, count = ref_merge(lab, 6, src, dst, w, threshold=0.0)
    assert region.tolist() == [[-1, -1, 0, -1, -1, 1]] and out.tolist() == [[[1, 1, 0], [-1, -1, 0]]]
    # cross-image and out-of-range entries are ignored; two images are independent
    lab = np.array([[[0, 1]], [[0, 1]]], np.int16)
    src = np.array([0, 1, 2, -1, 0, 3], np.int64)
    dst = np.array([1, 2, 3, 0, 4, 9], np.int64)
    w = np.array([np.nan, 0.0, 1.0, 0.0, 0.0, 0.0], np.float32)
    _, region, count = ref_merge(lab, 2, src, dst, w, num_regions=1)
    assert region.tolist() == [[0, 1], [0, 0]] and count.tolist() == [2, 1]
    # K = 1: one region per image that has a pixel of label 0
    lab = np.array([[[0, 3]], [[2, 2]]], np.int16)
    out, region, count = ref_merge(lab, 1, np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros(0, np.float32),
                                   num_regions=1)
    assert region.tolist() == [[0], [-1]] and count.tolist() == [1, 0] and out.tolist() == [[[0, -1]], [[-1, -1]]]


def test_region_ids_above_32767_read_as_uint16():
    K = 40000
    lab = np.arange(K, dtype=np.int64).astype(np.uint16).view(np.int16).reshape(1, 1, K)
    out, region, count = ref_merge(lab, K, np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros(0, np.float32),
                                   threshold=0.0)
    assert count.tolist() == [K] and np.array_equal(out.view(np.uint16), lab.view(np.uint16))
