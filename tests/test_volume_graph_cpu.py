"""Region adjacency graphs and shapes of label volumes without a GPU: the numpy restatement (volume_graph_cases.py)
against brute-force loops over voxels, its agreement with the 2-D restatements at D = 1, the graph's invariance under
axis permutations, the ABI, the scratch sizes and limits, and the argument checks (they come before any device
work)."""
import collections
import itertools
import os
import re

import numpy as np
import pytest
import torch

from geometry_cases import ref_properties
from rag_cases import ref_rag
from volume_graph_cases import (FIELDS_3D, forward_offsets, pair_count, ref_properties_3d, ref_rag3d, ref_rag3d_volume,
                                voxel_pairs)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NONE = 2 ** 64 - 1
ARGC = {"fslic_b200_rag3d_batch_scratch_bytes": 7, "fslic_b200_rag3d_batch_count": 15,
        "fslic_b200_rag3d_batch_fill": 18, "fslic_b200_props3d_batch": 15}


def test_abi_declares_and_binds_the_volume_entry_points():
    from fast_slic_b200 import _lib
    L = _lib.lib()
    header = open(os.path.join(ROOT, "include", "fslic_b200.h")).read()
    declared = set(re.findall(r"\b(fslic_b200_\w+)\s*\(", header))
    for sym, argc in ARGC.items():
        assert sym in declared and sym in _lib.EXPORTED_SYMBOLS, sym
        assert len(getattr(L, sym).argtypes) == argc, sym
    assert L.fslic_b200_rag3d_batch_scratch_bytes.restype is not None
    # the 2-D entry points keep their arguments
    assert len(L.fslic_b200_rag_batch_scratch_bytes.argtypes) == 6
    assert len(L.fslic_b200_rag_batch_count.argtypes) == 14
    assert len(L.fslic_b200_rag_batch_fill.argtypes) == 17
    assert len(L.fslic_b200_props_batch.argtypes) == 14


def test_scratch_bytes():
    from fast_slic_b200 import _lib
    L = _lib.lib()
    f, f2 = L.fslic_b200_rag3d_batch_scratch_bytes, L.fslic_b200_rag_batch_scratch_bytes
    assert f(0, 4, 5, 5, 10, 6, 0) == 256 and f(3, 0, 5, 5, 10, 18, 0) == 256 and f(3, 5, 5, 0, 10, 26, 1) == 256
    for args in ((1, 4, 5, 5, 0, 6, 0), (1, 4, 5, 5, 65535, 6, 0), (-1, 4, 5, 5, 10, 6, 0), (1, -1, 5, 5, 10, 6, 0),
                 (1, 4, 5, 5, 10, 4, 0), (1, 4, 5, 5, 10, 8, 0), (1, 4, 5, 5, 10, 27, 0),
                 (1, 2, 2 ** 14, 2 ** 14 + 1, 10, 6, 0),     # more than 2^29 voxels
                 (1, 2 ** 30, 2 ** 30, 2 ** 30, 10, 6, 0),   # no overflow of D * H * W on the way
                 (40000, 2, 2, 2, 65534, 6, 0),              # B * K + 1 > 2^31 - 1
                 (1, 512, 1024, 1024, 10, 18, 0),            # 2^29 voxels: P > 2^31 - 1 at 18 and 26
                 (1, 512, 1024, 1024, 10, 26, 0),
                 (1, 512, 512, 512, 65534, 26, 1)):          # an exact table over 2^31 slots
        assert f(*args) == NONE, args
    assert pair_count(512, 1024, 1024, 6) < 2 ** 31 and f(1, 512, 1024, 1024, 1600, 6, 0) != NONE
    assert pair_count(512, 512, 512, 26) < 2 ** 31 and f(1, 512, 512, 512, 16384, 26, 0) != NONE
    # at D = 1 the pairs of 6 are those of 4, of 18 and 26 those of 8: the same tables
    for B, H, W, K, e in ((1, 61, 77, 65534, 1), (3, 61, 77, 65534, 0), (2, 240, 320, 300, 0), (1, 720, 1280, 1600, 0)):
        assert f(B, 1, H, W, K, 6, e) == f2(B, H, W, K, 4, e)
        assert f(B, 1, H, W, K, 18, e) == f(B, 1, H, W, K, 26, e) == f2(B, H, W, K, 8, e)
    # exact tables: a power of two >= 2 * min(K (K - 1) / 2, voxel pairs) per volume; the graph's is 2^21 at K = 65534
    p = pair_count(20, 30, 40, 26)
    t = 1 << (2 * p - 1).bit_length()
    assert 8 * t <= f(1, 20, 30, 40, 65534, 26, 1) < 8 * t + 16 * 65535 + 65536 and t < 1 << 21
    assert f(1, 20, 30, 40, 65534, 26, 0) == f(1, 20, 30, 40, 65534, 26, 1)


def test_chunks(monkeypatch):
    from fast_slic_b200 import _lib, region_graph
    f = _lib.lib().fslic_b200_rag3d_batch_scratch_bytes
    assert region_graph.rag3d_chunk(8, 100, 192, 192, 4000, 26) == 8
    monkeypatch.setattr(region_graph, "RAG_SCRATCH_CAP", 3 * f(1, 100, 192, 192, 4000, 6, 0))
    c = region_graph.rag3d_chunk(8, 100, 192, 192, 4000, 6)
    assert 1 <= c <= 3 and f(c, 100, 192, 192, 4000, 6, 0) <= region_graph.RAG_SCRATCH_CAP
    with pytest.raises(ValueError, match="too large"):
        region_graph.rag3d_chunk(1, 512, 1024, 1024, 10, 26)


def test_pair_counts():
    from fast_slic_b200.region_graph import RAG3D_OFFSETS, voxel_pairs as lib_pairs
    assert len(forward_offsets(6)) == 3 and len(forward_offsets(18)) == 9 and len(forward_offsets(26)) == 13
    for conn, n in ((6, 3), (18, 9), (26, 13)):
        assert sorted(RAG3D_OFFSETS[:n]) == sorted(forward_offsets(conn))
    lab = np.zeros((4, 5, 7), np.int64)
    for conn in (6, 18, 26):
        assert voxel_pairs(lab, conn)[0].size == pair_count(4, 5, 7, conn) == lib_pairs(4, 5, 7, conn)
        for shape in ((1, 1, 1), (1, 9, 1), (0, 3, 3), (512, 512, 512), (512, 1024, 1024)):
            assert pair_count(*shape, conn) == lib_pairs(*shape, conn)


def test_argument_errors():
    from fast_slic_b200.geometry import region_properties_3d
    from fast_slic_b200.region_graph import region_adjacency_3d
    l = torch.zeros((2, 3, 5, 7), dtype=torch.int16)
    huge = torch.zeros((1, 1, 1, 1), dtype=torch.int16).expand(1, 2, 2 ** 14, 2 ** 14 + 1)  # over 2^29 voxels
    dense = torch.zeros((1, 1, 1, 1), dtype=torch.int16).expand(1, 512, 1024, 1024)       # 2^29 voxels
    bad = [
        ((l.numpy(), 10), "torch.from_numpy"),
        ((l.int(), 10), "int16"),
        ((l[0], 10), "dimensions"),
        ((l[None], 10), "dimensions"),
        ((l, 0), "K must be"),
        ((l, 65535), "K must be"),
        ((l, 3.0), "K must be"),
        ((l, 10, 4), "connectivity"),
        ((l, 10, 8), "connectivity"),
        ((l, 10, 6.0), "connectivity"),
        ((l, 10, "6"), "connectivity"),
        ((huge, 10), "exceed"),
        ((dense, 10, 18), "int32"),
        ((dense, 10, 26), "int32"),
        ((l, 10), "cuda"),
        ((l, 10, 26), "cuda"),
        ((dense, 10, 6), "cuda"),  # 2^29 voxels at 6-connectivity are allowed past the size checks
    ]
    for args, msg in bad:
        with pytest.raises(ValueError, match=msg):
            region_adjacency_3d(*args)
    long_side = torch.zeros((1, 1, 1, 1), dtype=torch.int16).expand(1, 1, 2, 32768)
    for args, msg in [((l.numpy(), 10), "torch.from_numpy"), ((l.int(), 10), "int16"), ((l[0], 10), "dimensions"),
                      ((l, 0), "K must be"), ((l, 65535), "K must be"), ((huge, 10), "32767"),
                      ((long_side, 10), "32767"), ((l, 10), "cuda"),
                      ((torch.zeros((1, 1, 1, 1), dtype=torch.int16).expand(1, 1, 16384, 32767), 10), "cuda")]:
        with pytest.raises(ValueError, match=msg):
            region_properties_3d(*args)


def _brute_graph(labels, K, connectivity):
    """Every voxel, every forward neighbour, in Python loops: {(a, c): pairs} over unordered label pairs."""
    D, H, W = labels.shape
    lab = labels.view(np.uint16)
    most = {6: 1, 18: 2, 26: 3}[connectivity]
    offsets = [o for o in itertools.product((-1, 0, 1), repeat=3)
               if o > (0, 0, 0) and sum(v != 0 for v in o) <= most]  # tuple order: first non-zero positive
    count = collections.Counter()
    for z, y, x in itertools.product(range(D), range(H), range(W)):
        for dz, dy, dx in offsets:
            z2, y2, x2 = z + dz, y + dy, x + dx
            if 0 <= z2 < D and 0 <= y2 < H and 0 <= x2 < W:
                a, c = int(lab[z, y, x]), int(lab[z2, y2, x2])
                if a < K and c < K and a != c:
                    count[min(a, c), max(a, c)] += 1
    return count


def _brute_properties(labels, K):
    """Every field of one [D,H,W] volume by a Python loop over voxels and faces, as exact Python numbers."""
    D, H, W = labels.shape
    lab = labels.view(np.uint16).astype(np.int64)
    area, surface, border = [0] * K, [0] * K, [0] * K
    m = [[0] * 9 for _ in range(K)]
    lo, hi = [[None] * 3 for _ in range(K)], [[None] * 3 for _ in range(K)]
    for z, y, x in itertools.product(range(D), range(H), range(W)):
        k = int(lab[z, y, x])
        if k >= K:
            continue
        area[k] += 1
        for f, v in enumerate((z, y, x, z * z, z * y, z * x, y * y, y * x, x * x)):
            m[k][f] += v
        for a, v in enumerate((z, y, x)):
            lo[k][a] = v if lo[k][a] is None else min(lo[k][a], v)
            hi[k][a] = v + 1 if hi[k][a] is None else max(hi[k][a], v + 1)
        for dz, dy, dx in ((-1, 0, 0), (1, 0, 0), (0, -1, 0), (0, 1, 0), (0, 0, -1), (0, 0, 1)):
            z2, y2, x2 = z + dz, y + dy, x + dx
            if not (0 <= z2 < D and 0 <= y2 < H and 0 <= x2 < W):
                surface[k] += 1
                border[k] += 1
            elif lab[z2, y2, x2] != k:
                surface[k] += 1
    bbox = [lo[k] + hi[k] if area[k] else [0] * 6 for k in range(K)]
    return area, bbox, m, surface, border


def _volumes(rng):
    D, H, W = 5, 6, 7
    zz, yy, xx = np.mgrid[:D, :H, :W]
    yield (zz // 2 * 100 + yy // 3 * 10 + xx // 4).astype(np.int16), 300
    yield rng.randint(0, 12, (D, H, W)).astype(np.int16), 12
    yield rng.randint(-1, 15, (D, H, W)).astype(np.int16), 12       # -1 and labels >= K
    yield rng.randint(-1, 2, (D, H, W)).astype(np.int16), 1         # K = 1
    yield rng.randint(0, 5, (1, 4, 9)).astype(np.int16), 5          # D = 1
    yield rng.randint(0, 5, (9, 1, 4)).astype(np.int16), 5          # H = 1
    yield rng.randint(0, 5, (4, 9, 1)).astype(np.int16), 5          # W = 1
    yield np.array([[[5]]], np.int16), 9
    yield ((zz + yy + xx) % 2).astype(np.int16), 2                  # 3-D checkerboard
    yield rng.choice(np.array([0, 3, 65533, 65535], np.uint16), (D, H, W)).view(np.int16), 65534


@pytest.mark.parametrize("connectivity", [6, 18, 26])
def test_graph_restatement_agrees_with_brute_force(connectivity):
    rng = np.random.RandomState(13)
    vols = list(_volumes(rng))
    for labels, K in vols:
        src, dst, w = ref_rag3d_volume(labels, K, connectivity)
        want = _brute_graph(labels, K, connectivity)
        got = {(s, d): c for s, d, c in zip(src.tolist(), dst.tolist(), w.tolist())}
        assert len(got) == len(src) == 2 * len(want)
        for (a, c), n in want.items():
            assert got[a, c] == got[c, a] == n
        assert sorted(zip(src.tolist(), dst.tolist())) == list(zip(src.tolist(), dst.tolist()))
    labels = np.stack([v for v, _ in vols[:3]])
    indptr, edge_index, boundary = ref_rag3d(labels, 300, connectivity)
    assert indptr.dtype == np.int64 and edge_index.dtype == np.int64 and boundary.dtype == np.int32
    assert indptr.shape == (3 * 300 + 1,) and edge_index.shape == (2, boundary.size) and indptr[-1] == boundary.size
    for n in range(3 * 300):
        assert (edge_index[0, indptr[n]:indptr[n + 1]] == n).all()
        assert (edge_index[1, indptr[n]:indptr[n + 1]] // 300 == n // 300).all()
    empty = ref_rag3d(np.zeros((0, 2, 4, 4), np.int16), 7, connectivity)
    assert empty[0].tolist() == [0] and empty[1].shape == (2, 0) and empty[2].shape == (0,)


def test_properties_restatement_agrees_with_brute_force():
    rng = np.random.RandomState(17)
    for labels, K in _volumes(rng):
        K = min(K, 400)
        got = ref_properties_3d(labels[None], K)
        area, bbox, m, surface, border = _brute_properties(labels, K)
        assert got["area"][0].tolist() == area and got["bbox"][0].tolist() == bbox
        assert got["moments"][0].tolist() == m and got["surface"][0].tolist() == surface
        assert got["border"][0].tolist() == border
        for k in range(K):
            if area[k]:
                c = [m[k][a] / area[k] for a in range(3)]
                assert got["centroid"][0, k].tolist() == pytest.approx(c, rel=1e-12, abs=1e-12)
                cov = [m[k][f] / area[k] - c[a] * c[b] for f, a, b in
                       ((3, 0, 0), (4, 0, 1), (5, 0, 2), (6, 1, 1), (7, 1, 2), (8, 2, 2))]
                assert got["covariance"][0, k].tolist() == pytest.approx(cov, rel=1e-9, abs=1e-9)
            else:
                assert not got["centroid"][0, k].any() and not got["covariance"][0, k].any()
    want = {"area": (np.int32, (2, 7)), "bbox": (np.int32, (2, 7, 6)), "moments": (np.int64, (2, 7, 9)),
            "surface": (np.int64, (2, 7)), "border": (np.int32, (2, 7)), "centroid": (np.float64, (2, 7, 3)),
            "covariance": (np.float64, (2, 7, 6))}
    out = ref_properties_3d(np.zeros((2, 3, 4, 5), np.int16), 7)
    assert tuple(out) == FIELDS_3D
    for f, (dt, shape) in want.items():
        assert out[f].dtype == dt and out[f].shape == shape, f


def test_one_slice_equals_the_2d_restatements():
    """At D = 1, 6-connectivity is 4 and 18 and 26 are 8; the properties have zero z moments, z centroid and z
    covariances, a (0, y0, x0, 1, y1, x1) box, surface = perimeter + 2 area and border = border_2d + 2 area."""
    rng = np.random.RandomState(5)
    maps = [(rng.randint(-1, 30, (3, 23, 29)).astype(np.int16), 25),
            (np.kron(rng.randint(0, 50, (2, 6, 8)), np.ones((1, 5, 4), np.int64)).astype(np.int16), 50),
            (rng.choice(np.array([0, 7, 65533, 65535], np.uint16), (2, 9, 40)).view(np.int16), 65534)]
    for lab2, K in maps:
        vol = lab2[:, None]
        for c3, c2 in ((6, 4), (18, 8), (26, 8)):
            for a, b in zip(ref_rag3d(vol, K, c3), ref_rag(lab2, K, c2)):
                assert a.dtype == b.dtype and np.array_equal(a, b)
        p3, p2 = ref_properties_3d(vol, K), ref_properties(lab2, K)
        assert np.array_equal(p3["area"], p2["area"])
        some = p2["area"] > 0
        want_box = np.zeros(p3["bbox"].shape, np.int32)
        want_box[..., 1], want_box[..., 2], want_box[..., 4], want_box[..., 5] = (p2["bbox"][..., f] for f in range(4))
        want_box[..., 3] = some
        assert np.array_equal(p3["bbox"], want_box)
        m = p3["moments"]
        assert not m[..., [0, 3, 4, 5]].any()
        assert np.array_equal(m[..., [1, 2, 6, 7, 8]], p2["moments"])
        assert np.array_equal(p3["surface"], p2["perimeter"].astype(np.int64) + 2 * p2["area"])
        assert np.array_equal(p3["border"], p2["border"] + 2 * p2["area"])
        assert not p3["centroid"][..., 0].any() and np.array_equal(p3["centroid"][..., 1:], p2["centroid"])
        assert not p3["covariance"][..., :3].any()
        assert np.array_equal(p3["covariance"][..., 3:], p2["covariance"])


@pytest.mark.parametrize("connectivity", [6, 18, 26])
def test_graph_is_invariant_under_axis_permutations(connectivity):
    """6-, 18- and 26-neighbourhoods are symmetric under any permutation of the axes, so the graph is too."""
    rng = np.random.RandomState(21)
    vol = np.kron(rng.randint(0, 40, (3, 4, 5)), np.ones((2, 3, 2), np.int64)).astype(np.int16)
    vol[rng.rand(*vol.shape) < 0.05] = -1
    want = ref_rag3d(vol[None], 40, connectivity)
    for perm in itertools.permutations(range(3)):
        got = ref_rag3d(np.ascontiguousarray(vol.transpose(perm))[None], 40, connectivity)
        for a, b in zip(got, want):
            assert np.array_equal(a, b), perm
