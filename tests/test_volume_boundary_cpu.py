"""Boundary statistics, outlines and segmentation scores of label volumes without a GPU: the numpy restatement
(volume_boundary_cases.py) against brute-force loops over voxels, its agreement with the 2-D restatements at D = 1,
the ABI, the scratch sizes and limits, the chunk helpers, and the argument checks (they come before any device
work)."""
import itertools
import math
import os
import re

import numpy as np
import pytest
import torch

from boundary_cases import ref_boundary
from groundtruth_cases import ref_boundaries, ref_scores
from volume_boundary_cases import (OFFSETS, dilate_3d, gt_boundary_map_3d, offsets, pair_ends_3d, ref_boundaries_3d,
                                   ref_boundary3d, ref_scores_3d)
from volume_graph_cases import pair_count, ref_rag3d

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NONE = 2 ** 64 - 1
ARGC = {"fslic_b200_boundary3d_select_scratch_bytes": 6, "fslic_b200_boundary3d_select_batch": 12,
        "fslic_b200_boundary3d_stats_scratch_bytes": 3, "fslic_b200_boundary3d_stats_batch": 27,
        "fslic_b200_gt_scores3d_scratch_bytes": 5, "fslic_b200_gt_scores3d_batch": 18,
        "fslic_b200_gt_boundaries3d_batch": 8}


def test_abi_declares_and_binds_the_volume_entry_points():
    from fast_slic_b200 import _lib
    L = _lib.lib()
    header = open(os.path.join(ROOT, "include", "fslic_b200.h")).read()
    declared = set(re.findall(r"\b(fslic_b200_\w+)\s*\(", header))
    for sym, argc in ARGC.items():
        assert sym in declared and sym in _lib.EXPORTED_SYMBOLS, sym
        assert len(getattr(L, sym).argtypes) == argc, sym
    for sym in ("fslic_b200_boundary3d_select_scratch_bytes", "fslic_b200_boundary3d_stats_scratch_bytes",
                "fslic_b200_gt_scores3d_scratch_bytes"):
        assert getattr(L, sym).restype is not None, sym
    # the 2-D entry points keep their arguments
    assert len(L.fslic_b200_boundary_select_scratch_bytes.argtypes) == 5
    assert len(L.fslic_b200_boundary_select_batch.argtypes) == 11
    assert len(L.fslic_b200_boundary_stats_scratch_bytes.argtypes) == 2
    assert len(L.fslic_b200_boundary_stats_batch.argtypes) == 25
    assert len(L.fslic_b200_gt_scores_scratch_bytes.argtypes) == 4
    assert len(L.fslic_b200_gt_scores_batch.argtypes) == 15
    assert len(L.fslic_b200_gt_boundaries_batch.argtypes) == 7


def test_offsets_are_region_adjacency_3d_s():
    from fast_slic_b200.region_graph import RAG3D_OFFSETS
    assert tuple(RAG3D_OFFSETS) == OFFSETS
    for conn, n in ((6, 3), (18, 9), (26, 13)):
        assert len(offsets(conn)) == n
        a, o, ords = pair_ends_3d(4, 5, 6, conn)
        assert a.size == pair_count(4, 5, 6, conn) and np.unique(ords).size == a.size
        assert (o > a).all()  # every forward offset is positive in linear index


def test_select_scratch_bytes():
    from fast_slic_b200 import _lib
    L = _lib.lib()
    f, s = L.fslic_b200_boundary3d_select_scratch_bytes, L.fslic_b200_boundary3d_stats_scratch_bytes
    assert f(0, 4, 5, 5, 10, 6) == 256 and f(3, 0, 5, 5, 10, 18) == 256 and f(3, 5, 5, 0, 10, 26) == 256
    for args in ((1, 4, 5, 5, 0, 6), (1, 4, 5, 5, 65535, 6), (-1, 4, 5, 5, 10, 6), (1, -1, 5, 5, 10, 6),
                 (1, 4, 5, 5, 10, 4), (1, 4, 5, 5, 10, 8), (1, 4, 5, 5, 10, 27),
                 (1, 2, 2 ** 14, 2 ** 14 + 1, 10, 6),     # more than 2^29 voxels
                 (1, 2 ** 30, 2 ** 30, 2 ** 30, 10, 6),   # no overflow of D * H * W on the way
                 (1, 512, 1024, 1024, 10, 18),            # 2^29 voxels: more than 2^31 - 1 pairs at 18 and 26
                 (1, 512, 1024, 1024, 10, 26),
                 (32, 256, 512, 512, 10, 6)):             # more than 2^31 - 1 voxels in one call
        assert f(*args) == NONE, args
    # a 2^29-voxel volume is taken at 6-connectivity; one CT volume's select stays far under 1 GiB at 26
    assert f(1, 512, 1024, 1024, 100, 6) != NONE
    ct = f(1, 256, 512, 512, 16384, 26)
    assert ct < 1 << 30 and 6 * 2 ** 26 <= ct <= 8 * 2 ** 26
    for conn in (6, 18, 26):  # sized per voxel, not per voxel pair
        assert f(1, 256, 512, 512, 16384, conn) == ct
    # stats: 4 bytes per voxel, 34 per pair, 24 per entry and the temporary storage
    assert s(0, 0, 0) > 0 and s(10, 100, 1000) > 4 * 10 + 34 * 100 + 24 * 1000
    for args in ((-1, 0, 0), (0, -1, 0), (0, 0, -1), (2 ** 31, 2 ** 31, 0), (1, 2 ** 31, 0), (0, 0, 2 ** 31),
                 (10, 9, 0), (10, 131, 0)):
        assert s(*args) == NONE, args


def test_gt_scratch_bytes():
    from fast_slic_b200 import _lib
    L = _lib.lib()
    f, f2 = L.fslic_b200_gt_scores3d_scratch_bytes, L.fslic_b200_gt_scores_scratch_bytes
    assert f(0, 4, 5, 5, 10) == 256 and f(3, 0, 5, 5, 10) == 256 and f(3, 5, 5, 0, 10) == 256
    for args in ((1, 4, 5, 5, 0), (1, 4, 5, 5, 65535), (-1, 4, 5, 5, 10), (1, -1, 5, 5, 10),
                 (1, 2, 2 ** 14, 2 ** 14 + 1, 10), (1, 2 ** 30, 2 ** 30, 2 ** 30, 10), (32, 256, 512, 512, 10),
                 (2 ** 17 + 1, 1, 1, 1, 10)):
        assert f(*args) == NONE, args
    # the 2-D layout with H = D * H and two more bitmaps
    for B, D, H, W, K in ((1, 1, 61, 77, 100), (3, 5, 40, 70, 300), (8, 155, 240, 240, 4000)):
        words = B * D * H * ((W + 31) // 32)
        assert f2(B, D * H, W, K) < f(B, D, H, W, K) <= f2(B, D * H, W, K) + 2 * (4 * words + 256)


def test_chunks(monkeypatch):
    from fast_slic_b200 import _lib, groundtruth, region_graph
    L = _lib.lib()
    f, g = L.fslic_b200_boundary3d_select_scratch_bytes, L.fslic_b200_gt_scores3d_scratch_bytes
    assert region_graph.boundary3d_chunk(8, 100, 192, 192, 4000, 26) == 8
    assert groundtruth.gt3d_chunk(8, 40, 96, 96, 4000) == 8
    monkeypatch.setattr(region_graph, "BOUNDARY_SCRATCH_CAP", 3 * f(1, 100, 192, 192, 4000, 26))
    c = region_graph.boundary3d_chunk(8, 100, 192, 192, 4000, 26)
    assert 1 <= c <= 3 and f(c, 100, 192, 192, 4000, 26) <= region_graph.BOUNDARY_SCRATCH_CAP
    monkeypatch.setattr(groundtruth, "GT_SCRATCH_CAP", 2 * g(1, 40, 96, 96, 4000))
    c = groundtruth.gt3d_chunk(8, 40, 96, 96, 4000)
    assert 1 <= c <= 2 and g(c, 40, 96, 96, 4000) <= groundtruth.GT_SCRATCH_CAP
    assert region_graph.boundary3d_chunk(1, 512, 1024, 1024, 10, 6) == 1  # a volume over the cap still runs alone
    with pytest.raises(ValueError, match="too large"):
        region_graph.boundary3d_chunk(1, 512, 1024, 1024, 10, 26)


def test_tolerance():
    from fast_slic_b200.groundtruth import check_tolerance_3d
    assert check_tolerance_3d(3) == (3, 3, 3) and check_tolerance_3d((0, 32, 5)) == (0, 32, 5)
    assert check_tolerance_3d([1, 2, 3]) == (1, 2, 3) and check_tolerance_3d(np.int64(4)) == (4, 4, 4)
    for bad in (-1, 33, 2.0, (1, 2), (1, 2, 3, 4), (1, 2, 33), (-1, 0, 0), (1, 2.5, 3), "2", None):
        with pytest.raises(ValueError, match="tolerance"):
            check_tolerance_3d(bad)


def test_argument_errors():
    from fast_slic_b200.groundtruth import boundaries_3d, segmentation_scores_3d
    from fast_slic_b200.region_graph import RegionGraph, boundary_stats_3d
    l = torch.zeros((2, 3, 5, 7), dtype=torch.int16)
    v = torch.zeros((2, 2, 3, 5, 7), dtype=torch.float32)
    g = RegionGraph(torch.zeros(2 * 10 + 1, dtype=torch.int64), torch.zeros((2, 4), dtype=torch.int64),
                    torch.zeros(4, dtype=torch.int32))
    huge = torch.zeros((1, 1, 1, 1), dtype=torch.int16).expand(1, 2, 2 ** 14, 2 ** 14 + 1)  # over 2^29 voxels
    hv = torch.zeros((1, 1, 1, 1, 1)).expand(1, 1, 2, 2 ** 14, 2 ** 14 + 1)
    dense = torch.zeros((1, 1, 1, 1), dtype=torch.int16).expand(1, 512, 1024, 1024)       # 2^29 voxels
    dv = torch.zeros((1, 1, 1, 1, 1)).expand(1, 1, 512, 1024, 1024)
    g1 = RegionGraph(torch.zeros(11, dtype=torch.int64), torch.zeros((2, 0), dtype=torch.int64),
                     torch.zeros(0, dtype=torch.int32))
    bad = [
        ((l.numpy(), 10, g, v), "torch.from_numpy"),
        ((l.int(), 10, g, v), "int16"),
        ((l[0], 10, g, v), "dimensions"),
        ((l, 10, g, v[0]), "dimensions"),
        ((l, 10, g, v.double()), "float32"),
        ((l, 10, g, v[:1]), "do not match"),
        ((l, 10, g, v[:, :, :2]), "do not match"),
        ((l, 10, g, v[:, :0]), "channel"),
        ((l, 0, g, v), "K must be"),
        ((l, 65535, g, v), "K must be"),
        ((l, 10, g, v, 4), "connectivity"),
        ((l, 10, g, v, 8), "connectivity"),
        ((l, 10, g, v, 6.0), "connectivity"),
        ((huge, 10, g1, hv), "exceed"),
        ((dense, 10, g1, dv, 18), "int32"),
        ((dense, 10, g1, dv, 26), "int32"),
        ((l, 11, g, v), "indptr"),
        ((l, 10, RegionGraph(g.indptr, g.edge_index.int(), g.boundary), v), "int64"),
        ((l, 10, RegionGraph(g.indptr, g.edge_index[:1], g.boundary), v), r"\[2,E\]"),
        ((l, 10, g, v), "cuda"),
        ((l, 10, g, v, 26), "cuda"),
        ((dense, 10, g1, dv, 6), "cuda"),  # 2^29 voxels at 6-connectivity are allowed past the size checks
    ]
    for args, msg in bad:
        with pytest.raises(ValueError, match=msg):
            boundary_stats_3d(*args)
    gt = torch.zeros((2, 3, 5, 7), dtype=torch.int64)
    for args, kw, msg in [((l.numpy(), gt, 10), {}, "torch.from_numpy"), ((l.int(), gt, 10), {}, "int16"),
                          ((l[0], gt[0], 10), {}, "dimensions"), ((l, gt.numpy(), 10), {}, "torch.from_numpy"),
                          ((l, gt.float(), 10), {}, "uint8, int16"), ((l, gt[:1], 10), {}, "does not match"),
                          ((l, gt, 0), {}, "K must be"), ((huge, huge, 10), {}, "exceed"),
                          ((l, gt, 10), {"tolerance": 33}, "tolerance"),
                          ((l, gt, 10), {"tolerance": (1, 2)}, "tolerance"),
                          ((l, gt, 10), {"tolerance": (1, 2, 33)}, "tolerance"),
                          ((l, gt, 10), {"tolerance": (-1, 2, 3)}, "tolerance"),
                          ((l, gt, 10), {"ignore_index": 1.5}, "ignore_index"),
                          ((l, gt, 10), {"tolerance": (0, 32, 1)}, "cuda")]:
        with pytest.raises(ValueError, match=msg):
            segmentation_scores_3d(*args, **kw)
    for args, msg in [(l.numpy(), "torch.from_numpy"), (l.int(), "int16"), (l[0], "dimensions"), (huge, "exceed"),
                      (l, "cuda")]:
        with pytest.raises(ValueError, match=msg):
            boundaries_3d(args)


def _brute_stats(labels, values, K, connectivity):
    """Every voxel in ordinal order and every direction, in Python loops: {(lo, hi): (mean, min, max) per channel,
    count}, the mean summed over 32 lanes and combined by the butterfly in float32."""
    D, H, W = labels.shape
    lab = labels.view(np.uint16)
    C = values.shape[0]
    seq = {}
    for z, y, x in itertools.product(range(D), range(H), range(W)):
        for dz, dy, dx in offsets(connectivity):
            z2, y2, x2 = z + dz, y + dy, x + dx
            if 0 <= z2 < D and 0 <= y2 < H and 0 <= x2 < W:
                a, c = int(lab[z, y, x]), int(lab[z2, y2, x2])
                if a < K and c < K and a != c:
                    seq.setdefault((min(a, c), max(a, c)), []).append(((z, y, x), (z2, y2, x2)))
    out = {}
    for key, pairs in seq.items():
        stats = []
        for ch in range(C):
            vals = [values[ch][p] for pr in pairs for p in pr]
            lanes = [np.float32(0.0)] * 32
            with np.errstate(invalid="ignore", over="ignore"):
                for j, x in enumerate(vals):
                    lanes[j % 32] = np.float32(lanes[j % 32] + x)
                for off in (16, 8, 4, 2, 1):
                    lanes = [np.float32(lanes[l] + lanes[l ^ off]) for l in range(32)]
                mean = np.float32(lanes[0] / np.float32(len(vals)))
            if any(math.isnan(x) for x in vals):
                mn = mx = np.float32("nan")
            else:
                order = sorted(vals, key=lambda x: (float(x), math.copysign(1.0, float(x))))
                mn, mx = order[0], order[-1]
            stats.append((mean, mn, mx))
        out[key] = (stats, len(pairs))
    return out


def _volumes(rng):
    D, H, W = 4, 5, 6
    zz, yy, xx = np.mgrid[:D, :H, :W]
    yield (zz // 2 * 100 + yy // 3 * 10 + xx // 4).astype(np.int16), 300
    yield rng.randint(0, 6, (D, H, W)).astype(np.int16), 6
    yield rng.randint(-1, 8, (D, H, W)).astype(np.int16), 6          # -1 and labels >= K
    yield rng.randint(0, 3, (1, 4, 9)).astype(np.int16), 3           # D = 1
    yield rng.randint(0, 3, (9, 1, 4)).astype(np.int16), 3           # H = 1
    yield rng.randint(0, 3, (4, 9, 1)).astype(np.int16), 3           # W = 1
    yield ((zz + yy + xx) % 2).astype(np.int16), 2                   # 3-D checkerboard
    yield rng.choice(np.array([0, 3, 65533, 65535], np.uint16), (D, H, W)).view(np.int16), 65534


def _values(rng, C, shape):
    v = rng.randn(C, *shape).astype(np.float32)
    v[rng.rand(*v.shape) < 0.03] = np.float32("nan")
    v[rng.rand(*v.shape) < 0.03] = np.float32("inf")
    v[rng.rand(*v.shape) < 0.03] = -np.float32("inf")
    v[rng.rand(*v.shape) < 0.05] = np.float32(-0.0)
    v[rng.rand(*v.shape) < 0.05] = np.float32(0.0)
    return v


@pytest.mark.parametrize("connectivity", [6, 18, 26])
def test_stats_restatement_agrees_with_brute_force(connectivity):
    rng = np.random.RandomState(31)
    for labels, K in _volumes(rng):
        values = _values(rng, 3, labels.shape)
        want = _brute_stats(labels, values, K, connectivity)
        _, (src, dst), w = ref_rag3d(labels[None], K, connectivity)
        mean, mn, mx, count = ref_boundary3d(labels[None], K, src, dst, values[None], connectivity)
        assert np.array_equal(count, w)  # count == the graph's boundary
        for e, (s, d) in enumerate(zip(src.tolist(), dst.tolist())):
            stats, n = want[min(s, d), max(s, d)]
            assert count[e] == n
            for ch, (m, lo, hi) in enumerate(stats):
                for got, ref in ((mean[e, ch], m), (mn[e, ch], lo), (mx[e, ch], hi)):
                    assert np.array([got], np.float32).view(np.int32)[0] == \
                        np.array([ref], np.float32).view(np.int32)[0] or (np.isnan(got) and np.isnan(ref))
    # entries across volumes, out of range, self loops, duplicates and absent pairs
    labels = np.stack([v for v, _ in list(_volumes(rng))[:2]])
    values = np.stack([_values(rng, 2, labels.shape[1:]) for _ in range(2)])
    K = 300
    src = np.array([0, 1, K + 1, -1, 5, 2 * K, 7, 0, 110, 110], np.int64)
    dst = np.array([1, 0, K + 2, 3, 5, 0, K + 7, 1, 111, 100], np.int64)
    mean, mn, mx, count = ref_boundary3d(labels, K, src, dst, values, connectivity)
    for e in (3, 4, 5, 6):
        assert count[e] == 0 and np.isnan(mean[e]).all() and np.isnan(mn[e]).all() and np.isnan(mx[e]).all()
    assert np.array_equal(mean[0].view(np.int32), mean[7].view(np.int32)) and count[0] == count[7]


def test_one_slice_equals_the_2d_restatements():
    """At D = 1, 6-connectivity is 4 and 18 and 26 are 8 in the same pair order; the outline and the scores with an
    int tolerance are the 2-D ones."""
    rng = np.random.RandomState(5)
    maps = [(rng.randint(-1, 30, (3, 23, 29)).astype(np.int16), 25),
            (np.kron(rng.randint(0, 50, (2, 6, 8)), np.ones((1, 5, 4), np.int64)).astype(np.int16), 50)]
    for lab2, K in maps:
        vol = lab2[:, None]
        values = np.stack([_values(rng, 5, lab2.shape[1:]) for _ in range(lab2.shape[0])])
        for c3, c2 in ((6, 4), (18, 8), (26, 8)):
            _, ei, _ = ref_rag3d(vol, K, c3)
            got = ref_boundary3d(vol, K, ei[0], ei[1], values[:, :, None], c3)
            want = ref_boundary(lab2, K, ei[0], ei[1], values, c2)
            for a, b in zip(got, want):
                assert a.dtype == b.dtype and np.array_equal(a.view(np.int32), b.view(np.int32))
        assert np.array_equal(ref_boundaries_3d(vol)[:, 0], ref_boundaries(lab2))
        gt = rng.randint(-1, 5, lab2.shape).astype(np.int32)
        for r in (0, 1, 3):
            for ignore in (None, 2):
                got, want = ref_scores_3d(vol, gt[:, None], K, (7, r, r), ignore), ref_scores(lab2, gt, K, r, ignore)
                for f, w in want.items():
                    assert np.array_equal(got[f], w, equal_nan=True), f


def test_scores_restatement_agrees_with_brute_force():
    """The dilation against a scan of every box, and the boundary maps against loops over voxels."""
    rng = np.random.RandomState(9)
    D, H, W = 5, 6, 7
    for _ in range(3):
        lab = rng.randint(0, 3, (D, H, W)).astype(np.int16)
        gt = rng.randint(-1, 3, (D, H, W)).astype(np.int64)
        sp = ref_boundaries_3d(lab[None])[0]
        gb = gt_boundary_map_3d(gt, 1)
        for z, y, x in itertools.product(range(D), range(H), range(W)):
            nb = [(z, y, x + 1), (z, y + 1, x), (z + 1, y, x)]
            inside = [(a, b, c) for a, b, c in nb if a < D and b < H and c < W]
            assert sp[z, y, x] == any(lab[p] != lab[z, y, x] for p in inside)
            ok = lambda p: 0 <= gt[p] and gt[p] != 1  # noqa: E731
            assert gb[z, y, x] == (ok((z, y, x)) and any(ok(p) and gt[p] != gt[z, y, x] for p in inside))
        for tol in ((0, 0, 0), (1, 0, 2), (2, 1, 0), (0, 3, 1), (4, 4, 4)):
            got = dilate_3d(sp, tol)
            rz, ry, rx = tol
            for z, y, x in itertools.product(range(D), range(H), range(W)):
                box = sp[max(0, z - rz):z + rz + 1, max(0, y - ry):y + ry + 1, max(0, x - rx):x + rx + 1]
                assert got[z, y, x] == box.any()
            res = ref_scores_3d(lab[None], gt[None], 3, tol, 1)
            valid = (gt >= 0) & (gt != 1)
            assert res["gt_boundary"][0] == gb.sum() and res["sp_boundary"][0] == (sp & valid).sum()
            assert res["gt_boundary_hits"][0] == (gb & got).sum()
            assert res["pixels"][0] == (valid & (lab.view(np.uint16) < 3)).sum()
