"""Superpixel shapes without a GPU: the ABI declaration, the argument checks (they come before any device work), the
numpy restatement against a per-pixel Python loop, hand-computed answers, and the perimeter against the region
adjacency graph's boundary lengths."""
import os
import re

import numpy as np
import pytest
import torch

from geometry_cases import ref_finish, ref_properties, ref_properties_image
from rag_cases import ref_rag_image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_abi_declares_and_binds_the_props_entry_point():
    from fast_slic_b200 import _lib
    L = _lib.lib()
    header = open(os.path.join(ROOT, "include", "fslic_b200.h")).read()
    declared = set(re.findall(r"\b(fslic_b200_\w+)\s*\(", header))
    assert "fslic_b200_props_batch" in declared and "fslic_b200_props_batch" in _lib.EXPORTED_SYMBOLS
    assert len(L.fslic_b200_props_batch.argtypes) == 14


def test_argument_errors():
    from fast_slic_b200.geometry import region_properties
    l = torch.zeros((2, 5, 7), dtype=torch.int16)
    one = torch.zeros((1, 1, 1), dtype=torch.int16)
    for lab, K, msg in [
        (l.numpy(), 10, "torch.from_numpy"),                       # numpy labels
        (l.int(), 10, "int16"),                                    # dtype
        (l.to(torch.uint8), 10, "int16"),
        (l[0], 10, "dimensions"),                                  # ndim
        (l[None], 10, "dimensions"),
        (l, 0, "K must be"), (l, 65535, "K must be"), (l, 3.0, "K must be"), (l, "5", "K must be"),
        (one.expand(1, 65536, 1), 10, "side"),                     # H just past the limit
        (one.expand(1, 1, 65536), 10, "side"),                     # W just past the limit
        (one.expand(2, 2 ** 15, 2 ** 14 + 1), 10, "exceed"),       # 2^29 + 2^15 pixels per image
        (l, 10, "cuda"),                                           # cpu tensor
    ]:
        with pytest.raises(ValueError, match=msg):
            region_properties(lab, K)
    # the exact limits pass every size check and are refused only as cpu tensors
    for shape in ((1, 65535, 1), (1, 1, 65535), (1, 65535, 8192), (1, 8192, 65535), (1, 2 ** 15, 2 ** 14),
                  (0, 65535, 8192)):
        with pytest.raises(ValueError, match="cuda"):
            region_properties(one.expand(*shape), 65534)
    with pytest.raises(ValueError, match="cuda"):
        region_properties(l, 1)


def _brute(labels, K):
    """Every pixel in Python loops, the float fields with Python floats (IEEE doubles) in the documented order."""
    H, W = labels.shape
    lab = labels.view(np.uint16).astype(int)
    f = {"area": [0] * K, "perimeter": [0] * K, "border": [0] * K, "moments": [[0] * 5 for _ in range(K)],
         "bbox": [[0] * 4 for _ in range(K)]}
    for y in range(H):
        for x in range(W):
            k = lab[y, x]
            if k >= K:
                continue
            if f["area"][k] == 0:
                f["bbox"][k] = [y, x, y + 1, x + 1]
            b = f["bbox"][k]
            f["bbox"][k] = [min(b[0], y), min(b[1], x), max(b[2], y + 1), max(b[3], x + 1)]
            f["area"][k] += 1
            for i, v in enumerate((y, x, y * y, x * y, x * x)):
                f["moments"][k][i] += v
            for ny, nx in ((y - 1, x), (y + 1, x), (y, x - 1), (y, x + 1)):
                outside = not (0 <= ny < H and 0 <= nx < W)
                if outside or lab[ny, nx] != k:
                    f["perimeter"][k] += 1
                f["border"][k] += outside
    cen, cov = [], []
    for k in range(K):
        n, m = f["area"][k], f["moments"][k]
        if n == 0:
            cen.append([0.0, 0.0])
            cov.append([0.0, 0.0, 0.0])
            continue
        cy, cx = float(m[0]) / float(n), float(m[1]) / float(n)
        cen.append([cy, cx])
        cov.append([float(m[2]) / float(n) - cy * cy, float(m[3]) / float(n) - cy * cx, float(m[4]) / float(n) - cx * cx])
    f["centroid"], f["covariance"] = cen, cov
    return f


def _maps(rng):
    H, W = 11, 13
    yy, xx = np.mgrid[:H, :W]
    yield (yy // 4 * 4 + xx // 5).astype(np.int16), 12
    yield rng.randint(-1, 25, (H, W)).astype(np.int16), 20                     # -1 and labels >= K
    yield rng.randint(0, 3, (H, W)).astype(np.int16), 3
    yield rng.randint(0, 4, (1, 40)).astype(np.int16), 4                       # H = 1
    yield rng.randint(0, 4, (40, 1)).astype(np.int16), 4                       # W = 1
    yield np.array([[3]], np.int16), 9
    yield np.full((H, W), -1, np.int16), 5                                     # no superpixel pixel
    yield ((yy * 7 + xx * 3) % 65534).astype(np.uint16).view(np.int16), 65534  # large labels
    yield rng.randint(0, 5, (37, 70)).astype(np.int16), 5                      # runs across 32-column words


def test_restatement_agrees_with_brute_force():
    rng = np.random.RandomState(4)
    for labels, K in _maps(rng):
        want = _brute(labels, K)
        got = ref_properties(labels[None], K)
        for f, v in want.items():
            assert np.array_equal(got[f][0], np.array(v).reshape(got[f].shape[1:])), (labels.shape, K, f)
        assert got["area"].dtype == np.int32 and got["bbox"].dtype == np.int32 and got["moments"].dtype == np.int64
        assert got["centroid"].dtype == np.float64 and got["covariance"].dtype == np.float64


def test_known_answers():
    # a single pixel: perimeter 4; border 2 in a corner, 1 on an edge, 0 inside
    for (y, x), border in (((0, 0), 2), ((4, 6), 2), ((0, 3), 1), ((2, 3), 0)):
        lab = np.zeros((5, 7), np.int16)
        lab[y, x] = 1
        p = ref_properties(lab[None], 2)
        assert p["area"][0, 1] == 1 and p["perimeter"][0, 1] == 4 and p["border"][0, 1] == border
        assert list(p["bbox"][0, 1]) == [y, x, y + 1, x + 1]
        assert list(p["moments"][0, 1]) == [y, x, y * y, x * y, x * x]
        assert list(p["centroid"][0, 1]) == [y, x] and not p["covariance"][0, 1].any()
    # one label over the whole image: perimeter = border = 2 (H + W), the pixel-grid centroid and variances
    for H, W in ((1, 1), (1, 9), (6, 1), (5, 8)):
        p = ref_properties(np.zeros((1, H, W), np.int16), 3)
        assert p["area"][0, 0] == H * W and p["perimeter"][0, 0] == p["border"][0, 0] == 2 * (H + W)
        assert list(p["bbox"][0, 0]) == [0, 0, H, W] and not p["area"][0, 1:].any() and not p["bbox"][0, 1:].any()
        assert list(p["centroid"][0, 0]) == [(H - 1) / 2, (W - 1) / 2]
        assert np.allclose(p["covariance"][0, 0], [(H * H - 1) / 12, 0.0, (W * W - 1) / 12])
    # a 2x2 checkerboard: every pixel its own run, every inner side a boundary
    p = ref_properties(np.array([[[0, 1], [1, 0]]], np.int16), 2)
    assert list(p["area"][0]) == [2, 2] and list(p["perimeter"][0]) == [8, 8] and list(p["border"][0]) == [4, 4]
    assert [list(b) for b in p["bbox"][0]] == [[0, 0, 2, 2], [0, 0, 2, 2]]
    assert [list(m) for m in p["moments"][0]] == [[1, 1, 1, 1, 1], [1, 1, 1, 0, 1]]
    assert [list(c) for c in p["covariance"][0]] == [[0.25, 0.25, 0.25], [0.25, -0.25, 0.25]]
    # a 1xW strip of runs a..b: perimeter 2 m + 2, border 2 m plus the ends on the image edge
    lab = np.array([[0, 0, 0, 1, 1, 2, 0, 0]], np.int16)
    p = ref_properties(lab[None], 3)
    assert list(p["area"][0]) == [5, 2, 1]
    assert list(p["perimeter"][0]) == [2 * 5 + 4, 2 * 2 + 2, 2 * 1 + 2]
    assert list(p["border"][0]) == [2 * 5 + 2, 2 * 2, 2 * 1]
    assert [list(b) for b in p["bbox"][0]] == [[0, 0, 1, 8], [0, 3, 1, 5], [0, 5, 1, 6]]
    assert list(p["moments"][0, 0]) == [0, 0 + 1 + 2 + 6 + 7, 0, 0, 0 + 1 + 4 + 36 + 49]
    # empty nodes: zeros, never NaN
    c, v = ref_finish(np.zeros(3, np.int32), np.zeros((3, 5), np.int64))
    assert not c.any() and not v.any() and not np.isnan(c).any()


def test_perimeter_is_border_plus_boundary_lengths():
    """perimeter - border = the 4-connectivity region adjacency boundary weights of k + sides facing labels outside
    [0, K)."""
    rng = np.random.RandomState(9)
    yy, xx = np.mgrid[:40, :50]
    maps = [((yy // 6) * 9 + xx // 6).astype(np.int16), rng.randint(-1, 14, (40, 50)).astype(np.int16),
            rng.randint(0, 3, (1, 60)).astype(np.int16), rng.randint(0, 3, (60, 1)).astype(np.int16)]
    for labels in maps:
        K = 12
        p = ref_properties_image(labels, K)
        src, _, w = ref_rag_image(labels, K, 4)
        rag = np.bincount(src, weights=w, minlength=K).astype(np.int64)
        lab = labels.view(np.uint16).astype(np.int64)
        outside = np.zeros(K, np.int64)
        for a, b in ((lab[:, :-1], lab[:, 1:]), (lab[:-1, :], lab[1:, :])):
            for u, v in ((a, b), (b, a)):
                sel = (u < K) & (v >= K)
                np.add.at(outside, u[sel], 1)
        assert np.array_equal(p["perimeter"] - p["border"], rag + outside)
