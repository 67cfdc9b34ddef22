"""Region adjacency graphs without a GPU: the ABI declarations, the argument checks (they come before any device work),
the scratch sizes and chunking, the overflow re-run's split, and the numpy restatement against a brute-force loop."""
import collections
import os
import re

import numpy as np
import pytest
import torch

from rag_cases import ref_rag, ref_rag_image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ("fslic_b200_rag_batch_scratch_bytes", "fslic_b200_rag_batch_count", "fslic_b200_rag_fill_scratch_bytes",
               "fslic_b200_rag_batch_fill")
NONE = 2 ** 64 - 1


def test_abi_declares_and_binds_the_rag_entry_points():
    from fast_slic_b200 import _lib
    L = _lib.lib()
    header = open(os.path.join(ROOT, "include", "fslic_b200.h")).read()
    declared = set(re.findall(r"\b(fslic_b200_\w+)\s*\(", header))
    for sym in NEW_SYMBOLS:
        assert sym in declared and sym in _lib.EXPORTED_SYMBOLS, sym
        assert getattr(L, sym).argtypes is not None, sym
    assert L.fslic_b200_rag_batch_scratch_bytes.restype is not None
    assert L.fslic_b200_rag_fill_scratch_bytes.restype is not None


def test_argument_errors():
    from fast_slic_b200.region_graph import region_adjacency
    l = torch.zeros((2, 5, 7), dtype=torch.int16)
    huge = torch.zeros((1, 1, 1), dtype=torch.int16).expand(2, 2 ** 15, 2 ** 14 + 1)  # 2^29 + 2^15 pixels per image
    assert huge.stride() == (0, 0, 0)
    bad = [
        ((l.numpy(), 10), "torch.from_numpy"),         # numpy labels
        ((l.int(), 10), "int16"),                      # dtype, before the device check
        ((l.to(torch.uint8), 10), "int16"),
        ((l[0], 10), "dimensions"),                    # ndim
        ((l[None], 10), "dimensions"),
        ((l, 0), "K must be"),                         # K range
        ((l, 65535), "K must be"),
        ((l, -1), "K must be"),
        ((l, 3.0), "K must be"),
        ((l, 10, 6), "connectivity"),                  # connectivity
        ((l, 10, 0), "connectivity"),
        ((l, 10, 4.0), "connectivity"),
        ((l, 10, "4"), "connectivity"),
        ((huge, 10), "int32"),                         # a boundary count could overflow int32
        ((l, 10), "cuda"),                             # cpu tensors
        ((l, 10, 8), "cuda"),
    ]
    for args, msg in bad:
        with pytest.raises(ValueError, match=msg):
            region_adjacency(*args)
    # the largest image is allowed past the size check (and refused as a cpu tensor)
    with pytest.raises(ValueError, match="cuda"):
        region_adjacency(torch.zeros((1, 1, 1), dtype=torch.int16).expand(1, 2 ** 15, 2 ** 14), 10)


def test_scratch_bytes_and_chunks(monkeypatch):
    from fast_slic_b200 import _lib, region_graph
    L = _lib.lib()
    f, g = L.fslic_b200_rag_batch_scratch_bytes, L.fslic_b200_rag_fill_scratch_bytes
    assert f(0, 5, 5, 10, 4, 0) == 256 and f(3, 0, 5, 10, 8, 0) == 256 and f(3, 5, 0, 10, 4, 1) == 256
    for args in ((1, 5, 5, 0, 4, 0), (1, 5, 5, 65535, 4, 0), (-1, 5, 5, 10, 4, 0), (1, 5, 5, 10, 6, 0),
                 (1, 2 ** 15, 2 ** 14 + 1, 10, 4, 0),     # more than 2^29 pixels
                 (40000, 2, 2, 65534, 4, 0),              # B * K + 1 > 2^31 - 1
                 (1, 2 ** 15, 2 ** 14, 65534, 8, 1)):     # an exact table over 2^31 slots
        assert f(*args) == NONE, args
    assert f(1, 2 ** 15, 2 ** 14, 1600, 8, 0) != NONE
    # superpixel maps: the graph's table, 2^16 slots for K = 1600; 8 bytes per slot, 16 per node
    for B, conn in ((1, 4), (32, 4), (32, 8)):
        assert f(B, 720, 1280, 1600, conn, 0) >= B * (8 * 65536 + 16 * 1600)
        assert f(B, 720, 1280, 1600, conn, 0) == f(B, 1080, 1920, 1600, conn, 0)
    # exact tables: a power of two >= 2 * min(K (K - 1) / 2, pixel pairs) per image
    pairs4 = 61 * 76 + 60 * 77
    assert 8 * 32768 <= f(1, 61, 77, 65534, 4, 1) < 8 * 32768 + 16 * 65535 + 65536 and 2 * pairs4 <= 32768
    assert f(1, 61, 77, 65534, 4, 0) == f(1, 61, 77, 65534, 4, 1)  # smaller than the graph's 2^21 slots
    assert f(1, 720, 1280, 65534, 8, 1) > 8 * 2 * 4 * 720 * 1280 > f(1, 720, 1280, 65534, 8, 0)
    assert f(1, 100, 100, 1, 8, 0) < 4096  # K = 1: no key can exist
    assert g(2, 10, 0) == 256 and g(2, 10, -1) == NONE and g(2, 10, 2 ** 31) == NONE and g(0, 10, 5) != NONE
    assert g(2, 10, 100) >= 1200 and g(2, 10, 2 ** 31 - 1) != NONE
    assert region_graph.rag_chunk(32, 720, 1280, 1600, 4) == 32
    monkeypatch.setattr(region_graph, "RAG_SCRATCH_CAP", 3 * f(1, 240, 320, 300, 4, 0))
    c = region_graph.rag_chunk(8, 240, 320, 300, 4)
    assert 1 <= c <= 3 and f(c, 240, 320, 300, 4, 0) <= region_graph.RAG_SCRATCH_CAP
    monkeypatch.setattr(region_graph, "RAG_SCRATCH_CAP", 1)
    assert region_graph.rag_chunk(8, 240, 320, 300, 8) == 1
    with pytest.raises(ValueError, match="too large"):
        region_graph.rag_chunk(1, 2 ** 15, 2 ** 15, 1, 4)


def test_overflow_split():
    from fast_slic_b200.region_graph import _split
    assert _split(4, [0, 1, 0, 0, 1]) == [(4, 1, 0), (5, 1, 1), (6, 2, 0), (8, 1, 1)]
    assert _split(0, [1]) == [(0, 1, 1)]
    assert _split(2, [1, 1, 0]) == [(2, 1, 1), (3, 1, 1), (4, 1, 0)]


def _brute(labels, K, connectivity):
    """Every pixel, every forward neighbour, in two Python loops: {(a, c): pairs} over unordered label pairs."""
    H, W = labels.shape
    lab = labels.view(np.uint16)
    offsets = [(0, 1), (1, 0)] + ([(1, 1), (1, -1)] if connectivity == 8 else [])
    count = collections.Counter()
    for i in range(H):
        for j in range(W):
            for di, dj in offsets:
                i2, j2 = i + di, j + dj
                if not (0 <= i2 < H and 0 <= j2 < W):
                    continue
                a, c = int(lab[i, j]), int(lab[i2, j2])
                if a < K and c < K and a != c:
                    count[min(a, c), max(a, c)] += 1
    return count


def _maps(rng):
    H, W = 13, 17
    yy, xx = np.mgrid[:H, :W]
    yield (yy // 4 * 10 + xx // 5).astype(np.int16), 40
    yield rng.randint(0, 20, (H, W)).astype(np.int16), 20
    yield rng.randint(-1, 25, (H, W)).astype(np.int16), 20     # -1 and labels >= K
    yield rng.randint(-1, 2, (H, W)).astype(np.int16), 1       # K = 1
    yield rng.randint(0, 6, (1, 40)).astype(np.int16), 6       # H = 1
    yield rng.randint(0, 6, (40, 1)).astype(np.int16), 6       # W = 1
    yield np.array([[5]], np.int16), 9
    yield ((yy + xx) % 2).astype(np.int16), 2                  # checkerboard
    yield rng.choice(np.array([0, 3, 65533, 65535], np.uint16), (H, W)).view(np.int16), 65534


@pytest.mark.parametrize("connectivity", [4, 8])
def test_restatement_agrees_with_brute_force(connectivity):
    rng = np.random.RandomState(11)
    maps = list(_maps(rng))
    for labels, K in maps:
        src, dst, w = ref_rag_image(labels, K, connectivity)
        want = _brute(labels, K, connectivity)
        got = collections.Counter()
        for s, d, c in zip(src.tolist(), dst.tolist(), w.tolist()):
            got[s, d] = c
        assert len(got) == len(src) == 2 * len(want)
        for (a, c), n in want.items():
            assert got[a, c] == got[c, a] == n
        assert sorted(zip(src.tolist(), dst.tolist())) == list(zip(src.tolist(), dst.tolist()))
    # the batch form: node ids b*K + label, CSR offsets over B*K rows
    labels = np.stack([m for m, _ in maps[:3]])
    indptr, edge_index, boundary = ref_rag(labels, 40, connectivity)
    assert indptr.dtype == np.int64 and edge_index.dtype == np.int64 and boundary.dtype == np.int32
    assert indptr.shape == (3 * 40 + 1,) and edge_index.shape == (2, boundary.size) and indptr[-1] == boundary.size
    for n in range(3 * 40):
        assert (edge_index[0, indptr[n]:indptr[n + 1]] == n).all()
        assert (edge_index[1, indptr[n]:indptr[n + 1]] // 40 == n // 40).all()
    empty = ref_rag(np.zeros((0, 4, 4), np.int16), 7, connectivity)
    assert empty[0].tolist() == [0] and empty[1].shape == (2, 0) and empty[2].shape == (0,)
