"""Batched label-map consumers without a GPU: argument checks (they come before any device work), the ABI
declarations and the documented size of the adjacency graph's scratch."""
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ("fslic_b200_connectivity_batch_scratch_bytes", "fslic_b200_get_connectivity_batch",
               "fslic_b200_get_mask_density_batch", "fslic_b200_cluster_density_to_mask_batch")


def _slic(K=10):
    from fast_slic_b200 import Slic
    return Slic(num_components=K)


def _clusters(B, K):
    from fast_slic_b200 import CLUSTER_DTYPE
    return np.zeros((B, K), CLUSTER_DTYPE)


def test_connectivity_argument_errors():
    s = _slic()
    lab = np.zeros((2, 8, 9), np.int16)
    for bad in (lab.astype(np.int32), lab.view(np.uint16), lab[0], lab[None], lab.tolist(), torch.from_numpy(lab)):
        with pytest.raises(ValueError):
            s.get_connectivity_batch(bad)


def test_mask_density_argument_errors():
    s = _slic(10)
    lab = np.zeros((2, 8, 9), np.int16)
    mask = np.zeros((2, 8, 9), np.uint8)
    cl = _clusters(2, 10)
    bad_calls = [
        (mask[:, :-1], lab, cl),                       # shape
        (mask[:1], lab, cl),                           # batch
        (mask.astype(np.int16), lab, cl),              # mask dtype
        (mask, lab.astype(np.uint8), cl),              # label dtype
        (mask, lab, _clusters(2, 9)),                  # K
        (mask, lab, _clusters(3, 10)),                 # B
        (mask, lab, cl.view(np.uint8).reshape(2, 10, 32).astype(np.float32)),
        (torch.from_numpy(mask), lab, cl),             # a cpu tensor
        (mask, lab, torch.from_numpy(cl.view(np.uint8).reshape(2, 10, 32).copy())),  # tensor clusters with numpy labels
    ]
    for args in bad_calls:
        with pytest.raises(ValueError):
            s.get_mask_density_batch(*args)


def test_broadcast_argument_errors():
    s = _slic(10)
    lab = np.zeros((2, 8, 9), np.int16)
    dens = np.zeros((2, 10), np.uint8)
    for d, l in ((dens[:, :-1], lab), (dens[:1], lab), (dens.astype(np.int32), lab), (dens[None], lab),
                 (dens, lab[0]), (torch.from_numpy(dens), lab)):
        with pytest.raises(ValueError):
            s.broadcast_density_to_mask_batch(d, l)


def test_abi_declares_and_binds_the_batch_entry_points():
    from fast_slic_b200 import _lib
    L = _lib.lib()
    header = open(os.path.join(ROOT, "include", "fslic_b200.h")).read()
    declared = set(re.findall(r"\b(fslic_b200_\w+)\s*\(", header))
    for sym in NEW_SYMBOLS:
        assert sym in declared and sym in _lib.EXPORTED_SYMBOLS, sym
        assert getattr(L, sym).argtypes is not None, sym  # bound: pointers and size_t must not pass as C ints
    assert L.fslic_b200_connectivity_batch_scratch_bytes.restype is not None


def _table_slots(K):
    t = 4096
    while t < 32 * K:
        t *= 2
    return t


def test_batch_scratch_grows_with_batch_and_components():
    from fast_slic_b200 import _lib
    f = _lib.lib().fslic_b200_connectivity_batch_scratch_bytes
    single = _lib.lib().fslic_b200_connectivity_scratch_bytes
    assert f(0, 4) == 256 and f(10, 0) == 256
    for K in (1, 128, 129, 1600, 65533):
        assert single(K) == f(K, 1), K
        prev = 0
        for B in (1, 2, 3, 32, 256):
            n = f(K, B)
            assert n >= 24 * _table_slots(K) * B + 4 * B, (K, B)
            assert n > prev
            prev = n
    assert f(1, 8) == f(128, 8)  # the table size is a power of two >= max(4096, 32 K)
    assert f(129, 8) > f(128, 8)
    assert f(1600, 8) < f(65533, 8)
    # more than 2^31 - 1 table slots cannot go through one radix sort: split the batch
    assert f(65535, 1023) < 2 ** 40 and f(65535, 1024) == 2 ** 64 - 1


def test_graph_chunk_respects_the_cap(monkeypatch):
    from fast_slic_b200 import _lib, graph_batch
    f = _lib.lib().fslic_b200_connectivity_batch_scratch_bytes
    assert graph_batch.graph_chunk(1600, 32) == 32
    c = graph_batch.graph_chunk(65533, 256)
    assert 1 <= c < 256 and f(65533, c) <= graph_batch.GRAPH_SCRATCH_CAP
    monkeypatch.setattr(graph_batch, "GRAPH_SCRATCH_CAP", 3 * f(300, 1))
    c = graph_batch.graph_chunk(300, 8)
    assert 1 <= c <= 3 and f(300, c) <= 3 * f(300, 1)
    monkeypatch.setattr(graph_batch, "GRAPH_SCRATCH_CAP", 1)
    assert graph_batch.graph_chunk(300, 8) == 1
