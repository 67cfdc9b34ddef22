"""Message passing over superpixel graphs (fast_slic_b200.message_passing) without a GPU: the numpy restatement
(message_passing_cases.py) against scalar loops and against float64 autograd of an independent dense implementation,
for values and every gradient; the argument checks; and the C ABI of the new entry points."""
import os
import re

import numpy as np
import pytest
import torch

from message_passing_cases import (F32, Graph, dense_torch, lane_sum, make_graph, nan_class_equal, okey, seq_max,
                                   seq_sum)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_ordered_sums_and_maxima_against_scalar_loops():
    rng = np.random.RandomState(1)
    seg = rng.randint(0, 7, 200)
    terms = (rng.randn(200, 3) * np.float32(10) ** rng.randint(-3, 4, (200, 1))).astype(F32)
    terms[5, 0], terms[9, 1], terms[11, 2] = -0.0, np.nan, -np.inf
    got = seq_sum(seg, terms, 9)
    best, arg = seq_max(seg, terms, np.arange(200), 9)
    for n in range(9):
        for c in range(3):
            acc, b, a = F32(0), F32(0), -1
            for i in np.nonzero(seg == n)[0]:
                acc = F32(acc + terms[i, c])
                v = terms[i, c]
                if a < 0 or (not np.isnan(b) and (np.isnan(v) or okey(v) > okey(b))):
                    b, a = v, i
            assert nan_class_equal(got[n, c], acc) and nan_class_equal(best[n, c], b) and arg[n, c] == a
    assert not np.signbit(got[7:]).any() and (arg[7:] == -1).all()
    # -0.0 < +0.0 in the order, and the first of equal values wins
    b, a = seq_max(np.zeros(4, np.int64), np.array([[-0.0], [0.0], [0.0], [-0.0]], F32), np.arange(4), 1)
    assert a[0, 0] == 1 and not np.signbit(b[0, 0])
    b, a = seq_max(np.zeros(3, np.int64), np.array([[1.0], [np.nan], [np.nan]], F32), np.arange(3), 1)
    assert a[0, 0] == 1 and np.isnan(b[0, 0])


def test_lane_sum_is_pools_order():
    rng = np.random.RandomState(2)
    for D in (1, 5, 16, 17, 32, 33, 70):
        t = rng.randn(3, 2, D).astype(F32)
        got = lane_sum(t)
        for m in range(3):
            for h in range(2):
                lanes = [F32(0)] * 32
                for j in range(D):
                    lanes[j % 32] = F32(lanes[j % 32] + t[m, h, j])
                for o in (16, 8, 4, 2, 1):
                    lanes = [F32(lanes[k] + lanes[k ^ o]) for k in range(32)]
                assert got[m, h].view(np.uint32) == lanes[0].view(np.uint32)


def test_restated_forwards_against_scalar_loops():
    indptr, t = make_graph(3, 12, invalid=0.2, self_loops=0.2, duplicates=0.2)
    g = Graph(indptr, t)
    rng = np.random.RandomState(3)
    x, w = rng.randn(12, 4).astype(F32), rng.randn(g.E, 2).astype(F32)
    out, deg, _ = g.aggregate(x, w, "sum")
    mean, _, _ = g.aggregate(x, w, "mean")
    sm = g.softmax(w)
    for n in range(12):
        es = [e for e in range(indptr[n], indptr[n + 1]) if 0 <= t[e] < 12]
        assert deg[n] == len(es)
        for c in range(4):
            acc = F32(0)
            for e in es:
                acc = F32(acc + F32(w[e, c // 2] * x[t[e], c]))
            assert out[n, c].view(np.uint32) == acc.view(np.uint32)
            want = F32(acc / F32(len(es))) if es else F32(0)
            assert mean[n, c].view(np.uint32) == want.view(np.uint32)
        if es:
            for h in range(2):
                m = max(w[es, h])
                y = [np.exp(F32(w[e, h] - m), dtype=F32) for e in es]
                Z = F32(0)
                for v in y:
                    Z = F32(Z + v)
                np.testing.assert_allclose(sm[es, h], np.array(y) / Z, rtol=1e-6)
    assert not sm[~g.valid].any() and not np.signbit(sm[~g.valid]).any()


def _check(restated, want, rtol=1e-4):
    want = want.detach().numpy().astype(np.float64)
    np.testing.assert_allclose(restated, want, rtol=rtol, atol=rtol * max(np.abs(want).max(), 1e-30))


@pytest.mark.parametrize("seed,N,H,C", [(10, 20, 1, 3), (11, 30, 2, 8), (12, 25, 6, 6), (13, 1, 1, 2)])
def test_restated_backward_against_float64_autograd(seed, N, H, C):
    """Every restated value and gradient against float64 autograd of dense_torch at the same float32 inputs.  Each
    restated operation is off by at most half an ulp (about 6e-8 relative) and the sums have at most a few dozen terms,
    so rtol 1e-4 (with an absolute term of 1e-4 times the largest magnitude) has a wide margin and still fails any
    wrong formula, which is off by O(1)."""
    indptr, t = make_graph(seed, N, invalid=0.15, self_loops=0.15, duplicates=0.15)
    g = Graph(indptr, t)
    rng = np.random.RandomState(seed)
    x, s = rng.randn(N, C).astype(F32), rng.randn(g.E, H).astype(F32)
    w = (rng.rand(g.E, H) + 0.5).astype(F32)
    gE, gN, gS = rng.randn(g.E, C).astype(F32), rng.randn(N, C).astype(F32), rng.randn(g.E, H).astype(F32)
    gather, softmax, aggregate = dense_torch(indptr, t)
    d = lambda a: torch.tensor(a, dtype=torch.float64, requires_grad=True)  # noqa: E731

    for end in ("target", "source"):
        X = d(x)
        y = gather(X, end)
        _check(g.gather(x, end), y)
        (y * torch.tensor(gE, dtype=torch.float64)).sum().backward()
        _check(g.gather_backward(gE, end), X.grad)

    S = d(s)
    y = softmax(S)
    out = g.softmax(s)
    _check(out, y)
    (y * torch.tensor(gS, dtype=torch.float64)).sum().backward()
    _check(g.softmax_backward(out, gS), S.grad)

    for reduce in ("sum", "mean", "max"):
        for weighted in (False, True):
            X, W = d(x), d(w)
            y = aggregate(X, W if weighted else None, reduce)
            out, deg, amax = g.aggregate(x, w if weighted else None, reduce)
            _check(out, y)
            (y * torch.tensor(gN, dtype=torch.float64)).sum().backward()
            gx, gw = g.aggregate_backward(x, w if weighted else None, gN, reduce, amax)
            _check(gx, X.grad)
            if weighted:
                _check(gw, W.grad)


def _graph(N, E):
    return type("G", (), {"indptr": torch.zeros(N + 1, dtype=torch.int64),
                          "edge_index": torch.zeros((2, E), dtype=torch.int64)})()


def test_argument_errors():
    from fast_slic_b200.message_passing import aggregate, edge_gather, edge_softmax
    x, g = torch.zeros((4, 6)), _graph(4, 10)
    w, s = torch.zeros(10), torch.zeros((10, 3))
    huge = type("G", (), {"indptr": torch.zeros(1, dtype=torch.int64).expand(2 ** 31 + 1),
                          "edge_index": torch.zeros((2, 1), dtype=torch.int64)})()
    bad_ei = type("G", (), {"indptr": g.indptr, "edge_index": torch.zeros((3, 10), dtype=torch.int64)})()
    many_e = type("G", (), {"indptr": torch.zeros(5, dtype=torch.int64),
                            "edge_index": torch.zeros((2, 1), dtype=torch.int64).expand(2, 2 ** 31)})()
    for fn, args, kw, msg in [
        (edge_gather, (x.numpy(), g), {}, "cuda tensor"), (edge_gather, (x.double(), g), {}, "float32"),
        (edge_gather, (x[0], g), {}, "dimensions"), (edge_gather, (x[:, :0], g), {}, "channel"),
        (edge_gather, (x, g), {"end": "both"}, "end must be"), (edge_gather, (x[:3], g), {}, "N \\+ 1"),
        (edge_gather, (x, object()), {}, "graph.indptr"), (edge_gather, (x, bad_ei), {}, "\\[2,E\\]"),
        (edge_gather, (x, type("G", (), {"indptr": g.indptr.int(), "edge_index": g.edge_index})()), {}, "int64"),
        (edge_gather, (x, type("G", (), {"indptr": g.indptr, "edge_index": g.edge_index.int()})()), {}, "int64"),
        (edge_gather, (x, type("G", (), {"indptr": g.indptr[:, None], "edge_index": g.edge_index})()), {},
         "dimensions"),
        (edge_gather, (x, many_e), {}, "2\\^31"), (edge_gather, (x, g), {}, "cuda"),
        (edge_softmax, (s.double(), g), {}, "float32"), (edge_softmax, (s[:9], g), {}, "E = 10"),
        (edge_softmax, (torch.zeros(10, 2, 2), g), {}, "float32 tensor"), (edge_softmax, (s[:, :0], g), {}, "H >= 1"),
        (edge_softmax, (torch.zeros(1), huge), {}, "2\\^31"), (edge_softmax, (s, g), {}, "cuda"),
        (aggregate, (x, g), {"reduce": "min"}, "reduce must be"), (aggregate, (x, g, w[:9]), {}, "E = 10"),
        (aggregate, (x, g, s[:, :1].expand(10, 4)), {}, "does not divide"), (aggregate, (x, g, w.half()), {}, "float32"),
        (aggregate, (x.int(), g), {}, "float32"), (aggregate, (torch.zeros(5, 6), g), {}, "N \\+ 1"),
        (aggregate, (x, g, w), {}, "cuda"), (aggregate, (x, g, s[:, :2]), {"reduce": "max"}, "cuda"),
    ]:
        with pytest.raises(ValueError, match=msg):
            fn(*args, **kw)


def test_abi_declares_and_binds_the_entry_points():
    from fast_slic_b200 import _lib
    L = _lib.lib()
    header = open(os.path.join(ROOT, "include", "fslic_b200.h")).read()
    declared = set(re.findall(r"\b(fslic_b200_\w+)\s*\(", header))
    for name, nargs in (("fslic_b200_mp_gather", 10), ("fslic_b200_mp_gather_backward_scratch_bytes", 2),
                        ("fslic_b200_mp_gather_backward", 12), ("fslic_b200_mp_softmax", 9),
                        ("fslic_b200_mp_softmax_backward", 10), ("fslic_b200_mp_aggregate", 14),
                        ("fslic_b200_mp_aggregate_backward_scratch_bytes", 4),
                        ("fslic_b200_mp_aggregate_backward", 18)):
        assert name in declared and name in _lib.EXPORTED_SYMBOLS
        assert len(getattr(L, name).argtypes) == nargs
    NO = 2 ** 64 - 1
    assert L.fslic_b200_mp_gather_backward_scratch_bytes(-1, 5) == NO
    assert L.fslic_b200_mp_gather_backward_scratch_bytes(5, 2 ** 31) == NO
    assert L.fslic_b200_mp_aggregate_backward_scratch_bytes(5, 5, 4, 3) == NO
    assert L.fslic_b200_mp_aggregate_backward_scratch_bytes(5, 5, 0, 0) == NO
    assert L.fslic_b200_mp_aggregate_backward_scratch_bytes(5, 5, 4, 1) > \
        L.fslic_b200_mp_aggregate_backward_scratch_bytes(5, 5, 4, 0) > 0
    # bad sizes, heads, ends and reductions are refused before any device work; nothing to do returns 0
    agg = L.fslic_b200_mp_aggregate
    for args in [(0, -1, 5, 4, 1, 0), (0, 2 ** 31, 5, 4, 1, 0), (0, 5, 2 ** 31, 4, 1, 0), (0, 5, 5, 0, 1, 0),
                 (0, 5, 5, 4, 3, 0), (0, 5, 5, 4, 0, 0), (0, 5, 5, 4, 1, 3), (0, 5, 5, 4, 1, -1)]:
        assert agg(*args, *[None] * 8) == -1, args
    assert agg(0, 0, 5, 4, 1, 0, *[None] * 8) == 0
    assert L.fslic_b200_mp_gather(0, 5, 5, 4, 2, *[None] * 5) == -1
    assert L.fslic_b200_mp_gather(0, 5, 0, 4, 0, *[None] * 5) == 0
    assert L.fslic_b200_mp_softmax(0, 5, 5, 0, *[None] * 5) == -1
    assert L.fslic_b200_mp_softmax(0, 0, 5, 2, *[None] * 5) == 0
