"""feature_slic without a GPU: the numpy restatement against a plain per-pixel loop, the argument checks (they come
before any device work), the ABI, and the enforcement step of the restatement through the CPU oracle."""
import os
import re

import numpy as np
import pytest
import torch

from feature_slic_cases import (F32, NAN_BITS, NO_LABEL, make_features, min_size_threshold, nan_class_equal,
                                ref_feature_slic, ref_feature_slic_image, seed_grid, superpixel_size, weight2)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NO_SIZE = 2 ** 64 - 1


def _pool_mean(values):
    """pool's order: 32 lanes left to right from +0, five butterfly steps, lane 0 over float32(count)."""
    lanes = [F32(0)] * 32
    for m, v in enumerate(values):
        lanes[m % 32] = F32(lanes[m % 32] + v)
    for off in (16, 8, 4, 2, 1):
        lanes = [F32(lanes[l] + lanes[l ^ off]) for l in range(32)]
    return F32(lanes[0] / F32(len(values)))


def loop_feature_slic(f, K, compactness, max_iter, stride, init=None):
    """The contract one pixel, one candidate and one channel at a time."""
    C, H, W = f.shape
    S = superpixel_size(H, W, K)
    w2 = weight2(compactness, S)
    if init is None:
        cy, cx = seed_grid(H, W, K)
        pos = [[F32(cy[k]), F32(cx[k])] for k in range(K)]
        mu = [[f[c, cy[k], cx[k]] for c in range(C)] for k in range(K)]
    else:
        pos = [[F32(min(max(v, 0), hi)) if v == v else F32(0) for v, hi in zip(init[0][k], (H - 1, W - 1))]
               for k in range(K)]
        mu = [list(init[1][k]) for k in range(K)]
    labels = np.full((H, W), NO_LABEL, np.uint16)

    def assign(rows):
        for i in rows:
            for j in range(W):
                best = None
                for k in range(K):
                    if abs(i - int(pos[k][0])) > S or abs(j - int(pos[k][1])) > S:
                        continue
                    fc = F32(0)
                    for c in range(C):
                        t = F32(f[c, i, j] - mu[k][c])
                        fc = F32(fc + F32(t * t))
                    ty, tx = F32(F32(i) - pos[k][0]), F32(F32(j) - pos[k][1])
                    d = F32(fc + F32(w2 * F32(F32(ty * ty) + F32(tx * tx))))
                    bits = NAN_BITS if np.isnan(d) else int(np.array(d).view(np.uint32))
                    key = bits << 32 | k
                    best = key if best is None or key < best else best
                if best is not None:
                    labels[i, j] = best & 0xFFFF

    count = [0] * K
    with np.errstate(invalid="ignore", over="ignore"):
        for t in range(max_iter):
            rows = list(range(t % stride, H, stride))
            assign(rows)
            for k in range(K):
                members = [(i, j) for i in rows for j in range(W) if labels[i, j] == k]
                count[k] = len(members)
                if members:
                    pos[k] = [F32(sum(i for i, _ in members) / len(members)),
                              F32(sum(j for _, j in members) / len(members))]
                    mu[k] = [_pool_mean([f[c, i, j] for i, j in members]) for c in range(C)]
        assign(range(H))
    return labels, np.array(pos, F32), np.array(mu, F32).reshape(K, C), np.array(count, np.int32)


def _same(a, b):
    for x, y in zip(a[1:], b[1:]):
        assert nan_class_equal(x, y) if x.dtype == np.float32 else np.array_equal(x, y)
    assert np.array_equal(a[0], b[0])


@pytest.mark.parametrize("case", [
    dict(seed=1, C=3, H=9, W=11, K=6, compactness=1.0, max_iter=3, stride=2),
    dict(seed=2, C=1, H=7, W=8, K=7, compactness=1e-3, max_iter=4, stride=3),
    dict(seed=3, C=5, H=6, W=5, K=30, compactness=1e3, max_iter=2, stride=1),   # K = H*W, S = 1
    dict(seed=4, C=2, H=1, W=13, K=3, compactness=2.0, max_iter=3, stride=2),   # one row
    dict(seed=5, C=2, H=12, W=1, K=4, compactness=2.0, max_iter=3, stride=5),   # one column
    dict(seed=6, C=4, H=8, W=9, K=5, compactness=1.0, max_iter=0, stride=3),    # seeds only
    dict(seed=7, C=3, H=8, W=8, K=4, compactness=1.0, max_iter=3, stride=2, kind="constant"),  # everything ties
    dict(seed=8, C=3, H=9, W=10, K=6, compactness=1.0, max_iter=3, stride=2, kind="nonfinite"),
])
def test_restatement_against_a_pixel_loop(case):
    case = dict(case)
    f = make_features(case.pop("seed"), 1, case.pop("C"), case.pop("H"), case.pop("W"), case.pop("kind", "smooth"))[0]
    args = (case["K"], case["compactness"], case["max_iter"], case["stride"])
    _same(ref_feature_slic_image(f, *args), loop_feature_slic(f, *args))


def test_uncovered_pixels_and_warm_start():
    f = make_features(11, 1, 2, 10, 10)[0]
    K = 6  # S = 4
    pos = np.zeros((K, 2), F32)
    pos[3] = [np.nan, 7.5]
    pos[4] = [1e9, -3]
    mu = np.arange(K * 2, dtype=F32).reshape(K, 2) / 3
    got = ref_feature_slic_image(f, K, 1.0, 2, 2, init=(pos, mu))
    _same(got, loop_feature_slic(f, K, 1.0, 2, 2, init=(pos, mu)))
    assert (got[0] == NO_LABEL).any() and (got[0] != NO_LABEL).any()  # rows far from every centre stay unlabelled
    # no pass: the clamped init comes back unchanged, every pixel within S of a centre gets a label
    lab, p, m, n = ref_feature_slic_image(f, K, 1.0, 0, 2, init=(pos, mu))
    assert p.tolist() == [[0, 0]] * 3 + [[0, 7.5], [9, 0], [0, 0]] and nan_class_equal(m, mu) and not n.any()


def test_ties_go_to_the_lower_index():
    f = np.zeros((1, 1, 5), F32)
    pos = np.array([[0, 2], [0, 2], [0, 0]], F32)
    mu = np.zeros((3, 1), F32)
    lab = ref_feature_slic_image(f, 3, 1.0, 0, 1, init=(pos, mu))[0]
    # S = 1: pixel 1 is as far from k = 0 (and k = 1) as from k = 2 and the lower index wins; pixel 4 has no candidate
    assert lab.tolist() == [[2, 0, 0, 0, NO_LABEL]]
    # a NaN distance (inf - inf) loses to +inf, and among NaNs the lower index wins
    f = np.array([[[np.inf, np.nan]]], F32)
    pos = np.array([[0, 0], [0, 1]], F32)
    mu = np.array([[np.inf], [0]], F32)
    assert ref_feature_slic_image(f, 2, 1.0, 0, 1, init=(pos, mu))[0].tolist() == [[1, 0]]
    assert loop_feature_slic(f, 2, 1.0, 0, 1, init=(pos, mu))[0].tolist() == [[1, 0]]


def test_enforcement_through_the_cpu_oracle():
    from oracle.oracle import Port
    f = make_features(21, 2, 3, 40, 50)
    K, msf = 30, 0.6
    final, pre, pos, mu, cnt = ref_feature_slic(f, K, 2.0, 4, 3, msf)
    thres = min_size_threshold(superpixel_size(40, 50, K), msf)
    assert thres == round(superpixel_size(40, 50, K) ** 2 * 0.6)
    for b in range(2):
        want = Port().enforce_connectivity(pre[b], K, thres).view(np.int16)
        assert np.array_equal(final[b], want)
        assert not np.array_equal(pre[b].view(np.int16), want)  # the map had small fragments to absorb
    assert final.dtype == np.int16 and final.min() >= 0 and final.max() < K


def test_threshold_rounding():
    assert min_size_threshold(4, 0.25) == 4 and min_size_threshold(3, 0.5) == 5  # 4.5 rounds away from zero
    assert min_size_threshold(24, 0.25) == 144 and min_size_threshold(7, 0.0) == 0
    assert superpixel_size(720, 1280, 1600) == 24 and superpixel_size(3, 3, 9) == 1


def test_abi_declares_and_binds_the_entry_points():
    from fast_slic_b200 import _lib
    L = _lib.lib()
    header = open(os.path.join(ROOT, "include", "fslic_b200.h")).read()
    declared = set(re.findall(r"\b(fslic_b200_\w+)\s*\(", header))
    for name, nargs in (("fslic_b200_feature_slic_scratch_bytes", 7), ("fslic_b200_feature_slic", 20)):
        assert name in declared and name in _lib.EXPORTED_SYMBOLS
        assert len(getattr(L, name).argtypes) == nargs
    f = L.fslic_b200_feature_slic_scratch_bytes
    for args in [(-1, 8, 8, 3, 4, 3, 10), (1, 0, 8, 3, 4, 3, 10), (1, 32768, 8, 3, 4, 3, 10), (1, 8, 8, 0, 4, 3, 10),
                 (1, 8, 8, 1025, 4, 3, 10), (1, 8, 8, 3, 0, 3, 10), (1, 8, 8, 3, 65, 3, 10), (1, 300, 300, 3, 65535, 3, 1),
                 (1, 8, 8, 3, 4, 0, 10), (1, 8, 8, 3, 4, 256, 10), (1, 8, 8, 3, 4, 3, -1),
                 (1, 32767, 32767, 1, 4, 3, 1),  # more than 2^29 pixels
                 (2 ** 15, 256, 256, 1, 2 ** 15 + 1, 3, 1),  # B*K > 2^30
                 (40000, 256, 256, 1, 4, 3, 1)]:  # more pixels than one sort takes
        assert int(f(*args)) == NO_SIZE, args
    assert int(f(0, 8, 8, 3, 4, 3, 10)) < NO_SIZE
    small, large = int(f(32, 720, 1280, 3, 1600, 3, 10)), int(f(32, 720, 1280, 64, 1600, 3, 10))
    assert 32 * 240 * 1280 * 16 <= small < large < NO_SIZE
    assert large - small == 32 * 1600 * 61 * 4


def test_argument_errors():
    from fast_slic_b200.feature_slic import feature_slic
    x = torch.zeros((2, 3, 8, 9))
    pos, feat = torch.zeros((2, 5, 2)), torch.zeros((2, 5, 3))
    for args, kw, msg in [
        ((x.numpy(), 5, 1.0), {}, "torch.from_numpy"), ((x.double(), 5, 1.0), {}, "float32"),
        ((x[0], 5, 1.0), {}, "dimensions"), ((x[:, :0], 5, 1.0), {}, "channels"),
        ((torch.zeros(1, 1025, 1, 1), 1, 1.0), {}, "channels"), ((x[:, :, :0], 5, 1.0), {}, "pixels"),
        ((torch.zeros(1, 1, 1, 32768), 5, 1.0), {}, "pixels"),
        ((torch.zeros(1, 1, 1, 1).expand(1, 1, 32767, 32767), 5, 1.0), {}, "pixels"),
        ((x, 0, 1.0), {}, "K must be"), ((x, 73, 1.0), {}, "K must be"), ((x, 5.0, 1.0), {}, "K must be an int"),
        ((torch.zeros(1, 1, 1, 1).expand(2 ** 15, 1, 256, 256), 2 ** 15 + 1, 1.0), {}, "B\\*K"),
        ((x, 5, 0.0), {}, "compactness"), ((x, 5, -1.0), {}, "compactness"), ((x, 5, float("nan")), {}, "compactness"),
        ((x, 5, float("inf")), {}, "compactness"), ((x, 5, 1e39), {}, "compactness"), ((x, 5, "1"), {}, "compactness"),
        ((x, 5, True), {}, "compactness"),
        ((x, 5, 1.0), {"max_iter": -1}, "max_iter"), ((x, 5, 1.0), {"max_iter": 2.0}, "max_iter"),
        ((x, 5, 1.0), {"subsample_stride": 0}, "subsample_stride"),
        ((x, 5, 1.0), {"subsample_stride": 256}, "subsample_stride"),
        ((x, 5, 1.0), {"min_size_factor": -0.1}, "min_size_factor"),
        ((x, 5, 1.0), {"min_size_factor": float("nan")}, "min_size_factor"),
        ((x, 5, 1.0), {"init": pos}, "init must be"), ((x, 5, 1.0), {"init": (pos, feat[:, :4])}, "init must be"),
        ((x, 5, 1.0), {"init": (pos, feat[..., :2])}, "init must be"),
        ((x, 5, 1.0), {"init": (pos.double(), feat)}, "float32"),
        ((x, 5, 1.0), {"init": (pos.numpy(), feat)}, "cuda tensor"),
        ((x, 5, 1.0), {}, "cuda"),  # cpu tensors, every other check passed
        ((x, 5, 1.0), {"init": (pos, feat)}, "cuda"),
    ]:
        with pytest.raises(ValueError, match=msg):
            feature_slic(*args, **kw)
    if torch.cuda.is_available():
        with pytest.raises(ValueError, match="init position is on"):
            feature_slic(x.cuda(), 5, 1.0, init=(pos, feat))
    # the limits themselves pass every check but the device one
    for args, kw in [((torch.zeros(1, 1024, 1, 1), 1, 1e-30), {}), ((torch.zeros(2, 1, 3, 3), 9, 1e30), {}),
                     ((torch.zeros(1, 1, 1, 1).expand(1, 1, 16384, 32767), 65534, 1.0), {"subsample_stride": 255}),
                     ((torch.zeros(1, 1, 1, 1).expand(2 ** 14, 1, 256, 256), 65534, 1.0), {"max_iter": 0}),
                     ((x[:0], 5, 1.0), {"min_size_factor": 0})]:
        with pytest.raises(ValueError, match="cuda"):
            feature_slic(*args, **kw)
