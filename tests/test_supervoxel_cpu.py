"""Supervoxels without a GPU: the numpy restatement (supervoxel_cases.py) against a plain per-voxel loop, its
enforcement against scipy's 6-connected labelling with the written rules and, at D = 1, against the CPU oracle's 2-D
enforcement; the grid rule, the argument checks (they come before any device work) and the ABI."""
import os
import re

import numpy as np
import pytest
import torch

from supervoxel_cases import (F32, NAN_BITS, NO_LABEL, block_labels, components, grid_of, make_volumes,
                              min_size_of, nan_class_equal, radii, ref_enforce, ref_supervoxel_volume, seeds,
                              weights2)

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


def loop_supervoxels(f, K, compactness, spacing, max_iter, stride):
    """The contract one voxel, one candidate and one channel at a time."""
    C, D, H, W = f.shape
    grid = grid_of(D, H, W, K, spacing)
    Kp = grid[0] * grid[1] * grid[2]
    R = radii(D, H, W, grid)
    w2 = weights2(D, H, W, grid, compactness, spacing)
    z, y, x = seeds(D, H, W, grid)
    pos = [[F32(z[k]), F32(y[k]), F32(x[k])] for k in range(Kp)]
    mu = [[f[c, z[k], y[k], x[k]] for c in range(C)] for k in range(Kp)]
    labels = np.full((D, H, W), NO_LABEL, np.uint16)

    def assign(rows):
        for vz in range(D):
            for vy in rows:
                for vx in range(W):
                    best = None
                    for k in range(Kp):
                        if any(abs(v - int(pos[k][a])) > R[a] for a, v in enumerate((vz, vy, vx))):
                            continue
                        fc = F32(0)
                        for c in range(C):
                            t = F32(f[c, vz, vy, vx] - mu[k][c])
                            fc = F32(fc + F32(t * t))
                        t = [F32(F32(v) - pos[k][a]) for a, v in enumerate((vz, vy, vx))]
                        sp = F32(F32(F32(w2[0] * F32(t[0] * t[0])) + F32(w2[1] * F32(t[1] * t[1]))) +
                                 F32(w2[2] * F32(t[2] * t[2])))
                        d = F32(fc + sp)
                        bits = NAN_BITS if np.isnan(d) else int(np.array(d).view(np.uint32))
                        key = bits << 32 | k
                        best = key if best is None or key < best else best
                    if best is not None:
                        labels[vz, vy, vx] = best & 0xFFFF

    count = [0] * Kp
    with np.errstate(invalid="ignore", over="ignore"):
        for t in range(max_iter):
            rows = list(range(t % stride, H, stride))
            assign(rows)
            for k in range(Kp):
                members = [(vz, vy, vx) for vz in range(D) for vy in rows for vx in range(W)
                           if labels[vz, vy, vx] == k]
                count[k] = len(members)
                if members:
                    pos[k] = [F32(sum(m[a] for m in members) / len(members)) for a in range(3)]
                    mu[k] = [_pool_mean([f[c][m] for m in members]) for c in range(C)]
        assign(range(H))
    return labels, np.array(pos, F32), np.array(mu, F32).reshape(Kp, C), np.array(count, np.int32)


def _same(a, b):
    for x, y in zip(a[1:4], b[1:4]):
        assert nan_class_equal(x, y) if x.dtype == np.float32 else np.array_equal(x, y)
    assert np.array_equal(a[0], b[0])


@pytest.mark.parametrize("case", [
    dict(seed=1, C=2, D=4, H=6, W=7, K=8, compactness=1.0, max_iter=3, stride=2),
    dict(seed=2, C=1, D=3, H=5, W=6, K=5, compactness=1e-3, max_iter=4, stride=3),
    dict(seed=3, C=3, D=2, H=3, W=4, K=24, compactness=1e3, max_iter=2, stride=1),      # one-voxel cells
    dict(seed=4, C=2, D=1, H=6, W=9, K=6, compactness=2.0, max_iter=3, stride=2),       # one slice
    dict(seed=5, C=2, D=7, H=1, W=5, K=4, compactness=2.0, max_iter=3, stride=2),       # one row per slice
    dict(seed=6, C=2, D=6, H=5, W=1, K=(3, 2, 1), compactness=1.0, max_iter=3, stride=3),  # explicit grid
    dict(seed=7, C=2, D=4, H=5, W=6, K=6, compactness=1.0, max_iter=0, stride=3),       # seeds only
    dict(seed=8, C=2, D=4, H=5, W=6, K=6, compactness=1.0, max_iter=3, stride=2, kind="constant"),  # ties
    dict(seed=9, C=3, D=4, H=6, W=6, K=6, compactness=1.0, max_iter=3, stride=2, kind="nonfinite"),
    dict(seed=10, C=2, D=3, H=8, W=8, K=6, compactness=1.0, max_iter=3, stride=2, spacing=(4.0, 1.0, 0.5)),
    dict(seed=11, C=1, D=1, H=1, W=1, K=1, compactness=1.0, max_iter=2, stride=1),      # one voxel
])
def test_restatement_against_a_voxel_loop(case):
    case = dict(case)
    f = make_volumes(case.pop("seed"), 1, case.pop("C"), case.pop("D"), case.pop("H"), case.pop("W"),
                     case.pop("kind", "smooth"))[0]
    args = (case["K"], case["compactness"], case.get("spacing", (1.0, 1.0, 1.0)), case["max_iter"], case["stride"])
    _same(ref_supervoxel_volume(f, *args), loop_supervoxels(f, *args))


def test_ties_uncovered_voxels_and_nan():
    from supervoxel_cases import assign
    f = np.zeros((1, 1, 1, 5), F32)
    pos = np.array([[0, 0, 2], [0, 0, 2], [0, 0, 0]], F32)
    mu = np.zeros((3, 1), F32)
    lab = np.full((1, 1, 5), NO_LABEL, np.uint16)
    assign(f, lab, np.arange(1), pos, mu, (1, 1, 1), np.ones(3, F32))
    # R = 1: voxel 1 is as far from k = 0 (and k = 1) as from k = 2 and the lower index wins; voxel 4 has no candidate
    assert lab.tolist() == [[[2, 0, 0, 0, NO_LABEL]]]
    f = np.array([[[[np.inf, np.nan]]]], F32)
    pos = np.array([[0, 0, 0], [0, 0, 1]], F32)
    mu = np.array([[np.inf], [0]], F32)
    lab = np.full((1, 1, 2), NO_LABEL, np.uint16)
    assign(f, lab, np.arange(1), pos, mu, (1, 1, 1), np.ones(3, F32))
    assert lab.tolist() == [[[1, 0]]]  # inf - inf is NaN and loses to +inf; among NaNs the lower index wins


def _scipy_enforce(lab, K, min_size):
    """The written rules over scipy.ndimage.label's 6-connected components, absorbing one component at a time."""
    from scipy import ndimage
    D, H, W = lab.shape
    N = lab.size
    comp_of = np.full(N, -1, np.int64)
    leaders, members = [], []
    for v in np.unique(lab):
        cc, n = ndimage.label(lab == v, structure=ndimage.generate_binary_structure(3, 1))
        flat = cc.ravel()
        for c in range(1, n + 1):
            idx = np.flatnonzero(flat == c)
            leaders.append(int(idx[0]))
            members.append(idx)
    order = np.argsort(leaders)
    leaders = [leaders[i] for i in order]
    members = [members[i] for i in order]
    for c, idx in enumerate(members):
        comp_of[idx] = c
    area = [len(m) for m in members]
    cand = [c for c in range(len(area)) if area[c] >= min_size]
    if len(cand) > K:
        cand = sorted(sorted(cand, key=lambda c: (-area[c], leaders[c]))[:K])
    sub = {c: i for i, c in enumerate(cand)}
    sub.setdefault(0, 0)
    for c in range(1, len(area)):
        if c in sub:
            continue
        p = leaders[c]
        q = p - 1 if p % W else p - W if (p // W) % H else p - H * W
        sub[c] = sub[int(comp_of[q])]
    return np.array([sub[int(c)] for c in comp_of], np.int16).reshape(D, H, W)


@pytest.mark.parametrize("seed,shape,nlab,block,K,min_size", [
    (1, (6, 7, 8), 3, (1, 1, 1), 50, 3),
    (2, (5, 9, 6), 4, (2, 1, 2), 20, 4),
    (3, (4, 6, 9), 2, (1, 2, 3), 5, 2),    # the cap binds
    (4, (3, 5, 5), 2, (1, 1, 1), 4, 1),    # the cap binds with many tied areas
    (5, (8, 4, 4), 3, (2, 2, 2), 1000, 0),  # every component kept
    (6, (1, 1, 30), 2, (1, 1, 1), 2, 2),
    (7, (30, 1, 1), 2, (1, 1, 1), 3, 2),
])
def test_enforcement_restatement_against_scipy(seed, shape, nlab, block, K, min_size):
    lab = block_labels(seed, *shape, nlab, block)
    want = _scipy_enforce(lab, K, min_size)
    got = ref_enforce(lab, K, min_size)
    assert np.array_equal(got, want)
    assert got.min() >= 0 and got.max() < K


def test_enforcement_of_a_checkerboard():
    D, H, W = 4, 5, 6
    z, y, x = np.mgrid[0:D, 0:H, 0:W]
    lab = ((z + y + x) % 2).astype(np.uint16)
    comp, leaders = components(lab)
    assert leaders.size == lab.size  # every voxel its own component
    assert np.array_equal(ref_enforce(lab, 65534, 1), np.arange(lab.size).reshape(D, H, W).astype(np.int16))
    assert np.array_equal(ref_enforce(lab, 7, 1), _scipy_enforce(lab, 7, 1))
    assert not ref_enforce(lab, 7, 2).any()  # nothing kept: everything takes component 0's label 0


@pytest.mark.parametrize("seed,H,W,nlab,K,thres", [(1, 30, 40, 6, 500, 4), (2, 17, 23, 3, 300, 2),
                                                   (3, 40, 33, 20, 2000, 3), (4, 25, 25, 4, 200, 0)])
def test_enforcement_at_one_slice_is_the_2d_oracle(seed, H, W, nlab, K, thres):
    from oracle.oracle import Port
    lab = block_labels(seed, 1, H, W, nlab, (1, 2, 2))
    comp, leaders = components(lab)
    area = np.bincount(comp)
    assert (area >= thres).sum() <= K  # the cap does not bind
    want = Port().enforce_connectivity(lab[0], K, thres).view(np.int16)
    assert np.array_equal(ref_enforce(lab, K, thres)[0], want)


def test_grid_rule():
    from fast_slic_b200.supervoxels import min_size_threshold, volume_grid
    assert volume_grid(64, 64, 64, 512) == (8, 8, 8)
    assert volume_grid(256, 512, 512, 16384) == grid_of(256, 512, 512, 16384) == (16, 32, 32)
    assert volume_grid(64, 512, 512, 4096, (3.0, 0.7, 0.7)) == grid_of(64, 512, 512, 4096, (3.0, 0.7, 0.7))
    assert volume_grid(1, 100, 100, 100) == (1, 22, 22)  # s0 = cbrt(100): n_z = floor(0.72) clamps up to 1
    assert volume_grid(2, 300, 4, 50) == grid_of(2, 300, 4, 50) and volume_grid(2, 300, 4, 50)[2] <= 4
    assert volume_grid(3, 4, 5, 10 ** 6) == (3, 4, 5)              # every n_a clamps to L_a: one-voxel cells
    assert volume_grid(10, 10, 10, 1) == (1, 1, 1)
    assert volume_grid(10, 10, 10, (2, 5, 10)) == (2, 5, 10)
    for args in [(64, 512, 512, 65535), (40, 40, 41, 65535), (100, 100, 100, (50, 50, 50))]:
        with pytest.raises(ValueError, match="more than 65534"):
            volume_grid(*args)
    for K in [(0, 1, 1), (11, 1, 1), (1, 2), 0, 2.0]:
        with pytest.raises(ValueError, match="K"):
            volume_grid(10, 10, 10, K)
    assert min_size_threshold(64, 64, 64, (8, 8, 8), 0.25) == 128 == min_size_of(64, 64, 64, (8, 8, 8), 0.25)
    assert min_size_threshold(3, 3, 3, (1, 1, 2), 0.5) == 7  # 6.5 rounds up
    assert min_size_threshold(10, 10, 10, (1, 1, 1), 0.0) == 0


def test_abi_declares_and_binds_the_entry_points():
    from fast_slic_b200 import _lib
    L = _lib.lib()
    header = open(os.path.join(ROOT, "include", "fslic_b200.h")).read()
    declared = set(re.findall(r"\b(fslic_b200_\w+)\s*\(", header))
    for name, nargs in (("fslic_b200_sv_enforce_scratch_bytes", 4), ("fslic_b200_sv_enforce", 12),
                        ("fslic_b200_sv_slic_scratch_bytes", 10), ("fslic_b200_sv_slic", 24)):
        assert name in declared and name in _lib.EXPORTED_SYMBOLS
        assert len(getattr(L, name).argtypes) == nargs
    e = L.fslic_b200_sv_enforce_scratch_bytes
    for args in [(-1, 4, 4, 4), (1, 0, 4, 4), (1, 4, 0, 4), (1, 4, 4, 32768), (1, 1024, 1024, 1024),
                 (70000, 1, 1, 1), (9, 1 << 8, 1 << 10, 1 << 10)]:  # more than 2^29 voxels; too many volumes or voxels
        assert int(e(*args)) == NO_SIZE, args
    assert int(e(0, 4, 4, 4)) < NO_SIZE
    assert 20 * 2 * 100 * 100 * 100 <= int(e(2, 100, 100, 100)) < NO_SIZE
    f = L.fslic_b200_sv_slic_scratch_bytes
    ok = (1, 16, 16, 16, 2, 2, 2, 2, 3, 10)
    assert int(f(*ok)) < NO_SIZE and int(f(0, *ok[1:])) < NO_SIZE
    for i, bad in [(0, -1), (1, 0), (4, 0), (4, 1025), (5, 0), (5, 17), (6, 17), (7, 0), (8, 0), (9, -1)]:
        args = list(ok)
        args[i] = bad
        assert int(f(*args)) == NO_SIZE, args
    assert int(f(1, 64, 64, 64, 1, 40, 40, 41, 3, 1)) == NO_SIZE  # K' > 65534
    assert int(f(1, 16, 16, 16, 1, 2, 2, 2, 256, 1)) == NO_SIZE
    assert int(f(2 ** 15, 64, 64, 64, 1, 64, 64, 9, 3, 0)) == NO_SIZE  # B*K' > 2^30
    # the passes and the enforcement share one scratch: the larger of the two
    small, large = int(f(1, 8, 64, 64, 1, 8, 32, 32, 1, 1)), int(f(1, 8, 64, 64, 1024, 8, 32, 32, 1, 1))
    assert int(e(1, 8, 64, 64)) <= small < large < NO_SIZE and large >= 8192 * 1024 * 4


def test_argument_errors():
    from fast_slic_b200.supervoxels import enforce_connectivity_3d, supervoxel_slic
    x = torch.zeros((2, 3, 4, 8, 9))
    for args, kw, msg in [
        ((x.numpy(), 8, 1.0), {}, "torch.from_numpy"), ((x.double(), 8, 1.0), {}, "float32"),
        ((x[0], 8, 1.0), {}, "dimensions"), ((x[:, :0], 8, 1.0), {}, "channels"),
        ((torch.zeros(1, 1025, 1, 1, 1), 1, 1.0), {}, "channels"), ((x[:, :, :0], 8, 1.0), {}, "voxels"),
        ((torch.zeros(1, 1, 1, 1, 32768), 1, 1.0), {}, "voxels"),
        ((torch.zeros(1, 1, 1, 1, 1).expand(1, 1, 1024, 1024, 1024), 8, 1.0), {}, "voxels"),
        ((x, 0, 1.0), {}, "K must be"), ((x, 8.0, 1.0), {}, "K must be an int"), ((x, (1, 2), 1.0), {}, "K must be"),
        ((x, (5, 1, 1), 1.0), {}, "K\\[0\\]"), ((x, (1, 1, 10), 1.0), {}, "K\\[2\\]"),
        ((torch.zeros(1, 1, 64, 512, 512), 65535, 1.0), {}, "more than 65534"),
        ((torch.zeros(1, 1, 1, 1, 1).expand(2 ** 15, 1, 64, 64, 64), (32, 32, 33), 1.0), {}, "B\\*K'"),
        ((x, 8, 0.0), {}, "compactness"), ((x, 8, -1.0), {}, "compactness"), ((x, 8, float("nan")), {}, "compactness"),
        ((x, 8, float("inf")), {}, "compactness"), ((x, 8, 1e30), {}, "overflows"), ((x, 8, "1"), {}, "compactness"),
        ((x, 8, True), {}, "compactness"),
        ((x, 8, 1.0), {"spacing": (1.0, 1.0)}, "spacing"), ((x, 8, 1.0), {"spacing": (1.0, 0.0, 1.0)}, "spacing"),
        ((x, 8, 1.0), {"spacing": (1.0, float("inf"), 1.0)}, "spacing"),
        ((x, 8, 1.0), {"spacing": (1.0, float("nan"), 1.0)}, "spacing"),
        ((x, 8, 1.0), {"spacing": (-1.0, 1.0, 1.0)}, "spacing"), ((x, 8, 1.0), {"spacing": 1.0}, "spacing"),
        ((x, 8, 1.0), {"max_iter": -1}, "max_iter"), ((x, 8, 1.0), {"max_iter": 2.0}, "max_iter"),
        ((x, 8, 1.0), {"subsample_stride": 0}, "subsample_stride"),
        ((x, 8, 1.0), {"subsample_stride": 256}, "subsample_stride"),
        ((x, 8, 1.0), {"min_size_factor": -0.1}, "min_size_factor"),
        ((x, 8, 1.0), {"min_size_factor": float("nan")}, "min_size_factor"),
        ((x, 8, 1.0), {"min_size_factor": float("inf")}, "min_size_factor"),
        ((x, 8, 1.0), {}, "cuda"),  # cpu tensors, every other check passed
    ]:
        with pytest.raises(ValueError, match=msg):
            supervoxel_slic(*args, **kw)
    # the limits themselves pass every check but the device one
    for args, kw in [((torch.zeros(1, 1024, 1, 1, 1), 1, 1e-30), {}), ((torch.zeros(2, 1, 3, 3, 3), 27, 1e10), {}),
                     ((torch.zeros(1, 1, 1, 1, 1).expand(1, 1, 1, 16384, 32767), (1, 2, 32767), 1.0),
                      {"subsample_stride": 255}),
                     ((torch.zeros(1, 1, 1, 1, 1).expand(2 ** 14, 1, 64, 64, 64), (2, 32767 // 1000, 1), 1.0), {}),
                     ((x[:0], 8, 1.0), {"min_size_factor": 0})]:
        with pytest.raises(ValueError, match="cuda"):
            supervoxel_slic(*args, **kw)
    lab = torch.zeros((2, 3, 4, 5), dtype=torch.int16)
    for args, msg in [((lab.numpy(), 4, 1), "torch.from_numpy"), ((lab.int(), 4, 1), "int16"),
                      ((lab[0], 4, 1), "dimensions"), ((lab[:, :0], 4, 1), "voxels"),
                      ((torch.zeros(1, 1, 1, 32768, dtype=torch.int16), 4, 1), "voxels"),
                      ((lab, 0, 1), "K must be"), ((lab, 65535, 1), "K must be"), ((lab, 4.0, 1), "K must be an int"),
                      ((lab, 4, -1), "min_size"), ((lab, 4, 1.5), "min_size"), ((lab, 4, 1), "cuda"),
                      ((lab, 65534, 0), "cuda")]:
        with pytest.raises(ValueError, match=msg):
            enforce_connectivity_3d(*args)
