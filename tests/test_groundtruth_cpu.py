"""Ground-truth scores without a GPU: the ABI declarations, the argument checks (they come before any device work), the
scratch sizes and chunking, the numpy restatement against brute-force per-pixel loops, and hand-computed answers."""
import os
import re

import numpy as np
import pytest
import torch

from groundtruth_cases import FIELDS, dilate, ref_boundaries, ref_class_histogram, ref_scores, ref_scores_image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ("fslic_b200_gt_histogram_batch", "fslic_b200_gt_scores_scratch_bytes", "fslic_b200_gt_scores_batch",
               "fslic_b200_gt_boundaries_batch")
NONE = 2 ** 64 - 1


def test_abi_declares_and_binds_the_groundtruth_entry_points():
    from fast_slic_b200 import _lib
    L = _lib.lib()
    header = open(os.path.join(ROOT, "include", "fslic_b200.h")).read()
    declared = set(re.findall(r"\b(fslic_b200_\w+)\s*\(", header))
    for sym in NEW_SYMBOLS:
        assert sym in declared and sym in _lib.EXPORTED_SYMBOLS, sym
        assert getattr(L, sym).argtypes is not None, sym
    assert L.fslic_b200_gt_scores_scratch_bytes.restype is not None
    codes = dict(re.findall(r"#define FSLIC_GT_(\w+) (\d+)", header))
    assert codes == {"UINT8": "1", "INT16": "2", "INT32": "4", "INT64": "8"}


def test_argument_errors():
    from fast_slic_b200.groundtruth import boundaries, class_histogram, segmentation_scores
    l = torch.zeros((2, 5, 7), dtype=torch.int16)
    g = torch.zeros((2, 5, 7), dtype=torch.uint8)
    huge = torch.zeros((1, 1, 1), dtype=torch.int16).expand(2, 2 ** 15, 2 ** 14 + 1)  # 2^29 + 2^15 pixels per image
    huge_g = torch.zeros((1, 1, 1), dtype=torch.uint8).expand(2, 2 ** 15, 2 ** 14 + 1)
    common = [
        ((g, l.numpy()), "torch.from_numpy"),        # numpy labels
        ((g.numpy(), l), "torch.from_numpy"),        # numpy gt
        ((g, l.int()), "int16"),                     # labels dtype
        ((g, l[0]), "dimensions"),                   # labels ndim
        ((g.float(), l), "uint8, int16, int32 or int64"),  # gt dtype
        ((g.bool(), l), "uint8, int16, int32 or int64"),
        ((g.to(torch.int8), l), "uint8, int16, int32 or int64"),
        ((g[:, :4], l), "does not match"),           # gt shape
        ((g[0], l), "does not match"),
        ((huge_g, huge), "exceed"),                  # a count could overflow int32
        ((g, l), "cuda"),                            # cpu tensors
        ((g.long(), l), "cuda"),
    ]
    for (gt, lab), msg in common:
        with pytest.raises(ValueError, match=msg):
            class_histogram(gt, lab, 10, 3)
        with pytest.raises(ValueError, match=msg):
            segmentation_scores(lab, gt, 10)
    for args, msg in [((g, l, 0, 3), "K must be"), ((g, l, 65535, 3), "K must be"), ((g, l, 3.0, 3), "K must be"),
                      ((g, l, 10, 0), "num_classes"), ((g, l, 10, 65537), "num_classes"),
                      ((g, l, 10, 2.0), "num_classes")]:
        with pytest.raises(ValueError, match=msg):
            class_histogram(*args)
    for kwargs, msg in [(dict(K=0), "K must be"), (dict(K=65535), "K must be"), (dict(K=10, tolerance=-1), "tolerance"),
                        (dict(K=10, tolerance=33), "tolerance"), (dict(K=10, tolerance=1.5), "tolerance"),
                        (dict(K=10, ignore_index=2 ** 63), "ignore_index"), (dict(K=10, ignore_index=1.0), "ignore_index"),
                        (dict(K=10, tolerance=32, ignore_index=-1), "cuda")]:
        with pytest.raises(ValueError, match=msg):
            segmentation_scores(l, g, **kwargs)
    for lab, msg in [(l.numpy(), "torch.from_numpy"), (l.int(), "int16"), (l[0], "dimensions"), (huge, "exceed"),
                     (l, "cuda")]:
        with pytest.raises(ValueError, match=msg):
            boundaries(lab)
    # the largest image is allowed past the size check (and refused as a cpu tensor)
    big = torch.zeros((1, 1, 1), dtype=torch.int16).expand(1, 2 ** 15, 2 ** 14)
    with pytest.raises(ValueError, match="cuda"):
        segmentation_scores(big, torch.zeros((1, 1, 1), dtype=torch.int32).expand(1, 2 ** 15, 2 ** 14), 10)


def test_scratch_bytes_and_chunks(monkeypatch):
    from fast_slic_b200 import _lib, groundtruth
    f = _lib.lib().fslic_b200_gt_scores_scratch_bytes
    assert f(0, 5, 5, 10) == 256 and f(3, 0, 5, 10) == 256 and f(3, 5, 0, 10) == 256
    for args in ((1, 5, 5, 0), (1, 5, 5, 65535), (-1, 5, 5, 10), (1, 2 ** 15, 2 ** 14 + 1, 10),
                 (5, 2 ** 15, 2 ** 14, 10),      # more than 2^31 - 1 pixels in one sort
                 (2 ** 17 + 1, 1, 1, 1)):        # more images than the key's 17 image bits
        assert f(*args) == NONE, args
    assert f(2 ** 17, 1, 1, 1) != NONE and f(3, 2 ** 15, 2 ** 14, 10) != NONE
    # 20 bytes per pixel (two key buffers and the run counts), 16 per (image, label), 3/8 per pixel of bitmaps
    for B, H, W in ((1, 720, 1280), (32, 720, 1280), (3, 97, 131)):
        n, words = B * H * W, B * H * ((W + 31) // 32)
        assert 20 * n + 16 * B * 1600 + 12 * words <= f(B, H, W, 1600) < 20 * n + 16 * B * 1600 + 12 * words + 48 * n
    assert groundtruth.gt_chunk(32, 720, 1280, 1600) == 32
    monkeypatch.setattr(groundtruth, "GT_SCRATCH_CAP", 3 * f(1, 240, 320, 300))
    c = groundtruth.gt_chunk(8, 240, 320, 300)
    assert 1 <= c <= 3 and f(c, 240, 320, 300) <= groundtruth.GT_SCRATCH_CAP
    monkeypatch.setattr(groundtruth, "GT_SCRATCH_CAP", 1)
    assert groundtruth.gt_chunk(8, 240, 320, 300) == 1
    monkeypatch.setattr(groundtruth, "GT_SCRATCH_CAP", 1 << 40)
    assert groundtruth.gt_chunk(2 ** 18, 1, 1, 1) == 2 ** 17
    with pytest.raises(ValueError, match="too large"):
        groundtruth.gt_chunk(1, 2 ** 15, 2 ** 15, 1)


def _brute_histogram(classes, labels, K, C):
    H, W = labels.shape
    out = np.zeros((K, C), np.int64)
    for i in range(H):
        for j in range(W):
            k, c = int(labels[i, j].view(np.uint16)), int(classes[i, j])
            if k < K and 0 <= c < C:
                out[k, c] += 1
    return out


def _brute_scores(labels, gt, K, r, ignore):
    """Every pixel in Python loops: the overlap counts in a dict, the windows by scanning the square."""
    H, W = labels.shape
    lab = labels.view(np.uint16).astype(int)
    g = gt.astype(np.int64)

    def valid(i, j):
        return 0 <= g[i, j] <= 2 ** 31 - 1 and (ignore is None or g[i, j] != ignore)

    def sp(i, j):
        return (j + 1 < W and lab[i, j + 1] != lab[i, j]) or (i + 1 < H and lab[i + 1, j] != lab[i, j])

    def gb(i, j):
        if not valid(i, j):
            return False
        return ((j + 1 < W and valid(i, j + 1) and g[i, j + 1] != g[i, j]) or
                (i + 1 < H and valid(i + 1, j) and g[i + 1, j] != g[i, j]))

    def near(pred, i, j):
        return any(pred(a, b) for a in range(max(0, i - r), min(H, i + r + 1)) for b in range(max(0, j - r), min(W, j + r + 1)))

    n = {}
    res = dict.fromkeys(FIELDS, 0)
    for i in range(H):
        for j in range(W):
            if valid(i, j) and lab[i, j] < K:
                res["pixels"] += 1
                n[lab[i, j], int(g[i, j])] = n.get((lab[i, j], int(g[i, j])), 0) + 1
            if gb(i, j):
                res["gt_boundary"] += 1
                res["gt_boundary_hits"] += near(sp, i, j)
            if sp(i, j) and valid(i, j):
                res["sp_boundary"] += 1
                res["sp_boundary_hits"] += near(gb, i, j)
    nk = {}
    for (k, _), c in n.items():
        nk[k] = nk.get(k, 0) + c
    res["asa_pixels"] = sum(max(c for (k2, _), c in n.items() if k2 == k) for k in nk)
    res["ue_pixels"] = sum(min(c, nk[k] - c) for (k, _), c in n.items())
    return res


def _maps(rng):
    H, W = 11, 13
    yy, xx = np.mgrid[:H, :W]
    blocks = (yy // 4 * 4 + xx // 5).astype(np.int16)
    regions = ((yy + 2) // 5 * 3 + (xx + 1) // 6).astype(np.int64)
    yield blocks, regions.astype(np.uint8), 12, None
    yield rng.randint(-1, 25, (H, W)).astype(np.int16), rng.randint(0, 4, (H, W)).astype(np.int16), 20, 3  # -1, >= K
    yield blocks, rng.choice(np.array([0, 1, 255], np.uint8), (H, W)), 12, 255
    yield blocks, rng.choice(np.array([-7, 0, 5, 2 ** 31 - 1, 2 ** 31, -2 ** 40], np.int64), (H, W)), 12, 5
    yield rng.randint(0, 3, (H, W)).astype(np.int16), rng.randint(-2, 3, (H, W)).astype(np.int32), 3, None
    yield rng.randint(0, 4, (1, 40)).astype(np.int16), rng.randint(0, 3, (1, 40)).astype(np.uint8), 4, None  # H = 1
    yield rng.randint(0, 4, (40, 1)).astype(np.int16), rng.randint(0, 3, (40, 1)).astype(np.int16), 4, None  # W = 1
    yield np.array([[3]], np.int16), np.array([[1]], np.uint8), 9, None
    yield np.full((H, W), -1, np.int16), regions.astype(np.int32), 5, None                   # no counted pixel


@pytest.mark.parametrize("tolerance", [0, 1, 2, 32])
def test_restatement_agrees_with_brute_force(tolerance):
    rng = np.random.RandomState(5)
    for labels, gt, K, ignore in _maps(rng):
        want = _brute_scores(labels, gt, K, tolerance, ignore)
        assert ref_scores_image(labels, gt, K, tolerance, ignore) == want, (labels.shape, gt.dtype, ignore)
        if tolerance == 0:
            C = 6
            h = ref_class_histogram(gt[None], labels[None], K, C)
            assert h.dtype == np.int32 and h.shape == (1, K, C)
            assert np.array_equal(h[0], _brute_histogram(gt, labels, K, C))
            H, W = labels.shape
            want_b = [[(j + 1 < W and labels[i, j + 1] != labels[i, j]) or (i + 1 < H and labels[i + 1, j] != labels[i, j])
                       for j in range(W)] for i in range(H)]
            assert np.array_equal(ref_boundaries(labels[None])[0], np.array(want_b, bool).reshape(H, W))


def test_dilation_is_the_square_binary_dilation():
    from scipy import ndimage
    rng = np.random.RandomState(2)
    for shape in ((11, 13), (1, 40), (40, 1), (70, 90)):
        mask = rng.rand(*shape) < 0.05
        for r in (0, 1, 2, 5, 32):
            want = ndimage.binary_dilation(mask, structure=np.ones((2 * r + 1, 2 * r + 1), bool)) if r else mask
            assert np.array_equal(dilate(mask, r), want), (shape, r)


def test_known_answers():
    rng = np.random.RandomState(8)
    # labels = a relabelled gt: ASA 1, UE 0, BR = BP = 1 at r = 0
    yy, xx = np.mgrid[:30, :40]
    gt = (yy // 7 * 6 + xx // 7).astype(np.int32)
    perm = rng.permutation(100)
    labels = perm[gt].astype(np.int16)
    s = ref_scores(labels[None], gt[None], 100, tolerance=0)
    assert s["asa"][0] == 1.0 and s["undersegmentation"][0] == 0.0 and s["ue_pixels"][0] == 0
    assert s["boundary_recall"][0] == 1.0 and s["boundary_precision"][0] == 1.0 and s["gt_boundary"][0] > 0
    # one superpixel over two gt halves of a and b pixels: ASA max(a,b)/(a+b), UE 2 min(a,b)/(a+b)
    for a_cols, b_cols in ((3, 7), (5, 5), (9, 1)):
        gt = np.zeros((4, a_cols + b_cols), np.uint8)
        gt[:, a_cols:] = 1
        a, b = 4 * a_cols, 4 * b_cols
        s = ref_scores(np.zeros((1,) + gt.shape, np.int16), gt[None], 1, tolerance=0)
        assert s["asa"][0] == max(a, b) / (a + b) and s["undersegmentation"][0] == 2 * min(a, b) / (a + b)
        assert s["sp_boundary"][0] == 0 and np.isnan(s["boundary_precision"][0]) and s["boundary_recall"][0] == 0.0
    # nothing counted: NaN ratios
    s = ref_scores(np.full((1, 3, 3), -1, np.int16), np.zeros((1, 3, 3), np.uint8), 4)
    assert s["pixels"][0] == 0 and np.isnan(s["asa"][0]) and np.isnan(s["undersegmentation"][0])
