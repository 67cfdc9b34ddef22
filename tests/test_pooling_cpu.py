"""Superpixel pooling without a GPU: the ABI declarations, the argument checks (they come before any device work),
the scratch size and chunking, and the numpy restatement of the summation order against float64 sums."""
import os
import re

import numpy as np
import pytest
import torch

from pool_cases import nan_class_equal, ref_pool, ref_pool_batch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ("fslic_b200_pool_batch_scratch_bytes", "fslic_b200_pool_batch", "fslic_b200_pool_unpool_batch",
               "fslic_b200_pool_paint_argmax_batch")


def test_abi_declares_and_binds_the_pool_entry_points():
    from fast_slic_b200 import _lib
    L = _lib.lib()
    header = open(os.path.join(ROOT, "include", "fslic_b200.h")).read()
    declared = set(re.findall(r"\b(fslic_b200_\w+)\s*\(", header))
    for sym in NEW_SYMBOLS:
        assert sym in declared and sym in _lib.EXPORTED_SYMBOLS, sym
        assert getattr(L, sym).argtypes is not None, sym
        assert not sym.startswith("fslic_b200_crf_") and "expf" not in sym
    assert L.fslic_b200_pool_batch_scratch_bytes.restype is not None


def _args(B=2, C=3, H=5, W=7, K=10, device="cpu"):
    feats = torch.zeros((B, C, H, W), dtype=torch.float32, device=device)
    labels = torch.zeros((B, H, W), dtype=torch.int16, device=device)
    return feats, labels, K


def test_pool_argument_errors():
    from fast_slic_b200.pooling import pool
    f, l, K = _args()
    bad = [
        ((f.numpy(), l, K), "torch.from_numpy"),                 # numpy features
        ((f, l.numpy(), K), "torch.from_numpy"),                 # numpy labels
        ((f.double(), l, K), "float32"),                         # dtype
        ((f.half(), l, K), "float32"),
        ((f, l.int(), K), "int16"),
        ((f, l.view(torch.uint8)[..., :7].contiguous(), K), "int16"),
        ((f[0], l, K), "dimensions"),                            # ndim
        ((f, l[0], K), "dimensions"),
        ((f[:, :, :-1], l, K), "do not match"),                  # shape
        ((f[:, :, :, :-1], l, K), "do not match"),
        ((f[:1], l, K), "do not match"),
        ((f[:, :0], l, K), "channel"),                           # C = 0
        ((f, l, 0), "K must be"),                                # K range
        ((f, l, 65535), "K must be"),
        ((f, l, -1), "K must be"),
        ((f, l, 3.0), "K must be"),
        ((f, l, K), "cuda"),                                     # cpu tensors
        ((f.to("meta"), l, K), "labels on cpu"),                 # mismatched devices
    ]
    for args, msg in bad:
        with pytest.raises(ValueError, match=msg):
            pool(*args)
    with pytest.raises(ValueError, match="reduce"):
        pool(f, l, K, reduce="max")


def test_unpool_and_paint_argument_errors():
    from fast_slic_b200.pooling import paint_argmax, unpool
    _, l, K = _args()
    v = torch.zeros((2, 3, K), dtype=torch.float32)
    for fn in (unpool, paint_argmax):
        for args, msg in [((v.numpy(), l), "torch.from_numpy"), ((v, l.numpy()), "torch.from_numpy"),
                          ((v.double(), l), "float32"), ((v, l.long()), "int16"), ((v[0], l), "dimensions"),
                          ((v[None], l), "dimensions"), ((v[:1], l), "do not match"), ((v[:, :0], l), "channel"),
                          ((v[:, :, :0], l), "K must be"), ((torch.zeros((2, 3, 65535)), l), "K must be"),
                          ((v, l), "cuda"), ((v.to("meta"), l), "labels on cpu")]:
            with pytest.raises(ValueError, match=msg):
                fn(*args)
    with pytest.raises(ValueError, match="32767"):
        paint_argmax(torch.zeros((2, 32768, 1)), l)


def test_scratch_bytes_and_chunks(monkeypatch):
    from fast_slic_b200 import _lib, pooling
    f = _lib.lib().fslic_b200_pool_batch_scratch_bytes
    none = 2 ** 64 - 1
    assert f(0, 5, 5, 10) == 256 and f(3, 0, 5, 10) == 256
    assert f(1, 5, 5, 0) == none and f(1, 5, 5, 65535) == none and f(-1, 5, 5, 10) == none
    for B, H, W, K in ((1, 240, 320, 300), (8, 240, 320, 300), (32, 720, 1280, 1600), (1, 4100, 4200, 1)):
        assert f(B, H, W, K) >= 16 * B * H * W + 8 * B * K
    assert f(1, 46341, 46341, 1) == none  # more than 2^31 - 1 pixels in one sort
    assert f(65537, 1, 1, 1) == none and f(65536, 1, 1, 1) != none
    assert pooling.pool_chunk(32, 720, 1280, 1600) == 32
    monkeypatch.setattr(pooling, "POOL_SCRATCH_CAP", 3 * f(1, 240, 320, 300))
    c = pooling.pool_chunk(8, 240, 320, 300)
    assert 1 <= c <= 3 and f(c, 240, 320, 300) <= pooling.POOL_SCRATCH_CAP
    monkeypatch.setattr(pooling, "POOL_SCRATCH_CAP", 1)
    assert pooling.pool_chunk(8, 240, 320, 300) == 1
    with pytest.raises(ValueError, match="too large"):
        pooling.pool_chunk(1, 46341, 46341, 1)


def _maps(rng):
    """Small label maps: blocky superpixels, noise, one label, out-of-range labels mixed in."""
    H, W = 13, 37
    yy, xx = np.mgrid[:H, :W]
    blocky = (yy // 4 * 10 + xx // 5).astype(np.int16)
    noise = rng.randint(0, 20, (H, W)).astype(np.int16)
    mixed = rng.randint(-1, 25, (H, W)).astype(np.int16)
    return [(blocky, 40), (noise, 20), (np.zeros((H, W), np.int16), 1), (mixed, 20), (np.full((H, W), 7, np.int16), 8)]


@pytest.mark.parametrize("C", [1, 3])
def test_restatement_agrees_with_float64_sums(C):
    rng = np.random.RandomState(3)
    for labels, K in _maps(rng):
        feats = rng.standard_normal((C,) + labels.shape).astype(np.float32)
        sums, means, counts = ref_pool(feats, labels, K)
        lab = labels.astype(np.int64).ravel()
        ok = (lab >= 0) & (lab < K)
        assert (counts == np.bincount(lab[ok], minlength=K)).all()
        want = np.zeros((C, K))
        for c in range(C):
            want[c] = np.bincount(lab[ok], weights=feats[c].ravel()[ok].astype(np.float64), minlength=K)
        np.testing.assert_allclose(sums, want, rtol=1e-5, atol=1e-5 * (1 + counts.max()))
        wm = np.where(counts > 0, want / np.maximum(counts, 1), 0.0)
        np.testing.assert_allclose(means, wm, rtol=1e-5, atol=1e-5)
        assert (means[:, counts == 0] == 0).all() and not np.signbit(sums[:, counts == 0]).any()


def test_restatement_special_values():
    labels = np.array([[0, 0, 1, 1, 2, 2, -1, 3]], np.int16)
    feats = np.array([[[-0.0, -0.0, np.nan, 1.0, np.inf, 2.0, np.nan, -np.inf]]], np.float32)
    sums, means, counts = ref_pool(feats, labels, 5)
    assert counts.tolist() == [2, 2, 2, 1, 0]
    want = np.array([[0.0, np.nan, np.inf, -np.inf, 0.0]], np.float32)
    assert nan_class_equal(sums, want) and not np.signbit(sums[0, 0])  # +0.0: the lanes start from +0.0
    assert nan_class_equal(means, want)
    # the batch form is image by image
    s2, m2, c2 = ref_pool_batch(np.concatenate([feats[None], feats[None]]), np.stack([labels, labels]), 5)
    assert nan_class_equal(s2[1], sums) and c2.dtype == np.int32


def test_restatement_lane_order():
    """40 members: lanes 0..7 add two members, the rest one; the butterfly then combines the lanes."""
    labels = np.zeros((1, 40), np.int16)
    feats = np.zeros((1, 1, 40), np.float32)
    feats[0, 0, 0], feats[0, 0, 32], feats[0, 0, 1] = 1.0, 2.0 ** -24, 2.0 ** -24
    sums = ref_pool(feats, labels, 1)[0]
    lanes = np.zeros(32, np.float32)
    lanes[0] = np.float32(1.0) + np.float32(2.0 ** -24)  # rounds to 1.0
    lanes[1] = np.float32(2.0 ** -24)
    v = lanes.copy()
    for off in (16, 8, 4, 2, 1):
        v = v + v[np.arange(32) ^ off]
    assert sums[0, 0] == v[0] == np.float32(1.0)
    assert np.float32(1.0) + np.float32(2.0 ** -23) != sums[0, 0]  # the two small members added first would show
