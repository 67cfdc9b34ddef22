"""Superpixel pooling on the GPU (fast_slic_b200.pooling): pool against the numpy restatement of its summation order
(pool_cases.py) bit for bit, NaN compared as a class; batch, chunk, stream and run invariance; adversarial label maps;
unpool and paint_argmax against torch gathers; autograd; and the SLIC -> SimpleCRFGroup -> paint_argmax loop."""
import numpy as np
import pytest
import torch

from cases import make_image
from pool_cases import nan_class_equal, ref_pool_batch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _needs_cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _np(x):
    return x.detach().cpu().numpy()


def _slic(H, W, K, B, msf, seed):
    from fast_slic_b200 import Slic
    imgs = torch.from_numpy(np.stack([make_image("syn", H, W, seed=seed + b) for b in range(B)])).cuda()
    return Slic(num_components=K, min_size_factor=msf).iterate_batch(imgs, return_clusters=True)


@pytest.fixture(scope="module", params=[0.0, 0.25], ids=["msf0", "msf.25"])
def slic_maps(request):
    labels, clusters = _slic(240, 320, 300, 8, request.param, seed=21)
    return labels, int(clusters.shape[1])


def _feats(B, C, H, W, seed):
    return torch.from_numpy(np.random.RandomState(seed).standard_normal((B, C, H, W)).astype(np.float32)).cuda()


def _check(feats, labels, K):
    """pool (sum, mean, counts) against the restatement, bit for bit; returns the device results."""
    from fast_slic_b200.pooling import pool
    sums, counts = pool(feats, labels, K, reduce="sum", return_counts=True)
    means, counts2 = pool(feats, labels, K, return_counts=True)
    assert sums.dtype == torch.float32 and counts.dtype == torch.int32 and sums.device == labels.device
    assert tuple(sums.shape) == (labels.shape[0], feats.shape[1], K) and tuple(counts.shape) == (labels.shape[0], K)
    ws, wm, wc = ref_pool_batch(_np(feats), _np(labels), K)
    assert (_np(counts) == wc).all() and (_np(counts2) == wc).all()
    assert nan_class_equal(_np(sums), ws)
    assert nan_class_equal(_np(means), wm)
    return sums, means, counts


@pytest.mark.parametrize("C", [1, 3, 21, 64])
def test_slic_maps(slic_maps, C):
    labels, K = slic_maps
    feats = _feats(labels.shape[0], C, 240, 320, seed=C)
    _, _, counts = _check(feats, labels, K)
    lab = _np(labels).astype(np.int64)
    for b in range(labels.shape[0]):
        assert (_np(counts[b]) == np.bincount(lab[b][(lab[b] >= 0) & (lab[b] < K)], minlength=K)).all()


def test_batch_chunk_and_stream_invariance(slic_maps, monkeypatch):
    from fast_slic_b200 import _lib, pooling
    from fast_slic_b200.pooling import pool
    labels, K = slic_maps
    B = labels.shape[0]
    feats = _feats(B, 5, 240, 320, seed=7)
    full, counts = pool(feats, labels, K, return_counts=True)
    sums = pool(feats, labels, K, reduce="sum")
    for b in range(B):  # a batch of one
        assert torch.equal(pool(feats[b:b + 1], labels[b:b + 1], K).view(torch.int32), full[b:b + 1].view(torch.int32))
    perm = torch.tensor([5, 2, 7, 0, 3, 1, 6, 4], device="cuda")
    assert torch.equal(pool(feats[perm], labels[perm], K).view(torch.int32), full[perm].view(torch.int32))
    assert torch.equal(pool(feats[perm], labels[perm], K, reduce="sum").view(torch.int32), sums[perm].view(torch.int32))
    # a second run, a run on a non-default stream, channels_last features
    assert torch.equal(pool(feats, labels, K).view(torch.int32), full.view(torch.int32))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        on_s = pool(feats, labels, K)
    s.synchronize()
    assert torch.equal(on_s.view(torch.int32), full.view(torch.int32))
    assert torch.equal(pool(feats.to(memory_format=torch.channels_last), labels, K).view(torch.int32),
                       full.view(torch.int32))
    # several chunks
    monkeypatch.setattr(pooling, "POOL_SCRATCH_CAP", 3 * _lib.lib().fslic_b200_pool_batch_scratch_bytes(1, 240, 320, K))
    assert pooling.pool_chunk(B, 240, 320, K) < B
    got, got_counts = pool(feats, labels, K, return_counts=True)
    assert torch.equal(got.view(torch.int32), full.view(torch.int32)) and torch.equal(got_counts, counts)
    assert torch.equal(pool(feats, labels, K, reduce="sum").view(torch.int32), sums.view(torch.int32))


def _adversarial():
    rng = np.random.RandomState(5)
    yield "noise", rng.randint(0, 5000, (2, 61, 77)).astype(np.int16), 5000
    yield "one label", np.zeros((2, 50, 70), np.int16), 1
    mixed = rng.randint(0, 40, (3, 45, 67)).astype(np.int16)
    mixed[rng.rand(*mixed.shape) < 0.2] = -1
    big = rng.rand(*mixed.shape) < 0.1
    mixed[big] = 40 + rng.randint(0, 30000, int(big.sum()))
    yield "out of range", mixed, 40
    yield "K=1 mixed", rng.randint(-1, 2, (2, 33, 65)).astype(np.int16), 1
    few = rng.choice(np.array([0, 17, 30000, 65533, 65535], np.uint16), (2, 40, 50)).view(np.int16)
    yield "K=65534 few labels", few, 65534
    yield "H=1", rng.randint(0, 9, (3, 1, 300)).astype(np.int16), 9
    yield "W=1", rng.randint(0, 9, (3, 300, 1)).astype(np.int16), 9
    yield "1x1", np.array([[[0]], [[-1]], [[2]]], np.int16), 3
    yield "W%32", rng.randint(0, 60, (2, 37, 95)).astype(np.int16) // 3, 20


@pytest.mark.parametrize("C", [1, 7])
def test_adversarial_maps(C):
    for name, labels, K in _adversarial():
        B, H, W = labels.shape
        feats = _feats(B, C, H, W, seed=B * H + W)
        _check(feats, torch.from_numpy(labels).cuda(), K)


def test_counts_above_2_24():
    H, W = 4100, 4200
    labels = np.zeros((1, H, W), np.int16)
    labels[0, :100, :100] = 1
    labels[0, -1, -7:] = -1
    feats = _feats(1, 1, H, W, seed=9)
    _, means, counts = _check(feats, torch.from_numpy(labels).cuda(), 2)
    n0 = H * W - 10000 - 7
    assert _np(counts).tolist() == [[n0, 10000]] and n0 > 2 ** 24 and float(np.float32(n0)) != n0


def test_special_values():
    rng = np.random.RandomState(8)
    B, C, H, W, K = 2, 4, 31, 45, 30
    labels = rng.randint(-1, K, (B, H, W)).astype(np.int16)
    f = rng.standard_normal((B, C, H, W)).astype(np.float32)
    f[0, 0][labels[0] == 3] = -0.0  # a superpixel of negative zeros
    f[1, 1][labels[1] < 5] = 0.0
    for val, frac in ((np.nan, 0.01), (np.inf, 0.01), (-np.inf, 0.01), (-0.0, 0.2)):
        f[rng.rand(B, C, H, W) < frac] = val
    _check(torch.from_numpy(f).cuda(), torch.from_numpy(labels).cuda(), K)


def test_empty_shapes():
    from fast_slic_b200.pooling import paint_argmax, pool, unpool
    for B, H, W in ((0, 5, 6), (2, 0, 6), (2, 5, 0)):
        labels = torch.zeros((B, H, W), dtype=torch.int16, device="cuda")
        s, c = pool(torch.ones((B, 3, H, W), device="cuda"), labels, 7, return_counts=True)
        assert tuple(s.shape) == (B, 3, 7) and not s.any() and tuple(c.shape) == (B, 7) and not c.any()
        u = unpool(torch.ones((B, 3, 7), device="cuda"), labels)
        assert tuple(u.shape) == (B, 3, H, W)
        assert tuple(paint_argmax(torch.ones((B, 3, 7), device="cuda"), labels).shape) == (B, H, W)


def _gather_want(values, labels):
    """torch restatement of unpool: values[b, :, label] where 0 <= label < K, else 0."""
    K = values.shape[2]
    lab = labels.long() & 0xFFFF
    valid = lab < K
    B, C = values.shape[:2]
    idx = torch.where(valid, lab, 0).view(B, 1, -1).expand(B, C, -1)
    g = torch.gather(values, 2, idx).view(B, C, *labels.shape[1:])
    return torch.where(valid[:, None], g, torch.zeros((), device=values.device)), valid


def test_unpool_and_paint_argmax():
    from fast_slic_b200.pooling import paint_argmax, unpool
    rng = np.random.RandomState(4)
    B, C, H, W, K = 3, 6, 37, 53, 50
    labels = torch.from_numpy(rng.randint(-1, K + 5, (B, H, W)).astype(np.int16)).cuda()
    q = rng.randint(0, 3, (B, C, K)).astype(np.float32)  # many ties
    q[0, 2, :10] = np.nan
    q[1, 4, 5:15] = np.nan
    q[1, 1, 10:12] = np.nan
    q[2, 0, :] = -0.0
    q[2, 1, :] = 0.0
    q[2, 2:, :] = -1.0
    q = torch.from_numpy(q).cuda()
    want, valid = _gather_want(q, labels)
    got = unpool(q, labels)
    assert torch.equal(got.view(torch.int32), want.view(torch.int32))
    cls = torch.argmax(q.cpu(), dim=1).cuda()  # [B, K]
    want_cls = torch.where(valid, torch.gather(cls, 1, torch.where(valid, labels.long() & 0xFFFF, 0).view(B, -1))
                           .view(B, H, W), -1).to(torch.int16)
    got_cls = paint_argmax(q, labels)
    assert got_cls.dtype == torch.int16 and torch.equal(got_cls, want_cls)
    assert (got_cls[2][valid[2]] == 0).all()  # -0.0 ties +0.0: the first index wins


def _f64_pool(f, labels, K):
    """float64 torch restatement with autograd: (sums, means) [B,C,K]."""
    B, C, H, W = f.shape
    lab = labels.long() & 0xFFFF
    idx = torch.where(lab < K, lab, K).view(B, 1, -1).expand(B, C, -1)
    sums = torch.zeros((B, C, K + 1), dtype=torch.float64, device=f.device).scatter_add(2, idx, f.reshape(B, C, -1))
    sums = sums[:, :, :K]
    counts = torch.zeros((B, K + 1), dtype=torch.float64, device=f.device).scatter_add(
        1, idx[:, 0], torch.ones_like(idx[:, 0], dtype=torch.float64))[:, :K]
    return sums, sums / counts.clamp(min=1)[:, None]


def test_autograd(slic_maps):
    from fast_slic_b200.pooling import pool, unpool
    labels, K = slic_maps
    labels = labels[:3].clone()
    labels[0, :5, :5] = -1
    B, C = 3, 4
    feats = _feats(B, C, 240, 320, seed=12)
    w = torch.from_numpy(np.random.RandomState(2).standard_normal((B, C, K)).astype(np.float32)).cuda()
    grads = {}
    for reduce in ("mean", "sum"):
        runs = []
        for _ in range(2):
            f = feats.clone().requires_grad_()
            out = pool(f, labels, K, reduce=reduce)
            (out * w).sum().backward()
            runs.append(f.grad)
        assert torch.equal(runs[0].view(torch.int32), runs[1].view(torch.int32)), reduce
        f64 = feats.double().requires_grad_()
        s64, m64 = _f64_pool(f64, labels, K)
        ((m64 if reduce == "mean" else s64) * w.double()).sum().backward()
        torch.testing.assert_close(runs[0].double(), f64.grad, rtol=1e-6, atol=0)
        assert (runs[0][0, :, :5, :5] == 0).all()
        grads[reduce] = runs[0]
    # the mean's backward is unpool(grad) / count, the sum's unpool(grad)
    _, counts = pool(feats, labels, K, return_counts=True)
    want_sum, valid = _gather_want(w, labels)
    assert torch.equal(grads["sum"].view(torch.int32), want_sum.view(torch.int32))
    cnt, _ = _gather_want(counts[:, None].float(), labels)
    want_mean = torch.where(valid[:, None], want_sum / cnt.clamp(min=1), torch.zeros((), device="cuda"))
    assert torch.equal(grads["mean"].view(torch.int32), want_mean.view(torch.int32))
    # unpool's backward is pool(grad, reduce="sum")
    g = torch.from_numpy(np.random.RandomState(6).standard_normal((B, C, 240, 320)).astype(np.float32)).cuda()
    runs = []
    for _ in range(2):
        v = w.clone().requires_grad_()
        (unpool(v, labels) * g).sum().backward()
        runs.append(v.grad)
    assert torch.equal(runs[0].view(torch.int32), runs[1].view(torch.int32))
    assert torch.equal(runs[0].view(torch.int32), pool(g, labels, K, reduce="sum").view(torch.int32))
    s64, _ = _f64_pool(g.double(), labels, K)
    torch.testing.assert_close(runs[0].double(), s64, rtol=1e-5, atol=1e-4)


def test_slic_crf_group_loop():
    """iterate_batch -> SimpleCRFGroup.push_label_frames -> set_proba(pool(softmax)) -> inference -> get_inferred ->
    paint_argmax, against SimpleCRFs fed the pooled probabilities through the host set_proba."""
    from fast_slic_b200.crf import SimpleCRF, SimpleCRFGroup
    from fast_slic_b200.pooling import paint_argmax, pool
    B, Cc, H, W = 3, 5, 240, 320
    labels, clusters = _slic(H, W, 300, B, 0.25, seed=50)
    K = int(clusters.shape[1])
    logits = _feats(B, Cc, H, W, seed=13) * 3
    pooled = pool(torch.softmax(logits, dim=1), labels, K)
    group = SimpleCRFGroup([SimpleCRF(Cc, K) for _ in range(B)])
    alone = [SimpleCRF(Cc, K) for _ in range(B)]
    group.push_label_frames(labels, clusters)
    group.set_proba(pooled)
    group.reset_inferred()
    group.inference(5)
    q = torch.empty((B, Cc, K), device="cuda")
    assert group.get_inferred(out=q) is q
    classes = paint_argmax(q, labels)
    lab = _np(labels).astype(np.int64)
    for b, crf in enumerate(alone):
        frame = crf.push_label_frames(labels[b], clusters[b])
        frame.set_proba(_np(pooled[b]))
        frame.reset_inferred()
        crf.inference(5)
        qb = frame.get_inferred()
        assert nan_class_equal(_np(q[b]), qb), b
        node = np.argmax(qb, axis=0)
        valid = (lab[b] >= 0) & (lab[b] < K)
        want = np.where(valid, node[np.where(valid, lab[b], 0)], -1).astype(np.int16)
        assert (_np(classes[b]) == want).all(), b
