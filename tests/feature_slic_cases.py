"""The contract of fast_slic_b200.feature_slic restated in numpy (DESIGN.md section 4.19), vectorised and float32-exact,
and a seeded generator of feature maps for the tests.

Every float operation below is one numpy float32 operation, which rounds like the device's separately rounded
intrinsics.  Keys are compared as uint32 bit patterns, a NaN distance taking the bits 0x7fffffff.  The feature means
are pool's, through pool_cases.ref_pool_batch.  The seed grid is initialize_clusters' grid, taken from the plain-C
oracle (oracle/slic_oracle.c), which the suite pins against the compiled reference.
"""
import math

import numpy as np

from pool_cases import ref_pool_batch

F32 = np.float32
NAN_BITS = 0x7FFFFFFF
NO_LABEL = 0xFFFF


def superpixel_size(H, W, K):
    return int(math.sqrt((H * W) // K))


def min_size_threshold(S, min_size_factor):
    x = float(S * S) * float(F32(min_size_factor))
    t = math.floor(x)
    return int(t + 1 if x - t >= 0.5 else t)


def seed_grid(H, W, K):
    """int64 (cy, cx) [K] of initialize_clusters' grid."""
    from oracle.oracle import Port
    cl = Port().initialize(np.zeros((H, W, 3), np.uint8), K)
    return cl["y"].astype(np.int64), cl["x"].astype(np.int64)


def weight2(compactness, S):
    w = F32(F32(compactness) / F32(S))
    return F32(w * w)


def keys_of(fc, i, j, pos, k, w2):
    """uint64 keys of (pixel (i, j), candidate k) pairs from their feature distances fc."""
    with np.errstate(invalid="ignore", over="ignore"):
        ty = i.astype(F32) - pos[k, 0]
        tx = j.astype(F32) - pos[k, 1]
        d = fc + w2 * (ty * ty + tx * tx)
    bits = d.view(np.uint32).copy()
    bits[np.isnan(d)] = NAN_BITS
    return bits.astype(np.uint64) << np.uint64(32) | k.astype(np.uint64)


def assign(f, labels, rows, pos, mu, S, w2, max_pairs=1 << 22):
    """Assigns the pixels of `rows` in place (labels uint16 [H,W]): the smallest key among the candidates."""
    C, H, W = f.shape
    K = pos.shape[0]
    row_in = np.zeros(H, bool)
    row_in[rows] = True
    cyi, cxi = pos[:, 0].astype(np.int64), pos[:, 1].astype(np.int64)
    d = np.arange(-S, S + 1)
    flat = f.reshape(C, -1)
    best = np.full(H * W, np.iinfo(np.uint64).max, np.uint64)
    step = max(1, max_pairs // (2 * S + 1) ** 2)
    for k0 in range(0, K, step):
        ks = np.arange(k0, min(K, k0 + step))
        i = (cyi[ks, None, None] + d[None, :, None]) + 0 * d[None, None, :]
        j = (cxi[ks, None, None] + d[None, None, :]) + 0 * d[None, :, None]
        k = np.broadcast_to(ks[:, None, None], i.shape)
        ok = (i >= 0) & (i < H) & (j >= 0) & (j < W)
        i, j, k = i[ok], j[ok], k[ok]
        keep = row_in[i]
        i, j, k = i[keep], j[keep], k[keep]
        p = i * W + j
        fc = np.zeros(p.size, F32)
        with np.errstate(invalid="ignore", over="ignore"):
            for c in range(C):
                t = flat[c][p] - mu[k, c]
                fc = fc + t * t
        np.minimum.at(best, p, keys_of(fc, i, j, pos, k, w2))
    hit = best != np.iinfo(np.uint64).max
    labels.reshape(-1)[hit] = (best[hit] & np.uint64(0xFFFF)).astype(np.uint16)


def update(f, labels, rows, pos, mu, K):
    """The update after a pass: returns the member counts and the pass's labels (0xffff off its rows), and moves pos
    and mu in place."""
    C, H, W = f.shape
    pass_labels = np.full((H, W), NO_LABEL, np.uint16)
    pass_labels[rows] = labels[rows]
    _, means, counts = ref_pool_batch(f[None], pass_labels.view(np.int16)[None], K)
    n = counts[0].astype(np.int64)
    lab = pass_labels.ravel().astype(np.int64)
    ok = lab < K
    ii, jj = np.divmod(np.arange(H * W), W)
    si = np.bincount(lab[ok], weights=ii[ok], minlength=K)  # exact: integer sums below 2^53
    sj = np.bincount(lab[ok], weights=jj[ok], minlength=K)
    nz = n > 0
    pos[nz, 0] = (si[nz] / n[nz]).astype(F32)
    pos[nz, 1] = (sj[nz] / n[nz]).astype(F32)
    mu[nz] = means[0][:, nz].T
    return n.astype(np.int32), pass_labels


def ref_feature_slic_image(f, K, compactness, max_iter=10, stride=3, init=None, with_pass_labels=False):
    """One image f float32 [C,H,W] -> (labels before enforcement uint16 [H,W], position f32 [K,2], features f32 [K,C],
    count int32 [K]), and with_pass_labels the labels of the last update (uint16 [H,W], None without one)."""
    f = np.ascontiguousarray(f, F32)
    C, H, W = f.shape
    S = superpixel_size(H, W, K)
    w2 = weight2(compactness, S)
    if init is None:
        cy, cx = seed_grid(H, W, K)
        pos = np.stack([cy, cx], 1).astype(F32)
        mu = np.ascontiguousarray(f[:, cy, cx].T)
    else:
        p0, m0 = init
        pos = np.stack([np.fmin(np.fmax(p0[:, 0], F32(0)), F32(H - 1)),
                        np.fmin(np.fmax(p0[:, 1], F32(0)), F32(W - 1))], 1).astype(F32)
        mu = np.array(m0, F32)
    labels = np.full((H, W), NO_LABEL, np.uint16)
    count = np.zeros(K, np.int32)
    pass_labels = None
    for t in range(max_iter):
        rows = np.arange(t % stride, H, stride)
        if rows.size:
            assign(f, labels, rows, pos, mu, S, w2)
        count, pass_labels = update(f, labels, rows, pos, mu, K)
    assign(f, labels, np.arange(H), pos, mu, S, w2)
    return (labels, pos, mu, count) + ((pass_labels,) if with_pass_labels else ())


def ref_feature_slic(features, K, compactness, max_iter=10, stride=3, min_size_factor=0.25, init=None):
    """[B,C,H,W] -> (labels after enforcement int16 [B,H,W], labels before uint16 [B,H,W], position [B,K,2],
    features [B,K,C], count [B,K]); enforcement by the plain-C oracle's enforce_connectivity."""
    from oracle.oracle import Port
    B, C, H, W = features.shape
    thres = min_size_threshold(superpixel_size(H, W, K), min_size_factor)
    port = Port()
    out = [ref_feature_slic_image(features[b], K, compactness, max_iter, stride,
                                  None if init is None else (init[0][b], init[1][b])) for b in range(B)]
    pre = np.stack([o[0] for o in out]) if B else np.zeros((0, H, W), np.uint16)
    final = np.stack([port.enforce_connectivity(p, K, thres) for p in pre]).view(np.int16) if B else pre.view(np.int16)
    pos = np.stack([o[1] for o in out]) if B else np.zeros((0, K, 2), F32)
    mu = np.stack([o[2] for o in out]) if B else np.zeros((0, K, C), F32)
    cnt = np.stack([o[3] for o in out]) if B else np.zeros((0, K), np.int32)
    return final, pre, pos, mu, cnt


def make_features(seed, B, C, H, W, kind="smooth"):
    """float32 [B,C,H,W]: "smooth" (sinusoids and blobs plus noise), "constant" (every pixel the same, everything
    ties), "nonfinite" (smooth with NaN, +inf and -inf pixels and whole NaN rows)."""
    rng = np.random.RandomState(seed)
    if kind == "constant":
        return np.full((B, C, H, W), F32(rng.randn()), F32)
    y, x = np.mgrid[0:H, 0:W].astype(F32)
    f = np.empty((B, C, H, W), F32)
    for b in range(B):
        for c in range(C):
            a, bb, ph = rng.rand(3) * F32(0.2) + F32(0.01)
            f[b, c] = np.sin(x * a + y * bb + ph * 10) * 3 + rng.randn(H, W).astype(F32) * F32(0.3)
    if kind == "nonfinite":
        n = max(1, f.size // 50)
        flat = f.reshape(-1)
        for v in (np.nan, np.inf, -np.inf):
            flat[rng.randint(0, f.size, n)] = v
        if H > 2:
            f[:, 0, rng.randint(0, H)] = np.nan
    return f


def nan_class_equal(a, b):
    """Bit-identical, except that any NaN equals any NaN."""
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    return bool((na == nb).all() and (a.view(np.uint32)[~na] == b.view(np.uint32)[~nb]).all())
