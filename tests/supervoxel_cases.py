"""The contract of fast_slic_b200.supervoxels restated in numpy (DESIGN.md section 4.22), vectorised and
float32-exact: grid, seeds, passes, assign, update and 6-connected enforcement; and seeded generators of volumes and
label volumes for the tests.

Every float operation below is one numpy float32 operation, which rounds like the device's separately rounded
intrinsics.  Keys are compared as uint32 bit patterns, a NaN distance taking the bits 0x7fffffff.  The feature means
are pool's, through pool_cases.ref_pool_batch over the volume viewed as [C, D*H, W].
"""
import math

import numpy as np

from pool_cases import ref_pool_batch

F32 = np.float32
NAN_BITS = 0x7FFFFFFF
NO_LABEL = 0xFFFF
MAX_K = 65534


def grid_of(D, H, W, K, spacing=(1.0, 1.0, 1.0)):
    """(nd, nh, nw): for an int K, n_a = clamp(floor(E_a / s0 + 0.5), 1, L_a), s0 = cbrt(prod E_a / K) in float64."""
    L = (D, H, W)
    if isinstance(K, tuple):
        return K
    E = [float(l) * float(s) for l, s in zip(L, spacing)]
    s0 = float(np.cbrt(E[0] * E[1] * E[2] / K))
    return tuple(min(max(int(math.floor(e / s0 + 0.5)), 1), l) for e, l in zip(E, L))


def weights2(D, H, W, grid, compactness, spacing):
    E = [float(l) * float(s) for l, s in zip((D, H, W), spacing)]
    s = float(np.cbrt((E[0] / grid[0]) * (E[1] / grid[1]) * (E[2] / grid[2])))
    q = [compactness * float(sp) / s for sp in spacing]
    return np.array([F32(v * v) for v in q], F32)


def radii(D, H, W, grid):
    return tuple(-(-l // n) for l, n in zip((D, H, W), grid))


def min_size_of(D, H, W, grid, min_size_factor):
    Kp = grid[0] * grid[1] * grid[2]
    return int(math.floor(float(F32(min_size_factor)) * ((D * H * W) // Kp) + 0.5))


def centres(L, n):
    i = np.arange(n)
    return (i * L // n + (i + 1) * L // n - 1) // 2


def seeds(D, H, W, grid):
    """int64 (z, y, x) [K'] of the seeds, k = (iz * nh + iy) * nw + ix."""
    cz, cy, cx = (centres(L, n) for L, n in zip((D, H, W), grid))
    z, y, x = np.meshgrid(cz, cy, cx, indexing="ij")
    return z.ravel(), y.ravel(), x.ravel()


def keys_of(fc, z, y, x, pos, k, w2):
    """uint64 keys of (voxel, candidate k) pairs from their feature distances fc."""
    with np.errstate(invalid="ignore", over="ignore"):
        tz = z.astype(F32) - pos[k, 0]
        ty = y.astype(F32) - pos[k, 1]
        tx = x.astype(F32) - pos[k, 2]
        d = fc + ((w2[0] * (tz * tz) + w2[1] * (ty * ty)) + w2[2] * (tx * tx))
    bits = d.view(np.uint32).copy()
    bits[np.isnan(d)] = NAN_BITS
    return bits.astype(np.uint64) << np.uint64(32) | k.astype(np.uint64)


def assign(f, labels, rows, pos, mu, R, w2, max_pairs=1 << 22):
    """Assigns the voxels of the rows `rows` of every slice in place (labels uint16 [D,H,W])."""
    C, D, H, W = f.shape
    K = pos.shape[0]
    row_in = np.zeros(H, bool)
    row_in[rows] = True
    ci = pos.astype(np.int64)  # (int) of non-negative positions
    dz, dy, dx = (np.arange(-r, r + 1) for r in R)
    box = (2 * R[0] + 1) * (2 * R[1] + 1) * (2 * R[2] + 1)
    oz, oy, ox = (v.ravel() for v in np.meshgrid(dz, dy, dx, indexing="ij"))
    flat = f.reshape(C, -1)
    best = np.full(D * H * W, np.iinfo(np.uint64).max, np.uint64)
    step = max(1, max_pairs // box)
    for k0 in range(0, K, step):
        ks = np.arange(k0, min(K, k0 + step))
        z = (ci[ks, 0, None] + oz[None]).ravel()
        y = (ci[ks, 1, None] + oy[None]).ravel()
        x = (ci[ks, 2, None] + ox[None]).ravel()
        k = np.repeat(ks, box)
        ok = (z >= 0) & (z < D) & (y >= 0) & (y < H) & (x >= 0) & (x < W)
        z, y, x, k = z[ok], y[ok], x[ok], k[ok]
        keep = row_in[y]
        z, y, x, k = z[keep], y[keep], x[keep], k[keep]
        p = (z * H + y) * W + x
        fc = np.zeros(p.size, F32)
        with np.errstate(invalid="ignore", over="ignore"):
            for c in range(C):
                t = flat[c][p] - mu[k, c]
                fc = fc + t * t
        np.minimum.at(best, p, keys_of(fc, z, y, x, pos, k, w2))
    hit = best != np.iinfo(np.uint64).max
    labels.reshape(-1)[hit] = (best[hit] & np.uint64(0xFFFF)).astype(np.uint16)


def update(f, labels, rows, pos, mu, K):
    """The update after a pass: returns the member counts, and moves pos and mu in place."""
    C, D, H, W = f.shape
    pass_labels = np.full((D, H, W), NO_LABEL, np.uint16)
    pass_labels[:, rows] = labels[:, rows]
    _, means, counts = ref_pool_batch(f.reshape(1, C, D * H, W), pass_labels.view(np.int16).reshape(1, D * H, W), K)
    n = counts[0].astype(np.int64)
    lab = pass_labels.ravel().astype(np.int64)
    ok = lab < K
    zz, rem = np.divmod(np.arange(D * H * W), H * W)
    yy, xx = np.divmod(rem, W)
    nz = n > 0
    for a, v in enumerate((zz, yy, xx)):
        s = np.bincount(lab[ok], weights=v[ok], minlength=K)  # exact: integer sums below 2^53
        pos[nz, a] = (s[nz] / n[nz]).astype(F32)
    mu[nz] = means[0][:, nz].T
    return n.astype(np.int32)


def ref_supervoxel_volume(f, K, compactness, spacing=(1.0, 1.0, 1.0), max_iter=10, stride=3):
    """One volume f float32 [C,D,H,W] -> (labels before enforcement uint16 [D,H,W], position f32 [K',3], features f32
    [K',C], count int32 [K'], grid)."""
    f = np.ascontiguousarray(f, F32)
    C, D, H, W = f.shape
    grid = grid_of(D, H, W, K, spacing)
    Kp = grid[0] * grid[1] * grid[2]
    R = radii(D, H, W, grid)
    w2 = weights2(D, H, W, grid, compactness, spacing)
    z, y, x = seeds(D, H, W, grid)
    pos = np.stack([z, y, x], 1).astype(F32)
    mu = np.ascontiguousarray(f[:, z, y, x].T)
    labels = np.full((D, H, W), NO_LABEL, np.uint16)
    count = np.zeros(Kp, np.int32)
    for t in range(max_iter):
        rows = np.arange(t % stride, H, stride)
        if rows.size:
            assign(f, labels, rows, pos, mu, R, w2)
        count = update(f, labels, rows, pos, mu, Kp)
    assign(f, labels, np.arange(H), pos, mu, R, w2)
    return labels, pos, mu, count, grid


def components(lab):
    """6-connected components of equal values of lab [D,H,W]: (component of each voxel int64 [N] numbered by leader
    order, leaders int64 [ncomp]).  Union-find by hooking roots to the smaller one, with pointer jumping."""
    D, H, W = lab.shape
    N = lab.size
    idx = np.arange(N).reshape(D, H, W)
    us, vs = [], []
    for a in range(3):
        lo = [slice(None)] * 3
        hi = [slice(None)] * 3
        lo[a], hi[a] = slice(0, -1), slice(1, None)
        same = lab[tuple(lo)] == lab[tuple(hi)]
        us.append(idx[tuple(lo)][same])
        vs.append(idx[tuple(hi)][same])
    u, v = np.concatenate(us), np.concatenate(vs)
    par = np.arange(N)
    while True:
        while True:
            nxt = par[par]
            if np.array_equal(nxt, par):
                break
            par = nxt
        pu, pv = par[u], par[v]
        diff = pu != pv
        if not diff.any():
            break
        m = np.minimum(pu[diff], pv[diff])
        np.minimum.at(par, pu[diff], m)
        np.minimum.at(par, pv[diff], m)
    roots = par == np.arange(N)
    number = np.cumsum(roots) - 1
    return number[par], np.flatnonzero(roots)


def ref_enforce(lab, K, min_size):
    """Enforcement of one label volume (any integer dtype, compared as uint16) -> int16 [D,H,W]."""
    lab = np.asarray(lab).astype(np.uint16)
    D, H, W = lab.shape
    comp, leaders = components(lab)
    nc = leaders.size
    area = np.bincount(comp, minlength=nc)
    cand = np.flatnonzero(area >= min_size)
    if cand.size > K:
        order = np.lexsort((leaders[cand], -area[cand]))
        cand = np.sort(cand[order[:K]])
    final = np.full(nc, -1, np.int64)
    final[cand] = np.arange(cand.size)
    if final[0] < 0:
        final[0] = 0
    # every other component points at its leader's predecessor's component; jump to a labelled one
    x = leaders % W
    y = (leaders // W) % H
    q = np.where(x > 0, leaders - 1, np.where(y > 0, leaders - W, leaders - H * W))
    target = np.where(final >= 0, np.arange(nc), comp[np.maximum(q, 0)])
    while True:
        nxt = target[target]
        if np.array_equal(nxt, target):
            break
        target = nxt
    return final[target][comp].reshape(D, H, W).astype(np.int16)


def ref_supervoxel_slic(volumes, K, compactness, spacing=(1.0, 1.0, 1.0), max_iter=10, stride=3,
                        min_size_factor=0.25):
    """[B,C,D,H,W] -> (labels after enforcement int16 [B,D,H,W], labels before uint16, position [B,K',3], features
    [B,K',C], count [B,K'], grid)."""
    B, C, D, H, W = volumes.shape
    out = [ref_supervoxel_volume(volumes[b], K, compactness, spacing, max_iter, stride) for b in range(B)]
    grid = grid_of(D, H, W, K, spacing)
    Kp = grid[0] * grid[1] * grid[2]
    thres = min_size_of(D, H, W, grid, min_size_factor)
    pre = np.stack([o[0] for o in out])
    final = np.stack([ref_enforce(p, Kp, thres) for p in pre])
    return (final, pre, np.stack([o[1] for o in out]), np.stack([o[2] for o in out]), np.stack([o[3] for o in out]),
            grid)


def make_volumes(seed, B, C, D, H, W, kind="smooth"):
    """float32 [B,C,D,H,W]: "smooth" (sinusoids plus noise), "constant" (every voxel the same, everything ties),
    "nonfinite" (smooth with NaN, +inf and -inf voxels and a whole NaN row)."""
    rng = np.random.RandomState(seed)
    if kind == "constant":
        return np.full((B, C, D, H, W), F32(rng.randn()), F32)
    z, y, x = np.mgrid[0:D, 0:H, 0:W].astype(F32)
    f = np.empty((B, C, D, H, W), F32)
    for b in range(B):
        for c in range(C):
            a, bb, cc, ph = rng.rand(4).astype(F32) * F32(0.25) + F32(0.01)
            f[b, c] = np.sin(x * a + y * bb + z * cc + ph * 10) * 3 + rng.randn(D, H, W).astype(F32) * F32(0.3)
    if kind == "nonfinite":
        n = max(1, f.size // 50)
        flat = f.reshape(-1)
        for v in (np.nan, np.inf, -np.inf):
            flat[rng.randint(0, f.size, n)] = v
        if H > 2:
            f[:, 0, rng.randint(0, D), rng.randint(0, H)] = np.nan
    return f


def block_labels(seed, D, H, W, nlab, block=(2, 2, 2)):
    """uint16 [D,H,W]: random labels in [0, nlab) constant on blocks, so components of many sizes and shapes."""
    rng = np.random.RandomState(seed)
    small = rng.randint(0, nlab, size=tuple(-(-L // b) for L, b in zip((D, H, W), block)))
    big = small.repeat(block[0], 0).repeat(block[1], 1).repeat(block[2], 2)
    return np.ascontiguousarray(big[:D, :H, :W]).astype(np.uint16)


def nan_class_equal(a, b):
    """Bit-identical, except that any NaN equals any NaN."""
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    return bool((na == nb).all() and (a.view(np.uint32)[~na] == b.view(np.uint32)[~nb]).all())
