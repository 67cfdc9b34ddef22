"""The contract of fast_slic_b200.soft_slic restated in numpy (DESIGN.md section 4.20), vectorised and float32-exact:
the grid, the 9 slots, the cell blocks, the forwards and backwards of soft_assign, soft_pool and soft_unpool, and
soft_slic's loop and argmax; and a seeded generator of feature maps for the tests.

Every float operation below is one numpy float32 operation, which rounds like the device's separately rounded
intrinsics.  expf is glibc's, through the library's host compile of the device clone (fslic_b200_debug_expf_host), one
call per run of nearby bit patterns.  Block sums use pool's lane order: a cell's block pixels in raster order are dealt
to 32 lanes, each summed left to right from +0.0, then the butterfly o = 16, 8, 4, 2, 1 (pool_cases.py).  Padding a lane
with +0.0 changes nothing, because a lane's partial sum starts at +0.0 and so is never -0.0.
"""
import ctypes

import numpy as np

from pool_cases import nan_class_equal, ref_pool_batch  # noqa: F401  (nan_class_equal: for the tests)

F32 = np.float32
SLOTS = 9
_ERR = dict(invalid="ignore", over="ignore", divide="ignore", under="ignore")


def expf(x):
    """glibc's expf of float32 x (any shape), bit for bit."""
    from fast_slic_b200 import _lib
    L = _lib.lib()
    L.fslic_b200_debug_expf_host.argtypes = [ctypes.c_uint32, ctypes.c_longlong, ctypes.c_void_p]
    x = np.ascontiguousarray(x, F32)
    bits, inv = np.unique(x.view(np.uint32).ravel(), return_inverse=True)
    out = np.empty(bits.size, F32)
    # one call per run of patterns less than 64 apart: the values in the gaps are computed and dropped
    cut = np.nonzero(np.diff(bits.astype(np.int64)) >= 64)[0] + 1
    for lo, hi in zip(np.r_[0, cut], np.r_[cut, bits.size]):
        first, n = int(bits[lo]), int(bits[hi - 1]) - int(bits[lo]) + 1
        buf = np.empty(n, F32)
        assert L.fslic_b200_debug_expf_host(first, n, buf.ctypes.data) == 0
        out[lo:hi] = buf[bits[lo:hi].astype(np.int64) - first]
    return out[inv].reshape(x.shape)


def cell_grid(H, W, K):
    """SSN's grid of an int K: nw = int(sqrt(K*W/H)), nh = int(sqrt(K*H/W)) in float64, clamped to [1, W] / [1, H]."""
    nw = min(max(int(np.sqrt(np.float64(K) * W / H)), 1), W)
    nh = min(max(int(np.sqrt(np.float64(K) * H / W)), 1), H)
    return nh, nw


def grid_labels(H, W, nh, nw):
    """int64 [H,W]: the own cell a*nw + b of every pixel."""
    return (np.arange(H) * nh // H)[:, None] * nw + (np.arange(W) * nw // W)[None, :]


def slots(H, W, nh, nw):
    """(k int64 [9,H,W], valid bool [9,H,W]): the cell of every slot, the pixel's own cell where the slot is invalid."""
    a = (np.arange(H) * nh // H)[None, :, None]
    b = (np.arange(W) * nw // W)[None, None, :]
    da = (np.arange(SLOTS) // 3 - 1)[:, None, None]
    db = (np.arange(SLOTS) % 3 - 1)[:, None, None]
    aa, bb = a + da, b + db
    valid = (aa >= 0) & (aa < nh) & (bb >= 0) & (bb < nw)
    own = np.broadcast_to(a * nw + b, (SLOTS, H, W))
    return np.where(valid, aa * nw + bb, own), valid


class Blocks:
    """The cell blocks of a grid, flattened: entry e is pixel pix[e] of the block of cell seg[e], at place pos[e] of
    the block's raster order, which sees the cell through its slot slot[e]."""

    def __init__(self, H, W, nh, nw):
        self.H, self.W, self.nh, self.nw, self.K = H, W, nh, nw, nh * nw
        row0 = -(-np.arange(nh + 1) * H // nh)  # first row of every cell row, and H
        col0 = -(-np.arange(nw + 1) * W // nw)
        ca, cb = np.arange(H) * nh // H, np.arange(W) * nw // W
        seg, pix, slot, pos = [], [], [], []
        for k in range(self.K):
            a, b = divmod(k, nw)
            i = np.arange(row0[max(a - 1, 0)], row0[min(a + 2, nh)])
            j = np.arange(col0[max(b - 1, 0)], col0[min(b + 2, nw)])
            ii, jj = np.repeat(i, j.size), np.tile(j, i.size)
            seg.append(np.full(ii.size, k))
            pix.append(ii * W + jj)
            slot.append((a - ca[ii] + 1) * 3 + (b - cb[jj] + 1))
            pos.append(np.arange(ii.size))
        self.seg, self.pix, self.slot, self.pos = (np.concatenate(x) for x in (seg, pix, slot, pos))
        self.rows = int(self.pos.max()) // 32 + 1

    def sum(self, terms):
        """terms float32 [C, N] (one per entry) -> float32 [C, K]: each cell's sum in pool's lane order."""
        C = terms.shape[0]
        out = np.zeros((C, self.K), F32)
        step = max(1, (1 << 25) // (self.K * self.rows * 32))
        lanes = np.arange(32)
        with np.errstate(**_ERR):
            for c0 in range(0, C, step):
                c1 = min(C, c0 + step)
                A = np.zeros((c1 - c0, self.K, self.rows, 32), F32)
                A[:, self.seg, self.pos // 32, self.pos % 32] = terms[c0:c1]
                v = np.zeros((c1 - c0, self.K, 32), F32)
                for r in range(self.rows):
                    v = v + A[:, :, r, :]
                for o in (16, 8, 4, 2, 1):
                    v = v + v[:, :, lanes ^ o]
                out[c0:c1] = v[:, :, 0]
        return out

    def at(self, x):
        """x [C,9,H,W] or [9,H,W] at every entry's (slot, pixel) -> [C, N] or [N]."""
        flat = x.reshape(x.shape[:-2] + (-1,))
        return flat[..., self.slot, self.pix]


def _slot_sum(terms, valid):
    """sum over the valid slots in n order from +0.0 of terms [9, ...] -> [...]"""
    acc = np.zeros(terms.shape[1:], F32)
    with np.errstate(**_ERR):
        for n in range(SLOTS):
            acc = np.where(valid[n], acc + terms[n], acc)
    return acc


class Image:
    """One image's grid: slots and blocks."""

    def __init__(self, H, W, nh, nw):
        self.H, self.W, self.nh, self.nw, self.K = H, W, nh, nw, nh * nw
        self.k, self.valid = slots(H, W, nh, nw)
        self.blocks = Blocks(H, W, nh, nw)

    def assign(self, f, mu):
        """f [C,H,W], mu [C,K] -> q [9,H,W]."""
        d = np.zeros((SLOTS, self.H, self.W), F32)
        with np.errstate(**_ERR):
            for c in range(f.shape[0]):
                t = f[c][None] - mu[c][self.k]
                d = d + t * t
            m = np.zeros((self.H, self.W), F32)
            seen = np.zeros((self.H, self.W), bool)
            for n in range(SLOTS):
                m = np.where(self.valid[n], np.where(seen, np.fmin(m, d[n]), d[n]), m)
                seen |= self.valid[n]
            e = expf(m[None] - d)
            s = _slot_sum(e, self.valid)
            return np.where(self.valid, e / s[None], F32(0))

    def pool(self, v, q):
        """v [C,H,W], q [9,H,W] -> (M [C,K], Z [K])."""
        w = self.blocks.at(q)
        vf = v.reshape(v.shape[0], -1)[:, self.blocks.pix]
        with np.errstate(**_ERR):
            A = self.blocks.sum(w[None] * vf)
            Z = self.blocks.sum(w[None])[0]
            return np.where(Z != 0, A / Z, F32(0)), Z

    def unpool(self, M, q):
        """M [C,K], q [9,H,W] -> [C,H,W]."""
        with np.errstate(**_ERR):
            return _slot_sum(q[:, None] * np.moveaxis(M[:, self.k], 0, 1), self.valid)

    def slot_dot(self, X, y, add=None):
        """sum_c X[c, k(n)] * y[c] (+ add[k(n)]) on the valid slots, +0.0 on the others -> [9,H,W]."""
        acc = np.zeros((SLOTS, self.H, self.W), F32)
        with np.errstate(**_ERR):
            for c in range(y.shape[0]):
                acc = acc + X[c][self.k] * y[c][None]
            if add is not None:
                acc = acc + add[self.k]
        return np.where(self.valid, acc, F32(0))

    def assign_backward(self, f, mu, q, g):
        """-> (gd [9,H,W], gF [C,H,W], gmu [C,K])."""
        with np.errstate(**_ERR):
            t = _slot_sum(q * g, self.valid)
            gd = np.where(self.valid, q * (t[None] - g), F32(0))
            diff = f[None] - np.moveaxis(mu[:, self.k], 0, 1)                      # [9,C,H,W]
            gf = F32(2) * _slot_sum(gd[:, None] * diff, self.valid)
            fb = f.reshape(f.shape[0], -1)[:, self.blocks.pix] - mu[:, self.blocks.seg]
            gmu = F32(-2) * self.blocks.sum(self.blocks.at(gd)[None] * fb)
        return gd, gf, gmu

    def pool_backward(self, v, q, M, Z, gM):
        """-> (gV [C,H,W], gQ [9,H,W])."""
        nz = Z != 0
        with np.errstate(**_ERR):
            gA = np.where(nz, gM / Z, F32(0))
            acc = np.zeros(self.K, F32)
            for c in range(M.shape[0]):
                acc = np.where(nz, acc + gA[c] * M[c], acc)
            gZ = np.where(nz, -acc, F32(0))
        return self.unpool(gA, q), self.slot_dot(gA, v, gZ)

    def unpool_backward(self, M, q, g):
        """-> (gM [C,K], gQ [9,H,W])."""
        gf = g.reshape(g.shape[0], -1)[:, self.blocks.pix]
        with np.errstate(**_ERR):
            gM = self.blocks.sum(self.blocks.at(q)[None] * gf)
        return gM, self.slot_dot(M, g)

    def argmax(self, q):
        """int64 [H,W]: the cell of the first largest q over the valid slots, a NaN counting as the maximum."""
        best = np.zeros((self.H, self.W), F32)
        cell = self.k[4].copy()
        seen = np.zeros((self.H, self.W), bool)
        for n in range(SLOTS):
            v = q[n]
            with np.errstate(**_ERR):
                take = self.valid[n] & ~(seen & np.isnan(best)) & (~seen | np.isnan(v) | (v > best))
            best = np.where(take, v, best)
            cell = np.where(take, self.k[n], cell)
            seen |= self.valid[n]
        return cell


def ref_soft_slic_image(f, grid, n_iter, with_history=False):
    """One image f [C,H,W] -> (argmax labels int64 [H,W], assoc [9,H,W], centroids [C,K]), and with_history also the
    list of (mu, q, M, Z) of every iteration (mu the centroids it assigned to)."""
    f = np.ascontiguousarray(f, F32)
    C, H, W = f.shape
    nh, nw = grid
    im = Image(H, W, nh, nw)
    mu = ref_pool_batch(f[None], grid_labels(H, W, nh, nw).astype(np.int16)[None], im.K)[1][0]
    hist = []
    for _ in range(n_iter):
        q = im.assign(f, mu)
        M, Z = im.pool(f, q)
        hist.append((mu, q, M, Z))
        mu = M
    out = (im.argmax(q), q, mu)
    return out + (hist,) if with_history else out


def dense_torch(H, W, grid):
    """An independent implementation in torch, for autograd in float64: (assign(F, mu), pool(V, q), unpool(M, q)) over
    [C,H,W] maps, [9, H*W] associations and [C,K] cell maps, by gathering the 9 slots of every pixel."""
    import torch
    nh, nw = grid
    K = nh * nw
    a = torch.arange(H)[:, None] * nh // H
    b = torch.arange(W)[None, :] * nw // W
    ks, oks = [], []
    for da in (-1, 0, 1):
        for db in (-1, 0, 1):
            aa, bb = a + da, b + db
            ok = (aa >= 0) & (aa < nh) & (bb >= 0) & (bb < nw)
            ks.append(torch.where(ok, aa * nw + bb, torch.zeros_like(aa * bb)).expand(H, W))
            oks.append(ok.expand(H, W))
    k, ok = torch.stack(ks).reshape(9, -1), torch.stack(oks).reshape(9, -1)

    def assign(F, mu):
        d = ((F.reshape(F.shape[0], 1, -1) - mu[:, k]) ** 2).sum(0)
        return torch.softmax(torch.where(ok, -d, torch.tensor(-float("inf"), dtype=d.dtype)), 0) * ok

    def pool(V, q):
        q = q * ok  # an invalid slot takes part in no sum, so its gradient is 0
        A = torch.zeros(V.shape[0], K, dtype=V.dtype).index_add(1, k[ok], (q[None] * V.reshape(V.shape[0], 1, -1))[:, ok])
        Z = torch.zeros(K, dtype=V.dtype).index_add(0, k[ok], q[ok])
        return A / Z

    def unpool(M, q):
        q = q * ok
        return (q[None] * M[:, k]).sum(1).reshape(M.shape[0], H, W)

    return assign, pool, unpool


def make_features(seed, B, C, H, W, kind="smooth", scale=1.0):
    """float32 [B,C,H,W]: "smooth" (sinusoids plus noise, times scale), "constant" (every pixel the same: everything
    ties), "nonfinite" (smooth with NaN, +inf and -inf pixels)."""
    rng = np.random.RandomState(seed)
    if kind == "constant":
        return np.full((B, C, H, W), F32(rng.randn()), F32)
    y, x = np.mgrid[0:H, 0:W].astype(F32)
    f = np.empty((B, C, H, W), F32)
    for b in range(B):
        for c in range(C):
            a, bb, ph = rng.rand(3) * F32(0.3) + F32(0.01)
            f[b, c] = (np.sin(x * a + y * bb + ph * 10) + rng.randn(H, W).astype(F32) * F32(0.2)) * F32(scale)
    if kind == "nonfinite":
        n = max(1, f.size // 40)
        flat = f.reshape(-1)
        for v in (np.nan, np.inf, -np.inf):
            flat[rng.randint(0, f.size, n)] = v
    return f
