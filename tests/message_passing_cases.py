"""The contract of fast_slic_b200.message_passing restated in numpy (DESIGN.md section 4.21), float32-exact and
scalar-ordered: edge_gather, edge_softmax and aggregate with their backward passes; an independent float64 torch
implementation over dense incidence matrices for autograd; and seeded generators of hand-made graphs.

Every float operation below is one numpy float32 operation, which rounds like the device's separately rounded
intrinsics.  Sums over a node's entries (or over the entries that target it) are taken rank by rank: step k adds the
k-th entry of every node, in increasing entry order, so each node's sum is the scalar left-to-right sum from +0.0.  A
masked-out term is added as +0.0, which changes no bit: a sum that starts at +0.0 is never -0.0 (x + y is -0.0 only
when both are), so adding +0.0 leaves it as it is.  expf is glibc's, through soft_slic_cases.expf."""
import numpy as np

from soft_slic_cases import expf  # noqa: F401  (glibc's expf, bit for bit)
from pool_cases import nan_class_equal  # noqa: F401  (for the tests)

F32 = np.float32
_ERR = dict(invalid="ignore", over="ignore", divide="ignore", under="ignore")


def rows_of(indptr, E):
    """int64 [E]: the row of every entry of a CSR offset array."""
    return np.searchsorted(np.asarray(indptr), np.arange(E), side="right") - 1


def _ranks(seg):
    """The entries of seg (in summation order) grouped by their rank inside their segment: a list of index arrays,
    step k holding the k-th entry of every segment that has one."""
    M = seg.size
    if M == 0:
        return []
    order = np.argsort(seg, kind="stable")
    s = seg[order]
    first = np.r_[True, s[1:] != s[:-1]]
    start = np.maximum.accumulate(np.where(first, np.arange(M), 0))
    rank = np.empty(M, np.int64)
    rank[order] = np.arange(M) - start
    by_rank = np.argsort(rank, kind="stable")
    counts = np.bincount(rank)
    return np.split(by_rank, np.cumsum(counts)[:-1])


def seq_sum(seg, terms, nseg):
    """terms [M, C] of entries listed in summation order, seg [M] their segments -> [nseg, C]: each segment's terms
    added left to right from +0.0."""
    out = np.zeros((nseg,) + terms.shape[1:], F32)
    with np.errstate(**_ERR):
        for sel in _ranks(seg):
            out[seg[sel]] = out[seg[sel]] + terms[sel]
    return out


def okey(v):
    """The total order of non-NaN floats with -0.0 < +0.0, as int32."""
    i = np.ascontiguousarray(v, F32).view(np.int32)
    return i ^ ((i >> 31) & 0x7fffffff)


def seq_max(seg, terms, ents, nseg):
    """(best [nseg, C], arg int32 [nseg, C]): per segment and channel the first maximal term (the first NaN wins;
    otherwise the total order of okey, a later entry only when strictly larger) and its entry ents[i]; (+0.0, -1)
    where the segment has no term."""
    C = terms.shape[1]
    best = np.zeros((nseg, C), F32)
    arg = np.full((nseg, C), -1, np.int32)
    for sel in _ranks(seg):
        n, v = seg[sel], terms[sel]
        b, a = best[n], arg[n]
        take = (a < 0) | (~np.isnan(b) & (np.isnan(v) | (okey(v) > okey(b))))
        best[n] = np.where(take, v, b)
        arg[n] = np.where(take, ents[sel][:, None].astype(np.int32), a)
    return best, arg


def lane_sum(terms):
    """terms [M, H, D] -> [M, H]: the sum over D in pool's lane order (term j to lane j mod 32, each lane left to right
    from +0.0, then the butterfly o = 16, 8, 4, 2, 1; lane 0's value)."""
    M, H, D = terms.shape
    R = -(-D // 32)
    A = np.zeros((M, H, R * 32), F32)
    A[:, :, :D] = terms
    A = A.reshape(M, H, R, 32)
    v = np.zeros((M, H, 32), F32)
    lanes = np.arange(32)
    with np.errstate(**_ERR):
        for r in range(R):
            v = v + A[:, :, r]
        for o in (16, 8, 4, 2, 1):
            v = v + v[:, :, lanes ^ o]
    return v[:, :, 0]


class Graph:
    """indptr int64 [N+1] (a CSR offset array) and targets int64 [E]: rows, valid entries and heads."""

    def __init__(self, indptr, targets):
        self.indptr = np.asarray(indptr, np.int64)
        self.t = np.asarray(targets, np.int64)
        self.N, self.E = self.indptr.size - 1, self.t.size
        self.row = rows_of(self.indptr, self.E)
        self.valid = (self.t >= 0) & (self.t < self.N)
        self.ev = np.nonzero(self.valid)[0]  # the valid entries, increasing
        self.deg = np.bincount(self.row[self.ev], minlength=self.N).astype(np.int64)

    # ---- edge_gather
    def gather(self, x, end):
        out = np.zeros((self.E, x.shape[1]), F32)
        src = self.t if end == "target" else self.row
        out[self.ev] = x[src[self.ev]]
        return out

    def gather_backward(self, g, end):
        seg = (self.t if end == "target" else self.row)[self.ev]
        return seq_sum(seg, g[self.ev], self.N)

    # ---- edge_softmax (scores [E,H])
    def softmax(self, s):
        ev, r = self.ev, self.row[self.ev]
        m, _ = seq_max(r, s[ev], ev, self.N)
        out = np.zeros_like(s)
        with np.errstate(**_ERR):
            y = expf(s[ev] - m[r])
            Z = seq_sum(r, y, self.N)
            out[ev] = y / Z[r]
        return out

    def softmax_backward(self, out, g):
        ev, r = self.ev, self.row[self.ev]
        res = np.zeros_like(out)
        with np.errstate(**_ERR):
            dot = seq_sum(r, out[ev] * g[ev], self.N)
            res[ev] = out[ev] * (g[ev] - dot[r])
        return res

    # ---- aggregate (w None or [E,H])
    def _terms(self, x, w, ents, src):
        """terms [M, C]: w[e, h(c)] * x[src, c] (one rounded product), x[src, c] without a weight."""
        v = x[src]
        if w is None:
            return v
        H = w.shape[1]
        with np.errstate(**_ERR):
            return np.repeat(w[ents], x.shape[1] // H, axis=1) * v

    def aggregate(self, x, w, reduce):
        """-> (out [N,C], deg int32 [N], amax int32 [N,C] or None)."""
        ev, r = self.ev, self.row[self.ev]
        terms = self._terms(x, w, ev, self.t[ev])
        amax = None
        if reduce == "max":
            out, amax = seq_max(r, terms, ev, self.N)
        else:
            out = seq_sum(r, terms, self.N)
            if reduce == "mean":
                with np.errstate(**_ERR):
                    out = np.where(self.deg[:, None] > 0, out / self.deg.astype(F32)[:, None], F32(0))
        return out, self.deg.astype(np.int32), amax

    def aggregate_backward(self, x, w, g, reduce, amax=None):
        """-> (grad_x [N,C], grad_w like w or None)."""
        N, C = x.shape
        G = g
        if reduce == "mean":
            with np.errstate(**_ERR):
                G = np.where(self.deg[:, None] > 0, g / self.deg.astype(F32)[:, None], F32(0))
        ev, r, t = self.ev, self.row[self.ev], self.t[self.ev]
        won = np.ones((ev.size, C), bool) if amax is None else amax[r] == ev[:, None]
        tx = np.where(won, self._terms(G, w, ev, r), F32(0))
        gx = seq_sum(t, tx, N)  # increasing e within each target
        gw = None
        if w is not None:
            H = w.shape[1]
            with np.errstate(**_ERR):
                p = np.where(won, G[r] * x[t], F32(0))
            gw = np.zeros_like(w)
            gw[ev] = lane_sum(p.reshape(ev.size, H, C // H))
        return gx, gw


def dense_torch(indptr, targets):
    """An independent float64 implementation over dense matrices, for autograd: (gather(x, end), softmax(s [E,H]),
    aggregate(x, w, reduce)).  P [E,N] selects each valid entry's target, S [N,E] each valid entry's row."""
    import torch
    g = Graph(indptr, targets)
    P = torch.zeros(g.E, g.N, dtype=torch.float64)
    S = torch.zeros(g.N, g.E, dtype=torch.float64)
    ev = torch.from_numpy(g.ev)
    P[ev, torch.from_numpy(g.t[g.ev])] = 1
    S[torch.from_numpy(g.row[g.ev]), ev] = 1
    deg = S.sum(1, keepdim=True)

    def gather(x, end):
        return P @ x if end == "target" else S.t() @ x

    def softmax(s):
        # [H, N, E]: the row's scores, -inf off the row
        a = torch.where(S[None] > 0, s.t()[:, None, :], torch.tensor(-float("inf"), dtype=s.dtype))
        p = torch.softmax(a, 2).nan_to_num(0.0)  # a node without entries has an all -inf row
        return (p * S[None]).sum(1).t()

    def aggregate(x, w, reduce):
        xt = P @ x                                         # [E,C]: x at every entry's target
        if w is not None:
            xt = xt * w.repeat_interleave(x.shape[1] // w.shape[1], 1)
        if reduce == "max":
            a = torch.where(S[:, :, None] > 0, xt[None], torch.tensor(-float("inf"), dtype=x.dtype))
            m = a.max(1).values
            return torch.where(deg > 0, m, torch.zeros_like(m))
        out = S @ xt
        return out / deg.clamp_min(1) if reduce == "mean" else out

    return gather, softmax, aggregate


def make_graph(seed, N, max_deg=8, invalid=0.0, self_loops=0.0, duplicates=0.0, empty=0.1, big=None):
    """(indptr int64 [N+1], targets int64 [E]) of a random CSR graph: rows of 0..max_deg entries (a share `empty` of
    them empty), a share `invalid` of the targets outside [0, N) (negative or >= N), self loops and repeated targets
    in about the given shares, and with big = (node, count) one node with `count` entries."""
    rng = np.random.RandomState(seed)
    deg = rng.randint(1, max_deg + 1, N)
    deg[rng.rand(N) < empty] = 0
    if big is not None:
        deg[big[0]] = big[1]
    indptr = np.r_[0, np.cumsum(deg)].astype(np.int64)
    E = int(indptr[-1])
    row = rows_of(indptr, E)
    t = rng.randint(0, max(N, 1), E).astype(np.int64)
    u = rng.rand(E)
    t = np.where(u < self_loops, row, t)
    dup = (u >= self_loops) & (u < self_loops + duplicates)
    prev = np.r_[0, t[:-1]]
    same_row = np.r_[False, row[1:] == row[:-1]]
    t = np.where(dup & same_row, prev, t)
    bad = rng.rand(E) < invalid
    t = np.where(bad, np.where(rng.rand(E) < 0.5, -1 - rng.randint(0, 5, E), N + rng.randint(0, 5, E)), t)
    return indptr, t


def special_values(rng, shape, share=0.05):
    """float32 randn with a share of NaN, +inf, -inf, -0.0 and +0.0 entries."""
    x = rng.randn(*shape).astype(F32)
    flat = x.reshape(-1)
    n = max(1, int(flat.size * share))
    for v in (np.nan, np.inf, -np.inf, -0.0, 0.0):
        flat[rng.randint(0, flat.size, n)] = v
    return x
