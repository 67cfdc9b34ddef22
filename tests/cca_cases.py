"""Label maps aimed at the branches of connectivity enforcement (fast_slic_b200/csrc/cca.cuh), and an exact host model of
what the stage's per-image counters must read on them.

Every map is built from a few integers (seeded where random), so nothing is stored but the SHA-256 of what the compiled
reference returns on them (tests/golden/cca_reference_digests.npz, tests/golden/make_cca_golden.py).

The model (`cca_model`) restates the reference's ConnectivityEnforcer (cca.cpp:178-265) the plain way: 4-connected
equal-label components numbered by their minimum raster index, candidates = area >= thres, the K largest candidates, and
what the GPU stage derives from them: the K-th largest area t, G = #(area > t), E = #(area == t), whether the kept set is
ambiguous (need_sim: std::partial_sort's tie order decides it), the number of heap replacements of that replay, which of
k_cca_threshold's three ways of finding t applies, and the total length of the absorb chains k_cca_absorb walks.
"""
import heapq

import numpy as np

HIST_BINS = 2048    # k_cca_threshold's exact histogram covers areas 0..2047; larger ones share one overflow bin
RADIX3_N = 1 << 22  # from this many pixels on the radix select needs its top digit (areas may exceed 2^22)


# ---- map builders --------------------------------------------------------------------------------------------------
def rect_grid(heights, widths, offset=0):
    """Block (i, j) is heights[i] x widths[j] and has label 2*(i%2) + (j%2) + offset: four labels coloured like a
    checkerboard, so no two blocks ever merge and every block's area is exactly heights[i] * widths[j]."""
    hi = np.repeat(np.arange(len(heights)), heights)
    wj = np.repeat(np.arange(len(widths)), widths)
    return np.ascontiguousarray((2 * (hi[:, None] % 2) + (wj[None, :] % 2) + offset).astype(np.uint16))


def random_rect_grid(H, W, hchoices, wchoices, seed, offset=0):
    """rect_grid with row heights / column widths drawn from the choices (the last row / column is cut to fit)."""
    rng = np.random.RandomState(seed)

    def sizes(total, choices):
        s = rng.choice(choices, total)  # (at least one per pixel: enough)
        c = np.cumsum(s)
        n = int(np.searchsorted(c, total)) + 1
        s = s[:n].copy()
        s[-1] -= int(c[n - 1]) - total
        return s

    return rect_grid(sizes(H, hchoices), sizes(W, wchoices), offset)


def spiral(H, W):
    """A 1-px path (label 1) winding inwards from the top-left corner, one pixel of background (label 0) between laps:
    two components that each reach across every 32 x 32 tile."""
    a = np.zeros((H, W), np.uint16)
    y = x = d = 0
    a[0, 0] = 1
    dirs = ((0, 1), (1, 0), (0, -1), (-1, 0))
    turns = 0
    while turns < 2:
        dy, dx = dirs[d]
        ny, nx, fy, fx = y + dy, x + dx, y + 2 * dy, x + 2 * dx
        ok = 0 <= ny < H and 0 <= nx < W and a[ny, nx] == 0 and not (0 <= fy < H and 0 <= fx < W and a[fy, fx] == 1)
        if ok:
            y, x = ny, nx
            a[y, x] = 1
            turns = 0
        else:
            d = (d + 1) % 4
            turns += 1
    return a


def serpentine(H, W):
    """Even rows are a path (label 1) joined at alternating ends through the odd rows; the rest of every odd row is a
    separate background run (label 0)."""
    a = np.zeros((H, W), np.uint16)
    a[0::2] = 1
    for y in range(1, H, 2):
        a[y, W - 1 if (y // 2) % 2 == 0 else 0] = 1
    return a


def comb(H, W):
    """Teeth (label 1) in the even columns, joined only along the bottom row; every odd column is its own component."""
    a = np.zeros((H, W), np.uint16)
    a[:, 0::2] = 1
    a[H - 1] = 1
    return a


def checkerboard(H, W):
    """Every pixel its own component: ncomp = N."""
    return np.ascontiguousarray(((np.arange(H)[:, None] + np.arange(W)[None, :]) % 2).astype(np.uint16))


def stripes(H, W, wide_every, wide_width):
    """1-px vertical stripes of alternating labels; every `wide_every`-th stripe is `wide_width` px wide instead.  With
    a threshold between H and H * wide_width the narrow ones are absorbed, each through the chain of narrow stripes to
    its left (their leaders sit in row 0)."""
    widths = [wide_width if i % wide_every == 0 else 1 for i in range(W)]
    c = np.cumsum(widths)
    widths = widths[:int(np.searchsorted(c, W)) + 1]
    widths[-1] -= int(np.sum(widths)) - W
    lab = np.repeat(np.arange(len(widths)) % 2, widths)
    return np.ascontiguousarray(np.broadcast_to(lab[None, :], (H, W)).astype(np.uint16))


def staircase(H, W, step):
    """Two-row bands that drop one row every `step` columns: band k >= 0 has its leader at (2k, 0) in column 0, so an
    absorbed band takes the label of the band above it."""
    y = np.arange(H)[:, None]
    xb = np.arange(W)[None, :] // step
    return np.ascontiguousarray((((y - xb) // 2) % 2).astype(np.uint16))


def blocky(H, W, nlab, seed, cell=3, speckle=0.15):
    """Random labels on cell x cell blocks plus speckle (tests/cases.py::cca_random_labels, any cell size)."""
    rng = np.random.RandomState(seed)
    small = rng.randint(0, nlab, (H // cell + 1, W // cell + 1))
    lab = np.kron(small, np.ones((cell, cell), int))[:H, :W]
    noise = rng.rand(H, W) < speckle
    lab[noise] = rng.randint(0, nlab, int(noise.sum()))
    return np.ascontiguousarray(lab.astype(np.uint16))


def with_ffff(lab, which):
    """Label `which` replaced by 0xFFFF (-1 as int16), a legal label the reference treats like any other."""
    out = lab.copy()
    out[lab == which] = 0xFFFF
    return out


def bands(H, W, rows):
    """Horizontal bands of the given row counts, alternating labels 0 / 1 (the last one takes the remaining rows)."""
    r = list(rows) + [H - sum(rows)]
    return np.ascontiguousarray(np.broadcast_to((np.repeat(np.arange(len(r)) % 2, r))[:, None], (H, W)).astype(np.uint16))


# ---- the host model ------------------------------------------------------------------------------------------------
def components(lab):
    """(comp[H*W], leader[ncomp], area[ncomp]): 4-connected equal-label components numbered in the order of their
    minimum raster index (the reference's component numbers, cca.cpp:118-134)."""
    H, W = lab.shape
    N = H * W
    flat = lab.ravel()
    values = np.unique(flat)
    if len(values) <= 8:  # few labels: one scipy.ndimage.label pass per label
        from scipy import ndimage
        ids = np.zeros(N, np.int64)
        base = 0
        for v in values:
            cc, n = ndimage.label(lab == v)
            m = cc.ravel() > 0
            ids[m] = cc.ravel()[m] - 1 + base
            base += n
    else:
        from scipy.sparse import coo_matrix
        from scipy.sparse.csgraph import connected_components
        idx = np.arange(N).reshape(H, W)
        eh = lab[:, 1:] == lab[:, :-1]
        ev = lab[1:, :] == lab[:-1, :]
        r = np.concatenate([idx[:, :-1][eh], idx[:-1, :][ev]])
        c = np.concatenate([idx[:, 1:][eh], idx[1:, :][ev]])
        g = coo_matrix((np.ones(len(r), np.int8), (r, c)), shape=(N, N))
        _, ids = connected_components(g, directed=False)
    _, first = np.unique(ids, return_index=True)  # first raster index of every id (ids are 0..n-1)
    order = np.argsort(first, kind="stable")
    rank = np.empty(len(order), np.int64)
    rank[order] = np.arange(len(order))
    comp = rank[ids]
    leader = first[order]
    area = np.bincount(comp, minlength=len(order))
    return comp, leader, area


def heap_replacements(cand_areas, K):
    """Heap replacements of std::partial_sort's __heap_select over the candidates in component order: the first K fill
    a min-heap, every later candidate larger than its top replaces it.  Which element sits on top among equal areas does
    not change the count, so heapq gives it without libstdc++'s tie order."""
    h = [int(a) for a in cand_areas[:K]]
    heapq.heapify(h)
    ops = 0
    for a in cand_areas[K:]:
        a = int(a)
        if a > h[0]:
            heapq.heapreplace(h, a)
            ops += 1
    return ops


def cca_model(lab, K, thres, port=None):
    """What connectivity enforcement of `lab` with (K, thres) must produce.  Returns a dict:
      ncomp, ncand, nkept, sel_mode, keep_thres, need_sim, heap_ops, kth_area  -- Engine.cca_counters() of the image
      t, G, E, n_big, branch ("all": ncand <= K; "hist": t from the 2048-bin histogram; "radix2" / "radix3": two- or
                                 three-pass radix select)
      hops     total absorb-chain length k_cca_absorb walks (every unkept component follows its chain to the end)
      labels   the output map, or None where the kept set depends on std::partial_sort's tie order and no `port` (an
               oracle.Port, whose std::partial_sort is libstdc++'s own) was given to resolve it."""
    lab = np.ascontiguousarray(lab).view(np.uint16)
    H, W = lab.shape
    N = H * W
    comp, leader, area = components(lab)
    ncomp = len(area)
    cands = np.nonzero(area >= thres)[0]
    ncand = len(cands)
    ca = area[cands]
    m = dict(ncomp=ncomp, ncand=ncand, t=0, G=0, E=0, n_big=int((ca >= HIST_BINS).sum()), heap_ops=0, kth_area=0,
             sel_mode=0, need_sim=0)
    kept = None
    if ncand <= K:
        m.update(branch="all", nkept=ncand, keep_thres=int(thres))
        kept = cands
    else:
        t = int(np.sort(ca)[::-1][K - 1])
        G, E = int((ca > t).sum()), int((ca == t).sum())
        m.update(t=t, G=G, E=E, kth_area=t, nkept=K)
        m["branch"] = "hist" if m["n_big"] < K else ("radix2" if N < RADIX3_N else "radix3")
        if E == K - G:
            m.update(keep_thres=t)
            kept = cands[ca >= t]
        else:
            m.update(need_sim=1, sel_mode=1, keep_thres=0, heap_ops=heap_replacements(ca, K))
            if port is not None:
                kept = np.sort(cands[port.stl_partial_sort(ca.astype(np.int32), K)])
    m["hops"] = None
    m["labels"] = None
    if kept is not None:
        # substitute[] of cca.cpp:229-255 by pointer doubling: an unkept component's neighbour component (left of its
        # leader, or above it for a leader in column 0) is always a smaller number, so every chain ends at a kept
        # component or at component 0 (which takes label 0 when unkept)
        is_kept = np.zeros(ncomp, bool)
        is_kept[kept] = True
        nbr = np.where(leader % W > 0, leader - 1, leader - W)
        walk = ~is_kept
        walk[0] = False
        nxt = np.arange(ncomp)
        nxt[walk] = comp[nbr[walk]]
        depth = walk.astype(np.int64)
        while True:
            nn = nxt[nxt]
            if (nn == nxt).all():
                break
            depth = depth + np.where(nxt != np.arange(ncomp), depth[nxt], 0)
            nxt = nn
        subst = np.zeros(ncomp, np.int64)
        subst[kept] = np.arange(len(kept))
        m["hops"] = int(depth.sum())
        m["labels"] = subst[nxt][comp].astype(np.uint16).reshape(H, W)
    return m


def k_for(area, thres, need_sim, at):
    """A K, below the number of candidates (components with area >= thres), whose K-th largest candidate area is `at`:
    with need_sim the K-th is one of several tied components that are not all kept (the choice among them is
    std::partial_sort's), otherwise exactly the components with area >= at are kept."""
    ca = area[area >= thres]
    G = int((ca > at).sum())
    E = int((ca == at).sum())
    K = G + E - 1 if need_sim else G + E
    assert E >= (2 if need_sim else 1) and 1 <= K < len(ca), "no such K at area %d" % at
    return K


# ---- the maps pinned to the compiled reference (tests/test_cca_cpu.py) ----------------------------------------------
# (name, builder, K, thres); K = None: max label + 1 (what the public enforce_connectivity passes)
def _grid2047():
    # rows 23 / 32 / 3 x columns 89 / 64 / 683: areas 2047 = 23*89, 2048 = 32*64, 2049 = 3*683 among others
    return rect_grid([23, 32, 3] * 6, [89, 64, 683] * 3)


def _ties_small(seed):
    # areas 1..6 in random component order: a tie-heavy heap replay with many replacements
    return random_rect_grid(600, 800, [1, 2], [1, 2, 3], seed)


def _radix2():
    # large blocks of four areas, 2400 / 2440 / 2460 / 2501, many of each: n_big >= K below 2^22 px
    return random_rect_grid(1500, 1600, [40, 41], [60, 61], 5)


def reference_map_cases():
    """The maps of the CPU digest test, each up to ~4 M px: [(name, label map u16, K, thres)]."""
    g = _grid2047()
    ga = components(g)[2]
    r2 = _radix2()
    r2a = components(r2)[2]
    out = [
        ("grid2047_hist_unamb", g, k_for(ga, 0, False, at=2047), 0),
        ("grid2047_hist_sim", g, k_for(ga, 0, True, at=2047), 0),
        ("grid2047_thres_t_sim", g, k_for(ga, 2047, True, at=2047), 2047),
        ("grid2047_K1", g, 1, 0),
        ("grid2047_K2", g, 2, 1),
        ("grid2047_thres_gt_N", g, 5, g.size + 1),
        ("radix2_unamb", r2, k_for(r2a, 0, False, at=2440), 0),
        ("radix2_sim", r2, k_for(r2a, 0, True, at=2460), 0),
        ("spiral_512", spiral(512, 512), 2, 1),
        ("serpentine_300x1000", serpentine(300, 1000), 20, 900),
        ("comb_256x512", comb(256, 512), 40, 200),
        ("checker_512_K65535", checkerboard(512, 512), 65535, 0),
        ("stripes_200x700", stripes(200, 700, 37, 4), 65535, 201),
        ("stairs_512x300_K5", staircase(512, 300, 7), 5, 0),
        ("stairs_512x300_absorb", staircase(512, 300, 7), 65535, 700),
        ("ffff_blocky_97x131", with_ffff(blocky(97, 131, 5, 21), 3), None, 4),
        ("ffff_grid2047", with_ffff(g, 2), 40, 10),
    ]
    for H, W in [(1, 1023), (1, 1024), (1, 1025), (33, 31), (32, 32), (31, 33), (70, 33), (70, 31), (64, 32)]:
        out.append(("blocky_%dx%d" % (H, W), blocky(H, W, 3, H * 7 + W, cell=2), None, 3))
    return out


# what each map of reference_map_cases is there for: (k_cca_threshold branch, need_sim), from the model
INTENDED = {
    "grid2047_hist_unamb": ("hist", 0), "grid2047_hist_sim": ("hist", 1), "grid2047_thres_t_sim": ("hist", 1),
    "grid2047_K1": ("radix2", 1), "grid2047_K2": ("radix2", 1), "grid2047_thres_gt_N": ("all", 0),
    "radix2_unamb": ("radix2", 0), "radix2_sim": ("radix2", 1), "spiral_512": ("all", 0),
    "serpentine_300x1000": ("hist", 1), "comb_256x512": ("hist", 1), "checker_512_K65535": ("hist", 1),
    "stripes_200x700": ("all", 0), "stairs_512x300_K5": ("hist", 1), "stairs_512x300_absorb": ("all", 0),
    "ffff_blocky_97x131": ("hist", 0), "ffff_grid2047": ("radix2", 1), "blocky_1x1023": ("hist", 1),
    "blocky_1x1024": ("hist", 0), "blocky_1x1025": ("hist", 0), "blocky_33x31": ("hist", 0), "blocky_32x32": ("hist", 0),
    "blocky_31x33": ("hist", 0), "blocky_70x33": ("hist", 0), "blocky_70x31": ("hist", 0), "blocky_64x32": ("hist", 1),
}


def default_k(lab):
    """K of the public enforce_connectivity: max label + 1 over labels != 0xFFFF (cfast_slic.pyx:377-382)."""
    lab = lab.view(np.uint16)
    v = lab[lab != 0xFFFF]
    return (int(v.max()) if v.size else 0) + 1


def cca_reference_outputs(impl, **kw):
    """(key prefix, {name: array}) of every map of reference_map_cases, enforced by `impl` (oracle.Port or oracle.Ref)."""
    for name, lab, K, thres in reference_map_cases():
        K = default_k(lab) if K is None else K
        yield "cca_maps/" + name, dict(labels=impl.enforce_connectivity(lab, K, thres, **kw))
