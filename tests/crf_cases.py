"""Seeded cases of the SimpleCRF tests, shared by the CPU suite, the GPU suite and tests/golden/make_crf_golden.py.

A case is a script of operations on one CRF (num_classes C, num_nodes N): push frames with clusters, a graph and
unaries, pop, initialize, inference, change params, snapshot.  `run_case(model, case)` plays it on any model with the
oracle_crf surface (oracle_crf.crf.Port / Ref, or the GPU adapter in tests/test_crf_gpu.py) and returns every snapshot
as named arrays: the unaries and q of each live frame and a sample of spatial and temporal pairwise energies.
"""
import numpy as np

from oracle.oracle import CLUSTER_DTYPE

_slic_cache = {}


def slic_frames(N, T, H, W):
    """Clusters and adjacency lists of T consecutive SLIC runs (the restatement of oracle/, warm-started) on seeded
    synthetic frames -- what push_slic_frame feeds the CRF."""
    key = (N, T, H, W)
    if key not in _slic_cache:
        from oracle.oracle import Port, synthetic_image
        port = Port()
        out = []
        cl = None
        for t in range(T):
            img = synthetic_image(H, W, seed=100 + t)
            if cl is None:
                cl = port.initialize(img, N)
            labels = port.iterate(img, cl, 5, 10.0, 0.25, 3, True)
            out.append((cl.copy(), port.get_connectivity(labels, N)))
        _slic_cache[key] = out
    return _slic_cache[key]


def random_clusters(rng, N, members):
    cl = np.zeros(N, CLUSTER_DTYPE)
    cl["y"] = rng.randint(0, 720, N)
    cl["x"] = rng.randint(0, 1280, N)
    for ch in "rgb":
        cl[ch] = rng.randint(0, 256, N)
    cl["number"] = np.arange(N) % 65536
    if members == "mixed":  # 0 (clamped to 1), ordinary counts and >= 2^31 (negative as int: clamped to 1)
        cl["num_members"] = rng.choice([0, 1, 7, 300, 4000, 2 ** 31, 2 ** 32 - 1], N)
    else:
        cl["num_members"] = rng.randint(1, 500, N)
    return cl


def random_graph(rng, N):
    """Self-loops, duplicates, isolated nodes and rows longer than 12."""
    lists = []
    for i in range(N):
        kind = rng.randint(5)
        if kind == 0:
            lists.append([])
        elif kind == 1:
            lists.append([i] + rng.randint(0, N, 3).tolist() + [i])
        elif kind == 2:
            lists.append(rng.randint(0, N, rng.randint(13, 30)).tolist())
        else:
            j = rng.randint(0, N, 4).tolist()
            lists.append(j + j[:2])
    return lists


def to_csr(lists):
    off = np.zeros(len(lists) + 1, np.int32)
    off[1:] = np.cumsum([len(x) for x in lists])
    nbr = np.array([j for x in lists for j in x], np.int32)
    return off, nbr


def unaries(rng, kind, C, N):
    """(setter, argument) of one frame's unaries."""
    if kind == "unbiased":
        return "set_unbiased", None
    if kind.startswith("mask"):
        return "set_mask", (rng.randint(0, C, N).astype(np.int32), float(kind[4:]))
    if kind == "proba":
        p = rng.dirichlet(np.ones(C), N).T.astype(np.float32)
        p[:, rng.rand(N) < 0.1] = 0  # -log 0 = inf unaries: every class of some nodes impossible
        p[0, rng.rand(N) < 0.1] = 0
        return "set_proba", np.ascontiguousarray(p)
    if kind == "raw":  # large negative unaries overflow expf: inf / inf = NaN in q
        u = rng.uniform(-3, 8, (C, N)).astype(np.float32)
        u[rng.rand(C, N) < 0.05] = -200.0
        u[0, 0] = -200.0
        return "set_unary", u
    if kind == "bigraw":  # exp(-unary) of every class of half the nodes sums below the 1e-5 clamp
        u = rng.uniform(0, 3, (C, N)).astype(np.float32)
        u[:, rng.rand(N) < 0.5] += 15.0
        return "set_unary", u
    if kind == "smallraw":
        return "set_unary", rng.uniform(0, 3, (C, N)).astype(np.float32)
    raise ValueError(kind)


# name, C, N, graph ("slic" or "rand"), members ("mixed" or "plain"), unary kinds (cycled over frames), params, script.
# Script ops: "F" push a frame with its data, "P" pop, "I" initialize, "i<k>" inference(k), "S" snapshot,
# "p<name>" apply PARAM_SETS[name], "r" reset_inferred on the last frame.
PARAM_SETS = {
    "smooth": dict(spatial_smooth_w=2.5, spatial_smooth_sxy=7.0),
    "neg": dict(spatial_w=-1.5, temporal_w=-0.75),
    "tiny": dict(spatial_srgb=0.01, temporal_srgb=0.01, spatial_sxy=0.01),  # every expf underflows: the 1e-5 clamp
    "mild": dict(spatial_w=0.5, temporal_w=1.25, spatial_srgb=20.0, spatial_sxy=40.0),
}
CRF_CASES = [
    ("c3_n100_t3_slic", 3, 100, "slic", "plain", ("unbiased", "proba", "mask0.5"), "FFFSIS i1S i3S"),
    ("c21_n1600_t5_slic", 21, 1600, "slic", "plain", ("proba", "mask0.5", "unbiased"), "FFFFFIS i2S"),
    ("c2_n100_t2_rand", 2, 100, "rand", "mixed", ("mask0", "mask1"), "FFSIS i1S i2S"),
    ("c3_n100_t3_smooth", 3, 100, "rand", "mixed", ("smallraw",), "FFF psmooth IS i2S"),
    ("c3_n100_t3_neg", 3, 100, "rand", "plain", ("smallraw", "proba"), "FFF pneg IS i2S"),
    ("c2_n100_t2_tiny", 2, 100, "rand", "plain", ("bigraw",), "FF ptiny IS i2S"),
    ("c1_n3_t2_nan", 1, 3, "rand", "mixed", ("raw",), "FFIS i2S"),
    ("c3_n100_t3_raw_nan", 3, 100, "rand", "mixed", ("raw",), "FFFIS i1S i2S"),
    ("c21_n100_t3_mask1", 21, 100, "rand", "mixed", ("mask1", "proba"), "FFFIS i2S"),
    ("c1_n1_t1", 1, 1, "rand", "plain", ("mask1",), "FIS i1S"),
    ("c2_n1_t5", 2, 1, "rand", "mixed", ("proba", "smallraw"), "FFFFFIS i2S"),
    ("c3_n3_t1_it0", 3, 3, "rand", "plain", ("proba",), "FIS i0S i1S"),
    ("c3_n100_t3_popush", 3, 100, "rand", "mixed", ("proba", "smallraw"), "FFFI i1 P F S r i1S P P F F I i2S"),
    ("c3_n100_t3_params", 3, 100, "slic", "plain", ("proba",), "FFFI i1S pmild i1S psmooth i1S"),
    ("c2_n100_t2_preinit", 2, 100, "rand", "plain", ("smallraw",), "FF i1S i1S IS"),
]
SLIC_SHAPES = {100: (120, 160), 1600: (480, 640)}
GPU_BIG_CASE = ("c21_n20000_t8_big", 21, 20000, "rand", "mixed", ("proba", "smallraw"), "FFFFFFFFI i3S")


def _frame_data(case, k, rng):
    C, N, graph, members, kinds = case[1:6]
    if graph == "slic":
        H, W = SLIC_SHAPES[N]
        cl, lists = slic_frames(N, 5, H, W)[k % 5]
    else:
        cl, lists = random_clusters(rng, N, members), random_graph(rng, N)
    return cl, lists, unaries(rng, kinds[k % len(kinds)], C, N)


def run_case(model, case, energies=True):
    """Plays `case` on `model`; returns {"<snapshot>/<array>": ndarray}."""
    name, C, N, script = case[0], case[1], case[2], case[6]
    rng = np.random.RandomState(sum(map(ord, name)))
    erng = np.random.RandomState(len(name))  # the energy sample: separate, so that energies=False sees the same data
    out = {}
    pushed = 0
    snap = 0
    for op in script.split():
        while op:
            if op[0] == "F":
                t = model.push()
                cl, lists, (setter, arg) = _frame_data(case, pushed, rng)
                pushed += 1
                model.set_clusters(t, cl)
                model.set_connectivity(t, *to_csr(lists))
                getattr(model, setter)(t, *(() if arg is None else (arg if isinstance(arg, tuple) else (arg,))))
                op = op[1:]
            elif op[0] == "P":
                model.pop()
                op = op[1:]
            elif op[0] == "I":
                model.initialize()
                op = op[1:]
            elif op[0] == "r":
                model.reset_inferred(model.last())
                op = op[1:]
            elif op[0] == "S":
                for t in range(model.first(), model.last() + 1):
                    out["s%d/t%d/unary" % (snap, t)] = model.get_unary(t)
                    out["s%d/t%d/q" % (snap, t)] = model.get_inferred(t)
                    if energies:
                        out["s%d/t%d/energy" % (snap, t)] = _energies(model, t, N, erng)
                snap += 1
                op = op[1:]
            elif op[0] == "p":
                model.set_params(**PARAM_SETS[op[1:]])
                op = ""
            elif op[0] == "i":
                model.inference(int(op[1:].rstrip("S")))
                op = "S" if op.endswith("S") else ""
            else:
                raise ValueError(op)
    return out


def _energies(model, t, N, rng):
    pairs = rng.randint(0, N, (8, 2))
    vals = [model.spatial(t, int(i), int(j)) for i, j in pairs]
    vals.append(model.spatial(t, 0, 0))
    for other in (t - 1, t, t + 1):
        if model.first() <= other <= model.last():
            vals += [model.temporal(t, int(i), other) for i in pairs[:, 0]]
    return np.array(vals, np.float32)


def nan_class_equal(a, b):
    """Bit-identical, except that any NaN equals any NaN (x86 and the GPU produce different NaN payloads)."""
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    if not (na == nb).all():
        return False
    return bool((a.view(np.uint32)[~na] == b.view(np.uint32)[~nb]).all())
