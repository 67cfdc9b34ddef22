"""Seeded inputs shared by the CPU and GPU parity tests."""
import hashlib

import numpy as np

from oracle.oracle import synthetic_image


def make_image(kind, H, W, seed=1, sigma=12.0):
    if kind == "syn":
        return synthetic_image(H, W, seed, sigma)
    if kind == "flat":
        return np.full((H, W, 3), 77, np.uint8)
    if kind == "noise":
        return np.random.RandomState(seed).randint(0, 256, (H, W, 3)).astype(np.uint8)
    if kind == "blocks":  # piecewise-constant patches: many exact distance ties
        rng = np.random.RandomState(seed)
        small = rng.randint(0, 4, (H // 8 + 1, W // 8 + 1, 3)) * 60
        return np.ascontiguousarray(np.kron(small, np.ones((8, 8, 1)))[:H, :W].astype(np.uint8))
    if kind == "tiled":  # large images without float64 H x W x 3 temporaries: a synthetic tile repeated + a coarse ramp
        base = synthetic_image(540, 960, seed, sigma)
        img = np.tile(base, ((H + 539) // 540, (W + 959) // 960, 1))[:H, :W]
        ramp = ((np.arange(H)[:, None] // 7 + np.arange(W)[None, :] // 5) % 23).astype(np.uint16)
        return np.ascontiguousarray(np.minimum(img + ramp[..., None], 255).astype(np.uint8))
    raise ValueError(kind)


# name, kind, H, W, K, kwargs
PIPELINE_CASES = [
    ("A_640x480_K200", "syn", 480, 640, 200, {}),
    ("odd_97x131_K37_msf.1", "syn", 97, 131, 37, dict(min_size_factor=0.1)),
    ("flat_97x131_K37", "flat", 97, 131, 37, dict(min_size_factor=0.5)),
    ("noise_120x160_K48_msf0", "noise", 120, 160, 48, dict(min_size_factor=0.0)),
    ("noise_120x160_K48_msf.25", "noise", 120, 160, 48, dict(min_size_factor=0.25)),
    ("blocks_200x300_K150_msf0", "blocks", 200, 300, 150, dict(min_size_factor=0.0)),
    ("thin_300x10_K4", "syn", 300, 10, 4, {}),
    ("thin_10x400_K5_it2", "syn", 10, 400, 5, dict(max_iter=2)),
    ("thin_301x17_K6_it1", "syn", 301, 17, 6, dict(max_iter=1)),
    ("one_cluster_64x64", "syn", 64, 64, 1, {}),
    ("rgb_path_150x200_K300", "syn", 150, 200, 300, dict(convert_to_lab=False, min_size_factor=0.0)),
    ("compact37.5_150x200_K30", "syn", 150, 200, 30, dict(compactness=37.5)),
    ("compact1_180x240_K150", "syn", 180, 240, 150, dict(compactness=1.0)),
    ("stride2_it1", "syn", 150, 200, 30, dict(subsample_stride=2, max_iter=1)),
    ("stride1_it3", "syn", 90, 120, 20, dict(subsample_stride=1, max_iter=3)),
    ("stride5_it7", "syn", 150, 200, 60, dict(subsample_stride=5, max_iter=7)),
    ("it0", "syn", 120, 160, 40, dict(max_iter=0)),
    ("bigS_generic_300x400_K2", "syn", 300, 400, 2, {}),
    ("dense_K_64x64_K1500", "noise", 64, 64, 1500, dict(min_size_factor=0.0)),
    ("speckle_240x320_K100_msf0", "syn", 240, 320, 100, dict(min_size_factor=0.0, sigma=40.0)),
]

# shapes and parameters off the beaten path (each verified oracle == compiled reference when added)
EDGE_CASES = [
    ("tiny_5x7_K3", "noise", 5, 7, 3, {}),
    ("row_1x200_K7", "syn", 1, 200, 7, {}),
    ("col_200x1_K7", "syn", 200, 1, 7, {}),
    ("denseK_96x128_K6000", "noise", 96, 128, 6000, dict(min_size_factor=0.0)),
    ("S1_20x20_K300", "noise", 20, 20, 300, dict(min_size_factor=0.0)),
    ("stride255_it3", "syn", 300, 200, 40, dict(subsample_stride=255, max_iter=3)),
    ("compact0.01", "syn", 120, 160, 30, dict(compactness=0.01)),
    ("compact2000", "syn", 120, 160, 30, dict(compactness=2000.0)),
    ("it25", "syn", 100, 140, 25, dict(max_iter=25)),
    ("msf3_everything_absorbed", "noise", 100, 140, 25, dict(min_size_factor=3.0)),
    ("w33", "syn", 70, 33, 9, {}),
    ("w31", "syn", 70, 31, 9, {}),
]

# shapes aimed at the TMA-staged assign kernel (W % 8 == 0): widths that are / are not multiples of the 32- and
# 128-column tiles, heights that leave ragged sub-row groups, small S (single-tile super tiles, list overflow),
# uncovered pixels, warm start is covered separately
TMA_CASES = [
    ("tma_97x136_K37", "syn", 97, 136, 37, dict(min_size_factor=0.1)),
    ("tma_123x200_K60_msf0", "syn", 123, 200, 60, dict(min_size_factor=0.0)),
    ("tma_250x264_K100", "noise", 250, 264, 100, {}),
    ("tma_131x128_K50_flat", "flat", 131, 128, 50, dict(min_size_factor=0.5)),
    ("tma_200x328_blocks_K150", "blocks", 200, 328, 150, dict(min_size_factor=0.0)),
    ("tma_S8_160x160_K400", "syn", 160, 160, 400, dict(min_size_factor=0.0)),
    ("tma_S16_256x256_K256", "noise", 256, 256, 256, dict(min_size_factor=0.0)),
    ("tma_S5_96x104_K350", "syn", 96, 104, 350, dict(min_size_factor=0.0)),
    ("tma_thin_13x520_K6", "syn", 13, 520, 6, {}),
    ("tma_thin_500x8_K5", "syn", 500, 8, 5, {}),
    ("tma_1row_1x256_K9", "syn", 1, 256, 9, {}),
    ("tma_compact40_300x400_K200", "syn", 300, 400, 200, dict(compactness=40.0)),
    ("tma_rgb_222x344_K99", "syn", 222, 344, 99, dict(convert_to_lab=False)),
    ("tma_it1_150x200_K30", "syn", 150, 200, 30, dict(max_iter=1)),
    ("tma_it2_150x200_K30", "syn", 150, 200, 30, dict(max_iter=2, min_size_factor=0.0)),
    ("tma_S60_700x1000_K190", "syn", 700, 1000, 190, dict(min_size_factor=0.0)),
    ("tma_S90_900x1200_K130", "syn", 900, 1200, 130, dict(min_size_factor=0.0)),
]

BIG_CASES = [
    ("B_1280x720_K1600_msf0", "syn", 720, 1280, 1600, dict(min_size_factor=0.0)),
    ("B_1280x720_K1600_msf.1_s40", "syn", 720, 1280, 1600, dict(min_size_factor=0.1, sigma=40.0)),
    ("C_1920x1080_K2000_msf0", "syn", 1080, 1920, 2000, dict(min_size_factor=0.0)),
    ("D_3840x2160_K4000_msf0", "tiled", 2160, 3840, 4000, dict(min_size_factor=0.0)),
    # > 2^24 pixels, a single image: k_ccl_number gets 64 CTAs, so 9 blocks per numbering warp and one trip of its
    # outer chunk loop (the second trip needs 8+ images above 16.7 M px: tests/test_cca_gpu.py)
    ("huge_4100x4200_K3000_msf.1", "tiled", 4100, 4200, 3000, dict(min_size_factor=0.1, sigma=20.0)),
]


def split_kwargs(kw):
    kw = dict(kw)
    sigma = kw.pop("sigma", 12.0)
    args = dict(max_iter=10, compactness=10.0, min_size_factor=0.25, subsample_stride=3, convert_to_lab=True)
    args.update(kw)
    return sigma, args


# ---- what the CPU tests compare the restatement with the compiled reference on ---------------------------------
# Each *_outputs function runs one case on `impl` (oracle.Port or oracle.Ref; `kw` are extra keyword arguments of
# impl.iterate, e.g. the reference's thread count) and returns {name: array}.  tests/golden/make_golden.py stores the
# SHA-256 of every array the compiled reference returns in tests/golden/reference_digests.npz under
# "<group>/<case id>/<name>"; tests/test_cpu.py recomputes them with the restatement.
REF_GRAPH_CASES = [(120, 160, 48, "syn", 0.25), (97, 131, 37, "noise", 0.0), (200, 300, 150, "blocks", 0.0),
                   (64, 64, 1500, "noise", 0.0), (180, 240, 70, "syn", 0.1), (480, 640, 200, "syn", 0.1),
                   (720, 1280, 1600, "syn", 0.0)]
REF_REAL_CASES = [("syn", 120, 160, 48, {}), ("noise", 97, 131, 37, dict(min_size_factor=0.0)),
                  ("syn", 240, 320, 150, dict(compactness=30.0)), ("blocks", 200, 300, 150, {}),
                  ("syn", 150, 200, 30, dict(subsample_stride=2, max_iter=3)), ("flat", 97, 131, 37, {}),
                  ("syn", 180, 240, 70, dict(convert_to_lab=False))]
REF_PREEMPT_CASES = [("syn", 120, 160, 48, 0.05, {}), ("syn", 200, 300, 150, 0.05, {}),
                     ("syn", 240, 320, 200, 0.2, dict(max_iter=15)),
                     ("syn", 181, 257, 90, 0.1, dict(subsample_stride=1, max_iter=6)),
                     ("blocks", 240, 320, 64, 0.5, dict(subsample_stride=2)),
                     ("syn", 300, 400, 300, 0.02, dict(sigma=4.0))]
REF_ARCHS = (("standard", 1), ("x64/avx2", 1), ("x64/avx2", 3))


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest()


def _args(a):
    return (a["max_iter"], a["compactness"], a["min_size_factor"], a["subsample_stride"], a["convert_to_lab"])


def pipeline_outputs(impl, case, seed, warm=False, **kw):
    """initialize + iterate with the stage dumps (Lab quad image, pre-CCA labels); `warm`: a second iterate on the
    clusters the first one left."""
    name, kind, H, W, K, ckw = case
    sigma, a = split_kwargs(ckw)
    img = make_image(kind, H, W, seed=seed, sigma=sigma)
    cl = impl.initialize(img, K)
    init = cl.copy()
    lab, quad, pre = impl.iterate(img, cl, *_args(a), stages=True, **kw)
    out = dict(init=init, quad=quad, pre=pre, labels=lab, clusters=cl.copy())
    if warm:
        lab, quad, pre = impl.iterate(img, cl, *_args(a), stages=True, **kw)
        out.update(quad2=quad, pre2=pre, labels2=lab, clusters2=cl)
    return out


def random_config_case(seed):
    """Seeded random shape / K / parameters (test_oracle_matches_compiled_reference_random_configs)."""
    rng = np.random.RandomState(1000 + seed)
    H, W = int(rng.randint(20, 160)), int(rng.randint(20, 200))
    K = int(rng.randint(1, max(2, H * W // 40)))
    kind = ["syn", "noise", "blocks"][seed % 3]
    args = dict(max_iter=int(rng.randint(0, 13)), compactness=float(rng.choice([0.5, 3.0, 10.0, 40.0])),
                min_size_factor=float(rng.choice([0.0, 0.1, 0.25, 1.0])), subsample_stride=int(rng.randint(1, 6)),
                convert_to_lab=bool(rng.randint(0, 2)))
    sigma = float(rng.choice([5.0, 12.0, 30.0]))
    return ("random%d" % seed, kind, H, W, K, dict(args, sigma=sigma))


def graph_outputs(impl, H, W, K, kind, msf, **kw):
    """Adjacency graph (12-neighbour cap included), mask density and density broadcast of a segmented image."""
    img = make_image(kind, H, W, seed=17)
    cl = impl.initialize(img, K)
    lab = impl.iterate(img, cl, 10, 10.0, msf, 3, True, **kw)

    def flat(conn):  # neighbour lists -> [counts..., neighbours...]
        return np.array([len(n) for n in conn] + [x for n in conn for x in n], np.int64)

    # saturated nodes (more than 12 distinct neighbours).  Labels >= K are left out: the reference reads
    # num_neighbors[source] before its range check (fast-slic.cpp:34-35), out of bounds for the 0xFFFF sentinel
    raw = (make_image("noise", H, W, seed=3)[..., 0].astype(np.uint16) % min(K, 40)).astype(np.uint16)
    mask = make_image("syn", H, W, seed=5)[..., 1]
    dens = impl.get_mask_density(cl, lab, mask)
    big = raw.copy()
    big[::7, ::5] = 0xFFFF
    return dict(labels=lab, clusters=cl, conn=flat(impl.get_connectivity(lab, K)),
                conn_raw=flat(impl.get_connectivity(raw, K)), density=dens, to_mask=impl.density_to_mask(K, lab, dens),
                to_mask_big=impl.density_to_mask(K, big, dens), density_big=impl.get_mask_density(cl, big, mask))


def real_dist_outputs(impl, variant, case):
    kind, H, W, K, ckw = case
    sigma, a = split_kwargs(ckw)
    img = make_image(kind, H, W, seed=31, sigma=sigma)
    cl = impl.initialize(img, K)
    lab, pre = impl.iterate_real(variant, img, cl, *_args(a), stages=True)
    return dict(pre=pre, labels=lab, clusters=cl)


def preemptive_outputs(impl, case, **kw):
    """preemptive=True, cold start then warm start on the records the first call left; `plain` = the same
    call without the option."""
    kind, H, W, K, thres, ckw = case
    sigma, a = split_kwargs(ckw)
    img = make_image(kind, H, W, seed=43, sigma=sigma)
    out = dict(plain=impl.iterate(img, impl.initialize(img, K), *_args(a), **kw))
    cl = impl.initialize(img, K)
    for round_ in range(2):
        lab, _, pre = impl.iterate(img, cl, *_args(a), stages=True, preemptive=True, preemptive_thres=thres, **kw)
        out.update({"pre%d" % round_: pre, "labels%d" % round_: lab, "clusters%d" % round_: cl.copy()})
    return out


# the cases of the GPU suite (tests/test_parity_gpu.py) that compare with the reference's outputs
GPU_REAL_CASES = REF_REAL_CASES + [("syn", 480, 640, 200, dict(min_size_factor=0.1)), ("thin", 10, 400, 5, {})]
GPU_PREEMPT_CASES = [("syn", 120, 160, 48, 0.05, {}), ("syn", 200, 300, 150, 0.05, {}),
                     ("syn", 240, 320, 200, 0.2, dict(max_iter=15)),
                     ("syn", 181, 257, 90, 0.1, dict(subsample_stride=1, max_iter=6)),
                     ("blocks", 240, 320, 64, 0.5, dict(subsample_stride=2)), ("syn", 300, 400, 300, 0.02, {}),
                     ("noise", 120, 160, 48, 0.05, dict(min_size_factor=0.0)),
                     ("syn", 480, 640, 400, 0.05, dict(sigma=4.0)), ("syn", 720, 1280, 1600, 0.05, dict(min_size_factor=0.0))]
GPU_CCA_CASES = [(60, 80, 6, 0, 1), (60, 80, 6, 5, 2), (100, 33, 3, 12, 3), (257, 515, 40, 30, 4), (64, 64, 2, 1, 5),
                 (1, 700, 4, 3, 6), (700, 1, 4, 3, 7), (720, 1280, 1600, 58, 8)]
LDG_FORCED_CASES = [PIPELINE_CASES[0], PIPELINE_CASES[3], TMA_CASES[1], TMA_CASES[5], BIG_CASES[0]]


def gpu_random_config_case(seed):
    """Seeded random shape (widths that are and are not multiples of 8), K, parameters, image kind; returns the case and
    the seed of its image (test_random_configurations)."""
    rng = np.random.RandomState(7000 + seed)
    H = int(rng.randint(24, 420))
    W = int(rng.randint(3, 70)) * 8 if seed % 2 == 0 else int(rng.randint(24, 560))
    K = int(rng.randint(1, max(2, H * W // 60)))
    kind = ["syn", "noise", "blocks", "syn"][seed % 4]
    args = dict(max_iter=int(rng.randint(0, 13)), compactness=float(rng.choice([0.5, 3.0, 10.0, 40.0])),
                min_size_factor=float(rng.choice([0.0, 0.1, 0.25, 1.0])), subsample_stride=int(rng.choice([1, 2, 3, 3, 3, 5])),
                convert_to_lab=bool(rng.randint(0, 2)))
    sigma = float(rng.choice([5.0, 12.0, 30.0]))
    return ("gpu_random%d" % seed, kind, H, W, K, dict(args, sigma=sigma)), 900 + seed


# ---- seeded sweeps of the float-distance, preemptive, Euclidean and LSC contexts --------------------------------------
# Wider than gpu_random_config_case: shapes from one row or column up to about 420 x 560 (widths that are and are not
# multiples of 8), K from 1 up to one cluster per pixel, parameters at the ends of their ranges, flat images.  Every
# sixth seed takes one regime of K: ordinary, dense (S = 1..3), S > 110, K > 4096, a one-row or one-column image.
SWEEP_KINDS = ("syn", "noise", "blocks", "flat")
SWEEP_COMPACTNESS = (0.01, 0.5, 3.0, 10.0, 40.0, 100.0)
SWEEP_MSF = (0.0, 0.1, 0.25, 1.0, 3.0)
SWEEP_STRIDES = (1, 2, 3, 5, 255)
SWEEP_THRES = (0.01, 0.05, 0.2, 0.5, 1.0)
K_MAX = 65533  # num_components < 65534 (cfast_slic.pyx:24-25)


def sweep_S(H, W, K):
    """The context's S (context.h:60: integer division first, then the square root, truncated)."""
    return int(np.sqrt(float(H * W // K)))


def sweep_turn(seed):
    """What the image kind and the float-distance variant cycle with: the seed plus one per round of six regimes, so
    that every regime meets every kind and variant (seed % 3 or seed % 4 alone would pair them with fixed regimes)."""
    return seed + seed // 6


def sweep_config(rng, seed):
    """(kind, H, W, K, kwargs) of sweep seed `seed`, drawn from `rng`."""
    regime = seed % 6

    def width(lo, hi):
        w = int(rng.randint(lo, hi + 1))
        return max(8, w - w % 8) if rng.randint(2) else w

    if regime == 1:    # dense: S = 1, 1, 2, 2 or 3
        H, W = int(rng.randint(6, 121)), width(6, 160)
        K = max(1, min(K_MAX, H * W // int(rng.choice([1, 2, 4, 6, 9]))))
    elif regime == 2:  # S > 110: k_assign_real / k_assign_lsc windows wider than any tile kernel's
        H, W = int(rng.randint(240, 421)), width(240, 560)
        K = int(rng.randint(1, H * W // (111 * 111) + 1))
    elif regime == 3:  # K > 4096: k_prepare instead of the in-tail prepare
        H, W = int(rng.randint(100, 421)), width(100, 560)
        K = int(rng.randint(4097, min(K_MAX, H * W // 2) + 1))
    elif regime == 4:  # one row or one column
        L = int(rng.randint(2, 561))
        H, W = (1, L) if rng.randint(2) else (L, 1)
        K = int(rng.randint(1, L // 2 + 1))
    else:
        H, W = int(rng.randint(1, 421)), width(1, 560)
        K = int(rng.randint(1, max(2, H * W // 60)))
    kind = SWEEP_KINDS[sweep_turn(seed) % 4]
    args = dict(max_iter=0 if seed % 7 == 3 else int(rng.randint(1, 16)),
                compactness=float(rng.choice(SWEEP_COMPACTNESS)), min_size_factor=float(rng.choice(SWEEP_MSF)),
                subsample_stride=int(rng.choice(SWEEP_STRIDES)), convert_to_lab=bool(rng.randint(0, 2)),
                sigma=float(rng.choice([5.0, 12.0, 30.0])))
    return kind, H, W, K, args


def real_sweep_case(seed, family=0):
    """Float-distance sweep: ((kind, H, W, K, kwargs), variant).  family 0: the Manhattan sweep (variants 0, 1, 2 by
    seed), 1: the Euclidean one (variants 0 and 2; "l2" ignores the flag)."""
    rng = np.random.RandomState(11000 + 1000 * family + seed)
    case = sweep_config(rng, seed)
    return case, (sweep_turn(seed) % 3 if family == 0 else (0, 2)[sweep_turn(seed) % 2])


def preempt_sweep_case(seed, family=0):
    """preemptive=True sweep: (kind, H, W, K, thres, kwargs); family 0 Manhattan, 1 Euclidean."""
    rng = np.random.RandomState(13008 + 1000 * family + seed)  # (a base at which both families reach every region)
    kind, H, W, K, args = sweep_config(rng, seed)
    return kind, H, W, K, float(rng.choice(SWEEP_THRES)), args


def sweep_regions(case):
    """The regions of the parameter space that the hand-picked case lists leave out and case (kind, H, W, K, [thres,]
    kwargs) falls in."""
    kind, H, W, K = case[:4]
    S, a = sweep_S(H, W, K), split_kwargs(case[-1])[1]
    long_run = a["subsample_stride"] == 1 or a["subsample_stride"] >= 5
    return {name for name, hit in (
        ("S <= 2", S <= 2), ("S > 110", S > 110), ("K > 4096", K > 4096), ("one row or column", H == 1 or W == 1),
        ("W % 8 == 0", W % 8 == 0 and W > 1), ("W % 8 != 0", W % 8 != 0), ("stride 1", a["subsample_stride"] == 1),
        ("stride >= 5", a["subsample_stride"] >= 5), ("max_iter 0", a["max_iter"] == 0),
        ("max_iter >= 13", a["max_iter"] >= 13), ("stride 1 or >= 5 with max_iter 0 or >= 13",
                                                 long_run and (a["max_iter"] == 0 or a["max_iter"] >= 13)),
        ("Lab off", not a["convert_to_lab"]), ("Lab on", a["convert_to_lab"]), ("msf >= 1", a["min_size_factor"] >= 1),
        ("compactness 0.01", a["compactness"] == 0.01), ("compactness 100", a["compactness"] == 100.0),
        ("flat image", kind == "flat")) if hit}


SWEEP_REGIONS = ("S <= 2", "S > 110", "K > 4096", "one row or column", "W % 8 == 0", "W % 8 != 0", "stride 1",
                 "stride >= 5", "max_iter 0", "max_iter >= 13", "stride 1 or >= 5 with max_iter 0 or >= 13", "Lab off",
                 "Lab on", "msf >= 1", "compactness 0.01", "compactness 100", "flat image")

REAL_SWEEP_SEEDS = range(24)
PREEMPT_SWEEP_SEEDS = range(16)


def sweep_case_id(case):
    """kind_HxW_K<K> plus the parameters that differ between seeds, for test ids."""
    kind, H, W, K = case[:4]
    a = split_kwargs(case[-1])[1]
    return "%s_%dx%d_K%d_it%d_c%g_m%g_s%d%s" % (kind, H, W, K, a["max_iter"], a["compactness"], a["min_size_factor"],
                                                 a["subsample_stride"], "" if a["convert_to_lab"] else "_rgb")


def real_dist_sweep_outputs(impl, variant, case):
    """real_dist_warm_outputs with the pre-CCA labels of both calls."""
    kind, H, W, K, ckw = case
    sigma, a = split_kwargs(ckw)
    img = make_image(kind, H, W, seed=41, sigma=sigma)
    cl = impl.initialize(img, K)
    out = {}
    for round_ in range(2):
        lab, pre = impl.iterate_real(variant, img, cl, *_args(a), stages=True)
        out.update({"pre%d" % round_: pre, "labels%d" % round_: lab, "clusters%d" % round_: cl.copy()})
    return out


def real_dist_warm_outputs(impl, variant, case):
    """A float-distance class called twice on one image (test_real_dist_variants): labels and clusters per call."""
    kind, H, W, K, ckw = case
    sigma, a = split_kwargs(ckw)
    img = make_image("syn" if kind == "thin" else kind, H, W, seed=41, sigma=sigma)
    cl = impl.initialize(img, K)
    out = {}
    for round_ in range(2):
        out["labels%d" % round_] = impl.iterate_real(variant, img, cl, *_args(a))
        out["clusters%d" % round_] = cl.copy()
    return out


def cca_random_labels(H, W, nlab, seed):
    """The blocky random label maps of test_enforce_connectivity_random."""
    rng = np.random.RandomState(seed)
    small = rng.randint(0, nlab, (H // 3 + 1, W // 3 + 1))
    lab = np.kron(small, np.ones((3, 3), int))[:H, :W]
    noise = rng.rand(H, W) < 0.15
    lab[noise] = rng.randint(0, nlab, noise.sum())
    return np.ascontiguousarray(lab.astype(np.int16))


def cca_range_labels():
    """The label maps of test_enforce_connectivity_label_range_beyond_pixel_count: few labels, large ids."""
    rng = np.random.RandomState(77)
    out = []
    for H, W, top in [(50, 50, 4000), (50, 50, 65000), (50, 50, 37), (9, 13, 30000)]:
        small = rng.randint(0, 12, (H // 4 + 1, W // 4 + 1))
        lab = np.kron(small, np.ones((4, 4), int))[:H, :W]
        ids = np.sort(rng.choice(top, 12, replace=False))
        ids[-1] = top  # the maximum label is `top`
        out.append((np.ascontiguousarray(ids[lab].astype(np.uint16).view(np.int16)), top + 1))
    return out


def cca_outputs(impl, **kw):
    """Connectivity enforcement alone on the maps of the GPU suite."""
    out = {}
    for H, W, nlab, thres, seed in GPU_CCA_CASES:
        lab = cca_random_labels(H, W, nlab, seed).view(np.uint16)
        out["random_%dx%d_t%d_s%d" % (H, W, thres, seed)] = impl.enforce_connectivity(lab, int(lab.max()) + 1, thres, **kw)
    for t, (lab, K) in enumerate(cca_range_labels()):
        out["range%d" % t] = impl.enforce_connectivity(lab.view(np.uint16), K, 3, **kw)
    return out


def gpu_suite_cases():
    """(key prefix, function(impl, **iterate_kw) -> {name: array}) for the GPU suite's comparisons with the reference."""
    cases = []
    for group, seed, lst in (("gpu_pipeline", 7, PIPELINE_CASES), ("tma", 23, TMA_CASES), ("ldg", 29, LDG_FORCED_CASES),
                             ("big", 11, BIG_CASES)):
        for case in lst:
            cases.append(("%s/%s" % (group, case[0]), lambda impl, c=case, s=seed, **kw: pipeline_outputs(impl, c, s, **kw)))
    cases.append(("warm/syn_200x260_K90", lambda impl, **kw: pipeline_outputs(
        impl, ("warm", "syn", 200, 260, 90, {}), 3, warm=True, **kw)))
    for seed in range(16):
        case, img_seed = gpu_random_config_case(seed)
        cases.append(("gpu_random/%d" % seed, lambda impl, c=case, s=img_seed, **kw: pipeline_outputs(impl, c, s, warm=True, **kw)))
    for variant in range(3):
        for case in GPU_REAL_CASES:
            cases.append(("gpu_real%d/%s_%dx%d_K%d" % ((variant,) + case[:4]),
                          lambda impl, v=variant, c=case, **kw: real_dist_warm_outputs(impl, v, c)))
    for case in GPU_PREEMPT_CASES:
        cases.append(("gpu_preempt/%s_%dx%d_K%d_t%g" % case[:5], lambda impl, c=case, **kw: preemptive_outputs(impl, c, **kw)))
    cases.append(("cca/gpu_suite", lambda impl, **kw: cca_outputs(impl, **kw)))
    for seed in REAL_SWEEP_SEEDS:
        case, variant = real_sweep_case(seed)
        cases.append(("gpu_real_sweep/%d" % seed, lambda impl, v=variant, c=case, **kw: real_dist_sweep_outputs(impl, v, c)))
    for seed in PREEMPT_SWEEP_SEEDS:
        cases.append(("gpu_preempt_sweep/%d" % seed,
                      lambda impl, c=preempt_sweep_case(seed), **kw: preemptive_outputs(impl, c, **kw)))
    return cases


def big_init_outputs(impl):
    """initialize_clusters above 2^24 pixels (the reference indexes the image with a float expression there)."""
    img = make_image("tiled", 4100, 4200, seed=11, sigma=20.0)
    return dict(init=impl.initialize(img, 3000))


def reference_outputs(impl, threads=2):
    """Every (key prefix, {name: array}) of reference_digests.npz, computed by the compiled reference `impl`."""
    kw = dict(num_threads=threads)
    for case in PIPELINE_CASES[:12]:
        yield "pipeline/" + case[0], pipeline_outputs(impl, case, 13, **kw)
    for case in EDGE_CASES:
        yield "edge/" + case[0], pipeline_outputs(impl, case, 5, **kw)
    for seed in range(10):
        yield "random/%d" % seed, pipeline_outputs(impl, random_config_case(seed), seed, **kw)
    for H, W, K, kind, msf in REF_GRAPH_CASES:
        yield "graph/%dx%d_K%d_%s_%g" % (H, W, K, kind, msf), graph_outputs(impl, H, W, K, kind, msf, **kw)
    for variant in range(3):
        for case in REF_REAL_CASES:
            yield "real%d/%s_%dx%d_K%d" % ((variant,) + case[:4]), real_dist_outputs(impl, variant, case)
    for arch in ("x64/avx2", "standard"):
        for case in REF_PREEMPT_CASES:
            yield "preemptive_%s/%s_%dx%d_K%d" % ((arch.replace("/", "_"),) + case[:4]), \
                preemptive_outputs(impl, case, arch=arch, **kw)
    img = make_image("syn", 120, 160, seed=3)
    for arch, nt in REF_ARCHS:
        cl = impl.initialize(img, 40)
        lab = impl.iterate(img, cl, 10, 10.0, 0.1, 3, True, arch=arch, num_threads=nt)
        yield "arch/%s_%d" % (arch.replace("/", "_"), nt), dict(labels=lab, clusters=cl)
    yield "init_2p24/tiled_4100x4200_K3000", big_init_outputs(impl)
    for prefix, fn in gpu_suite_cases():
        yield prefix, fn(impl, **kw)
