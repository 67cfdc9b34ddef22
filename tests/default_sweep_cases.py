"""Seeded inputs of the default integer path (Slic, and Slic(manhattan_spatial_dist=False): the u16 distance with its
spatial patch), shared by tests/test_default_sweep_cpu.py, tests/test_default_sweep_gpu.py and
tests/golden/make_default_sweep_golden.py.

* the seeded sweep (tests/cases.py::sweep_config) at two bases at which each family reaches every region of
  SWEEP_REGIONS: Manhattan and Euclidean;
* the two ends of the compactness range on shapes from S = 1 to S > 110: the largest compactness the library accepts
  (in-window distances then come within 2 of FSLIC_BIGSP, the out-of-window marker and high half of the assign
  kernels' sort keys) and compactness 0 (every spatial term is 0: distances tie over whole flat patches, so the labels
  rest on the rank tie-break alone)."""
import numpy as np

from cases import K_MAX, pipeline_outputs, sweep_config, sweep_S

DEFAULT_SWEEP_SEEDS = (range(24), range(12))   # per family: 0 Manhattan, 1 Euclidean
FAMILIES = ("manhattan", "euclid")
ARCHS = ("x64/avx2", "standard")
BIGSP = 64770                                  # FSLIC_BIGSP (csrc/common.cuh)
COLOR_MAX = 766                                # 3 * 255 + 1: the colour term stays below it
SWEEP_IMAGE_SEED = 50                          # image seed of sweep seed s: 50 + s
LIMIT_IMAGE_SEED = 61


def default_sweep_case(seed, family=0):
    """("sweep<seed>", kind, H, W, K, kwargs) of sweep seed `seed`; family 0 Manhattan, 1 Euclidean."""
    rng = np.random.RandomState((21000, 22100)[family] + seed)
    kind, H, W, K, kw = sweep_config(rng, seed)
    return ("sweep%d" % seed, kind, H, W, K, kw)


def _accepts(S, compactness, convert_to_lab):
    """check_params (csrc/capi.cu) in float32, same operations in the same order: 1 / (S / c), times 1 << shift,
    times 2S, below FSLIC_BIGSP - 766."""
    f = np.float32
    with np.errstate(divide="ignore"):
        coef = f(1) / (f(S) / f(compactness))
    coef = coef * f(1 << (1 if convert_to_lab else 0))
    return bool(coef * f(2 * S) < f(BIGSP - COLOR_MAX))


def compactness_limit(S, convert_to_lab):
    """The largest float32 compactness the library accepts for a context of this S (bisection over bit patterns:
    non-negative floats are ordered like their bits)."""
    lo, hi = 0, int(np.float32(1e9).view(np.uint32))
    assert _accepts(S, 0.0, convert_to_lab) and not _accepts(S, 1e9, convert_to_lab)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if _accepts(S, np.uint32(mid).view(np.float32), convert_to_lab):
            lo = mid
        else:
            hi = mid
    return float(np.uint32(lo).view(np.float32))


def next_float_up(c):
    return float(np.nextafter(np.float32(c), np.float32(np.inf)))


# name, kind, H, W, K, kwargs of the shapes; S = 1, 2, 3, about 20 and above 110; W % 8 == 0 (TMA assign kernel) and
# != 0 (LDG kernel); S > 110 takes the generic kernel
LIMIT_SHAPES = [
    ("S1_noise_24x40_K900", "noise", 24, 40, 900, dict(min_size_factor=0.0)),
    ("S2_blocks_50x61_K700", "blocks", 50, 61, 700, {}),
    ("S3_syn_63x96_K600", "syn", 63, 96, 600, dict(min_size_factor=0.0)),
    ("S20_syn_200x264_K130", "syn", 200, 264, 130, {}),
    ("S19_flat_180x237_K110", "flat", 180, 237, 110, {}),
    ("S20_blocks_160x200_K80", "blocks", 160, 200, 80, dict(min_size_factor=0.0)),
    ("S125_noise_300x420_K8", "noise", 300, 420, 8, {}),
    ("S128_syn_260x256_K4", "syn", 260, 256, 4, dict(max_iter=3)),
]


def limit_case(shape, convert_to_lab, at_limit):
    name, kind, H, W, K, kw = shape
    c = compactness_limit(sweep_S(H, W, K), convert_to_lab) if at_limit else 0.0
    return ("%s_%s_%s" % (name, "lab" if convert_to_lab else "rgb", "limit" if at_limit else "c0"), kind, H, W, K,
            dict(kw, compactness=c, convert_to_lab=convert_to_lab))


LIMIT_CASES = [limit_case(s, lab, lim) for s in LIMIT_SHAPES for lab in (True, False) for lim in (True, False)]


def all_cases(family):
    """(group, case, image seed) of one family: the sweep, then the limit cases."""
    return [("sweep", default_sweep_case(s, family), SWEEP_IMAGE_SEED + s) for s in DEFAULT_SWEEP_SEEDS[family]] + \
           [("limit", c, LIMIT_IMAGE_SEED) for c in LIMIT_CASES]


def case_key(family, group, case):
    return "%s/%s/%s" % (FAMILIES[family], group, case[0])


def accepted(case):
    """The configurations the product takes: S >= 1, K below the u16 label limit, compactness within the u16 range."""
    _, _, H, W, K, kw = case
    S = sweep_S(H, W, K) if K <= H * W else 0
    c = kw.get("compactness", 10.0)
    return 1 <= K <= min(K_MAX, H * W) and S >= 1 and _accepts(S, c, kw.get("convert_to_lab", True))


def default_sweep_reference_outputs(ref_manhattan, ref_euclid, threads=2):
    """Every (key prefix, {name: array}) of default_sweep_reference_digests.npz: pipeline_outputs(..., warm=True) of
    every case of both families, from the compiled reference in both of its arch contexts (prefix "<arch>/...")."""
    for arch in ARCHS:
        top = arch.replace("/", "_")
        for family, impl in enumerate((ref_manhattan, ref_euclid)):
            for group, case, seed in all_cases(family):
                yield "%s/%s" % (top, case_key(family, group, case)), \
                    pipeline_outputs(impl, case, seed, warm=True, arch=arch, num_threads=threads)
