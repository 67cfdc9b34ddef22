"""Seeded inputs of the LSC (linear spectral clustering) tests, shared by the CPU suite, the GPU suite and
tests/golden/make_lsc_golden.py.

Each case runs one LSC context twice on one image: cold start from initialize_clusters, then warm start on the records
the first call left ("...0" / "...1" outputs)."""
import numpy as np

from cases import make_image, split_kwargs, sweep_case_id, sweep_config

# name, image kind, H, W, K, kwargs (split_kwargs: max_iter, compactness, min_size_factor, subsample_stride,
# convert_to_lab, sigma).  Shapes with W % 8 != 0 are among them; S = (int)sqrt(H W / K).
LSC_CASES = [
    ("syn_120x160_K48", "syn", 120, 160, 48, {}),
    ("noise_97x131_K37_msf0", "noise", 97, 131, 37, dict(min_size_factor=0.0)),
    ("rgb_180x240_K70", "syn", 180, 240, 70, dict(convert_to_lab=False)),
    ("S1_20x20_K300", "syn", 20, 20, 300, {}),  # S = 1, S / 4 = 0: one-pixel centroid windows; empty clusters
    ("S3_60x84_K500", "syn", 60, 84, 500, dict(max_iter=5)),  # S = 3, S / 4 = 0
    ("compact0.01_120x160_K30", "syn", 120, 160, 30, dict(compactness=0.01)),
    ("compact100_150x200_K60", "syn", 150, 200, 60, dict(compactness=100.0)),
    ("blocks_200x300_K150", "blocks", 200, 300, 150, {}),
    ("stride2_it3_150x200_K30", "syn", 150, 200, 30, dict(subsample_stride=2, max_iter=3)),
    ("stride1_it4_90x100_K20", "syn", 90, 100, 20, dict(subsample_stride=1, max_iter=4)),
    ("it0_64x80_K12", "syn", 64, 80, 12, dict(max_iter=0)),
    ("thin_12x403_K8", "syn", 12, 403, 8, dict(compactness=40.0)),
]
# a cluster of these ends a pass without pixels: its centroid features become 0/0 = NaN (lsc.cpp:305)
LSC_NAN_CASES = ("S1_20x20_K300", "S3_60x84_K500")
# GPU suite only (the CPU checker is slow on it; it is the bench's image shape)
LSC_BIG_CASE = ("hd_720x1280_K1600", "syn", 720, 1280, 1600, {})


def lsc_sweep_case(seed):
    """Seeded random LSC case (tests/cases.py::sweep_config) in the form of LSC_CASES."""
    kind, H, W, K, kw = sweep_config(np.random.RandomState(17000 + seed), seed)
    return ("sweep%d_%s" % (seed, sweep_case_id((kind, H, W, K, kw))), kind, H, W, K, kw)


LSC_SWEEP_CASES = [lsc_sweep_case(seed) for seed in range(16)]


def lsc_args(a):
    return (a["max_iter"], a["compactness"], a["min_size_factor"], a["subsample_stride"], a["convert_to_lab"])


def lsc_image(case):
    name, kind, H, W, K, ckw = case
    sigma, a = split_kwargs(ckw)
    return make_image(kind, H, W, seed=61, sigma=sigma), K, a


def lsc_outputs(impl, case, stages=("means", "weights", "cinit", "cfinal"), **kw):
    """{name: array} of one case on a checker of oracle_lsc.lsc (`kw`: extra keyword arguments of its iterate_lsc)."""
    img, K, a = lsc_image(case)
    cl = impl.initialize(img, K)
    out = {"init": cl.copy()}
    for round_ in range(2):
        lab, st = impl.iterate_lsc(img, cl, *lsc_args(a), stages=True, **kw)
        out.update({"labels%d" % round_: lab, "pre%d" % round_: st["pre"], "clusters%d" % round_: cl.copy()})
        out.update({"%s%d" % (s, round_): st[s] for s in stages})
    return out


def lsc_reference_outputs(impl):
    """Every (key prefix, {name: array}) of tests/golden/lsc_reference_digests.npz, computed by the compiled reference
    `impl` (oracle_lsc.lsc.Ref) with num_threads = 1."""
    for case in LSC_CASES + LSC_SWEEP_CASES:
        yield "lsc/" + case[0], lsc_outputs(impl, case, num_threads=1)
