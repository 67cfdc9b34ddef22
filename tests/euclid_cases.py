"""Seeded inputs of the manhattan_spatial_dist=False tests (Euclidean spatial term), shared by the CPU suite, the GPU
suite and tests/golden/make_euclid_golden.py.  Every case here gives a different result than with the Manhattan term, so
each one exercises the option (tests/test_euclidean_cpu.py checks that).

The *_outputs functions run one case on `impl`: a checker of oracle_euclid.euclid (Euclidean) or of oracle.oracle (the
same case with the Manhattan term, for comparison); `kw` are extra keyword arguments of its iterate call."""
from cases import (EDGE_CASES, PIPELINE_CASES, TMA_CASES, make_image, pipeline_outputs, preempt_sweep_case,
                   real_sweep_case, split_kwargs)

_BY_NAME = {c[0]: c for c in PIPELINE_CASES + EDGE_CASES + TMA_CASES}

# (group, case, image seed).  Groups name the assign path the CUDA side takes: "tma" W % 8 == 0 with stride 3 and
# Lab (k_assign5), "ldg" W % 8 != 0 (k_assign_warp), "pipeline" either (the GPU suite also forces the LDG kernel on
# them), "generic" S > 110, "dense" K so large for the image that warp tiles overflow their candidate list and take
# assign_pixel_generic, "edge" shapes and parameters off the beaten path.
EUCLID_CASES = [("tma", _BY_NAME[n], 23) for n in ("tma_97x136_K37", "tma_250x264_K100", "tma_S8_160x160_K400",
                                                    "tma_S5_96x104_K350", "tma_S60_700x1000_K190")] + \
               [("pipeline", _BY_NAME[n], 7) for n in ("A_640x480_K200", "noise_120x160_K48_msf0")] + \
               [("ldg", _BY_NAME[n], 7) for n in ("odd_97x131_K37_msf.1", "blocks_200x300_K150_msf0", "w33")] + \
               [("generic", _BY_NAME["bigS_generic_300x400_K2"], 7)] + \
               [("dense", _BY_NAME[n], 5) for n in ("dense_K_64x64_K1500", "denseK_96x128_K6000")] + \
               [("edge", _BY_NAME[n], 5) for n in ("S1_20x20_K300", "tiny_5x7_K3", "thin_10x400_K5_it2",
                                                    "thin_301x17_K6_it1", "it0", "stride2_it1",
                                                    "stride5_it7", "stride255_it3", "rgb_path_150x200_K300",
                                                    "compact37.5_150x200_K30", "compact1_180x240_K150")]
# compactness 0.01 on the u16 path: coef * hypot(di, dj) <= 0.04 truncates to 0 just like coef * (|di| + |dj|), so the
# result is the Manhattan one -- kept as a parity case, with that equality as its check
EUCLID_SAME_CASES = [("edge", _BY_NAME["compact0.01"], 5)]
EUCLID_WARM_CASE = ("warm_syn_200x264_K90", "syn", 200, 264, 90, {})

# float-distance contexts: variants 0 ("standard") and 2 ("noq") change with the flag, variant 1 ("l2") ignores it
EUCLID_REAL_CASES = [("syn", 120, 160, 48, {}), ("noise", 97, 131, 37, dict(min_size_factor=0.0)),
                     ("syn", 240, 320, 150, dict(compactness=30.0)), ("blocks", 200, 300, 150, {}),
                     ("syn", 150, 200, 30, dict(subsample_stride=2, max_iter=3)),
                     ("syn", 180, 240, 70, dict(convert_to_lab=False)), ("syn", 12, 400, 8, dict(compactness=40.0)),
                     ("syn", 120, 160, 30, dict(compactness=0.01))]
EUCLID_L2_CASES = EUCLID_REAL_CASES[:3]
EUCLID_PREEMPT_CASES = [("syn", 120, 160, 48, 0.05, {}), ("syn", 240, 320, 200, 0.2, dict(max_iter=15)),
                        ("syn", 181, 257, 90, 0.1, dict(subsample_stride=1, max_iter=6)),
                        ("blocks", 240, 320, 64, 0.5, dict(subsample_stride=2))]
EUCLID_ARCHS = ("x64/avx2", "standard")

# seeded sweeps (tests/cases.py::sweep_config): float-distance variants 0 and 2, and preemptive.  Unlike the lists above
# a sweep case need not change with the flag (flat images, max_iter 0, ...): it is a parity case only.
EUCLID_REAL_SWEEP = [real_sweep_case(seed, family=1) for seed in range(12)]   # ((kind, H, W, K, kw), variant)
EUCLID_PREEMPT_SWEEP = [preempt_sweep_case(seed, family=1) for seed in range(8)]


def real_sweep_id(seed):
    return "real_sweep/%d" % seed


def preempt_sweep_id(seed):
    return "preempt_sweep/%d" % seed


def case_id(group, case):
    return "%s/%s" % (group, case[0])


def real_case_id(variant, case):
    return "real%d/%s_%dx%d_K%d" % ((variant,) + case[:4])


def preempt_case_id(case):
    return "preemptive/%s_%dx%d_K%d_t%g" % case[:5]


def _args(a):
    return (a["max_iter"], a["compactness"], a["min_size_factor"], a["subsample_stride"], a["convert_to_lab"])


def euclid_pipeline_outputs(impl, group, case, seed, **kw):
    return pipeline_outputs(impl, case, seed, warm=group == "warm", **kw)


def euclid_real_outputs(impl, variant, case, **kw):
    """A float-distance context called twice on one image (cold, then warm on the records the first call left)."""
    kind, H, W, K, ckw = case
    sigma, a = split_kwargs(ckw)
    img = make_image(kind, H, W, seed=47, sigma=sigma)
    cl = impl.initialize(img, K)
    out = {}
    for round_ in range(2):
        lab, pre = impl.iterate_real(variant, img, cl, *_args(a), stages=True, **kw)
        out.update({"pre%d" % round_: pre, "labels%d" % round_: lab, "clusters%d" % round_: cl.copy()})
    return out


def euclid_preempt_outputs(impl, case, **kw):
    """preemptive=True, cold start then warm start on the records the first call left."""
    kind, H, W, K, thres, ckw = case
    sigma, a = split_kwargs(ckw)
    img = make_image(kind, H, W, seed=53, sigma=sigma)
    cl = impl.initialize(img, K)
    out = {}
    for round_ in range(2):
        lab, _, pre = impl.iterate(img, cl, *_args(a), stages=True, preemptive=True, preemptive_thres=thres, **kw)
        out.update({"pre%d" % round_: pre, "labels%d" % round_: lab, "clusters%d" % round_: cl.copy()})
    return out


def euclid_reference_outputs(impl, threads=2):
    """Every (key prefix, {name: array}) of tests/golden/euclid_reference_digests.npz, computed by the compiled reference
    `impl` (oracle_euclid.euclid.Ref) for both of its arch contexts (prefix "euclid_<arch>/..."; the float-distance contexts have one arch)."""
    for arch in EUCLID_ARCHS:
        top = "euclid_" + arch.replace("/", "_")
        kw = dict(arch=arch, num_threads=threads)
        for group, case, seed in EUCLID_CASES + EUCLID_SAME_CASES:
            yield "%s/%s" % (top, case_id(group, case)), euclid_pipeline_outputs(impl, group, case, seed, **kw)
        yield "%s/%s" % (top, case_id("warm", EUCLID_WARM_CASE)), \
            euclid_pipeline_outputs(impl, "warm", EUCLID_WARM_CASE, 3, **kw)
        for case in EUCLID_PREEMPT_CASES:
            yield "%s/%s" % (top, preempt_case_id(case)), euclid_preempt_outputs(impl, case, **kw)
        for seed, case in enumerate(EUCLID_PREEMPT_SWEEP):
            yield "%s/%s" % (top, preempt_sweep_id(seed)), euclid_preempt_outputs(impl, case, **kw)
    for variant in (0, 2):
        for case in EUCLID_REAL_CASES:
            yield "euclid/" + real_case_id(variant, case), euclid_real_outputs(impl, variant, case, num_threads=threads)
    for case in EUCLID_L2_CASES:  # the "l2" context ignores the flag: these must equal its Manhattan outputs
        yield "euclid/" + real_case_id(1, case), euclid_real_outputs(impl, 1, case, num_threads=threads)
    for seed, (case, variant) in enumerate(EUCLID_REAL_SWEEP):
        yield "euclid/" + real_sweep_id(seed), euclid_real_outputs(impl, variant, case, num_threads=threads)
