"""Seeded cases of the debug_mode recorder sweep (tests/test_recorder_sweep_*.py,
tests/golden/make_recorder_sweep_golden.py).

The hand-picked recorder cases (tests/recorder_cases.py) keep compactness at 10, S >= 13, K <= 1600 and stride <= 5.
These draw from tests/cases.py::sweep_config instead, one RandomState base per family, with each family's own
conventions:

* "manhattan" / "euclid": Slic with either spatial distance;
* "real": SlicRealDist, SlicRealDistL2 and SlicRealDistNoQ, cycled like real_sweep_case, Euclidean on every other
  group of three seeds;
* "preemptive": Slic(preemptive=True), the threshold drawn from SWEEP_THRES after the configuration as
  preempt_sweep_case does;
* "lsc": LSC(num_threads=1) on lsc_cases' image (seed 61).

The start cycles with the seed: cold, warm (after an untraced iterate with max_iter 2) or the `clusters` setter, with
every even cluster's centre below the image and others up to 40 pixels outside it (recorder_cases.setter_clusters).
The traced Slic cases of default_sweep_cases.LIMIT_CASES follow, with both spatial distances: the largest compactness
the library accepts, which puts u16 min_dists within 2 of FSLIC_BIGSP, and compactness 0.  Last comes one NoQ case
built so that a float centroid's window reaches S + 1 columns past its truncated centre (NOQ_WINDOW_CASE)."""
import collections

import numpy as np

from cases import K_MAX, SWEEP_THRES, make_image, split_kwargs, sweep_case_id, sweep_config, sweep_regions, sweep_S, \
    sweep_turn
from default_sweep_cases import LIMIT_CASES, LIMIT_IMAGE_SEED, _accepts
from recorder_cases import setter_clusters as _setter_clusters

Case = collections.namedtuple("Case", "name family cls kind H W K max_iter stride compactness msf lab manhattan "
                                      "preemptive thres start sigma seed")

FAMILIES = ("manhattan", "euclid", "real", "preemptive", "lsc")
# RandomState base of each family: sweep seed s draws its configuration from RandomState(base + s).  Chosen so that
# every family reaches every region of cases.SWEEP_REGIONS.
BASES = {"manhattan": 30144, "euclid": 31395, "real": 32559, "preemptive": 33230, "lsc": 34034}
SEEDS = range(16)
STARTS = ("cold", "warm", "setter")
REAL_CLASSES = ("SlicRealDist", "SlicRealDistL2", "SlicRealDistNoQ")
# recorder_shim.cpp context of each class (the preemptive family is Slic too)
REF_KIND = {"Slic": "standard", "SlicRealDist": "real_standard", "SlicRealDistL2": "real_l2",
            "SlicRealDistNoQ": "real_noq", "LSC": "lsc"}
# image seed of each family: the seeds of real_dist_sweep_outputs, preemptive_outputs and lsc_image; the Slic
# families take default_sweep_cases' 50 + s
IMAGE_SEED = {"real": 41, "preemptive": 43, "lsc": 61}


def sweep_case(family, seed):
    rng = np.random.RandomState(BASES[family] + seed)
    kind, H, W, K, kw = sweep_config(rng, seed)
    thres = float(rng.choice(SWEEP_THRES)) if family == "preemptive" else 0.05
    sigma, a = split_kwargs(kw)
    cls, manhattan = "Slic", True
    if family == "euclid":
        manhattan = False
    elif family == "real":
        cls, manhattan = REAL_CLASSES[sweep_turn(seed) % 3], (seed // 3) % 2 == 0
    elif family == "preemptive":
        manhattan = seed % 2 == 0
    elif family == "lsc":
        cls = "LSC"
    name = "%s/sweep%d_%s_%s" % (family, seed, sweep_case_id((kind, H, W, K, kw)), STARTS[seed % 3])
    return Case(name, family, cls, kind, H, W, K, a["max_iter"], a["subsample_stride"], a["compactness"],
                a["min_size_factor"], a["convert_to_lab"], manhattan, family == "preemptive", thres, STARTS[seed % 3],
                sigma, IMAGE_SEED.get(family, 50 + seed))


def limit_case(case, manhattan):
    name, kind, H, W, K, kw = case
    sigma, a = split_kwargs(kw)
    family = "manhattan" if manhattan else "euclid"
    return Case("%s/limit/%s" % (family, name), family, "Slic", kind, H, W, K, a["max_iter"], a["subsample_stride"],
                a["compactness"], a["min_size_factor"], a["convert_to_lab"], manhattan, False, 0.05, "cold", sigma,
                LIMIT_IMAGE_SEED)


# SlicRealDistNoQ windows are cut from float centres: rows (int)(cy - S) .. (int)(cy + S + 1) - 1 (context.cpp:471).
# When cy + S rounds up to the next integer, the last column lies S + 1 past the truncated centre the cell grid files
# the cluster under, so the assign and trace kernels look one cell column further.  Here S = G = 64; the 66 setter
# centres sit at row 32, x = 64 t.  Cluster 64 (x = 4096) is the only colour-A one: its pass-0 members (colour A, even
# rows, mean x 4096 - 1/4064) leave cx = 4096 - 2^-12 in float, cx + 64 rounds to 4160 and the window ends at column
# 4160, 65 past cx's column 4095: a search S columns wide from 4160 starts at cell 64 and misses cell 63.  Odd rows
# (pass 1) have colour A in column 4160 only, which cluster 64 wins at distance 0; the colour-B clusters cover the rest.
NOQ_WINDOW_CASE = Case("real/noq_window_edge_64x4224_K66", "real", "SlicRealDistNoQ", "noq_window", 64, 4224, 66, 2, 2,
                       0.0, 0.0, False, True, False, 0.05, "setter", 12.0, 0)


def _noq_window_image(case):
    img = np.zeros((case.H, case.W, 3), np.uint8)
    img[..., 2] = 255                              # colour B
    a = np.zeros((case.H, case.W), bool)
    a[0::2, 4033:4160] = True                      # mean column 4096 ...
    a[0, 4033], a[0, 4032] = False, True           # ... less 1 / 4064
    a[1::2, 4160] = True
    img[a] = (255, 0, 0)                           # colour A
    return img


def setter_clusters(case):
    """The `clusters` setter input of a "setter" case."""
    if case.kind != "noq_window":
        return _setter_clusters(case)
    return [dict(yx=(32, 64 * t), color=(0, 0, 0), num_members=0) for t in range(case.K)]


def setter_records(case, dtype):
    """What SlicModel's `clusters` setter makes of setter_clusters."""
    recs = np.zeros(case.K, dtype)
    for i, d in enumerate(setter_clusters(case)):
        recs[i]["number"] = i
        recs[i]["y"], recs[i]["x"] = d["yx"]
        recs[i]["r"], recs[i]["g"], recs[i]["b"] = d["color"]
        recs[i]["num_members"] = d["num_members"]
        recs[i]["is_active"] = 1
        recs[i]["is_updatable"] = 1
    return recs


SWEEP_CASES = [sweep_case(f, s) for f in FAMILIES for s in SEEDS]
LIMIT_RECORDER_CASES = [limit_case(c, m) for m in (True, False) for c in LIMIT_CASES]
CASES = SWEEP_CASES + LIMIT_RECORDER_CASES + [NOQ_WINDOW_CASE]


def regions(case):
    """cases.sweep_regions of the case's configuration."""
    return sweep_regions((case.kind, case.H, case.W, case.K, dict(
        max_iter=case.max_iter, compactness=case.compactness, min_size_factor=case.msf,
        subsample_stride=case.stride, convert_to_lab=case.lab)))


def accepted(case):
    """A configuration the product takes: 1 <= K <= min(K_MAX, H W), S >= 1, the compactness within check_params'
    u16 range, a stride of 1..255 and max_iter >= 0."""
    S = sweep_S(case.H, case.W, case.K) if case.K <= case.H * case.W else 0
    return (1 <= case.K <= min(K_MAX, case.H * case.W) and S >= 1 and _accepts(S, case.compactness, case.lab)
            and 1 <= case.stride <= 255 and case.max_iter >= 0)


def image(case, seed=None, kind=None):
    if case.kind == "noq_window":
        return _noq_window_image(case)
    return make_image(kind or case.kind, case.H, case.W, seed=case.seed if seed is None else seed, sigma=case.sigma)


def ref_kwargs(case):
    return dict(compactness=case.compactness, min_size_factor=case.msf, stride=case.stride, convert_to_lab=case.lab,
                manhattan=case.manhattan, preemptive=case.preemptive, preemptive_thres=case.thres, num_threads=1)


def reference_report(case, ref, kind=None):
    """The compiled reference's report bytes of `case` (oracle.recorder.RecorderRef); `kind` overrides the context."""
    from oracle.oracle import CLUSTER_DTYPE, Port
    img = image(case)
    cl = setter_records(case, CLUSTER_DTYPE) if case.start == "setter" else Port().initialize(img, case.K)
    kw = ref_kwargs(case)
    kind = kind or REF_KIND[case.cls]
    if case.start == "warm":
        ref.iterate(kind, img, cl, max_iter=2, **kw)
    rep, _ = ref.iterate(kind, img, cl, max_iter=case.max_iter, **kw)
    return rep


def make_slic(case, debug_mode=True):
    """The product-side object of `case`, ready for .iterate(image(case), case.max_iter)."""
    import fast_slic_b200 as fs
    s = getattr(fs, case.cls)(num_components=case.K, compactness=case.compactness, min_size_factor=case.msf,
                              subsample_stride=case.stride, convert_to_lab=case.lab, preemptive=case.preemptive,
                              preemptive_thres=case.thres, manhattan_spatial_dist=case.manhattan,
                              debug_mode=debug_mode, num_threads=1)
    if case.start == "setter":
        s.slic_model.clusters = setter_clusters(case)
    elif case.start == "warm":
        s.slic_model.debug_mode = False
        s.iterate(image(case), 2)
        s.slic_model.debug_mode = debug_mode
    return s
