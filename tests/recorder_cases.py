"""Cases of the debug_mode recorder tests (tests/test_recorder_*.py, tests/golden/make_recorder_golden.py).

Each case is one SlicModel.iterate with debug_mode=True, optionally after a warm-up call (debug off) or with cluster
records set through the `clusters` setter.  `ref_kind` names the reference context (oracle/recorder_shim.cpp) and
`kernel` the assign kernel family the device takes on the update passes (Engine.DISPATCH_KERNELS).
"""
import collections

import numpy as np

Case = collections.namedtuple("Case", "name cls H W K max_iter stride compactness lab manhattan preemptive thres start kernel seed")

_D = dict(stride=3, compactness=10.0, lab=True, manhattan=True, preemptive=False, thres=0.05, start="cold", seed=7)


def _c(name, cls, H, W, K, max_iter, kernel, **kw):
    d = dict(_D)
    d.update(kw)
    return Case(name, cls, H, W, K, max_iter, d["stride"], d["compactness"], d["lab"], d["manhattan"], d["preemptive"],
                d["thres"], d["start"], kernel, d["seed"])


CASES = [
    _c("tma_10", "Slic", 96, 128, 48, 10, "tma"),
    _c("ldg_2", "Slic", 90, 122, 40, 2, "ldg"),
    _c("generic_2", "Slic", 60, 500, 2, 2, "generic", stride=2),
    _c("iter0", "Slic", 64, 80, 30, 0, None),
    _c("iter1_stride1", "Slic", 64, 80, 30, 1, None, stride=1),
    _c("warm_stride2", "Slic", 64, 80, 30, 10, None, stride=2, start="warm"),
    _c("euclid_stride5", "Slic", 72, 96, 36, 4, None, stride=5, manhattan=False),
    _c("rgb", "Slic", 64, 64, 20, 3, None, lab=False),
    _c("thin_uncovered", "Slic", 8, 300, 3, 5, None, stride=2),
    _c("setter_out_of_range", "Slic", 48, 64, 6, 2, None, start="setter"),
    _c("preempt_freeze", "Slic", 96, 128, 48, 10, "preemptive", preemptive=True, thres=0.5),
    _c("preempt_euclid", "Slic", 64, 96, 24, 3, "preemptive", stride=2, preemptive=True, manhattan=False),
    _c("real_standard", "SlicRealDist", 64, 80, 30, 3, "real_standard"),
    _c("real_l2", "SlicRealDistL2", 64, 80, 30, 2, "real_l2", stride=2),
    _c("real_noq_warm", "SlicRealDistNoQ", 64, 80, 30, 4, "real_noq", start="warm"),
    _c("real_euclid", "SlicRealDist", 48, 72, 20, 2, "real_standard", manhattan=False),
    _c("noq_euclid", "SlicRealDistNoQ", 48, 72, 20, 3, "real_noq", manhattan=False),
    _c("avx2_class", "SlicAvx2", 90, 122, 40, 3, "ldg"),
    _c("lsc_3", "LSC", 64, 80, 30, 3, "lsc"),
    _c("lsc_stride2_warm", "LSC", 72, 96, 36, 5, "lsc", stride=2, start="warm"),
    _c("lsc_rgb_iter1", "LSC", 48, 64, 12, 1, "lsc", lab=False),
    _c("lsc_emptied_cluster", "LSC", 48, 64, 8, 3, "lsc", start="setter_dup"),
    _c("hd_720p", "Slic", 720, 1280, 1600, 2, "tma"),
]

# recorder_shim.cpp context of each class; Slic's "x64/avx2" report is byte-identical to "standard" on every Slic case
# (checked by make_recorder_golden.py), so one device path serves both classes.
REF_KIND = {"Slic": "standard", "SlicAvx2": "x64/avx2", "SlicRealDist": "real_standard", "SlicRealDistL2": "real_l2",
            "SlicRealDistNoQ": "real_noq", "LSC": "lsc"}


def image(case):
    from oracle.oracle import synthetic_image
    return synthetic_image(case.H, case.W, seed=case.seed)


def setter_clusters(case):
    """The `clusters` setter input of a "setter" case: centres partly outside the image.  A "setter_dup" case puts every
    odd cluster on the centre of the one before it: it loses every tie to it and ends up without members."""
    rng = np.random.RandomState(case.seed)
    out = []
    if case.start == "setter_dup":
        for k in range(case.K):
            yx = (int(rng.randint(0, case.H)), int(rng.randint(0, case.W))) if k % 2 == 0 else out[-1]["yx"]
            out.append(dict(yx=yx, color=(0, 0, 0), num_members=0))
        return out
    for k in range(case.K):
        y = int(rng.randint(0, case.H + 40)) if k % 2 else case.H + 7
        x = int(rng.randint(0, case.W + 40))
        out.append(dict(yx=(y, x), color=tuple(int(v) for v in rng.randint(0, 256, 3)), num_members=k))
    return out


def setter_records(case, dtype):
    """What SlicModel's `clusters` setter makes of setter_clusters (base_slic.py / cfast_slic.pyx:68-98)."""
    recs = np.zeros(case.K, dtype)
    for i, d in enumerate(setter_clusters(case)):
        recs[i]["number"] = i
        recs[i]["y"], recs[i]["x"] = d["yx"]
        recs[i]["r"], recs[i]["g"], recs[i]["b"] = d["color"]
        recs[i]["num_members"] = d["num_members"]
        recs[i]["is_active"] = 1
        recs[i]["is_updatable"] = 1
    return recs


def reference_report(case, ref, kind=None):
    """The compiled reference's report bytes of `case` (oracle.recorder.RecorderRef)."""
    from oracle.oracle import Port
    img = image(case)
    if case.start in ("setter", "setter_dup"):
        from oracle.oracle import CLUSTER_DTYPE
        cl = setter_records(case, CLUSTER_DTYPE)
    else:
        cl = Port().initialize(img, case.K)
    kw = dict(compactness=case.compactness, min_size_factor=0.25, stride=case.stride, convert_to_lab=case.lab,
              manhattan=case.manhattan, preemptive=case.preemptive, preemptive_thres=case.thres, num_threads=1)
    kind = kind or REF_KIND[case.cls]
    if case.start == "warm":
        ref.iterate(kind, img, cl, max_iter=2, **kw)
    rep, _ = ref.iterate(kind, img, cl, max_iter=case.max_iter, **kw)
    return rep


def make_slic(case, debug_mode=True):
    """The product-side object of `case`, ready for .iterate(image(case), case.max_iter)."""
    import fast_slic_b200 as fs
    import fast_slic_b200.avx2 as fs_avx2
    cls = getattr(fs_avx2 if case.cls == "SlicAvx2" else fs, case.cls)
    s = cls(num_components=case.K, compactness=case.compactness, subsample_stride=case.stride, convert_to_lab=case.lab,
            preemptive=case.preemptive, preemptive_thres=case.thres, manhattan_spatial_dist=case.manhattan,
            debug_mode=debug_mode, num_threads=1)
    if case.start in ("setter", "setter_dup"):
        s.slic_model.clusters = setter_clusters(case)
    elif case.start == "warm":
        s.slic_model.debug_mode = False
        s.iterate(image(case), 2)
        s.slic_model.debug_mode = debug_mode
    return s


def first_difference(got, want):
    """Where two reports first differ, for assertion messages."""
    import json
    try:
        g, w = json.loads(got), json.loads(want)
    except ValueError:  # e.g. "nan" in an LSC report: name the first differing byte instead
        i = next((i for i, (a, b) in enumerate(zip(got, want)) if a != b), min(len(got), len(want)))
        return "byte %d: %r vs %r" % (i, got[max(0, i - 40):i + 40], want[max(0, i - 40):i + 40])
    for key in ("height", "width"):
        if g[key] != w[key]:
            return "%s: %r vs %r" % (key, g[key], w[key])
    if len(g["snapshots"]) != len(w["snapshots"]):
        return "%d snapshots vs %d" % (len(g["snapshots"]), len(w["snapshots"]))
    for gs, ws in zip(g["snapshots"], w["snapshots"]):
        for field in ("iteration", "clusters", "assignment", "min_dists"):
            if gs[field] != ws[field]:
                where = ""
                if isinstance(gs[field], list):
                    i = next(i for i, (a, b) in enumerate(zip(gs[field], ws[field])) if a != b)
                    where = " [%d]: %r vs %r" % (i, gs[field][i], ws[field][i])
                return "snapshot of iteration %d, field %s%s" % (ws["iteration"], field, where)
    return "same JSON values, different text"
