"""debug_mode on the GPU over the seeded recorder sweep (tests/recorder_sweep_cases.py): every family's report against
the compiled reference's bytes (oracle/_ref, where it is built) or its pinned digests
(tests/golden/recorder_sweep_reference_digests.npz), the trace kernel's own check of the assign kernels, the same labels
and clusters as untraced, batched tracing through Engine.set_trace (image b of a batch == the image alone, up to the
K > 4096 prepare kernels and TPS = 4 super tiles), and graph replay around a traced call at K > 4096."""
import ctypes as C
import hashlib
import os

import numpy as np
import pytest
import torch

from cases import SWEEP_KINDS
from default_sweep_cases import compactness_limit
from recorder_cases import first_difference
from recorder_sweep_cases import (CASES, FAMILIES, SEEDS, Case, image, make_slic, reference_report, setter_records,
                                  sweep_case)

pytestmark = pytest.mark.gpu

GOLDEN = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden",
                              "recorder_sweep_reference_digests.npz"))
DIGEST = {n: (s, int(l)) for n, s, l in zip(GOLDEN["names"].tolist(), GOLDEN["sha256"].tolist(),
                                              GOLDEN["length"].tolist())}
REAL_VARIANT = {"SlicRealDist": "standard", "SlicRealDistL2": "l2", "SlicRealDistNoQ": "noq"}

# what the traced calls of this file reached: ("update", kernel name), ("prepare", code), ("fused", count)
REACHED = set()


def _record(eng):
    d = eng.dispatch()
    REACHED.add(("update", eng.DISPATCH_KERNELS[d["update"]["kernel"]]))
    if d["prepare"]:
        REACHED.add(("prepare", d["prepare"]))
    REACHED.add(("fused", d["fused_prepares"]))
    return d


def _mismatches(eng):
    """The trace kernel's count of pixels whose label the assign kernels set differently from its argmin, read
    directly (Engine.trace_snapshots raises on a nonzero count instead of returning it)."""
    bad = C.c_uint32(0xFFFFFFFF)
    with eng.lock:
        eng._L.fslic_b200_trace_snapshots(eng._h, 0, None, None, None, C.byref(bad))
    return int(bad.value)


def _check_report(case, got):
    from oracle.recorder import RecorderRef
    if RecorderRef.available():
        want = reference_report(case, RecorderRef())
        assert got == want, case.name + ": " + first_difference(got, want)
    assert (hashlib.sha256(got).hexdigest(), len(got)) == DIGEST[case.name], \
        case.name + ": report differs from the reference digest"


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_report_matches_reference(case):
    from fast_slic_b200 import get_engine
    s = make_slic(case)
    labels = s.iterate(image(case), case.max_iter)
    eng = get_engine(case.H, case.W, case.K)
    _record(eng)
    assert _mismatches(eng) == 0, case.name + ": the assign kernels disagree with the trace kernel's argmin"
    _check_report(case, s.slic_model.last_recorder_report)
    # the same call untraced: identical labels and cluster records
    off = make_slic(case, debug_mode=False)
    assert (off.iterate(image(case), case.max_iter) == labels).all(), case.name + ": labels differ from untraced"
    assert off.slic_model.cluster_array.tobytes() == s.slic_model.cluster_array.tobytes(), \
        case.name + ": clusters differ from untraced"


# ---- batched tracing through Engine.set_trace -------------------------------------------------------------------------
def _params(case, max_iter):
    from fast_slic_b200 import Engine
    return Engine.params(case.compactness, case.msf, case.stride, case.lab, max_iter)


def _run(eng, case, imgs, cl, max_iter, labels=None):
    """The device entry point of the case's class."""
    p, kw = _params(case, max_iter), dict(manhattan_spatial_dist=case.manhattan)
    if case.preemptive:
        return eng.iterate_preemptive(imgs, cl, p, case.thres, labels, **kw)
    if case.cls == "Slic":
        return eng.iterate(imgs, cl, p, labels, **kw)
    if case.cls == "LSC":
        return eng.iterate_lsc(imgs, cl, p, labels, **kw)
    return eng.iterate_real(REAL_VARIANT[case.cls], imgs, cl, p, labels, **kw)


def _start(eng, case, imgs):
    """Cluster records of every image in the case's start state: seeded, warmed by an untraced call with max_iter 2,
    or the setter's records."""
    from fast_slic_b200 import CLUSTER_DTYPE
    if case.start == "setter":
        recs = setter_records(case, CLUSTER_DTYPE).view(np.uint8).reshape(1, case.K, 32)
        return torch.from_numpy(np.repeat(recs, imgs.shape[0], 0)).to(imgs.device)
    cl = eng.initialize_clusters(imgs)
    if case.start == "warm":
        _run(eng, case, imgs, cl, 2)
    return cl


def _traced(eng, case, imgs):
    """(labels, clusters, dispatch) of one traced call from the case's start; the trace kernel agreed on every pixel."""
    cl = _start(eng, case, imgs)
    eng.set_trace(True)
    try:
        lab = _run(eng, case, imgs, cl, case.max_iter)
    finally:
        eng.set_trace(False)
    d = _record(eng)
    assert _mismatches(eng) == 0, case.name + ": the assign kernels disagree with the trace kernel's argmin"
    return lab, cl, d


def _check_batch(case, imgs, snapshots=False):
    """Image b of a traced batch against the image traced alone: report bytes (or, with `snapshots`, the snapshot
    arrays the report is formatted from), and the untraced batch's labels and clusters.  -> (traced, untraced)
    dispatch of the batch."""
    from fast_slic_b200 import Engine
    B = imgs.shape[0]
    batch, single = Engine(case.H, case.W, case.K, max_batch=B), Engine(case.H, case.W, case.K, max_batch=1)
    try:
        d = torch.from_numpy(imgs).cuda()
        lab, cl, dt = _traced(batch, case, d)
        got = [batch.trace_snapshots(b) if snapshots else batch.recorder_report(b) for b in range(B)]
        cl_off = _start(batch, case, d)
        lab_off = _run(batch, case, d, cl_off, case.max_iter)
        du = batch.dispatch()
        assert torch.equal(lab, lab_off) and torch.equal(cl, cl_off), case.name + ": traced batch differs from untraced"
        for b in range(B):
            one = d[b:b + 1].contiguous()
            _traced(single, case, one)
            if snapshots:
                want = single.trace_snapshots(0)
                for k in ("assignment", "min_dists", "clusters"):
                    assert want[k].tobytes() == got[b][k].tobytes(), "%s: image %d of %d, %s" % (case.name, b, B, k)
            else:
                want = single.recorder_report(0)
                assert got[b] == want, "%s: image %d of %d: %s" % (case.name, b, B, first_difference(got[b], want))
        return dt, du
    finally:
        batch.close()
        single.close()


def _three_kinds(kind):
    return (kind,) + tuple(k for k in SWEEP_KINDS if k != kind)[:2]


BATCH_CASES = [sweep_case(f, s) for f in FAMILIES for s in SEEDS if s % 4 == 0]


@pytest.mark.parametrize("case", BATCH_CASES, ids=[c.name for c in BATCH_CASES])
def test_batch_of_three_equals_singles(case):
    imgs = np.stack([image(case, case.seed + 7 * b, k) for b, k in enumerate(_three_kinds(case.kind))])
    _check_batch(case, imgs)


def _bigk_case(manhattan):
    """K > 4096 (S = 3) at the compactness limit, warm start."""
    return Case("bigK_240x320_K5000_%s" % ("manhattan" if manhattan else "euclid"), "manhattan", "Slic", "syn", 240,
                320, 5000, 5, 3, compactness_limit(3, True), 0.0, True, manhattan, False, 0.05, "warm", 12.0, 400)


@pytest.mark.parametrize("B,prepare,manhattan", [(3, 2, True), (8, 1, False)], ids=["B3_k_prepare2", "B8_k_prepare"])
def test_large_K_batches(B, prepare, manhattan):
    """K > 4096: k_prepare2 below 8 images, k_prepare from 8 up, every pass through run_prepare under trace."""
    case = _bigk_case(manhattan)
    imgs = np.stack([image(case, 400 + b, SWEEP_KINDS[b % 4]) for b in range(B)])
    dt, du = _check_batch(case, imgs)
    assert dt["prepare"] == du["prepare"] == prepare and dt["fused_prepares"] == 0


def test_tps4_batch():
    """Eight 720p images, K = 1600: the untraced call's update passes take super tiles of 4 warp tiles; the traced call
    makes the same launch decisions and each image's snapshots equal the image traced alone.  max_iter 2 keeps the
    snapshot buffer (T B (32 K + N (2 + 2)) bytes) near 90 MB."""
    case = Case("hd_720x1280_K1600_it2", "manhattan", "Slic", "syn", 720, 1280, 1600, 2, 3, 10.0, 0.25, True, True,
                False, 0.05, "cold", 12.0, 500)
    imgs = np.stack([image(case, 500 + b, ("syn", "blocks", "noise")[b % 3]) for b in range(8)])
    dt, du = _check_batch(case, imgs, snapshots=True)
    assert du["update"]["tps"] == 4 and du["update"]["kernel"] == 5, du["update"]
    assert (dt["update"], dt["full"], dt["prepare"]) == (du["update"], du["full"], du["prepare"])


def test_trace_leaves_untraced_calls_alone_large_K():
    """off, off, on, off at K > 4096 on one context and stream: the second call captures a graph, the traced third
    neither replays nor recaptures it, the fourth replays it; the untraced calls around the traced one agree on
    launches, dispatch, labels and clusters, and the traced one leaves the same labels and clusters."""
    from fast_slic_b200 import Engine
    case = _bigk_case(True)
    eng = Engine(case.H, case.W, case.K, max_batch=1)
    try:
        st = torch.cuda.Stream()
        img = torch.from_numpy(image(case)).cuda()[None]
        params = _params(case, case.max_iter)
        seeds = eng.initialize_clusters(img)
        cl = torch.empty_like(seeds)
        lab = torch.empty((1, case.H, case.W), dtype=torch.int16, device=seeds.device)
        torch.cuda.synchronize()
        out = []
        with torch.cuda.stream(st):
            for trace in (False, False, True, False):
                cl.copy_(seeds)
                eng.set_trace(trace)
                eng.iterate(img, cl, params, labels=lab)
                eng.set_trace(False)
                st.synchronize()
                out.append((eng.launches_last_iterate(), _record(eng) if trace else eng.dispatch(),
                            lab.cpu().numpy(), cl.cpu().numpy(), eng.graph_counts()))
                if trace:
                    assert _mismatches(eng) == 0
        assert [o[4] for o in out] == [(0, 0), (1, 0), (1, 0), (1, 1)]
        (l1, d1, lab1, cl1, _), (l3, d3, lab3, cl3, _) = out[1], out[3]
        assert l1 == l3 and d1 == d3 and d1["prepare"] == 2
        assert (lab1 == lab3).all() and cl1.tobytes() == cl3.tobytes()
        assert (out[2][2] == lab1).all() and out[2][3].tobytes() == cl1.tobytes()
    finally:
        eng.close()


# ---- what the file reached --------------------------------------------------------------------------------------------
NEEDED = [("update", k) for k in ("tma", "ldg", "generic", "real_standard", "real_l2", "real_noq", "preemptive", "lsc")] \
    + [("prepare", p) for p in (1, 2, 3)]


def test_kernel_coverage(request):
    """The traced calls above reached every update kernel and every prepare kernel, and none of them fused a prepare
    into an assign tail.  Runs last; skipped when tests of this file were deselected."""
    mine = [i for i in request.session.items if i.module is request.module and i.name != request.node.name]
    from_file = [n for n in dir(request.module) if n.startswith("test_") and n != "test_kernel_coverage"]
    if {i.originalname for i in mine} != set(from_file) or len(REACHED) == 0:
        pytest.skip("only part of the file ran")
    print("traced calls reached:", sorted(REACHED, key=str))
    missed = [k for k in NEEDED if k not in REACHED]
    assert not missed, "never reached under trace: %s" % missed
    assert {r[1] for r in REACHED if r[0] == "fused"} == {0}, "a traced call fused a prepare into an assign tail"
