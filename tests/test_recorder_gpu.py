"""debug_mode on the GPU: SlicModel.last_recorder_report against the compiled reference's bytes (oracle/_ref, where it is
built) or its pinned SHA-256 digests (tests/golden/recorder_reference_digests.npz), plus the guarantees of tracing:
same labels and clusters as untraced, no effect on later untraced calls (graph replay included), batch = singles, host
entry points refused."""
import hashlib
import os

import numpy as np
import pytest
import torch

from recorder_cases import CASES, first_difference, image, make_slic, reference_report

pytestmark = pytest.mark.gpu

GOLDEN = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "recorder_reference_digests.npz"))
DIGEST = dict(zip(GOLDEN["names"].tolist(), GOLDEN["sha256"].tolist()))


def _check_report(case, got):
    from oracle.recorder import RecorderRef
    if RecorderRef.available():
        want = reference_report(case, RecorderRef())
        assert got == want, case.name + ": " + first_difference(got, want)
    assert hashlib.sha256(got).hexdigest() == DIGEST[case.name], case.name + ": report differs from the reference digest"


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_report_matches_reference(case):
    s = make_slic(case)
    labels = s.iterate(image(case), case.max_iter)
    _check_report(case, s.slic_model.last_recorder_report)
    if case.kernel is not None:
        from fast_slic_b200.base_slic import get_engine
        eng = get_engine(case.H, case.W, case.K)
        assert eng.DISPATCH_KERNELS[eng.dispatch()["update"]["kernel"]] == case.kernel
    # the same call untraced: identical labels and cluster records
    off = make_slic(case, debug_mode=False)
    assert (off.iterate(image(case), case.max_iter) == labels).all()
    assert off.slic_model.cluster_array.tobytes() == s.slic_model.cluster_array.tobytes()
    assert off.slic_model.last_recorder_report == b'{"snapshots":[]}'


def _engine_case():
    return next(c for c in CASES if c.name == "tma_10")


def test_trace_leaves_untraced_calls_alone():
    """off, off, on, off on one context and stream: the second call captures a graph, the traced third neither replays nor
    recaptures it, the fourth replays it; the untraced calls around the traced one agree on launches, dispatch, labels
    and clusters."""
    from fast_slic_b200 import Engine
    case = _engine_case()
    eng = Engine(case.H, case.W, case.K, max_batch=1)
    st = torch.cuda.Stream()
    img = torch.from_numpy(image(case)).cuda()[None]
    params = Engine.params(case.compactness, 0.25, case.stride, case.lab, case.max_iter)
    seeds = eng.initialize_clusters(img)
    # fixed cluster and label buffers: the graph is keyed on them
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
            out.append((eng.launches_last_iterate(), eng.dispatch(), lab.cpu().numpy(), cl.cpu().numpy(),
                        eng.graph_counts()))
            if trace:
                snap = eng.trace_snapshots(0)
                assert snap["mismatches"] == 0
    assert [o[4] for o in out] == [(0, 0), (1, 0), (1, 0), (1, 1)]
    (l1, d1, lab1, cl1, _), (l3, d3, lab3, cl3, _) = out[1], out[3]
    assert l1 == l3 and d1 == d3
    assert (lab1 == lab3).all() and cl1.tobytes() == cl3.tobytes()
    assert (out[2][2] == lab1).all() and out[2][3].tobytes() == cl1.tobytes()
    eng.close()


def test_batch_of_three_equals_singles():
    from fast_slic_b200 import Engine
    from oracle.oracle import synthetic_image
    case = next(c for c in CASES if c.name == "ldg_2")
    imgs = np.stack([synthetic_image(case.H, case.W, seed=s) for s in (1, 2, 3)])
    params = Engine.params(case.compactness, 0.25, case.stride, case.lab, 3)
    batch = Engine(case.H, case.W, case.K, max_batch=3)
    single = Engine(case.H, case.W, case.K, max_batch=1)
    d = torch.from_numpy(imgs).cuda()
    batch.set_trace(True)
    batch.iterate(d, batch.initialize_clusters(d), params)
    single.set_trace(True)
    for b in range(3):
        one = d[b:b + 1].contiguous()
        single.iterate(one, single.initialize_clusters(one), params)
        assert single.recorder_report(0) == batch.recorder_report(b), "image %d" % b
    batch.close()
    single.close()


def test_host_entry_points_refused_while_tracing():
    from fast_slic_b200 import Engine
    case = _engine_case()
    eng = Engine(case.H, case.W, case.K, max_batch=1)
    img = image(case)[None]
    cl = eng.initialize_clusters_host(img)
    eng.set_trace(True)
    with pytest.raises(ValueError):
        eng.iterate_host(img, cl, Engine.params())
    eng.set_trace(False)
    eng.iterate_host(img, cl, Engine.params())
    eng.close()
