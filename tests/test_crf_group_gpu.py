"""SimpleCRFGroup on the GPU: every group call against the members' own calls on an identical second set of CRFs,
bit for bit (NaN compares as a class), plus one member against the CRF checker, chunked groups, refusals that change
nothing, and the members' own entry points after group calls."""
import ctypes as C

import numpy as np
import pytest

from crf_cases import nan_class_equal, run_case

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _needs_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _torch():
    import torch
    return torch


def _gpu_adapter(C_, N):
    from test_crf_gpu import Gpu
    return Gpu(C_, N)


def _case(name, C_, N, T, param=None, odd=False):
    """A crf_cases script: T frames of random clusters, graph and unaries, optional params, initialize, and with
    `odd` one inference(1) of the member alone, so that its ping-pong parity is odd when the group takes over."""
    script = "F" * T + (" p" + param if param else "") + " I" + (" i1" if odd else "")
    return (name, C_, N, "rand", "mixed", ("proba", "smallraw", "raw"), script)


def _specs(C_, N):
    return [_case("g%d_%d_t1" % (C_, N), C_, N, 1), _case("g%d_%d_t2" % (C_, N), C_, N, 2, "neg"),
            _case("g%d_%d_t3" % (C_, N), C_, N, 3, "smooth", odd=True), _case("g%d_%d_t5" % (C_, N), C_, N, 5, "mild")]


def _build(cases):
    """Two identical sets of members, played from the seeded cases."""
    sets = []
    for _ in range(2):
        members = []
        for case in cases:
            g = _gpu_adapter(case[1], case[2])
            run_case(g, case, energies=False)
            members.append(g.crf)
        sets.append(members)
    return sets


def _frames(crf):
    return [crf.get_frame(t) for t in range(crf.first_time, crf.last_time + 1)] if crf.num_frames else []


def _raw(frame):
    from fast_slic_b200 import CLUSTER_DTYPE
    cl = np.zeros(frame.num_nodes, CLUSTER_DTYPE)
    frame._call("get_clusters", cl.ctypes.data_as(C.c_void_p))
    return cl.tobytes()


def assert_members_equal(got, want, what, records=False):
    for m, (a, b) in enumerate(zip(got, want)):
        assert (a.first_time, a.last_time) == (b.first_time, b.last_time), (what, m)
        for fa, fb in zip(_frames(a), _frames(b)):
            assert nan_class_equal(fa.get_inferred(), fb.get_inferred()), "%s: q of member %d frame %d" % (
                what, m, fa.time)
            assert nan_class_equal(fa.unaries, fb.unaries), "%s: unaries of member %d frame %d" % (what, m, fa.time)
            if records:
                assert _raw(fa) == _raw(fb), (what, m, fa.time)
                assert fa.get_connectivity() == fb.get_connectivity(), (what, m, fa.time)


@pytest.mark.parametrize("C_,N", [(21, 1600), (2, 100), (1, 3), (2, 1)])
def test_group_inference_equals_member_inference(C_, N):
    from fast_slic_b200.crf import SimpleCRFGroup
    grouped, alone = _build(_specs(C_, N))
    group = SimpleCRFGroup(grouped)
    for k in (3, 2):
        group.inference(k)
        for crf in alone:
            crf.inference(k)
        assert_members_equal(grouped, alone, "inference(%d)" % k)
    # the members' own inference carries on from the group's state
    for a, b in zip(grouped, alone):
        a.inference(1), b.inference(1)
    assert_members_equal(grouped, alone, "member inference after the group's")


def test_group_member_equals_checker():
    from fast_slic_b200.crf import SimpleCRFGroup
    from oracle_crf.crf import Port
    cases = _specs(2, 100)
    grouped, _ = _build(cases)
    SimpleCRFGroup(grouped).inference(3)
    case = cases[2]  # three frames, smooth params, odd parity
    want = run_case(Port(case[1], case[2]), case[:6] + (case[6] + " i3S",), energies=False)
    for f in _frames(grouped[2]):
        assert nan_class_equal(f.get_inferred(), want["s0/t%d/q" % f.time]), f.time


def test_group_over_the_chunk_boundary():
    """70 members: two launch sets of the chain kernels and of the per-frame setters."""
    torch = _torch()
    from fast_slic_b200.crf import SimpleCRFGroup
    cases = [_case("chunk%d" % m, 2, 5, 1 + m % 3, odd=m % 4 == 1) for m in range(70)]
    grouped, alone = _build(cases)
    group = SimpleCRFGroup(grouped)
    rng = np.random.RandomState(7)
    proba = torch.from_numpy(rng.rand(70, 2, 5).astype(np.float32)).cuda()
    group.set_proba(proba), group.reset_inferred(), group.inference(3)
    for b, crf in enumerate(alone):
        f = crf.get_frame(crf.last_time)
        f.set_proba(proba[b]), f.reset_inferred(), crf.inference(3)
    assert_members_equal(grouped, alone, "70 members")
    q = group.get_inferred()
    for b, crf in enumerate(alone):
        assert nan_class_equal(q[b].cpu().numpy(), crf.get_frame(crf.last_time).get_inferred()), b


def _slic_batch(B, K, seed):
    from fast_slic_b200 import Slic
    from oracle.oracle import synthetic_image
    images = _torch().from_numpy(np.stack([synthetic_image(240, 320, seed=seed + b) for b in range(B)])).cuda()
    return Slic(num_components=K).iterate_batch(images, return_clusters=True)


@pytest.mark.parametrize("several_chunks", [False, True])
def test_group_push_equals_member_push(monkeypatch, several_chunks):
    """Records, CSR, unaries and q of group pushes against each member's own push, over a sliding window with pops,
    with setters, inference and get_inferred(out=) on the way; members start with different frame counts."""
    torch = _torch()
    from fast_slic_b200 import _lib, graph_batch
    from fast_slic_b200.crf import SimpleCRF, SimpleCRFGroup
    B, K, Cc = 3, 300, 4
    if several_chunks:
        monkeypatch.setattr(graph_batch, "GRAPH_SCRATCH_CAP",
                            2 * _lib.lib().fslic_b200_connectivity_batch_scratch_bytes(K, 1))
        assert graph_batch.graph_chunk(K, B) < B
    grouped, alone = [[SimpleCRF(Cc, K) for _ in range(B)] for _ in range(2)]
    labels, clusters = _slic_batch(B, K, seed=30)
    for b in range(1, B):  # member b starts with b frames
        for crfs in (grouped, alone):
            crfs[b].push_label_frames(labels[:b], clusters[:b])
    group = SimpleCRFGroup(grouped)
    rng = np.random.RandomState(11)
    for step in range(4):
        labels, clusters = _slic_batch(B, K, seed=40 + 10 * step)
        frames = group.push_label_frames(labels, clusters)
        own = [crf.push_label_frames(labels[b], clusters[b]) for b, crf in enumerate(alone)]
        assert [f.time for f in frames] == [f.time for f in own]
        assert all(f.parent_crf is crf for f, crf in zip(frames, grouped))
        proba = torch.from_numpy(rng.dirichlet(np.ones(Cc), (B, K)).transpose(0, 2, 1).astype(np.float32).copy()).cuda()
        group.set_proba(proba), group.reset_inferred(), group.inference(5)
        for b, crf in enumerate(alone):
            own[b].set_proba(proba[b]), own[b].reset_inferred(), crf.inference(5)
        q = torch.full((B, Cc, K), -3.0, device="cuda")
        assert group.get_inferred(out=q) is q
        for b in range(B):
            assert nan_class_equal(q[b].cpu().numpy(), own[b].get_inferred(out=torch.empty(Cc, K, device="cuda"))
                                   .cpu().numpy()), (step, b)
        assert_members_equal(grouped, alone, "step %d" % step, records=True)
        if step >= 1:
            assert group.pop_frame() == [crf.pop_frame() for crf in alone]
    # the members' own calls after group calls
    for a, b in zip(grouped, alone):
        a.initialize(), b.initialize()
        a.inference(2), b.inference(2)
    assert_members_equal(grouped, alone, "own calls afterwards", records=True)


def test_pop_of_members_without_frames():
    from fast_slic_b200.crf import SimpleCRF, SimpleCRFGroup
    crfs = [SimpleCRF(2, 4) for _ in range(3)]
    crfs[1].push_frame(), crfs[1].push_frame(), crfs[2].push_frame()
    group = SimpleCRFGroup(crfs)
    assert group.pop_frame() == [-1, 0, 0]
    assert [c.num_frames for c in crfs] == [0, 1, 0]
    assert group.pop_frame() == [-1, 1, -1]
    assert group.pop_frame() == [-1, -1, -1]


def test_refusals_change_nothing():
    torch = _torch()
    from fast_slic_b200 import crf as crf_mod
    from fast_slic_b200.crf import SimpleCRF, SimpleCRFGroup
    cases = _specs(2, 100)[:3]
    grouped, alone = _build(cases)
    group = SimpleCRFGroup(grouped)
    B, Cc, N = 3, 2, 100
    before = [[f.get_inferred() for f in _frames(c)] for c in grouped]
    with pytest.raises(ValueError):
        SimpleCRFGroup([grouped[0], grouped[1], grouped[0]])
    for other in (SimpleCRF(3, N), SimpleCRF(Cc, N + 1)):
        with pytest.raises(ValueError):
            SimpleCRFGroup(grouped + [other])
    elsewhere = SimpleCRF(Cc, N)
    elsewhere.device = 1  # as a member on another device would look
    with pytest.raises(ValueError):
        SimpleCRFGroup(grouped + [elsewhere])
    elsewhere.device = 0
    # the C entry points refuse a repeated member and a mismatched one themselves
    L = crf_mod._L()
    for members in ([grouped[0], grouped[0]], [grouped[0], SimpleCRF(3, N)]):
        handles = (C.c_void_p * 2)(*[c._h.value for c in members])
        assert L.fslic_b200_crfgroup_inference(handles, 2, 1, None) != 0
        assert L.fslic_b200_crfdev_group_reset_inferred(handles, 2, None) != 0
    # a member without frames
    empty = SimpleCRFGroup(grouped + [SimpleCRF(Cc, N)])
    for call in (lambda: empty.inference(2), empty.reset_inferred,
                 lambda: empty.set_proba(torch.rand(B + 1, Cc, N, device="cuda")),
                 lambda: empty.get_inferred()):
        with pytest.raises(IndexError):
            call()
    empty.inference(0)  # a no-op, as for a single CRF
    # wrong shapes, dtypes and devices
    for bad in (torch.rand(B, Cc, N + 1, device="cuda"), torch.rand(B - 1, Cc, N, device="cuda"),
                torch.rand(B, Cc, N, device="cuda", dtype=torch.float64), torch.rand(B, Cc, N),
                torch.rand(Cc, N, device="cuda")):
        with pytest.raises(ValueError):
            group.set_proba(bad)
        with pytest.raises(ValueError):
            group.get_inferred(out=bad)
    with pytest.raises(ValueError):
        group.get_inferred(out=torch.rand(B, Cc, 2 * N, device="cuda")[:, :, ::2])
    labels, clusters = _slic_batch(B, N, seed=60)
    for lab, cl in ((labels[:2], clusters), (labels, clusters[:, :99]), (labels.int(), clusters),
                    (labels, clusters.float()), (labels.cpu(), clusters.cpu()), (labels[0], clusters[0])):
        with pytest.raises(ValueError):
            group.push_label_frames(lab, cl)
    after = [[f.get_inferred() for f in _frames(c)] for c in grouped]
    assert all(nan_class_equal(x, y) for a, b in zip(before, after) for x, y in zip(a, b))
    assert [c.num_frames for c in grouped] == [1, 2, 3]
    # and the members still run exactly as the untouched set does
    group.inference(2)
    for crf in alone:
        crf.inference(2)
    assert_members_equal(grouped, alone, "after refusals")


def test_group_on_a_non_blocking_side_stream():
    torch = _torch()
    from fast_slic_b200.crf import SimpleCRF, SimpleCRFGroup
    B, K, Cc = 2, 300, 3
    labels, clusters = _slic_batch(B, K, seed=70)
    proba = torch.rand(B, Cc, K, device="cuda")
    grouped, alone = [[SimpleCRF(Cc, K) for _ in range(B)] for _ in range(2)]
    group = SimpleCRFGroup(grouped)
    out = torch.empty(B, Cc, K, device="cuda")
    side = torch.cuda.Stream()  # created with cudaStreamNonBlocking
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        group.push_label_frames(labels, clusters)
        group.set_proba(proba), group.reset_inferred(), group.inference(4)
        group.get_inferred(out=out)
    side.synchronize()
    for b, crf in enumerate(alone):
        f = crf.push_label_frames(labels[b], clusters[b])
        f.set_proba(proba[b]), f.reset_inferred(), crf.inference(4)
        assert nan_class_equal(out[b].cpu().numpy(), f.get_inferred()), b
    assert_members_equal(grouped, alone, "side stream", records=True)
