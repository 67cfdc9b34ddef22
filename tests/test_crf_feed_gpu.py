"""The CRF fed from device tensors (SimpleCRF.push_label_frames and the tensor setters / getter of SimpleCRFFrame) on
the GPU: every device-fed frame against the host path (push_slic_frame and the numpy setters) fed the same values,
at tolerance 0 (NaN compares as a class), the device logf clone on every input, the host copies of a device-pushed
frame, and the absence of host copies on the device path."""
import ctypes as C
import hashlib
import json
import os
import tempfile
import types

import numpy as np
import pytest

from crf_cases import nan_class_equal

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOGF_DIGESTS = os.path.join(ROOT, "tests", "golden", "logf_reference_digests.npz")
REF_LIB = os.path.join(ROOT, "oracle_crf", "_ref", "libfslic_ref_crf.so")


@pytest.fixture(scope="module", autouse=True)
def _needs_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _torch():
    import torch
    return torch


def _crf(C_, N):
    from fast_slic_b200.crf import SimpleCRF
    return SimpleCRF(C_, N)


def _records(cl):
    """uint8 [..., K, 32] cuda tensor of structured records."""
    torch = _torch()
    return torch.from_numpy(np.ascontiguousarray(cl).view(np.uint8).reshape(cl.shape + (32,)).copy()).cuda()


def _struct(t):
    from fast_slic_b200 import CLUSTER_DTYPE
    return t.cpu().numpy().view(CLUSTER_DTYPE).reshape(t.shape[:-1])


def host_push(crf, labels, clusters):
    """push_slic_frame of a Slic whose last_assignment is `labels` (int16 [H,W]) and whose records are `clusters`."""
    from fast_slic_b200 import SlicModel
    model = SlicModel(crf._N)
    model._clusters = clusters
    with np.errstate(invalid="ignore"):  # NaN / inf / out-of-range records: numpy's cast gives INT_MIN
        return crf.push_slic_frame(types.SimpleNamespace(slic_model=model, last_assignment=labels))


def both(labels, clusters, C_=5):
    """(device-fed CRF, its frames, host-fed CRF, its frames) for cuda labels [B,H,W] and records [B,K,32]."""
    K = clusters.shape[1]
    dev, host = _crf(C_, K), _crf(C_, K)
    df = dev.push_label_frames(labels, clusters)
    lab, cl = labels.cpu().numpy(), _struct(clusters)
    hf = [host_push(host, lab[b], cl[b]) for b in range(lab.shape[0])]
    return dev, df, host, hf


def raw(frame):
    from fast_slic_b200 import CLUSTER_DTYPE
    cl = np.zeros(frame.num_nodes, CLUSTER_DTYPE)
    frame._call("get_clusters", cl.ctypes.data_as(C.c_void_p))
    return cl.tobytes()


def same(a, b, what):
    assert nan_class_equal(a, b), what


def assert_frames_equal(dfs, hfs):
    for t, (d, h) in enumerate(zip(dfs, hfs)):
        assert d.time == h.time
        assert raw(d) == raw(h), "records of frame %d" % t
        assert d.get_yxmrgb() == h.get_yxmrgb(), t
        assert d.get_connectivity() == h.get_connectivity(), "graph of frame %d" % t
        same(d.unaries, h.unaries, "unaries of frame %d" % t)


def assert_crfs_equal(dev, df, host, hf, pairs=64):
    """Frames, q after initialize() and after inference 1 and 5, and both pairwise energies."""
    assert_frames_equal(df, hf)
    dev.initialize(), host.initialize()
    for it in (0, 1, 4):
        dev.inference(it), host.inference(it)
        for t, (d, h) in enumerate(zip(df, hf)):
            same(d.get_inferred(), h.get_inferred(), "q of frame %d after %d more iterations" % (t, it))
    rng = np.random.RandomState(3)
    N = dev._N
    for t, (d, h) in enumerate(zip(df, hf)):
        conn = d.get_connectivity()
        ij = [(i, conn[i][0]) for i in range(min(N, pairs)) if conn[i]] + \
            [tuple(x) for x in rng.randint(0, N, (pairs, 2))]
        for i, j in ij:
            same(np.float32(d.spatial_pairwise_energy(i, j)), np.float32(h.spatial_pairwise_energy(i, j)), (t, i, j))
        if t:
            for i in rng.randint(0, N, pairs):
                same(np.float32(d.temporal_pairwise_energy(i, df[t - 1])),
                     np.float32(h.temporal_pairwise_energy(i, hf[t - 1])), (t, i))


def _images(B, H=240, W=320, seed=0):
    from oracle.oracle import synthetic_image
    return _torch().from_numpy(np.stack([synthetic_image(H, W, seed=seed + b) for b in range(B)])).cuda()


def _slic(kind, K):
    from fast_slic_b200 import LSC, Slic, SlicRealDistNoQ
    if kind == "slic":
        return Slic(num_components=K)
    if kind == "noq":
        return SlicRealDistNoQ(num_components=K)
    return LSC(num_components=K, num_threads=1)


def test_device_logf_on_every_input():
    """The device compile of glibc_logf.cuh over all 2^32 bit patterns hashes to glibc's digest: bit-identical to
    glibc (and to the host compile), NaN sign and payload included."""
    torch = _torch()
    from fast_slic_b200 import crf as crf_mod
    L = crf_mod._L()
    z = np.load(LOGF_DIGESTS)
    want = bytes(z["sha"][z["keys"].tolist().index("logf/all")])
    chunk = 1 << 28
    buf = torch.empty(chunk, dtype=torch.float32, device="cuda:0")
    host = torch.empty(chunk, dtype=torch.float32, pin_memory=True)
    h = hashlib.sha256()
    for first in range(0, 1 << 32, chunk):
        st = torch.cuda.current_stream(0)
        assert L.fslic_b200_debug_logf_device(0, first, chunk, C.c_void_p(buf.data_ptr()),
                                              C.c_void_p(st.cuda_stream)) == 0
        host.copy_(buf)
        h.update(host.numpy().tobytes())
    assert h.digest() == want


@pytest.mark.parametrize("kind,B", [("slic", 1), ("slic", 8), ("noq", 3), ("lsc", 2)])
def test_push_matches_push_slic_frame(kind, B):
    """Labels and records of Slic, SlicRealDistNoQ (fractional centroids) and LSC, pushed from the device, against
    push_slic_frame of the same values."""
    K = 300
    labels, clusters = _slic(kind, K).iterate_batch(_images(B, seed=10 * B), return_clusters=True)
    if kind == "noq":
        frac = _struct(clusters)
        assert (frac["y"] != np.trunc(frac["y"])).any()
    assert_crfs_equal(*both(labels, clusters))


def test_single_image_gives_one_frame():
    from fast_slic_b200.crf import SimpleCRFFrame
    labels, clusters = _slic("slic", 200).iterate_batch(_images(1), return_clusters=True)
    dev, host = _crf(3, 200), _crf(3, 200)
    f = dev.push_label_frames(labels[0], clusters[0])
    assert isinstance(f, SimpleCRFFrame) and f.time == 0
    h = host_push(host, labels[0].cpu().numpy(), _struct(clusters)[0])
    assert_crfs_equal(dev, [f], host, [h])


def test_batch_over_several_scratch_chunks(monkeypatch):
    from fast_slic_b200 import _lib, graph_batch
    K = 300
    monkeypatch.setattr(graph_batch, "GRAPH_SCRATCH_CAP", 2 * _lib.lib().fslic_b200_connectivity_batch_scratch_bytes(K, 1))
    assert graph_batch.graph_chunk(K, 5) < 5
    labels, clusters = _slic("slic", K).iterate_batch(_images(5, seed=3), return_clusters=True)
    assert_crfs_equal(*both(labels, clusters))


def test_labels_outside_the_range_and_overflow_replay():
    """-1 and >= K labels are ignored; a noise map takes the graph's overflow replay."""
    torch = _torch()
    from fast_slic_b200 import Slic
    K = 300
    labels, clusters = _slic("slic", K).iterate_batch(_images(2, 512, 512, seed=5), return_clusters=True)
    rng = np.random.RandomState(4)
    noise = rng.randint(0, K, (512, 512)).astype(np.int16)
    odd = labels[1].cpu().numpy().copy()
    odd[rng.rand(512, 512) < 0.1] = -1
    odd[rng.rand(512, 512) < 0.1] = K + 7
    labels = torch.from_numpy(np.stack([noise, odd, labels[0].cpu().numpy()])).cuda()
    clusters = torch.cat([clusters, clusters[:1]])
    _, _, rep = Slic(num_components=K).get_connectivity_batch(labels, return_replayed=True)
    assert rep.tolist() == [1, 0, 0]
    assert_crfs_equal(*both(labels, clusters))


def test_one_node():
    torch = _torch()
    from fast_slic_b200 import CLUSTER_DTYPE
    cl = np.zeros((2, 1), CLUSTER_DTYPE)
    cl["y"], cl["x"], cl["num_members"], cl["r"] = 3.5, 2.0, 40, 100.0
    lab = np.zeros((2, 6, 7), np.int16)
    lab[1, 2:4] = -1
    assert_crfs_equal(*both(torch.from_numpy(lab).cuda(), _records(cl), C_=2), pairs=2)


def test_hand_made_records():
    """NaN, ±inf, negative, >= 2^31 and fractional fields; num_members 0, 2^31 and 2^32 - 1: numpy's x86 cast."""
    torch = _torch()
    from fast_slic_b200 import CLUSTER_DTYPE
    K = 24
    specials = np.array([np.nan, np.inf, -np.inf, -3.7, -0.5, 0.99, 2.0 ** 31, 3e9, -2.0 ** 31, -2.0 ** 31 - 256,
                         2.0 ** 31 - 128, 1e30, -1e30, 7.5, 0.0, -0.0], np.float32)
    rng = np.random.RandomState(9)
    cl = np.zeros((2, K), CLUSTER_DTYPE)
    for ch in ("y", "x", "r", "g", "b", "a"):
        cl[ch] = rng.choice(specials, (2, K))
    cl["num_members"] = rng.choice(np.array([0, 1, 5, 2 ** 31 - 1, 2 ** 31, 2 ** 32 - 1], np.uint32), (2, K))
    cl["number"], cl["is_active"], cl["is_updatable"] = 77, 1, 2
    lab = rng.randint(0, K, (2, 16, 20)).astype(np.int16)
    dev, df, host, hf = both(torch.from_numpy(lab).cuda(), _records(cl))
    got = np.frombuffer(raw(df[0]), CLUSTER_DTYPE)
    assert (got["y"][np.isnan(cl["y"][0])] == -2.0 ** 31).all()
    assert (got["num_members"][cl["num_members"][0] >= 2 ** 31] == 2 ** 31).all()
    assert_crfs_equal(dev, df, host, hf, pairs=K)


def test_refusals_push_nothing():
    torch = _torch()
    labels, clusters = _slic("slic", 100).iterate_batch(_images(2), return_clusters=True)
    crf = _crf(3, 100)
    bad = [
        (labels, clusters[:, :99]),                      # K != num_nodes
        (labels.int(), clusters),                        # label dtype
        (labels, clusters.float()),                      # record dtype
        (labels[:1], clusters),                          # batch
        (labels, clusters[0]),                           # rank
        (labels.cpu(), clusters.cpu()),                  # host tensors
        (labels.cpu().numpy(), clusters),                # numpy
    ]
    for lab, cl in bad:
        with pytest.raises(ValueError):
            crf.push_label_frames(lab, cl)
    assert crf.num_frames == 0 and crf.first_time == -1
    other = _crf(3, 99)
    with pytest.raises(ValueError):
        other.push_label_frames(labels, clusters)
    assert other.num_frames == 0
    assert crf.push_label_frames(labels[:0], clusters[:0]) == []
    assert crf.num_frames == 0


def test_tensor_setters_equal_host_setters():
    torch = _torch()
    N = 40
    rng = np.random.RandomState(1)
    for C_ in (1, 2, 21):
        dev, host = _crf(C_, N), _crf(C_, N)
        d, h = dev.push_frame(), host.push_frame()
        p = rng.rand(C_, N).astype(np.float32)
        flat = p.reshape(-1)
        flat[:14] = np.array([0, -0.0, 1e-45, 1e-40, 1.17e-38, 1, 1.5, 3e38, -1, -1e-40, np.inf, -np.inf, np.nan, 0.5],
                             np.float32)[:flat.size][:14]
        if flat.size > 14:
            flat[14] = np.frombuffer(np.uint32(0xffa12345).tobytes(), np.float32)[0]  # a signalling NaN with payload
        d.set_proba(torch.from_numpy(p).cuda()), h.set_proba(p)
        same(d.unaries, h.unaries, "set_proba C=%d" % C_)
        u = rng.randn(C_, N).astype(np.float32)
        d.unaries, h.unaries = torch.from_numpy(u).cuda(), u
        assert d.unaries.tobytes() == h.unaries.tobytes() == u.tobytes()
        for conf in (0.0, 0.5, 1.0):
            cls = rng.randint(0, C_, N).astype(np.int32)
            d.set_mask(torch.from_numpy(cls).cuda(), conf), h.set_mask(cls, conf)
            same(d.unaries, h.unaries, "set_mask C=%d confidence %g" % (C_, conf))
        before = d.unaries
        cls = rng.randint(0, C_, N).astype(np.int32)
        cls[N // 2] = C_
        with pytest.raises(ValueError):
            d.set_mask(torch.from_numpy(cls).cuda(), 0.5)
        cls[N // 2] = -1
        with pytest.raises(ValueError):
            d.set_mask(torch.from_numpy(cls).cuda(), 0.5)
        assert d.unaries.tobytes() == before.tobytes()
        dev.initialize(), host.initialize()
        dev.inference(2), host.inference(2)
        out = torch.full((C_, N), -7.0, device="cuda")
        assert d.get_inferred(out=out) is out
        same(out.cpu().numpy(), h.get_inferred(), "get_inferred(out=) C=%d" % C_)
        for bad in (torch.zeros(C_, N + 1, device="cuda"), torch.zeros(C_, N, device="cuda", dtype=torch.float64),
                    torch.zeros(C_, 2 * N, device="cuda")[:, ::2]):
            with pytest.raises(ValueError):
                d.get_inferred(out=bad)
        for bad in (torch.zeros(C_, N + 1, device="cuda"), torch.zeros(C_, N, device="cuda", dtype=torch.float64)):
            with pytest.raises(ValueError):
                d.set_proba(bad)
        with pytest.raises(ValueError):
            d.set_mask(torch.zeros(N, device="cuda", dtype=torch.int64), 0.5)


def test_set_connectivity_with_fewer_rows_keeps_the_rest():
    K = 300
    labels, clusters = _slic("slic", K).iterate_batch(_images(2, seed=7), return_clusters=True)
    dev, df, host, hf = both(labels, clusters)
    rows = [[1, 2], [], [0, 0, 5]]
    for f in (df[1], hf[1]):
        from fast_slic_b200 import NodeConnectivity
        counts = np.array([len(r) for r in rows], np.int32)
        nb = np.zeros((3, 12), np.int32)
        for i, r in enumerate(rows):
            nb[i, :len(r)] = r
        f.set_connectivity(NodeConnectivity(counts, nb))
    assert df[1].get_connectivity()[:3] == rows
    assert_crfs_equal(dev, df, host, hf)


def test_sliding_window_with_pool_reuse():
    """push, set_proba, inference, pop over a window of 3: the device-fed CRF gives the host-fed one's q, frame after
    frame, through slots popped and reused (some first used by host pushes)."""
    torch = _torch()
    K, Cc = 300, 6
    slic = _slic("slic", K)
    labels, clusters = slic.iterate_batch(_images(8, seed=20), return_clusters=True)
    lab, cl = labels.cpu().numpy(), _struct(clusters)
    dev, host = _crf(Cc, K), _crf(Cc, K)
    rng = np.random.RandomState(2)
    for i in range(8):
        if i == 2:  # a host push on the device-fed CRF too: its slot is later reused by a device push
            d, h = host_push(dev, lab[i], cl[i]), host_push(host, lab[i], cl[i])
        else:
            d, h = dev.push_label_frames(labels[i], clusters[i]), host_push(host, lab[i], cl[i])
        p = rng.dirichlet(np.ones(Cc), K).T.astype(np.float32).copy()
        d.set_proba(torch.from_numpy(p).cuda()), h.set_proba(p)
        d.reset_inferred(), h.reset_inferred()
        dev.inference(5), host.inference(5)
        out = torch.empty(Cc, K, device="cuda")
        same(d.get_inferred(out=out).cpu().numpy(), h.get_inferred(), "q at frame %d" % i)
        if dev.num_frames >= 3:
            assert dev.pop_frame() == host.pop_frame()
    live = [dev.get_frame(t) for t in range(dev.first_time, dev.last_time + 1)]
    assert_frames_equal(live, [host.get_frame(t) for t in range(host.first_time, host.last_time + 1)])


def test_device_path_makes_no_host_copies():
    """On a non-default stream, a profiler trace of push + set_proba + set_mask + inference + get_inferred(out=) has
    no device-to-host copy larger than set_mask's 4-byte flag."""
    torch = _torch()
    from torch.profiler import ProfilerActivity, profile
    K, Cc = 300, 4
    labels, clusters = _slic("slic", K).iterate_batch(_images(2, seed=40), return_clusters=True)
    crf = _crf(Cc, K)
    crf.push_label_frames(labels, clusters)  # slots allocated outside the trace
    crf.pop_frame(), crf.pop_frame()
    proba = torch.rand(Cc, K, device="cuda")
    cls = torch.randint(0, Cc, (K,), device="cuda", dtype=torch.int32)
    out = torch.empty(Cc, K, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            frames = crf.push_label_frames(labels, clusters)
            frames[0].set_mask(cls, 0.7)
            frames[1].set_proba(proba)
            crf.initialize()
            crf.inference(5)
            frames[1].get_inferred(out=out)
            side.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        events = json.load(open(path))["traceEvents"]
    copies = [e for e in events if e.get("cat") == "gpu_memcpy"]
    assert copies, "the trace recorded no copies at all"
    big = [(e["name"], e.get("args", {}).get("bytes")) for e in copies
           if "DtoH" in e["name"] and e.get("args", {}).get("bytes", 1 << 30) > 4]
    assert not big, big
    # the host-side readers of the frames pushed on the side stream see them exactly
    host = _crf(Cc, K)
    for b, f in enumerate(frames):
        h = host_push(host, labels[b].cpu().numpy(), _struct(clusters)[b])
        assert raw(f) == raw(h) and f.get_connectivity() == h.get_connectivity(), b


@pytest.mark.skipif(not os.path.exists(REF_LIB), reason="oracle_crf/_ref is built only where FSLIC_REFERENCE is set")
def test_device_fed_crf_against_compiled_reference():
    """Three SLIC frames pushed from the device, set_proba from a tensor, inference(5): unaries and q equal the
    reference's SimpleCRF fed the same records (converted as push_slic_frame does) and the reference-checked graph."""
    torch = _torch()
    from oracle.oracle import Port as SlicPort
    from oracle_crf.crf import Ref
    from crf_cases import to_csr
    K, Cc = 300, 5
    labels, clusters = _slic("noq", K).iterate_batch(_images(3, seed=50), return_clusters=True)
    crf, ref = _crf(Cc, K), Ref(Cc, K)
    frames = crf.push_label_frames(labels, clusters)
    lab, cl = labels.cpu().numpy(), _struct(clusters)
    rng = np.random.RandomState(5)
    for b, f in enumerate(frames):
        t = ref.push()
        rec = np.zeros(K, cl.dtype)
        for name in ("y", "x", "r", "g", "b"):
            rec[name] = cl[b][name].astype(np.float64).astype(np.int32)
        rec["num_members"] = cl[b]["num_members"].astype(np.float64).astype(np.int32).astype(np.uint32)
        rec["number"] = np.arange(K)
        ref.set_clusters(t, rec)
        ref.set_connectivity(t, *to_csr(SlicPort().get_connectivity(lab[b].view(np.uint16), K)))
        p = rng.dirichlet(np.ones(Cc), K).T.astype(np.float32).copy()
        f.set_proba(torch.from_numpy(p).cuda())
        ref.set_proba(t, p)
    crf.initialize(), ref.initialize()
    crf.inference(5), ref.inference(5)
    for b, f in enumerate(frames):
        same(f.unaries, ref.get_unary(b), "unaries %d" % b)
        same(f.get_inferred(), ref.get_inferred(b), "q %d" % b)
