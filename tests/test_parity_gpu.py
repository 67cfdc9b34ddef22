"""GPU parity: the CUDA path (through the C ABI) against the CPU oracle, bit-exact.

Tolerance: 0 for label maps (pre- and post-CCA), the Lab quad image and every Cluster field
(they are integers on this path).
"""
import numpy as np
import pytest
import torch

from cases import (BIG_CASES, EDGE_CASES, LDG_FORCED_CASES, PIPELINE_CASES, PREEMPT_SWEEP_SEEDS, REAL_SWEEP_SEEDS,
                   SWEEP_KINDS, TMA_CASES, cca_random_labels, cca_range_labels, gpu_random_config_case, make_image,
                   preempt_sweep_case, real_sweep_case, split_kwargs, sweep_case_id)
from class_checks import LSC, PREEMPT, REAL_KERNELS, assert_kernel, check_class_call

pytestmark = pytest.mark.gpu


def _engine(H, W, K, B=1):
    from fast_slic_b200 import get_engine
    return get_engine(H, W, K, B, 0)


def _run_cuda(img, K, args, iterate_twice=False):
    H, W, _ = img.shape
    eng = _engine(H, W, K)
    t = torch.from_numpy(img).cuda()[None].contiguous()
    cl = eng.initialize_clusters(t)
    init = cl.cpu().numpy().copy()
    p = eng.params(args["compactness"], args["min_size_factor"], args["subsample_stride"], args["convert_to_lab"],
                   args["max_iter"])
    lab = eng.iterate(t, cl, p)
    if iterate_twice:
        lab = eng.iterate(t, cl, p)
    quad, pre = eng.debug_stages(1)
    torch.cuda.synchronize()
    return init, lab[0].cpu().numpy().view(np.uint16), quad[0].cpu().numpy(), pre[0].cpu().numpy().view(np.uint16), \
        cl[0].cpu().numpy()


def _run_oracle(checker, img, K, args, iterate_twice=False):
    cl = checker.initialize(img, K)
    init = cl.copy()
    out, quad, pre = checker.iterate(img, cl, args["max_iter"], args["compactness"], args["min_size_factor"],
                                  args["subsample_stride"], args["convert_to_lab"], stages=True)
    if iterate_twice:
        out, quad, pre = checker.iterate(img, cl, args["max_iter"], args["compactness"], args["min_size_factor"],
                                      args["subsample_stride"], args["convert_to_lab"], stages=True)
    return init, out, quad, pre, cl


def _compare(name, got, want):
    ginit, glab, gquad, gpre, gcl = got
    winit, wlab, wquad, wpre, wcl = want
    assert ginit.tobytes() == winit.tobytes(), name + ": initialize_clusters differs"
    assert (gquad == wquad).all(), name + ": quad image differs (%d px)" % (gquad != wquad).any(-1).sum()
    assert (gpre == wpre).all(), name + ": pre-CCA labels differ (%d px)" % (gpre != wpre).sum()
    gc = gcl.view(wcl.dtype).reshape(-1)
    for f in ("y", "x", "r", "g", "b", "num_members", "number", "is_active", "is_updatable"):
        assert (gc[f] == wcl[f]).all(), name + ": cluster field %s differs" % f
    assert (glab == wlab).all(), name + ": final labels differ (%d px)" % (glab != wlab).sum()


@pytest.mark.parametrize("case", PIPELINE_CASES, ids=[c[0] for c in PIPELINE_CASES])
def test_pipeline_parity(checker, case):
    name, kind, H, W, K, kw = case
    sigma, args = split_kwargs(kw)
    img = make_image(kind, H, W, seed=7, sigma=sigma)
    _compare(name, _run_cuda(img, K, args), _run_oracle(checker, img, K, args))


@pytest.mark.parametrize("case", EDGE_CASES, ids=[c[0] for c in EDGE_CASES])
def test_pipeline_parity_edge(checker, case):
    name, kind, H, W, K, kw = case
    sigma, args = split_kwargs(kw)
    img = make_image(kind, H, W, seed=5, sigma=sigma)
    _compare(name, _run_cuda(img, K, args), _run_oracle(checker, img, K, args))


@pytest.mark.parametrize("case", TMA_CASES, ids=[c[0] for c in TMA_CASES])
def test_pipeline_parity_tma_kernel(checker, case):
    name, kind, H, W, K, kw = case
    sigma, args = split_kwargs(kw)
    img = make_image(kind, H, W, seed=23, sigma=sigma)
    _compare(name, _run_cuda(img, K, args), _run_oracle(checker, img, K, args))
    eng = _engine(H, W, K)
    assert eng.S > 110 or eng.assign_impl() == 5, "the TMA-staged kernel did not run (impl %d)" % eng.assign_impl()


@pytest.mark.parametrize("case", LDG_FORCED_CASES, ids=lambda c: "%s-W%d" % (c[0], c[3] - 1))
def test_pipeline_parity_ldg_kernel_by_width(checker, case):
    """The round-1 LDG kernel on these shapes one column narrower: W % 8 != 0 rules out the TMA kernel's tensor maps,
    so the dispatch takes the LDG kernel (the path of every such image) where it would take the TMA one."""
    name, kind, H, W, K, kw = case
    W -= 1
    sigma, args = split_kwargs(kw)
    img = make_image(kind, H, W, seed=29, sigma=sigma)
    _compare(name, _run_cuda(img, K, args), _run_oracle(checker, img, K, args))
    assert _engine(H, W, K).assign_impl() == 4


def test_rejects_what_the_reference_cannot_do():
    """K > H*W makes S = 0: the reference divides by zero there (preemptive.h:37-38); compactness beyond the u16
    distance range is undefined behaviour in the reference (context.cpp:30).  Both are refused, not guessed."""
    from fast_slic_b200 import Slic
    from fast_slic_b200._lib import FslicError
    with pytest.raises(ValueError):
        Slic(num_components=50).iterate(np.zeros((6, 6, 3), np.uint8))
    # (the exact bound, and that a refused call writes nothing: tests/test_default_sweep_gpu.py)
    for lab in (True, False):
        s = Slic(num_components=30, compactness=1e6, convert_to_lab=lab)
        with pytest.raises(FslicError, match="compactness too large"):
            s.iterate(np.zeros((64, 64, 3), np.uint8))


@pytest.mark.parametrize("case", BIG_CASES, ids=[c[0] for c in BIG_CASES])
def test_pipeline_parity_big(checker, case):
    name, kind, H, W, K, kw = case
    sigma, args = split_kwargs(kw)
    img = make_image(kind, H, W, seed=11, sigma=sigma)
    _compare(name, _run_cuda(img, K, args), _run_oracle(checker, img, K, args))


def test_warm_start_second_iterate(checker):
    img = make_image("syn", 200, 260, seed=3)
    _, args = split_kwargs({})
    _compare("warm", _run_cuda(img, 90, args, iterate_twice=True), _run_oracle(checker, img, 90, args, iterate_twice=True))


def test_batch_matches_single(checker):
    H, W, K, B = 180, 240, 70, 5
    imgs = np.stack([make_image("syn" if b % 2 == 0 else "noise", H, W, seed=20 + b) for b in range(B)])
    from fast_slic_b200 import Slic
    s = Slic(num_components=K, min_size_factor=0.1)
    labels, clusters = s.iterate_batch(torch.from_numpy(imgs).cuda(), return_clusters=True)
    labels = labels.cpu().numpy().view(np.uint16)
    labels_h, clusters_h = s.iterate_batch(imgs, return_clusters=True)
    for b in range(B):
        cl = checker.initialize(imgs[b], K)
        want = checker.iterate(imgs[b], cl, 10, 10.0, 0.1, 3, True)
        assert (labels[b] == want).all(), "device batch image %d" % b
        assert (labels_h[b].view(np.uint16) == want).all(), "host batch image %d" % b
        assert clusters[b].cpu().numpy().tobytes() == cl.tobytes() == clusters_h[b].tobytes()


def test_sub_batched_paths(checker, monkeypatch):
    """Forces the CCA sub-batch loop (scratch smaller than the batch) and the multi-chunk host pipeline."""
    from fast_slic_b200 import Slic, clear_engine_cache
    monkeypatch.setenv("FSLIC_CCA_BATCH", "2")
    monkeypatch.setenv("FSLIC_HOST_CHUNK", "3")
    clear_engine_cache()
    try:
        H, W, K, B = 120, 160, 40, 7
        imgs = np.stack([make_image("noise" if b % 3 == 0 else "syn", H, W, seed=40 + b) for b in range(B)])
        s = Slic(num_components=K, min_size_factor=0.0)
        lab_d = s.iterate_batch(torch.from_numpy(imgs).cuda()).cpu().numpy().view(np.uint16)
        lab_h = s.iterate_batch(imgs).view(np.uint16)
        for b in range(B):
            cl = checker.initialize(imgs[b], K)
            want = checker.iterate(imgs[b], cl, 10, 10.0, 0.0, 3, True)
            assert (lab_d[b] == want).all() and (lab_h[b] == want).all(), b
    finally:
        clear_engine_cache()


def test_streaming_matches_blocking(checker):
    """SlicStream (iterate_host_async / wait on two alternating contexts) == the oracle, batch by batch, with
    pinned and pageable inputs, ragged last batch and more batches than slots."""
    from fast_slic_b200 import SlicStream
    H, W, K, B = 120, 160, 40, 4
    batches = [np.stack([make_image("noise" if (b + t) % 3 == 0 else "syn", H, W, seed=70 + 10 * t + b)
                         for b in range(B if t != 4 else 2)]) for t in range(5)]
    st = SlicStream(H, W, K, batch=B, depth=2, min_size_factor=0.0)
    pinned = st.pinned_images()
    pinned[...] = batches[1]
    feed = [batches[0], pinned] + batches[2:]
    got = list(st.map(feed))
    assert st.in_flight == 0 and len(got) == 5
    for t, labs in enumerate(got):
        assert labs.shape == (batches[t].shape[0], H, W)
        for b in range(labs.shape[0]):
            cl = checker.initialize(batches[t][b], K)
            want = checker.iterate(batches[t][b], cl, 10, 10.0, 0.0, 3, True)
            assert (labs[b].view(np.uint16) == want).all(), (t, b)
    # explicit submit / collect: clusters come back too, and over-submitting is refused
    st.submit(batches[0]); st.submit(batches[2])
    with pytest.raises(RuntimeError):
        st.submit(batches[3])
    labs, cls = st.collect()
    cl = checker.initialize(batches[0][1], K)
    want = checker.iterate(batches[0][1], cl, 10, 10.0, 0.0, 3, True)
    assert (labs[1].view(np.uint16) == want).all() and cls[1].tobytes() == cl.tobytes()
    st.close()


def test_async_same_context_serialises(checker):
    """Two _async calls on ONE context: the second waits for the first instead of overwriting its staging."""
    from fast_slic_b200 import Engine, CLUSTER_DTYPE
    H, W, K, B = 96, 128, 30, 3
    eng = Engine(H, W, K, B)
    p = eng.params(10.0, 0.1, 3, True, 10)
    bufs = []
    for t in range(2):
        imgs = torch.from_numpy(np.stack([make_image("syn", H, W, seed=90 + 5 * t + b) for b in range(B)])).pin_memory()
        cl = torch.from_numpy(eng.initialize_clusters_host(imgs.numpy()).view(np.uint8).reshape(B, K, 32)).pin_memory()
        lab = torch.empty((B, H, W), dtype=torch.int16).pin_memory()
        bufs.append((imgs, cl, lab))
    for imgs, cl, lab in bufs:
        eng.iterate_host_async(imgs.numpy(), cl.numpy(), p, lab.numpy())
    eng.wait()
    eng.wait()  # idempotent
    for imgs, cl, lab in bufs:
        for b in range(B):
            c0 = checker.initialize(imgs.numpy()[b], K)
            want = checker.iterate(imgs.numpy()[b], c0, 10, 10.0, 0.1, 3, True)
            assert (lab.numpy()[b].view(np.uint16) == want).all()
            assert cl.numpy()[b].tobytes() == c0.tobytes()
    eng.close()


def test_graph_replay_small_host_batches(checker):
    """Host calls with fewer than 4 images replay one captured CUDA graph.  Same results as the plain launches for
    changing images (replay), changing parameters (re-capture) and the async entry point."""
    from fast_slic_b200 import Engine
    H, W, K = 120, 160, 40
    eng = Engine(H, W, K, 2)
    for msf in (0.0, 0.3):
        p = eng.params(10.0, msf, 3, True, 10)
        for t in range(3):
            imgs = np.stack([make_image("noise" if (t + b) % 2 else "syn", H, W, seed=300 + 7 * t + b) for b in range(2)])
            cl = eng.initialize_clusters_host(imgs)
            lab = eng.iterate_host(imgs, cl, p)
            for b in range(2):
                c0 = checker.initialize(imgs[b], K)
                want = checker.iterate(imgs[b], c0, 10, 10.0, msf, 3, True)
                assert (lab[b].view(np.uint16) == want).all(), (msf, t, b)
                assert cl[b].tobytes() == c0.tobytes()
    # one image, async entry point, same context: a third graph
    p = eng.params(10.0, 0.1, 3, True, 10)
    for t in range(2):
        img = torch.from_numpy(make_image("syn", H, W, seed=400 + t)[None]).pin_memory()
        cl = torch.from_numpy(eng.initialize_clusters_host(img.numpy()).view(np.uint8).reshape(1, K, 32)).pin_memory()
        lab = torch.empty((1, H, W), dtype=torch.int16).pin_memory()
        eng.iterate_host_async(img.numpy(), cl.numpy(), p, lab.numpy())
        eng.wait()
        c0 = checker.initialize(img.numpy()[0], K)
        want = checker.iterate(img.numpy()[0], c0, 10, 10.0, 0.1, 3, True)
        assert (lab.numpy()[0].view(np.uint16) == want).all() and cl.numpy()[0].tobytes() == c0.tobytes()
    eng.close()


def test_lab_full_colour_cube(port):
    """All 2^24 colours as one 4096x4096 image, against the oracle (which is pinned to the reference)."""
    v = np.arange(1 << 24, dtype=np.uint32)
    img = np.stack([(v >> 16) & 255, (v >> 8) & 255, v & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)
    eng = _engine(4096, 4096, 1000)
    got = eng.rgb_to_quad(torch.from_numpy(img).cuda()[None]).cpu().numpy()[0]
    want = port.rgb_to_quad(img, True)
    assert (got == want).all()
    import hashlib
    cube = np.ascontiguousarray(got[..., :3]).tobytes()
    assert hashlib.sha256(cube).hexdigest() == "016250467c2bd57f2ef75f61bb0571a9ab8d6558f69eca0ac0831d20db948624"
    from fast_slic_b200 import clear_engine_cache
    clear_engine_cache()


@pytest.mark.parametrize("n,middle,maxarea", [(50, 7, 3), (1000, 100, 4), (5000, 1600, 6), (20000, 300, 2),
                                              (100000, 4000, 50), (4097, 4096, 3), (300, 300, 5), (9000, 1, 4)])
def test_heap_select_device_vs_stl(port, n, middle, maxarea):
    rng = np.random.RandomState(n + middle)
    area = rng.randint(1, maxarea + 1, n).astype(np.int32)
    area[rng.randint(0, n, max(1, n // 50))] += rng.randint(0, 1000, max(1, n // 50)).astype(np.int32)
    eng = _engine(64, 64, 8)
    kept = eng.debug_heap_select(torch.from_numpy(area), middle).cpu().numpy()
    want = port.stl_partial_sort(area, middle)
    assert (np.nonzero(kept)[0] == want).all()


def test_enforce_connectivity_known_answer():
    """Input of the reference's only live CCA gtest (src/cpptest/test_cca.cpp:178-204).  That test's EXPECT_EQ
    values are stale against the reference's own current code (labels are renumbered in leader order,
    cca.cpp:229-237); the expected map below is what the compiled reference returns (tests/golden/make_golden.py)."""
    from fast_slic_b200 import enforce_connectivity
    x = 9
    lab = np.array([[0, 0, 0, 0, 0], [1, 1, x, 0, 0], [1, x, 0, x, 4], [2, 2, x, x, 4], [2, 3, 3, 3, 3]], np.int16)
    want = np.array([[0, 0, 0, 0, 0], [1, 1, 2, 0, 0], [1, 3, 4, 5, 6], [7, 7, 5, 5, 6], [7, 8, 8, 8, 8]], np.int16)
    out = enforce_connectivity(lab.copy(), 0)
    assert (out == want).all()


@pytest.mark.parametrize("H,W,nlab,thres,seed", [(60, 80, 6, 0, 1), (60, 80, 6, 5, 2), (100, 33, 3, 12, 3),
                                                 (257, 515, 40, 30, 4), (64, 64, 2, 1, 5), (1, 700, 4, 3, 6),
                                                 (700, 1, 4, 3, 7), (720, 1280, 1600, 58, 8)])
def test_enforce_connectivity_random(checker, H, W, nlab, thres, seed):
    from fast_slic_b200 import enforce_connectivity
    lab = cca_random_labels(H, W, nlab, seed)
    K = int(lab.max()) + 1
    want = checker.enforce_connectivity(lab.view(np.uint16), K, thres)
    got = enforce_connectivity(lab.copy(), thres).view(np.uint16)
    assert (got == want).all(), "%d px differ" % (got != want).sum()


def test_enforce_connectivity_label_range_beyond_pixel_count(checker):
    """ADVICE r1: a small crop with large label ids (K = max label + 1 > H*W) is legal for the reference's
    ConnectivityEnforcer (K only bounds the kept set, cca.cpp:176,225); varying K must not build new contexts."""
    from fast_slic_b200 import base_slic, enforce_connectivity
    for trial, (lab, K) in enumerate(cca_range_labels()):
        want = checker.enforce_connectivity(lab.view(np.uint16), K, 3)
        got = enforce_connectivity(lab.copy(), 3).view(np.uint16)
        assert (got == want).all(), "trial %d: %d px differ" % (trial, (got != want).sum())
    assert sum(1 for k in base_slic._engines if k[0] == "cca" and k[2:] == (50, 50)) == 1


def test_engine_cache_is_bounded():
    from fast_slic_b200 import base_slic, get_engine
    base_slic.clear_engine_cache()
    first = get_engine(40, 40, 5)
    for i in range(base_slic.ENGINE_CACHE_SIZE + 3):
        get_engine(40 + 8 * (i + 1), 48, 6)
    assert len(base_slic._engines) == base_slic.ENGINE_CACHE_SIZE
    assert first._h is None  # evicted contexts are closed, not leaked
    base_slic.clear_engine_cache()


def test_python_surface_matches_reference_api():
    """Mirrors fast-slic/test/test_slic.py:41-65."""
    from fast_slic_b200 import Slic
    x = np.zeros([480, 640, 3], np.uint8)
    slic = Slic(num_components=100)
    out = slic.iterate(x)
    assert out.dtype == np.int16 and out.shape == (480, 640)
    for i, cluster in enumerate(slic.slic_model.clusters):
        assert cluster["number"] == i
        assert isinstance(cluster, dict)
        assert len(cluster["yx"]) == 2 and isinstance(cluster["yx"], tuple)
        assert len(cluster["color"]) == 3 and isinstance(cluster["color"], tuple)
        assert isinstance(cluster["num_members"], int)
    orig = slic.slic_model.clusters
    slic.slic_model.clusters = orig[:10]
    assert len(slic.slic_model.clusters) == 10
    assert slic.slic_model.clusters == orig[:10]
    assert slic.slic_model.num_components == 10 and slic.num_components == 10
    import json
    rep = json.loads(slic.slic_model.last_timing_report)
    assert rep["name"] == "iterate" and len(rep["children"]) == 5
    cca = rep["children"][4]["children"][0]   # enforce_connectivity -> cca -> the reference's six sub-sections
    assert cca["name"] == "cca" and [c["name"] for c in cca["children"]] == [
        "build_disjoint_set", "flatten", "threshold_by_area", "sort", "substitute", "output"]
    assert sum(c["duration"] for c in cca["children"]) > 0


def test_single_image_api_parity(checker):
    from fast_slic_b200 import Slic
    img = make_image("syn", 240, 320, seed=5)
    s = Slic(num_components=120, min_size_factor=0.1)
    got = s.iterate(img).view(np.uint16)
    cl = checker.initialize(img, 120)
    want = checker.iterate(img, cl, 10, 10.0, 0.1, 3, True)
    assert (got == want).all()
    assert s.slic_model.cluster_array.tobytes() == cl.tobytes()
    got2 = s.iterate(img).view(np.uint16)  # warm start
    want2 = checker.iterate(img, cl, 10, 10.0, 0.1, 3, True)
    assert (got2 == want2).all()


@pytest.mark.parametrize("H,W,K,kind,msf", [(120, 160, 48, "syn", 0.25), (97, 131, 37, "noise", 0.0), (200, 300, 150, "blocks", 0.0),
                                            (64, 64, 1500, "noise", 0.0), (480, 640, 200, "syn", 0.1), (720, 1280, 1600, "syn", 0.0)])
def test_graph_and_density_consumers(checker, H, W, K, kind, msf):
    """SlicModel.get_connectivity / get_mask_density / broadcast_density_to_mask (cfast_slic.pyx:262-320) on the GPU ==
    the reference's fast-slic.cpp functions, exactly (neighbour ORDER included; the 12-neighbour cap is exercised by the
    msf = 0 and the synthetic saturated maps)."""
    from fast_slic_b200 import Slic
    img = make_image(kind, H, W, seed=17)
    s = Slic(num_components=K, min_size_factor=msf)
    lab = s.iterate(img)
    m = s.slic_model
    assert m.get_connectivity(lab).tolist() == checker.get_connectivity(lab.view(np.uint16), K)
    raw = (make_image("noise", H, W, seed=3)[..., 0].astype(np.uint16) % min(K, 40)).astype(np.uint16).view(np.int16)
    assert m.get_connectivity(np.ascontiguousarray(raw)).tolist() == checker.get_connectivity(raw.view(np.uint16), K)
    mask = np.ascontiguousarray(make_image("syn", H, W, seed=5)[..., 1])
    cl = m.cluster_array
    dens = m.get_mask_density(mask, lab)
    assert (dens == checker.get_mask_density(cl, lab.view(np.uint16), mask)).all()
    holes = lab.copy()
    holes[::7, ::5] = -1
    assert (m.get_mask_density(mask, holes) == checker.get_mask_density(cl, holes.view(np.uint16), mask)).all()
    assert (m.broadcast_density_to_mask(dens, holes) == checker.density_to_mask(K, holes.view(np.uint16), dens)).all()
    with pytest.raises(ValueError):
        m.get_mask_density(mask[:-1], lab)
    with pytest.raises(ValueError):
        m.broadcast_density_to_mask(dens[:-1], lab)
    with pytest.raises(NotImplementedError):
        m.get_knn_connectivity(lab, 4)


@pytest.mark.parametrize("H,W", [(0, 40), (40, 0)])
def test_graph_and_density_consumers_refuse_an_empty_map(H, W):
    """A label map without rows or columns is refused by all three single-image SlicModel methods."""
    from fast_slic_b200 import SlicModel
    K = 10
    m = SlicModel(K)
    lab = np.zeros((H, W), np.int16)
    with pytest.raises(ValueError):
        m.get_connectivity(lab)
    with pytest.raises(ValueError):
        m.get_mask_density(np.zeros((H, W), np.uint8), lab)
    with pytest.raises(ValueError):
        m.broadcast_density_to_mask(np.zeros(K, np.uint8), lab)


def test_connectivity_table_overflow_falls_back_to_the_scan(checker):
    """A label map with far more distinct adjacent pairs than a superpixel map has: the pair table overflows and the
    single-thread replay of the reference's loop takes over (exact, slow)."""
    from fast_slic_b200 import SlicModel
    H, W, K = 256, 256, 3000   # ~196 000 distinct adjacent pairs > the 131 072-entry table of K = 3000
    rng = np.random.RandomState(9)
    lab = rng.randint(0, K, (H, W)).astype(np.uint16).view(np.int16)
    m = SlicModel(K)
    assert m.get_connectivity(lab).tolist() == checker.get_connectivity(lab.view(np.uint16), K)


def test_stream_warm_start_is_the_reference_second_iterate(checker):
    """SlicStream(warm_start=True): image b of batch t+1 starts from the clusters image b of batch t ended with ==
    calling the reference's iterate() again on the same model (cfast_slic.pyx:160 keeps the clusters)."""
    from fast_slic_b200 import SlicStream
    H, W, K, B, T = 120, 160, 40, 3, 4
    frames = [np.stack([make_image("syn", H, W, seed=500 + 10 * b + t, sigma=10.0 + t) for b in range(B)]) for t in range(T)]
    st = SlicStream(H, W, K, batch=B, depth=2, min_size_factor=0.1, warm_start=True)
    got = list(st.map(frames))
    assert len(got) == T and st.in_flight == 0
    for b in range(B):
        cl = checker.initialize(frames[0][b], K)
        for t in range(T):
            want = checker.iterate(frames[t][b], cl, 10, 10.0, 0.1, 3, True)   # cl carries over, like the reference
            assert (got[t][b].view(np.uint16) == want).all(), (b, t)
    st.close()


def test_graph_replay_device_api_rotating_images(checker):
    """fslic_b200_iterate with fewer than 4 images: from the second call with the same cluster / label buffers and
    parameters everything after the Lab kernel is a replayed CUDA graph, whatever image buffer comes in (a video stream).
    Four frames per stream, two streams of images in one batch, on a non-default stream; warm start across frames."""
    from fast_slic_b200 import Engine
    H, W, K, B, T = 120, 160, 40, 2, 5
    eng = Engine(H, W, K, B)
    p = eng.params(10.0, 0.1, 3, True, 10)
    frames = [np.stack([make_image("syn" if (t + b) % 2 else "noise", H, W, seed=700 + 10 * b + t) for b in range(B)])
              for t in range(T)]
    d_frames = [torch.from_numpy(f).cuda() for f in frames]       # a different device buffer every call
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        cl = eng.initialize_clusters(d_frames[0])
        lab = torch.empty((B, H, W), dtype=torch.int16, device="cuda")
        outs = []
        for t in range(T):
            eng.iterate(d_frames[t], cl, p, lab)
            outs.append((lab.clone(), cl.clone()))
    st.synchronize()
    for b in range(B):
        c0 = checker.initialize(frames[0][b], K)
        for t in range(T):
            want = checker.iterate(frames[t][b], c0, 10, 10.0, 0.1, 3, True)   # clusters carry over (warm start)
            assert (outs[t][0][b].cpu().numpy().view(np.uint16) == want).all(), (b, t)
            assert outs[t][1][b].cpu().numpy().tobytes() == c0.tobytes(), (b, t)
    eng.close()


def test_cython_stub_parity(checker, tmp_path):
    """The reference-side Cython binding of INTEGRATION.md section 2 (integration/cfast_slic_b200.pyx), built on the box
    and driven like cfast_slic.SlicModel: same labels and clusters as the compiled reference, cold and warm start."""
    import importlib, os, subprocess, sys
    pytest.importorskip("Cython")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    subprocess.check_call(["bash", os.path.join(root, "integration", "build_stub.sh"), str(tmp_path)],
                          stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    sys.path.insert(0, str(tmp_path))
    try:
        m = importlib.import_module("cfast_slic_b200")
    finally:
        sys.path.pop(0)
    img = make_image("syn", 240, 320, seed=61)
    model = m.SlicModelCuda(120)
    model.convert_to_lab = True
    model.initialize(img)
    cl = checker.initialize(img, 120)
    for _ in range(2):
        got = model.iterate(img, 10, 10.0, 0.1, 3)
        want = checker.iterate(img, cl, 10, 10.0, 0.1, 3, True)
        assert got.dtype == np.int16 and (got.view(np.uint16) == want).all()
        for k, c in enumerate(model.clusters):
            assert c["number"] == k and c["yx"] == (float(cl[k]["y"]), float(cl[k]["x"])) and c["num_members"] == int(cl[k]["num_members"])


REAL_CASES = [("syn", 120, 160, 48, {}), ("noise", 97, 131, 37, dict(min_size_factor=0.0)),
              ("syn", 240, 320, 150, dict(compactness=30.0)), ("blocks", 200, 300, 150, {}),
              ("syn", 150, 200, 30, dict(subsample_stride=2, max_iter=3)), ("flat", 97, 131, 37, {}),
              ("syn", 180, 240, 70, dict(convert_to_lab=False)), ("syn", 480, 640, 200, dict(min_size_factor=0.1)),
              ("thin", 10, 400, 5, {})]


REAL_VARIANTS = ("standard", "l2", "noq")

# the hand-picked cases under every variant, then the seeded sweep (tests/cases.py::real_sweep_case), variant by seed
REAL_SWEEP = [(REAL_VARIANTS[v], c) for c, v in (real_sweep_case(s) for s in REAL_SWEEP_SEEDS)]
REAL_PARAMS = [(v, c) for c in REAL_CASES for v in REAL_VARIANTS] + REAL_SWEEP
REAL_IDS = ["%s_%dx%d_K%d-%s" % (c[:4] + (v,)) for c in REAL_CASES for v in REAL_VARIANTS] + \
           ["sweep%d_%s-%s" % (s, sweep_case_id(c), v) for s, (v, c) in enumerate(REAL_SWEEP)]


@pytest.mark.parametrize("variant,case", REAL_PARAMS, ids=REAL_IDS)
def test_real_dist_variants(checker, variant, case):
    """SlicRealDist / SlicRealDistL2 / SlicRealDistNoQ (fast_slic/base_slic.py:64-85 -> context.cpp:394-499) on the GPU:
    float distances, every operation in the reference's order and rounding -- labels, pre-CCA labels and raw Cluster
    bytes (float centroids of the NoQ variant included) identical to the compiled reference, cold start and warm start,
    on k_assign_real of the variant."""
    import fast_slic_b200 as fs
    kind, H, W, K, kw = case
    kind = "syn" if kind == "thin" else kind
    sigma, args = split_kwargs(kw)
    img = make_image(kind, H, W, seed=41, sigma=sigma)
    cls = {"standard": fs.SlicRealDist, "l2": fs.SlicRealDistL2, "noq": fs.SlicRealDistNoQ}[variant]
    s = cls(num_components=K, compactness=args["compactness"], min_size_factor=args["min_size_factor"],
            subsample_stride=args["subsample_stride"], convert_to_lab=args["convert_to_lab"])
    v = REAL_VARIANTS.index(variant)
    cl = checker.initialize(img, K)
    for round_ in range(2):
        got = s.iterate(img, args["max_iter"]).view(np.uint16)
        want, want_pre = checker.iterate_real(v, img, cl, args["max_iter"], args["compactness"], args["min_size_factor"],
                                              args["subsample_stride"], args["convert_to_lab"], stages=True)
        check_class_call("%s round %d" % (variant, round_), s, got, want, want_pre, cl, REAL_KERNELS[variant],
                          args["max_iter"])


PREEMPT_CASES = [("syn", 120, 160, 48, 0.05, {}), ("syn", 200, 300, 150, 0.05, {}), ("syn", 240, 320, 200, 0.2, dict(max_iter=15)),
                 ("syn", 181, 257, 90, 0.1, dict(subsample_stride=1, max_iter=6)), ("blocks", 240, 320, 64, 0.5, dict(subsample_stride=2)),
                 ("syn", 300, 400, 300, 0.02, {}), ("noise", 120, 160, 48, 0.05, dict(min_size_factor=0.0)),
                 ("syn", 480, 640, 400, 0.05, dict(sigma=4.0)), ("syn", 720, 1280, 1600, 0.05, dict(min_size_factor=0.0))]


PREEMPT_SWEEP = [preempt_sweep_case(s) for s in PREEMPT_SWEEP_SEEDS]
PREEMPT_IDS = ["%s_%dx%d_K%d_t%g" % c[:5] for c in PREEMPT_CASES] + \
              ["sweep%d_%s_t%g" % (s, sweep_case_id(c), c[4]) for s, c in enumerate(PREEMPT_SWEEP)]


@pytest.mark.parametrize("case", PREEMPT_CASES + PREEMPT_SWEEP, ids=PREEMPT_IDS)
def test_preemptive(checker, case):
    """Slic(preemptive=True, preemptive_thres=t) (fast_slic/base_slic.py:12-13 -> preemptive.h, context.cpp:218,307-385):
    clusters that stopped moving drop out of assign and update.  Labels, pre-CCA labels and the raw Cluster records --
    including the is_updatable countdown the reference leaves in them -- identical to the compiled reference, cold and
    warm start, with k_assign_preempt on the update passes; on the hand-picked cases the option really bites (the result
    differs from the non-preemptive one), the seeded sweep (tests/cases.py::preempt_sweep_case) is parity only."""
    import fast_slic_b200 as fs
    kind, H, W, K, thres, kw = case
    sigma, args = split_kwargs(kw)
    img = make_image(kind, H, W, seed=43, sigma=sigma)
    s = fs.Slic(num_components=K, compactness=args["compactness"], min_size_factor=args["min_size_factor"],
                subsample_stride=args["subsample_stride"], convert_to_lab=args["convert_to_lab"], preemptive=True,
                preemptive_thres=thres)
    cl = checker.initialize(img, K)
    plain = checker.iterate(img, checker.initialize(img, K), args["max_iter"], args["compactness"], args["min_size_factor"],
                            args["subsample_stride"], args["convert_to_lab"])
    for round_ in range(2):
        got = s.iterate(img, args["max_iter"]).view(np.uint16)
        want, _, want_pre = checker.iterate(img, cl, args["max_iter"], args["compactness"], args["min_size_factor"],
                                            args["subsample_stride"], args["convert_to_lab"], stages=True, preemptive=True,
                                            preemptive_thres=thres)
        check_class_call("round %d" % round_, s, got, want, want_pre, cl, PREEMPT, args["max_iter"])
        if round_ == 0 and kind != "noise" and case in PREEMPT_CASES:
            assert (want != plain).any(), "the case does not exercise the option"


@pytest.mark.parametrize("K", [900, 3500, 5000])
def test_fused_prepare_tail(checker, K):
    """Batches of one or two images: the last CTA of every assign+update launch does the bookkeeping of the next pass
    (prepare_in_tail, K <= 4096; larger K keeps the k_prepare launch).  Labels and Cluster bytes against the compiled
    reference for one and two images per call, cold and warm start."""
    from fast_slic_b200 import Engine
    H, W = 240, 320
    for B in (1, 2):
        eng = Engine(H, W, K, B)
        p = eng.params(10.0, 0.1, 3, True, 10)
        imgs = np.stack([make_image("syn" if b == 0 else "blocks", H, W, seed=500 + 3 * b + K) for b in range(B)])
        cl = eng.initialize_clusters_host(imgs)
        refcl = [checker.initialize(imgs[b], K) for b in range(B)]
        for round_ in range(2):
            lab = eng.iterate_host(imgs, cl, p)
            for b in range(B):
                want = checker.iterate(imgs[b], refcl[b], 10, 10.0, 0.1, 3, True)
                assert (lab[b].view(np.uint16) == want).all(), (K, B, round_, b)
                assert cl[b].tobytes() == refcl[b].tobytes(), (K, B, round_, b)
        eng.close()


@pytest.mark.parametrize("seed", range(16))
def test_random_configurations(checker, seed):
    """Seeded random shapes (widths that are and are not multiples of 8: TMA and LDG assign kernels), K, compactness,
    min_size_factor, stride, Lab on/off, iteration counts, image kinds: every stage against the compiled reference,
    cold start and warm start."""
    (_, kind, H, W, K, kw), img_seed = gpu_random_config_case(seed)
    sigma, args = split_kwargs(kw)
    img = make_image(kind, H, W, seed=img_seed, sigma=sigma)
    name = "seed%d %dx%d K%d %s %r" % (seed, H, W, K, kind, args)
    _compare(name, _run_cuda(img, K, args), _run_oracle(checker, img, K, args))
    _compare(name + " warm", _run_cuda(img, K, args, iterate_twice=True), _run_oracle(checker, img, K, args, iterate_twice=True))


@pytest.fixture(scope="module")
def sweep_checkers(checker):
    """(Euclidean checker, its extra iterate keyword arguments, LSC checker), chosen as test_euclidean_gpu.py and
    test_lsc_gpu.py choose them: the compiled reference where it was built, else the restatement."""
    from oracle_euclid.euclid import Port as EPort, Ref as ERef
    from oracle_lsc.lsc import Port as LPort, Ref as LRef
    ekw = dict(arch="x64/avx2", num_threads=checker._threads) if ERef.available() else {}
    return ERef() if ERef.available() else EPort(), ekw, LRef() if LRef.available() else LPort()


def _batch_specs():
    """(family, float-distance variant, case (kind, H, W, K, [thres,] kwargs), image kinds, image seed) per input of
    test_iterate_batch_variants: the original three classes on one shape, then every fourth seed of each sweep with three
    images of different kinds."""
    from euclid_cases import EUCLID_PREEMPT_SWEEP, EUCLID_REAL_SWEEP
    from lsc_cases import LSC_SWEEP_CASES
    base, kinds = ("syn", 120, 160, 48, {}), ("syn", "blocks", "syn")
    specs = [("l2", ("real", 1, base, kinds, 610)), ("noq", ("real", 2, base, kinds, 610)),
             ("preemptive", ("preemptive", None, base[:4] + (0.1, {}), kinds, 610))]
    sweeps = [("real", [(v, c) for c, v in (real_sweep_case(s) for s in REAL_SWEEP_SEEDS)]),
              ("preemptive", [(None, c) for c in PREEMPT_SWEEP]),
              ("euclid_real", [(v, c) for c, v in EUCLID_REAL_SWEEP]),
              ("euclid_preemptive", [(None, c) for c in EUCLID_PREEMPT_SWEEP]),
              ("lsc", [(None, c[1:]) for c in LSC_SWEEP_CASES])]
    for family, cases in sweeps:
        for seed in range(0, len(cases), 4):
            v, c = cases[seed]
            three = (c[0],) + tuple(k for k in SWEEP_KINDS if k != c[0])[:2]
            specs.append(("%s_sweep%d%s" % (family, seed, "" if v is None else "_v%d" % v),
                          (family, v, c, three, 620 + seed)))
    return specs


BATCH_SPECS = _batch_specs()


def test_iterate_batch_variants(checker, sweep_checkers):
    """iterate_batch() of the float-distance classes, of Slic(preemptive=True), of both with manhattan_spatial_dist=False
    and of LSC(num_threads=1), on every input of BATCH_SPECS: every image of a host batch and of a device batch equals the
    single-image result of the checker -- labels, pre-CCA labels, Cluster bytes -- and the batch entry ran the class's
    kernel (it must not fall back to the default integer path).  Every input runs; the failure names all that failed."""
    failed = []
    for name, spec in BATCH_SPECS:
        try:
            _check_batch(checker, sweep_checkers, spec)
        except AssertionError as e:
            failed.append("%s: %s" % (name, (str(e).splitlines() or ["assertion failed"])[0]))
    assert not failed, "%d of %d inputs differ:\n%s" % (len(failed), len(BATCH_SPECS), "\n".join(failed))


def _check_batch(checker, sweep_checkers, spec):
    import fast_slic_b200 as fs
    from fast_slic_b200 import get_engine
    family, v, case, kinds, img_seed = spec
    euclid, ekw, lsc_checker = sweep_checkers
    kind, H, W, K = case[:4]
    thres = case[4] if len(case) == 6 else None
    sigma, a = split_kwargs(case[-1])
    args = (a["max_iter"], a["compactness"], a["min_size_factor"], a["subsample_stride"], a["convert_to_lab"])
    B = len(kinds)
    imgs = np.stack([make_image(k, H, W, seed=img_seed + b, sigma=sigma) for b, k in enumerate(kinds)])
    real_cls = (fs.SlicRealDist, fs.SlicRealDistL2, fs.SlicRealDistNoQ)
    cls, ckw, kernel, run = {
        "real": (real_cls[v or 0], {}, 10 + (v or 0),
                 lambda im, cl: checker.iterate_real(v, im, cl, *args, stages=True)),
        "preemptive": (fs.Slic, dict(preemptive=True, preemptive_thres=thres), PREEMPT,
                       lambda im, cl: checker.iterate(im, cl, *args, stages=True, preemptive=True,
                                                      preemptive_thres=thres)[::2]),
        "euclid_real": (real_cls[v or 0], dict(manhattan_spatial_dist=False), 10 + (v or 0),
                        lambda im, cl: euclid.iterate_real(v, im, cl, *args, stages=True)),
        "euclid_preemptive": (fs.Slic, dict(preemptive=True, preemptive_thres=thres, manhattan_spatial_dist=False), PREEMPT,
                              lambda im, cl: euclid.iterate(im, cl, *args, stages=True, preemptive=True,
                                                            preemptive_thres=thres, **ekw)[::2]),
        "lsc": (fs.LSC, dict(num_threads=1), LSC,
                lambda im, cl: (lambda lab, st: (lab, st["pre"]))(*lsc_checker.iterate_lsc(im, cl, *args, stages=True))),
    }[family]
    obj = cls(num_components=K, compactness=a["compactness"], min_size_factor=a["min_size_factor"],
              subsample_stride=a["subsample_stride"], convert_to_lab=a["convert_to_lab"], **ckw)
    want = []
    for b in range(B):
        cl = checker.initialize(imgs[b], K)
        lab, pre = run(imgs[b], cl)
        want.append((lab, pre, cl.tobytes()))
    for where, src in (("host", imgs), ("device", torch.from_numpy(imgs).cuda())):
        lab, cl = obj.iterate_batch(src, max_iter=a["max_iter"], return_clusters=True)
        eng = get_engine(H, W, K, B)
        pre = eng.debug_stages(B)[1].cpu().numpy().view(np.uint16)
        assert_kernel("%s %s" % (family, where), eng.dispatch(), kernel, a["max_iter"])
        if where == "device":
            lab, cl = lab.cpu().numpy(), cl.cpu().numpy()
        for b, (wlab, wpre, wcl) in enumerate(want):
            name = "%s %s image %d (%s)" % (family, where, b, kinds[b])
            assert (pre[b] == wpre).all(), "%s: pre-CCA labels differ (%d px)" % (name, int((pre[b] != wpre).sum()))
            assert (lab[b].view(np.uint16) == wlab).all(), "%s: labels differ" % name
            assert cl[b].tobytes() == wcl, "%s: Cluster bytes differ" % name
