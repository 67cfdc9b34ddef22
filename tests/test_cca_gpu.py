"""Connectivity enforcement on the GPU against the compiled reference (conftest.Checker) at tolerance 0, on maps aimed at
the branches of fast_slic_b200/csrc/cca.cuh that real images rarely reach: the selection heap in global memory, each way
k_cca_threshold finds the K-th largest area, long-range topology, batches mixing replayed and settled images, and SLIC at
large K.  Every case also compares each image's counters (Engine.cca_counters) with the host model of tests/cca_cases.py
and asserts the branch it is there for, from the model and from the launch read-back (Engine.dispatch()["cca"]): a
case that drifts out of its branch fails.
"""
import numpy as np
import pytest
import torch

from cases import make_image
from cca_cases import INTENDED, bands, blocky, cca_model, default_k, random_rect_grid, reference_map_cases

pytestmark = pytest.mark.gpu

COUNTERS = ("ncomp", "ncand", "nkept", "sel_mode", "keep_thres", "need_sim", "heap_ops", "kth_area")
MAX_HOPS = 10 ** 8  # absorb-chain steps per case (k_cca_absorb walks chains without path compression)
_engines = {}


@pytest.fixture(scope="module", autouse=True)
def _free_contexts():
    yield
    from fast_slic_b200 import clear_engine_cache
    for e in _engines.values():
        e.close()
    _engines.clear()
    clear_engine_cache()


def _engine(H, W, B=1):
    from fast_slic_b200 import Engine
    key = (H, W, B)
    if key not in _engines:
        _engines[key] = Engine(H, W, max_batch=B, cca_only=True)
    return _engines[key]


def _close(H, W, B=1):
    e = _engines.pop((H, W, B), None)
    if e is not None:
        e.close()


def _run(eng, maps, K, thres):
    """enforce_connectivity of the u16 maps [B,H,W] on `eng` with an explicit K -> (labels u16 [B,H,W], ms)."""
    t = torch.from_numpy(np.ascontiguousarray(maps).view(np.int16)).to(eng.device)
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    eng.enforce_connectivity(t, K, thres)
    end.record()
    torch.cuda.synchronize()
    return t.cpu().numpy().view(np.uint16), start.elapsed_time(end)


def _check_counters(eng, slot, m, what):
    got = eng.cca_counters(slot)
    assert {k: got[k] for k in COUNTERS} == {k: int(m[k]) for k in COUNTERS}, what


def _check_labels(got, want, what):
    assert (got == want).all(), "%s: %d px differ from the reference" % (what, int((got != want).sum()))


@pytest.fixture(scope="module")
def max_k():
    """The largest K whose selection heap fits shared memory on this device (from the launch read-back)."""
    eng = _engine(8, 8)
    _run(eng, np.zeros((1, 8, 8), np.uint16), 5, 0)
    d = eng.dispatch()["cca"]
    assert d["heap_smem"] == 1 and d["heap_smem_max_k"] >= 1000, d
    return d["heap_smem_max_k"]


def _resolve_k(spec, max_k):
    return {"max_k": max_k, "max_k+1": max_k + 1}.get(spec, spec)


# ---- the std::partial_sort heap in global memory -------------------------------------------------------------------
@pytest.mark.parametrize("middle", ["max_k", "max_k+1", 20000, 65535])
def test_heap_select_device_vs_stl_large_middle(port, max_k, middle):
    """k_debug_heap_select at and beyond the shared-memory limit: 2^20 areas drawn from 1..6, so tens of thousands
    of tie-heavy heap replacements, against libstdc++'s std::partial_sort."""
    middle = _resolve_k(middle, max_k)
    rng = np.random.RandomState(middle)
    area = rng.randint(1, 7, 1 << 20).astype(np.int32)
    kept = _engine(8, 8).debug_heap_select(torch.from_numpy(area), middle).cpu().numpy()
    want = port.stl_partial_sort(area, middle)
    got = np.nonzero(kept)[0]
    assert len(got) == middle and (got == want).all()


@pytest.fixture(scope="module")
def ties_map():
    return random_rect_grid(600, 800, [1, 2], [1, 2, 3], 11)  # ~160 000 components of areas 1..6


@pytest.mark.parametrize("K", ["max_k", "max_k+1", 30000, 65535])
def test_enforce_heap_placement(checker, port, max_k, ties_map, K):
    """need_sim images at K on both sides of the shared-memory limit: the replay runs with the heap in shared memory
    at max_k, in global memory above it."""
    K = _resolve_k(K, max_k)
    lab = ties_map
    m = cca_model(lab, K, 0, port=port)
    assert m["need_sim"] == 1 and m["heap_ops"] > 1000 and m["hops"] <= MAX_HOPS, m
    eng = _engine(*lab.shape)
    got, _ = _run(eng, lab[None], K, 0)
    d = eng.dispatch()["cca"]
    assert d["heap_smem"] == (1 if K <= max_k else 0) and d["heap_smem_max_k"] == max_k, d
    _check_labels(got[0], checker.enforce_connectivity(lab, K, 0), "K=%d" % K)
    _check_labels(got[0], m["labels"], "K=%d (model)" % K)
    _check_counters(eng, 0, m, "K=%d" % K)


# ---- the maps pinned to the compiled reference (threshold branches, topology, widths) ------------------------------
MAPS = reference_map_cases()


@pytest.mark.parametrize("case", MAPS, ids=[c[0] for c in MAPS])
def test_reference_maps(checker, port, max_k, case):
    """Explicit K on an Engine(cca_only=True); the maps without one go through the public enforce_connectivity (K =
    max label + 1 over labels != 0xFFFF)."""
    name, lab, K, thres = case
    H, W = lab.shape
    explicit = K is not None
    K = K if explicit else default_k(lab)
    m = cca_model(lab, K, thres, port=port)
    assert (m["branch"], m["need_sim"]) == INTENDED[name], (name, m["branch"], m["need_sim"])
    assert m["hops"] <= MAX_HOPS
    if explicit:
        eng = _engine(H, W)
        got, ms = _run(eng, lab[None], K, thres)
        got = got[0]
    else:
        from fast_slic_b200 import base_slic, enforce_connectivity
        got = enforce_connectivity(lab.copy().view(np.int16), thres).view(np.uint16)
        eng = base_slic.get_cca_engine(H, W)
        ms = float("nan")
    d = eng.dispatch()["cca"]
    assert d["heap_smem"] == (1 if K <= max_k else 0) and d["sub_batches"] == 1 and d["split"] == 0, d
    print("\n%s: %dx%d K=%d thres=%d branch=%s need_sim=%d heap_ops=%d hops=%d, %.2f ms" % (
        name, H, W, K, thres, m["branch"], m["need_sim"], m["heap_ops"], m["hops"], ms))
    _check_labels(got, checker.enforce_connectivity(lab, K, thres), name)
    _check_counters(eng, 0, m, name)


@pytest.mark.parametrize("K,need_sim", [(1, 1), (2, 0)])
def test_three_pass_radix_select(checker, K, need_sim):
    """N >= 2^22 and n_big >= K: the three-pass radix select.  Two bands of 4 200 000 px (t = 0x401640: all three
    11-bit digits non-zero) and one of 600 000 px on a 3000 x 3000 map; K = 1 ties the two bands (need_sim, K = 1
    skips make_heap), K = 2 keeps exactly them."""
    lab = bands(3000, 3000, [1400, 1400])
    m = cca_model(lab, K, 0)
    assert (m["branch"], m["need_sim"], m["t"], m["n_big"]) == ("radix3", need_sim, 4200000, 3), m
    assert all((m["t"] >> s) & 2047 for s in (0, 11, 22))
    eng = _engine(3000, 3000)
    got, _ = _run(eng, lab[None], K, 0)
    _check_labels(got[0], checker.enforce_connectivity(lab, K, 0), "K=%d" % K)
    _check_counters(eng, 0, m, "K=%d" % K)
    _close(3000, 3000)


# ---- batches of the standalone entry point -------------------------------------------------------------------------
BATCH_K = 5000


def _mixed_batch():
    """8 maps of 256 x 256: even images are tie-heavy grids of ~22 000 components (need_sim at K = 5000), odd ones
    coarse blocks with fewer candidates than K (settled)."""
    return np.stack([random_rect_grid(256, 256, [1, 2], [1, 2, 3], 40 + b) if b % 2 == 0 else
                     blocky(256, 256, 4, 50 + b, cell=16, speckle=0.0) for b in range(8)])


@pytest.fixture(scope="module")
def mixed(checker, port):
    maps = _mixed_batch()
    models = [cca_model(maps[b], BATCH_K, 0, port=port) for b in range(8)]
    assert [m["need_sim"] for m in models] == [1, 0] * 4
    want = [checker.enforce_connectivity(maps[b], BATCH_K, 0) for b in range(8)]
    return maps, models, want


def test_batch_mixing_replayed_and_settled_images(mixed):
    """One sub-batch of 8, split: the settled images' tail runs on the side stream (which = 0) while the replay runs,
    the replayed images' tail after it (which = 1)."""
    maps, models, want = mixed
    eng = _engine(256, 256, 8)
    got, _ = _run(eng, maps, BATCH_K, 0)
    d = eng.dispatch()["cca"]
    assert d["sub_batches"] == 1 and d["split"] == 1 and d["heap_smem"] == 1, d
    for b in range(8):
        _check_labels(got[b], want[b], "image %d" % b)
        _check_counters(eng, b, models[b], "image %d" % b)


def test_batch_in_sub_batches(monkeypatch, mixed):
    """The same batch on a context whose scratch holds 3 images (FSLIC_CCA_BATCH is read at context creation): sub-
    batches of 3, 3, 2 images, none split; the counters are those of the last sub-batch."""
    from fast_slic_b200 import Engine
    maps, models, want = mixed
    monkeypatch.setenv("FSLIC_CCA_BATCH", "3")
    eng = Engine(256, 256, max_batch=8, cca_only=True)
    try:
        got, _ = _run(eng, maps, BATCH_K, 0)
        d = eng.dispatch()["cca"]
        assert d["sub_batches"] == 3 and d["split"] == 0, d
        for b in range(8):
            _check_labels(got[b], want[b], "image %d" % b)
        for slot, b in enumerate((6, 7)):
            _check_counters(eng, slot, models[b], "image %d" % b)
    finally:
        eng.close()


def test_batch_large_images_numbering_chunks(checker, port):
    """8 images of 4096 x 4100 (16.8 M px): k_ccl_number's warps own more than 32 blocks each, so its outer chunk loop
    takes a second trip.  Two maps alternate: ~150 000 components with a tie at K = 65535 (need_sim), and 4096 coarse
    blocks (settled)."""
    H, W, K = 4096, 4100, 65535
    a = blocky(H, W, 4, 61, cell=8, speckle=0.002)
    b = blocky(H, W, 4, 62, cell=64, speckle=0.0)
    ma, mb = cca_model(a, K, 0, port=port), cca_model(b, K, 0, port=port)
    assert (ma["need_sim"], mb["need_sim"]) == (1, 0) and ma["hops"] + mb["hops"] <= MAX_HOPS / 4
    wa, wb = checker.enforce_connectivity(a, K, 0), checker.enforce_connectivity(b, K, 0)
    maps = np.stack([a, b] * 4)
    eng = _engine(H, W, 8)
    got, ms = _run(eng, maps, K, 0)
    del maps
    d = eng.dispatch()["cca"]
    assert d["number_nb"] > 32 and d["sub_batches"] == 1 and d["split"] == 1 and d["heap_smem"] == 0, d
    print("\n4096x4100 x 8, K=65535: %s, %.1f ms" % (d, ms))
    for i in range(8):
        _check_labels(got[i], (wa, wb)[i % 2], "image %d" % i)
        _check_counters(eng, i, (ma, mb)[i % 2], "image %d" % i)
    _close(H, W, 8)


# ---- SLIC at large K -----------------------------------------------------------------------------------------------
def _slic_case(checker, imgs, K, batch_device):
    """Slic(num_components=K, min_size_factor=0) on `imgs` against the reference: final labels, pre-CCA labels and
    Cluster bytes of every image, the connectivity counters against the model on the pre-CCA labels, and the read-back."""
    from fast_slic_b200 import Slic, get_engine
    B, H, W, _ = imgs.shape
    slic = Slic(num_components=K, min_size_factor=0.0)
    if batch_device:
        lab, cl = slic.iterate_batch(torch.from_numpy(imgs).cuda(), return_clusters=True)
        lab, cl = lab.cpu().numpy().view(np.uint16), cl.cpu().numpy()
    else:
        lab, cl = slic.iterate(imgs[0])[None].view(np.uint16), slic.slic_model.cluster_array[None]
    eng = get_engine(H, W, K, B)
    d = eng.dispatch()
    _, pre = eng.debug_stages(B)
    pre = pre.cpu().numpy().view(np.uint16)
    for b in range(B):
        wcl = checker.initialize(imgs[b], K)
        wlab, _, wpre = checker.iterate(imgs[b], wcl, 10, 10.0, 0.0, 3, True, stages=True)
        _check_labels(pre[b], wpre, "pre-CCA labels of image %d" % b)
        _check_labels(lab[b], wlab, "labels of image %d" % b)
        assert cl[b].tobytes() == wcl.tobytes(), "clusters of image %d" % b
        m = cca_model(pre[b], K, 0)
        _check_counters(eng, b, m, "image %d" % b)
    return d


def test_slic_k20000_1080p(checker):
    img = make_image("syn", 1080, 1920, seed=71)[None]
    d = _slic_case(checker, img, 20000, False)
    assert d["prepare"] == 2 and d["cca"]["heap_smem"] == 0, d


def test_slic_k20000_1080p_batch8(checker):
    imgs = np.stack([make_image("syn", 1080, 1920, seed=80 + b, sigma=(12.0, 40.0)[b % 2]) for b in range(8)])
    d = _slic_case(checker, imgs, 20000, True)
    assert d["prepare"] == 1 and d["cca"]["heap_smem"] == 0 and d["cca"]["split"] == 1, d


def test_slic_k65533_4k(checker):
    from fast_slic_b200 import clear_engine_cache
    img = make_image("tiled", 2160, 3840, seed=91)[None]
    d = _slic_case(checker, img, 65533, False)
    assert d["prepare"] == 2 and d["cca"]["heap_smem"] == 0, d
    clear_engine_cache()
