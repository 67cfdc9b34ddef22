"""Absorption of unkept components on the GPU (k_ccl_flatten's predecessor roots, k_kept_label, k_cca_absorb) against the
compiled reference (conftest.Checker) and the host model of tests/cca_cases.py, tolerance 0.  The maps put component
leaders where the predecessor root is found in different ways: at lane 0 of a 32-pixel chunk and at the start of a
1024-pixel block (ccl_find across the chunk or block boundary), in column 0 (the root above), on images whose pixel
count is not a multiple of 1024, and in absorb chains that run through many blocks.
"""
import numpy as np
import pytest
import torch

from cca_cases import blocky, cca_model, components, random_rect_grid, serpentine, staircase, stripes, with_ffff

pytestmark = pytest.mark.gpu

COUNTERS = ("ncomp", "ncand", "nkept", "sel_mode", "keep_thres", "need_sim", "heap_ops", "kth_area")
_engines = {}


@pytest.fixture(scope="module", autouse=True)
def _free_contexts():
    yield
    for e in _engines.values():
        e.close()
    _engines.clear()


def _engine(H, W, B=1):
    from fast_slic_b200 import Engine
    key = (H, W, B)
    if key not in _engines:
        _engines[key] = Engine(H, W, max_batch=B, cca_only=True)
    return _engines[key]


def _run(eng, maps, K, thres):
    t = torch.from_numpy(np.ascontiguousarray(maps).view(np.int16)).to(eng.device)
    eng.enforce_connectivity(t, K, thres)
    torch.cuda.synchronize()
    return t.cpu().numpy().view(np.uint16)


def _check(eng, slot, got, lab, K, thres, checker, port, what):
    m = cca_model(lab, K, thres, port=port)
    want = checker.enforce_connectivity(lab, K, thres)
    assert (got == want).all(), "%s: %d px differ from the reference" % (what, int((got != want).sum()))
    assert (got == m["labels"]).all(), "%s: %d px differ from the model" % (what, int((got != m["labels"]).sum()))
    c = eng.cca_counters(slot)
    assert {k: c[k] for k in COUNTERS} == {k: int(m[k]) for k in COUNTERS}, what
    return m


def _run1(lab, K, thres, checker, port, what):
    H, W = lab.shape
    eng = _engine(H, W)
    got = _run(eng, lab[None], K, thres)[0]
    return _check(eng, 0, got, lab, K, thres, checker, port, what)


def chunk_runs(H, W, seed):
    """Rows of runs whose lengths are multiples of 32 px and labels that differ from the run above: with W a multiple of
    32 every run starts at lane 0 of a chunk, many of them at the start of a 1024-pixel block."""
    rng = np.random.RandomState(seed)
    lab = np.zeros((H, W), np.uint16)
    for y in range(H):
        x = 0
        while x < W:
            n = 32 * int(rng.randint(1, 4))
            lab[y, x:x + n] = (y % 2) * 4 + int(rng.randint(0, 4))
            x += n
    return lab


@pytest.mark.parametrize("H,W,K,thres", [(64, 1024, 3, 0), (96, 96, 10, 40), (40, 2048, 1, 0), (33, 320, 7, 33)])
def test_roots_at_chunk_and_block_starts(checker, port, H, W, K, thres):
    lab = chunk_runs(H, W, H + W)
    _, leader, _ = components(lab)
    assert (leader % 32 == 0).all() and ((leader % 1024 == 0) & (leader > 0)).any()
    m = _run1(lab, K, thres, checker, port, "chunk_runs %dx%d" % (H, W))
    assert m["nkept"] < m["ncomp"]


@pytest.mark.parametrize("W", [1, 33, 1281])
@pytest.mark.parametrize("kind", ["staircase", "blocky"])
def test_column0_leaders(checker, port, W, kind):
    """Leaders in column 0 take the component above them (cca.cpp:246)."""
    H = 300
    lab = staircase(H, W, 5) if kind == "staircase" else blocky(H, W, 3, W, cell=2)
    _, leader, area = components(lab)
    assert ((leader % W == 0) & (leader > 0)).any()
    K = max(1, len(area) // 7)
    m = _run1(lab, K, 0, checker, port, "%s W=%d" % (kind, W))
    assert m["nkept"] < m["ncomp"]


@pytest.mark.parametrize("H,W", [(37, 33), (1, 1023), (129, 1025), (7, 3001)])
def test_pixel_count_not_a_multiple_of_1024(checker, port, H, W):
    lab = blocky(H, W, 4, H * 31 + W, cell=3)
    assert (H * W) % 1024 != 0
    _run1(lab, max(1, H * W // 300), 2, checker, port, "blocky %dx%d" % (H, W))


def test_chains_through_many_blocks(checker, port):
    """Narrow stripes absorbed through the chain of narrow stripes to their left: chains of up to 1500 components
    whose leaders lie in row 0, across two 1024-pixel blocks; and a serpentine whose background runs are absorbed
    into the path."""
    lab = stripes(40, 3100, 1500, 5)
    m = _run1(lab, 65535, 41, checker, port, "stripes")
    assert m["hops"] > 1000000, m["hops"]
    _run1(serpentine(301, 777), 1, 0, checker, port, "serpentine")


@pytest.mark.parametrize("H,W", [(200, 300), (1, 1)])
def test_all_unkept_at_k1(checker, port, H, W):
    """No candidate at all (threshold above every area): every component, component 0 included, ends up 0."""
    lab = blocky(H, W, 5, 3, cell=4)
    m = _run1(lab, 1, H * W + 1, checker, port, "all unkept %dx%d" % (H, W))
    assert m["nkept"] == 0 and m["ncand"] == 0


def test_label_ffff_in_input(checker, port):
    lab = with_ffff(blocky(150, 257, 6, 9, cell=3), 2)
    assert (lab == 0xFFFF).any()
    _run1(lab, 40, 5, checker, port, "ffff")


def test_mixed_batch_of_eight(checker, port):
    """8 maps of 200 x 300 (not a multiple of 1024 px): even images need the std::partial_sort replay, odd ones are
    settled by k_cca_threshold, so the settled tail runs on the side stream while the replay runs.  Threshold 2: the
    single-pixel specks of the odd images are absorbed too."""
    K, thres = 4000, 2
    maps = np.stack([random_rect_grid(200, 300, [1, 2], [1, 2, 3], 70 + b) if b % 2 == 0 else
                     blocky(200, 300, 4, 80 + b, cell=5, speckle=0.05) for b in range(8)])
    eng = _engine(200, 300, 8)
    got = _run(eng, maps, K, thres)
    d = eng.dispatch()["cca"]
    assert d["sub_batches"] == 1 and d["split"] == 1, d
    sims = []
    for b in range(8):
        m = _check(eng, b, got[b], maps[b], K, thres, checker, port, "image %d" % b)
        assert m["nkept"] < m["ncomp"]
        sims.append(m["need_sim"])
    assert sims == [1, 0] * 4, sims
