"""Connectivity enforcement on the CPU: the plain-C restatement (oracle.Port, what the GPU tests compare with where the
compiled reference is absent) against the compiled reference's digests on the maps of tests/cca_cases.py, and the host
model of tests/cca_cases.py (what the GPU tests compare the stage's counters with) against a plain BFS and against the
restatement's output."""
import os
import re
from collections import deque

import numpy as np
import pytest

from cases import digest
from cca_cases import (INTENDED, blocky, cca_model, cca_reference_outputs, checkerboard, comb, components, default_k,
                       heap_replacements, random_rect_grid, reference_map_cases, serpentine, spiral, staircase, stripes,
                       with_ffff)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIGESTS = os.path.join(ROOT, "tests", "golden", "cca_reference_digests.npz")


@pytest.fixture(scope="module")
def ref_sha():
    z = np.load(REF_DIGESTS)
    return {k: bytes(v) for k, v in zip(z["keys"].tolist(), z["sha"])}


def test_port_reproduces_reference_digests(port, ref_sha):
    seen = 0
    for prefix, outputs in cca_reference_outputs(port):
        for name, arr in outputs.items():
            key = "%s/%s" % (prefix, name)
            assert key in ref_sha, key
            assert digest(arr) == ref_sha[key], key + " differs from the compiled reference"
            seen += 1
    assert seen == len(ref_sha)


def _bfs_components(lab):
    """Reference-free: 4-connected equal-label components by BFS in raster order of their first pixel."""
    H, W = lab.shape
    comp = np.full((H, W), -1, np.int64)
    leader, area = [], []
    for y0 in range(H):
        for x0 in range(W):
            if comp[y0, x0] >= 0:
                continue
            c = len(leader)
            leader.append(y0 * W + x0)
            comp[y0, x0] = c
            q = deque([(y0, x0)])
            n = 0
            while q:
                y, x = q.popleft()
                n += 1
                for ny, nx in ((y - 1, x), (y + 1, x), (y, x - 1), (y, x + 1)):
                    if 0 <= ny < H and 0 <= nx < W and comp[ny, nx] < 0 and lab[ny, nx] == lab[y, x]:
                        comp[ny, nx] = c
                        q.append((ny, nx))
            area.append(n)
    return comp.ravel(), np.array(leader), np.array(area)


SMALL_MAPS = [("spiral", spiral(37, 45)), ("serpentine", serpentine(21, 40)), ("comb", comb(16, 33)),
              ("checker", checkerboard(13, 17)), ("stripes", stripes(9, 50, 7, 3)), ("stairs", staircase(40, 30, 3)),
              ("grid", random_rect_grid(40, 50, [1, 2, 5], [1, 3, 4], 3)), ("ffff", with_ffff(blocky(30, 41, 4, 9), 2)),
              ("many_labels", blocky(35, 29, 40, 4, cell=2)), ("row", blocky(1, 77, 3, 5, cell=2)),
              ("col", blocky(61, 1, 3, 6, cell=2))]


@pytest.mark.parametrize("name,lab", SMALL_MAPS, ids=[m[0] for m in SMALL_MAPS])
def test_model_components_match_bfs(name, lab):
    comp, leader, area = components(lab)
    bcomp, bleader, barea = _bfs_components(lab)
    assert (comp == bcomp).all() and (leader == bleader).all() and (area == barea).all()


@pytest.mark.parametrize("name,lab", SMALL_MAPS, ids=[m[0] for m in SMALL_MAPS])
@pytest.mark.parametrize("K,thres", [(1, 0), (2, 1), (3, 3), (10, 2), (65535, 5), (4, 10 ** 6)])
def test_model_labels_match_restatement(port, name, lab, K, thres):
    """The model's output map (kept set resolved by libstdc++'s std::partial_sort where ties make it ambiguous) and its
    branch bookkeeping are consistent with the restatement's output."""
    m = cca_model(lab, K, thres, port=port)
    assert (m["labels"] == port.enforce_connectivity(lab, K, thres)).all()
    assert m["nkept"] == min(K, m["ncand"]) and int(m["labels"].max()) < max(1, m["nkept"])
    if m["branch"] != "all":
        assert m["G"] < K <= m["G"] + m["E"] and m["need_sim"] == (m["E"] != K - m["G"])


def test_heap_replacements_match_a_plain_replay():
    """heapq's count against a literal list-based __heap_select (pop the minimum, push the new element)."""
    rng = np.random.RandomState(3)
    for n, K, top in [(50, 7, 3), (400, 1, 4), (400, 2, 2), (1000, 333, 6), (64, 64, 5)]:
        a = rng.randint(1, top + 1, n)
        h = sorted(a[:K].tolist())
        ops = 0
        for v in a[K:]:
            if v > h[0]:
                h[0] = int(v)
                h.sort()
                ops += 1
        assert heap_replacements(a, K) == ops


def test_reference_maps_reach_their_branches(port):
    """Each map of the digest set reaches what its name says (if a builder drifts, this fails rather than the digest
    test silently covering something else)."""
    cases = reference_map_cases()
    assert sorted(INTENDED) == sorted(c[0] for c in cases)
    for name, lab, K, thres in cases:
        m = cca_model(lab, default_k(lab) if K is None else K, thres)
        assert (m["branch"], m["need_sim"]) == INTENDED[name], name
        if name.startswith(("grid2047_hist", "grid2047_thres_t")):
            assert m["t"] == 2047 and m["branch"] == "hist", name
    cases = {c[0]: c for c in reference_map_cases()}
    g = cases["grid2047_hist_unamb"][1]
    area = components(g)[2]
    assert {2047, 2048, 2049} <= set(area.tolist())
    assert cases["grid2047_K1"][2] == 1 and cases["grid2047_K2"][2] == 2
    assert cases["grid2047_thres_gt_N"][3] > g.size


def test_abi_declares_the_connectivity_read_back():
    """fslic_b200_debug_cca_dispatch: exported, bound with a pointer argument, and documented field by field in the
    header in the order Engine.dispatch()["cca"] names them."""
    from fast_slic_b200 import _lib
    L = _lib.lib()
    assert "fslic_b200_debug_cca_dispatch" in _lib.EXPORTED_SYMBOLS
    assert L.fslic_b200_debug_cca_dispatch.argtypes is not None
    header = open(os.path.join(ROOT, "include", "fslic_b200.h")).read()
    assert "int fslic_b200_debug_cca_dispatch(const fslic_ctx* ctx, int32_t* out, int count);" in header
    assert re.search(r"#define FSLIC_CCA_DISPATCH_COUNT (\d+)", header).group(1) == str(_lib.CCA_DISPATCH_COUNT)
    for i, name in enumerate(_lib.CCA_DISPATCH_FIELDS):
        assert re.search(r"\[%d\]\s+%s:" % (i, name), header), name
