"""debug_mode without a GPU: the host-only report formatter (fslic_b200_format_report) against a Python restatement of
recorder.h's text, its number formatting corner cases, the C header, and the pinned reference digests."""
import os
import re

import numpy as np
import pytest

from fast_slic_b200 import CLUSTER_DTYPE, _lib
from recorder_cases import CASES

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _g(v):
    """ostream << float with default flags == printf %.6g of the value as a double."""
    return "%.6g" % float(np.float32(v))


def _python_report(H, W, assignment, min_dists, clusters):
    snaps = []
    for s in range(clusters.shape[0]):
        cl = ",".join(
            '{"yx": [%s,%s], "color": [%s,%s,%s], "is_updatable": %d, "is_active": %d, "number": %d, "num_members": %d}'
            % (_g(c["y"]), _g(c["x"]), _g(c["r"]), _g(c["g"]), _g(c["b"]), c["is_updatable"], c["is_active"],
               c["number"], c["num_members"]) for c in clusters[s])
        fmt = _g if min_dists.dtype == np.float32 else str
        snaps.append('{"iteration": %d, "clusters": [%s], "assignment": [%s], "min_dists": [%s]}' % (
            s - 1, cl, ",".join(str(int(a)) for a in assignment[s].ravel()),
            ",".join(fmt(d) for d in min_dists[s].ravel())))
    return ('{"height": %d, "width": %d, "snapshots": [%s]}' % (H, W, ",".join(snaps))).encode()


def _random_snapshots(T, H, W, K, dist_dtype, rng):
    assignment = rng.randint(0, 65536, size=(T, H * W)).astype(np.uint16)
    if dist_dtype == np.uint16:
        dist = rng.randint(0, 65536, size=(T, H * W)).astype(np.uint16)
    else:
        dist = (rng.standard_normal((T, H * W)) * 10.0 ** rng.randint(-8, 9, size=(T, H * W))).astype(np.float32)
    cl = np.zeros((T, K), CLUSTER_DTYPE)
    for f in ("y", "x", "r", "g", "b"):
        cl[f] = (rng.random_sample((T, K)) * 300).astype(np.float32)
    cl["y"][:, ::2] = np.round(cl["y"][:, ::2])
    cl["number"] = rng.randint(0, 65536, size=(T, K))
    cl["is_active"] = rng.randint(0, 256, size=(T, K))
    cl["is_updatable"] = rng.randint(0, 3, size=(T, K))
    cl["num_members"] = rng.randint(0, 2 ** 32, size=(T, K), dtype=np.uint64)
    return assignment, dist, cl


@pytest.mark.parametrize("dist_dtype", [np.uint16, np.float32])
def test_formatter_matches_recorder_text(dist_dtype):
    rng = np.random.RandomState(3)
    H, W, K, T = 5, 7, 4, 3
    a, d, cl = _random_snapshots(T, H, W, K, dist_dtype, rng)
    assert _lib.format_recorder_report(H, W, a, d, cl) == _python_report(H, W, a, d, cl)


def test_formatter_number_corner_cases():
    specials = np.array([65535, np.finfo(np.float32).max, -0.0, 0.0, 1e-5, 12.345678, 1e6, 999999, -3.5, np.inf,
                         -np.inf, 123456.7, 2 ** 24, 1.17549435e-38], np.float32)
    H, W = 1, len(specials)
    cl = np.zeros((1, 1), CLUSTER_DTYPE)
    cl["y"], cl["x"], cl["r"] = 12.3456789, -0.0, 1e-5  # non-integer NoQ-style centroids
    a = np.full((1, W), 65535, np.uint16)
    rep = _lib.format_recorder_report(H, W, a, specials[None], cl)
    assert rep == _python_report(H, W, a, specials[None], cl)
    text = rep.decode()
    assert '"yx": [12.3457,-0]' in text and '"color": [1e-05,0,0]' in text
    assert ('"min_dists": [65535,3.40282e+38,-0,0,1e-05,12.3457,1e+06,999999,-3.5,inf,-inf,123457,1.67772e+07,'
            '1.17549e-38]') in text
    u16 = _lib.format_recorder_report(H, W, a, np.full((1, W), 65535, np.uint16), cl).decode()
    assert u16.endswith('"min_dists": [' + ",".join(["65535"] * W) + ']}]}')


def test_formatter_max_iter_zero_and_empty():
    cl = np.zeros((1, 2), CLUSTER_DTYPE)
    a = np.full((1, 6), 65535, np.uint16)
    d = np.zeros((1, 6), np.uint16)
    rep = _lib.format_recorder_report(2, 3, a, d, cl)
    assert rep.startswith(b'{"height": 2, "width": 3, "snapshots": [{"iteration": -1, "clusters": [{"yx": [0,0]')
    assert rep.endswith(b'"assignment": [65535,65535,65535,65535,65535,65535], "min_dists": [0,0,0,0,0,0]}]}')
    empty = _lib.format_recorder_report(2, 3, a[:0], d[:0], cl[:0])
    assert empty == b'{"height": 2, "width": 3, "snapshots": []}'
    # no pixels and no clusters: the report is all fixed text, which the buffer must hold on its own
    T = 200
    z = np.zeros((T, 0), np.uint16)
    rep = _lib.format_recorder_report(0, 0, z, z, np.zeros((T, 0), CLUSTER_DTYPE))
    assert rep == _python_report(0, 0, z, z, np.zeros((T, 0), CLUSTER_DTYPE))


def test_formatter_longest_values():
    """Every pixel at its longest text: assignment 65535 and a 12-character float min_dist, 19 bytes with their
    separators, few clusters to pad the buffer.  A buffer sized for one 16-byte value per pixel ran past its end here
    (an LSC report of a stride-255 call with K = 2: unreached rows keep 65535 and FLT_MAX)."""
    H, W, T = 40, 50, 3
    a = np.full((T, H * W), 65535, np.uint16)
    d = np.full((T, H * W), -1.17549435e-38, np.float32)
    d[:, ::3] = np.finfo(np.float32).max
    cl = np.zeros((T, 1), CLUSTER_DTYPE)
    rep = _lib.format_recorder_report(H, W, a, d, cl)
    assert rep == _python_report(H, W, a, d, cl)
    assert len(rep) > T * H * W * 18


def test_new_symbols_declared_in_header():
    header = open(os.path.join(ROOT, "include", "fslic_b200.h")).read()
    declared = set(re.findall(r"\b(fslic_b200_\w+)\s*\(", header))
    for sym in ("fslic_b200_set_trace", "fslic_b200_trace_info", "fslic_b200_trace_snapshots",
                "fslic_b200_format_report", "fslic_b200_free_report", "fslic_b200_debug_graph_counts"):
        assert sym in declared and sym in _lib.EXPORTED_SYMBOLS, sym


def test_reference_digests_cover_every_case():
    g = np.load(os.path.join(ROOT, "tests", "golden", "recorder_reference_digests.npz"))
    assert sorted(g["names"].tolist()) == sorted(c.name for c in CASES)
    assert all(len(h) == 64 for h in g["sha256"].tolist())


def test_reference_report_matches_digest_where_built():
    """The compiled reference (where oracle/_ref holds it) still gives the pinned bytes."""
    import hashlib
    from oracle.recorder import RecorderRef
    from recorder_cases import reference_report
    if not RecorderRef.available():
        pytest.skip("oracle/_ref/libfslic_ref_recorder.so is not built (make -C oracle -f recorder.mk ref)")
    g = np.load(os.path.join(ROOT, "tests", "golden", "recorder_reference_digests.npz"))
    digest = dict(zip(g["names"].tolist(), g["sha256"].tolist()))
    ref = RecorderRef()
    for case in CASES:
        assert hashlib.sha256(reference_report(case, ref)).hexdigest() == digest[case.name], case.name


def test_debug_mode_selects_the_traced_path():
    """debug_mode=False keeps the empty report; debug_mode=True traces every class (LSC at num_threads=1 included)."""
    import fast_slic_b200 as fs
    from fast_slic_b200.avx2 import SlicAvx2
    from fast_slic_b200.base_slic import EMPTY_RECORDER_REPORT
    assert EMPTY_RECORDER_REPORT == b'{"snapshots":[]}'
    for cls in (fs.Slic, SlicAvx2, fs.SlicRealDist, fs.SlicRealDistL2, fs.SlicRealDistNoQ, fs.LSC):
        for debug in (False, True):
            m = cls(num_components=8, debug_mode=debug, num_threads=1).slic_model
            m._unsupported()
            assert m._traced() is debug, (cls.__name__, debug)
