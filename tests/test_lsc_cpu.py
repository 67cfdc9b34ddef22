"""LSC (linear spectral clustering, the reference's ContextLSC) on the CPU: the restatement (oracle_lsc) against the
compiled reference's digests, the evidence behind the num_threads=1 contract, and the refusal rules."""
import os

import numpy as np
import pytest

from cases import digest
from lsc_cases import LSC_CASES, LSC_NAN_CASES, LSC_SWEEP_CASES, lsc_args, lsc_image, lsc_outputs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIGESTS = os.path.join(ROOT, "tests", "golden", "lsc_reference_digests.npz")


@pytest.fixture(scope="module")
def lport():
    from oracle_lsc.lsc import Port
    return Port()


@pytest.fixture(scope="module")
def ref_sha():
    z = np.load(REF_DIGESTS)
    return {k: bytes(v) for k, v in zip(z["keys"].tolist(), z["sha"])}


@pytest.mark.parametrize("case", LSC_CASES + LSC_SWEEP_CASES, ids=[c[0] for c in LSC_CASES + LSC_SWEEP_CASES])
def test_oracle_lsc_matches_compiled_reference(lport, ref_sha, case):
    """Initial clusters, pre-CCA and final labels, Cluster bytes, feature means, pixel weights and the centroid
    features after before_iteration and at the end equal the reference's ContextLSC with num_threads=1, cold and warm."""
    prefix = "lsc/" + case[0]
    want = {k[len(prefix) + 1:]: v for k, v in ref_sha.items() if k.startswith(prefix + "/")}
    got = {k: digest(v) for k, v in lsc_outputs(lport, case).items()}
    assert want and set(got) == set(want), (sorted(got), sorted(want))
    bad = sorted(k for k in got if got[k] != want[k])
    assert not bad, "%s: %s differ from the compiled reference" % (case[0], bad)


def test_cases_reach_the_empty_cluster_path(lport):
    """A cluster that ends a pass without pixels gets 0/0 = NaN centroid features (lsc.cpp:305) and never wins again."""
    for case in LSC_CASES:
        out = lsc_outputs(lport, case)
        nan = any(np.isnan(out["cfinal%d" % r]).any() for r in (0, 1))
        assert nan == (case[0] in LSC_NAN_CASES), case[0]


def test_sweep_reaches_the_empty_cluster_path(lport):
    """The seeded LSC sweep has cases that leave NaN centroid features and cases that do not."""
    nan = [any(np.isnan(out["cfinal%d" % r]).any() for r in (0, 1))
           for out in (lsc_outputs(lport, case) for case in LSC_SWEEP_CASES)]
    assert any(nan) and not all(nan), nan


def test_reference_with_four_threads_changes_the_centroids():
    """The evidence for the num_threads=1 contract: the reference's after_update merges per-thread partial sums
    (lsc.cpp:245-303), so 4 threads give other centroid features than 1."""
    from oracle_lsc.lsc import Ref
    if not os.path.exists(os.path.join(ROOT, "oracle_lsc", "_ref", "libfslic_ref_lsc.so")):
        pytest.skip("oracle_lsc/_ref is built only where FSLIC_REFERENCE names a fast-slic checkout")
    ref = Ref()
    img, K, a = lsc_image(LSC_CASES[0])
    got = []
    for threads in (1, 4):
        cl = ref.initialize(img, K)
        _, st = ref.iterate_lsc(img, cl, *lsc_args(a), stages=True, num_threads=threads)
        got.append(st["cfinal"])
    assert (got[0].view(np.uint32) != got[1].view(np.uint32)).any()


def test_lsc_refusal_rules():
    import torch
    import fast_slic_b200 as fs
    from fast_slic_b200.avx2 import LSCAvx2
    img = np.zeros((16, 16, 3), np.uint8)
    with pytest.raises(NotImplementedError, match="num_threads=1"):
        fs.LSC(num_components=4).iterate(img)  # the default num_threads=-1
    with pytest.raises(NotImplementedError, match="num_threads=1"):
        fs.LSC(num_components=4, num_threads=4).iterate(img)
    with pytest.raises(NotImplementedError, match="rcp_ps"):
        LSCAvx2(num_components=4, num_threads=1).iterate(img)
    with pytest.raises(NotImplementedError, match="preemptive"):
        fs.LSC(num_components=4, num_threads=1, preemptive=True).iterate(img)
    with pytest.raises(NotImplementedError):
        fs.LSC(num_components=4).iterate_batch(img[None])
    ok = fs.LSC(num_components=4, num_threads=1, manhattan_spatial_dist=False, convert_to_lab=False)
    ok.slic_model._unsupported()
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError):
            ok.iterate(img)


def test_abi_declares_the_lsc_entry_points():
    from fast_slic_b200 import _lib
    for sym in ("fslic_b200_iterate_lsc", "fslic_b200_debug_lsc_stages"):
        assert sym in _lib.EXPORTED_SYMBOLS
        assert hasattr(_lib.lib(), sym)
    header = open(os.path.join(ROOT, "include", "fslic_b200.h")).read()
    assert "int fslic_b200_iterate_lsc(" in header and "int fslic_b200_debug_lsc_stages(" in header
