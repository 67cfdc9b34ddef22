"""SimpleCRF on the CPU: the restatement (oracle_crf) and, where it is built, the compiled reference against the
reference's digests; the expf clone's host compile against glibc on every input; refusal rules that need no device;
the ABI."""
import hashlib
import os

import numpy as np
import pytest

from cases import digest
from crf_cases import CRF_CASES, run_case

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIGESTS = os.path.join(ROOT, "tests", "golden", "crf_reference_digests.npz")
REF_LIB = os.path.join(ROOT, "oracle_crf", "_ref", "libfslic_ref_crf.so")


@pytest.fixture(scope="module")
def ref_sha():
    z = np.load(REF_DIGESTS)
    return {k: bytes(v) for k, v in zip(z["keys"].tolist(), z["sha"])}


def _check_case(model_cls, ref_sha, case):
    prefix = "crf/" + case[0] + "/"
    want = {k[len(prefix):]: v for k, v in ref_sha.items() if k.startswith(prefix)}
    got = {k: digest(v) for k, v in run_case(model_cls(case[1], case[2]), case).items()}
    assert want and set(got) == set(want), (sorted(got), sorted(want))
    bad = sorted(k for k in got if got[k] != want[k])
    assert not bad, "%s: %s differ from the compiled reference" % (case[0], bad)


@pytest.mark.parametrize("case", CRF_CASES, ids=[c[0] for c in CRF_CASES])
def test_oracle_crf_matches_compiled_reference(ref_sha, case):
    """Unaries, q after initialize() and after each inference(), and the pairwise energies of the restatement are
    byte-identical (NaN payloads included) to the reference's."""
    from oracle_crf.crf import Port
    _check_case(Port, ref_sha, case)


@pytest.mark.parametrize("case", CRF_CASES, ids=[c[0] for c in CRF_CASES])
def test_reference_shim_reproduces_the_digests(ref_sha, case):
    if not os.path.exists(REF_LIB):
        pytest.skip("oracle_crf/_ref is built only where FSLIC_REFERENCE names a fast-slic checkout")
    from oracle_crf.crf import Ref
    _check_case(Ref, ref_sha, case)


def test_cases_reach_nan_and_the_clamp():
    from oracle_crf.crf import Port
    by_name = {c[0]: c for c in CRF_CASES}
    for name in ("c1_n3_t2_nan", "c3_n100_t3_raw_nan"):
        out = run_case(Port(*by_name[name][1:3]), by_name[name], energies=False)
        assert any(np.isnan(v).any() for k, v in out.items() if k.endswith("/q")), name
    out = run_case(Port(*by_name["c2_n100_t2_tiny"][1:3]), by_name["c2_n100_t2_tiny"], energies=False)
    # clamped sums: some node's q sums to well below 1 after inference
    q = out["s1/t0/q"]
    assert (q.sum(0) < 0.5).any()


def test_host_expf_clone_equals_glibc_on_every_input(ref_sha):
    """The host compile of glibc_expf.cuh equals glibc's expf on all 2^32 bit patterns, and the stream of glibc's
    outputs still hashes to the pinned digest.  About a minute."""
    import ctypes as C
    from fast_slic_b200 import crf  # binds the debug entry points
    from oracle_crf.crf import glibc_expf_range
    L = crf._L()
    h = hashlib.sha256()
    chunk = 1 << 26
    out = np.empty(chunk, np.float32)
    for first in range(0, 1 << 32, chunk):
        assert L.fslic_b200_debug_expf_host(first, chunk, out.ctypes.data_as(C.c_void_p)) == 0
        want = glibc_expf_range(first, chunk)
        bad = np.flatnonzero(out.view(np.uint32) != want.view(np.uint32))
        assert not len(bad), "expf clone differs at %d inputs, first 0x%08x" % (len(bad), first + int(bad[0]))
        h.update(out.tobytes())
    assert h.digest() == ref_sha["expf/all"]


def test_refusals_before_the_device():
    from fast_slic_b200.crf import SimpleCRF
    with pytest.raises(OverflowError):
        SimpleCRF(-1, 3)
    with pytest.raises(OverflowError):
        SimpleCRF(3, -1)
    with pytest.raises(TypeError):
        SimpleCRF(3)


def test_abi_declares_the_crf_entry_points():
    from fast_slic_b200 import _lib
    header = open(os.path.join(ROOT, "include", "fslic_b200.h")).read()
    syms = [s for s in _lib.EXPORTED_SYMBOLS if s.startswith("fslic_b200_crf_") or "expf" in s]
    assert len(syms) == 24
    for sym in syms:
        assert hasattr(_lib.lib(), sym)
        assert "int %s(" % sym in header, sym


def test_package_exports_the_crf():
    import fast_slic_b200
    from fast_slic_b200.crf import SimpleCRF, SimpleCRFFrame
    assert fast_slic_b200.SimpleCRF is SimpleCRF and fast_slic_b200.SimpleCRFFrame is SimpleCRFFrame
    src = open(os.path.join(ROOT, "fast_slic_b200", "crf.py")).read()
    assert "import oracle" not in src and "from oracle" not in src
