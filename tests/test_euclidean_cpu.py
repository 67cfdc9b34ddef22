"""manhattan_spatial_dist=False (the Euclidean spatial term, context.cpp:23-40, :462-496) on the CPU: the restatement
(oracle_euclid) against the compiled reference's digests, the kernels' square root against glibc's hypotf, and the
option's effect (the Manhattan restatement, oracle/, on the same cases)."""
import os

import numpy as np
import pytest

from cases import digest
from euclid_cases import (EUCLID_ARCHS, EUCLID_CASES, EUCLID_L2_CASES, EUCLID_PREEMPT_CASES, EUCLID_PREEMPT_SWEEP,
                          EUCLID_REAL_CASES, EUCLID_REAL_SWEEP, EUCLID_SAME_CASES, EUCLID_WARM_CASE, case_id,
                          euclid_pipeline_outputs, euclid_preempt_outputs, euclid_real_outputs, preempt_case_id,
                          preempt_sweep_id, real_case_id, real_sweep_id)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIGESTS = os.path.join(ROOT, "tests", "golden", "euclid_reference_digests.npz")
ARCH_PREFIXES = ["euclid_" + a.replace("/", "_") for a in EUCLID_ARCHS]


@pytest.fixture(scope="module")
def eport():
    from oracle_euclid.euclid import Port
    return Port()


@pytest.fixture(scope="module")
def ref_sha():
    z = np.load(REF_DIGESTS)
    return {k: bytes(v) for k, v in zip(z["keys"].tolist(), z["sha"])}


def _check_ref(ref_sha, prefix, outputs):
    want = {k[len(prefix) + 1:]: v for k, v in ref_sha.items() if k.startswith(prefix + "/")}
    got = {k: digest(v) for k, v in outputs.items()}
    assert want and set(got) == set(want), (prefix, sorted(got), sorted(want))
    bad = sorted(k for k in got if got[k] != want[k])
    assert not bad, "%s: %s differ from the compiled reference" % (prefix, bad)


def _differs(a, b, skip=("init", "quad")):
    return any(digest(a[k]) != digest(b[k]) for k in a if not k.startswith(skip))


def test_hypotf_equals_the_kernels_square_root(eport):
    """The kernels replace hypotf (CUDA's is not correctly rounded) by the correctly rounded square root of the exact
    integer square sum.  glibc's hypotf, which the reference calls, agrees on every offset a context can produce:
    |di|, |dj| <= S <= 32767 (H, W <= 32767), exhaustively for the non-negative quadrant, and for both signs near 0."""
    assert eport.hypotf_mismatches(0, 32767) == 0
    assert eport.hypotf_mismatches(-1500, 1500) == 0


ALL_CASES = EUCLID_CASES + EUCLID_SAME_CASES + [("warm", EUCLID_WARM_CASE, 3)]


@pytest.mark.parametrize("group,case,seed", ALL_CASES, ids=[case_id(g, c) for g, c, _ in ALL_CASES])
def test_oracle_euclidean_matches_compiled_reference(eport, port, ref_sha, group, case, seed):
    """Slic / SlicAvx2 with manhattan_spatial_dist=False: the u16 patch (u16)(coef * hypotf(di, dj)) -- initial and
    final clusters, Lab quad image, pre-CCA and final labels equal the reference's, both arch contexts -- and the
    option changes the result (compactness 0.01 excepted: both spatial terms truncate to 0 there)."""
    got = euclid_pipeline_outputs(eport, group, case, seed)
    for top in ARCH_PREFIXES:
        _check_ref(ref_sha, "%s/%s" % (top, case_id(group, case)), got)
    manhattan = euclid_pipeline_outputs(port, group, case, seed)
    if (group, case, seed) in EUCLID_SAME_CASES:
        assert not _differs(got, manhattan)
    else:
        assert _differs(got, manhattan), "the case does not exercise the option"


@pytest.mark.parametrize("case", EUCLID_PREEMPT_CASES, ids=[preempt_case_id(c) for c in EUCLID_PREEMPT_CASES])
def test_oracle_euclidean_preemptive_matches_compiled_reference(eport, port, ref_sha, case):
    got = euclid_preempt_outputs(eport, case)
    for top in ARCH_PREFIXES:
        _check_ref(ref_sha, "%s/%s" % (top, preempt_case_id(case)), got)
    assert _differs(got, euclid_preempt_outputs(port, case)), "the case does not exercise the option"


@pytest.mark.parametrize("variant", [0, 2])
@pytest.mark.parametrize("case", EUCLID_REAL_CASES, ids=lambda c: "%s_%dx%d_K%d" % c[:4])
def test_oracle_euclidean_real_dist_matches_compiled_reference(eport, port, ref_sha, variant, case):
    """SlicRealDist (coef * hypotf, untruncated) and SlicRealDistNoQ (squared differences, fused as the reference's
    object code fuses them) with manhattan_spatial_dist=False, cold and warm start."""
    got = euclid_real_outputs(eport, variant, case)
    _check_ref(ref_sha, "euclid/" + real_case_id(variant, case), got)
    assert _differs(got, euclid_real_outputs(port, variant, case)), "the case does not exercise the option"


@pytest.mark.parametrize("seed", range(len(EUCLID_REAL_SWEEP)))
def test_oracle_euclidean_real_dist_sweep_matches_compiled_reference(eport, ref_sha, seed):
    """The seeded sweep of SlicRealDist / SlicRealDistNoQ with the flag off (tests/cases.py::sweep_config), cold and warm."""
    case, variant = EUCLID_REAL_SWEEP[seed]
    _check_ref(ref_sha, "euclid/" + real_sweep_id(seed), euclid_real_outputs(eport, variant, case))


@pytest.mark.parametrize("seed", range(len(EUCLID_PREEMPT_SWEEP)))
def test_oracle_euclidean_preemptive_sweep_matches_compiled_reference(eport, ref_sha, seed):
    got = euclid_preempt_outputs(eport, EUCLID_PREEMPT_SWEEP[seed])
    for top in ARCH_PREFIXES:
        _check_ref(ref_sha, "%s/%s" % (top, preempt_sweep_id(seed)), got)


def test_oracle_l2_variant_ignores_the_flag(port, eport, ref_sha):
    """ContextRealDistL2::set_spatial_patch does not read manhattan_spatial_dist (context.cpp:435-445): what the compiled
    reference returns with the flag off is the Manhattan restatement's output."""
    for case in EUCLID_L2_CASES:
        _check_ref(ref_sha, "euclid/" + real_case_id(1, case), euclid_real_outputs(port, 1, case))
        _check_ref(ref_sha, "euclid/" + real_case_id(1, case), euclid_real_outputs(eport, 1, case))


def test_euclidean_is_no_longer_refused():
    """Every class takes manhattan_spatial_dist=False; without a GPU the call fails for want of one, not for the option.
    `preemptive` together with a float-distance class stays refused."""
    import torch
    import fast_slic_b200 as fs
    img = np.zeros((16, 16, 3), np.uint8)
    for cls in (fs.Slic, fs.SlicRealDist, fs.SlicRealDistL2, fs.SlicRealDistNoQ):
        s = cls(num_components=4, manhattan_spatial_dist=False)
        s.slic_model._unsupported()
        if not torch.cuda.is_available():
            with pytest.raises(RuntimeError):
                s.iterate(img)
    with pytest.raises(NotImplementedError):
        fs.SlicRealDist(num_components=4, preemptive=True, manhattan_spatial_dist=False).slic_model._unsupported()


def test_abi_declares_the_setter():
    from fast_slic_b200 import _lib
    assert "fslic_b200_set_manhattan_spatial_dist" in _lib.EXPORTED_SYMBOLS
    assert hasattr(_lib.lib(), "fslic_b200_set_manhattan_spatial_dist")
