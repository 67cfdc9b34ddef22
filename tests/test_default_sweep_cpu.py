"""The default integer path's seeded sweep and compactness edges on the CPU: the restatement (oracle/, oracle_euclid/)
against the compiled reference's digests, the sweep's coverage, and the u16 distance limit that check_params enforces."""
import os

import numpy as np
import pytest

from cases import SWEEP_REGIONS, digest, pipeline_outputs, sweep_regions, sweep_S
from default_sweep_cases import (ARCHS, BIGSP, COLOR_MAX, DEFAULT_SWEEP_SEEDS, LIMIT_CASES, LIMIT_SHAPES, _accepts,
                                 accepted, all_cases, case_key, compactness_limit, default_sweep_case, next_float_up)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIGESTS = os.path.join(ROOT, "tests", "golden", "default_sweep_reference_digests.npz")


@pytest.fixture(scope="module")
def ref_sha():
    z = np.load(REF_DIGESTS)
    return {k: bytes(v) for k, v in zip(z["keys"].tolist(), z["sha"])}


@pytest.fixture(scope="module")
def eport():
    from oracle_euclid.euclid import Port
    return Port()


def _check_ref(ref_sha, prefix, outputs):
    want = {k[len(prefix) + 1:]: v for k, v in ref_sha.items() if k.startswith(prefix + "/")}
    got = {k: digest(v) for k, v in outputs.items()}
    assert want and set(got) == set(want), (prefix, sorted(got), sorted(want))
    bad = sorted(k for k in got if got[k] != want[k])
    assert not bad, "%s: %s differ from the compiled reference" % (prefix, bad)


PARAMS = [(f, g, c, s) for f in (0, 1) for g, c, s in all_cases(f)]


@pytest.mark.parametrize("family,group,case,seed", PARAMS, ids=[case_key(f, g, c) for f, g, c, _ in PARAMS])
def test_restatement_matches_compiled_reference(port, eport, ref_sha, family, group, case, seed):
    """Initial clusters, Lab quad image, pre-CCA and final labels and Cluster bytes of a cold and a warm call equal the
    compiled reference's in both of its arch contexts."""
    got = pipeline_outputs((port, eport)[family], case, seed, warm=True)
    for arch in ARCHS:
        _check_ref(ref_sha, "%s/%s" % (arch.replace("/", "_"), case_key(family, group, case)), got)


def test_digests_cover_every_case(ref_sha):
    """The file holds the cases of tests/default_sweep_cases.py and nothing else (a case dropped from the lists, or a
    stale file, fails here)."""
    names = ("init", "quad", "pre", "labels", "clusters", "quad2", "pre2", "labels2", "clusters2")
    want = {"%s/%s/%s" % (a.replace("/", "_"), case_key(f, g, c), n)
            for a in ARCHS for f, g, c, _ in PARAMS for n in names}
    assert set(ref_sha) == want


@pytest.mark.parametrize("family", [0, 1])
def test_sweep_reaches_every_region(family):
    """Each family's sweep has a case in every region of SWEEP_REGIONS, and only configurations the product accepts."""
    cases = [default_sweep_case(s, family) for s in DEFAULT_SWEEP_SEEDS[family]]
    reached = set().union(*[sweep_regions(c[1:]) for c in cases])
    assert not set(SWEEP_REGIONS) - reached, sorted(set(SWEEP_REGIONS) - reached)
    for c in cases:
        assert accepted(c), c


def test_limit_cases_cover_their_regions():
    """S = 1, 2, 3, about 20 and above 110; Lab on and off; every image kind; W % 8 == 0 and != 0; both compactness ends
    on every shape."""
    S = {sweep_S(*s[2:5]) for s in LIMIT_SHAPES}
    assert {1, 2, 3} <= S and any(18 <= s <= 22 for s in S) and any(s > 110 for s in S)
    assert {c[1] for c in LIMIT_CASES} == {"syn", "noise", "blocks", "flat"}
    assert {c[3] % 8 == 0 for c in LIMIT_CASES} == {True, False}
    assert {(c[-1]["convert_to_lab"], c[-1]["compactness"] == 0) for c in LIMIT_CASES} == \
        {(True, True), (True, False), (False, True), (False, False)}
    for c in LIMIT_CASES:
        assert accepted(c), c


@pytest.mark.parametrize("lab", [True, False])
@pytest.mark.parametrize("S", [1, 2, 3, 19, 20, 24, 125, 128, 1000])
def test_compactness_limit_is_the_last_accepted_float(port, S, lab):
    """compactness_limit is accepted and the next float32 above it is not; at the limit the largest spatial patch entry
    (u16)(coef * 2S) is at least 64000, so an in-window distance (spatial + colour < 766) comes within 2 of FSLIC_BIGSP;
    the limit is about 16001 with Lab on and about 32002 with Lab off, whatever S is."""
    c = compactness_limit(S, lab)
    assert _accepts(S, c, lab) and not _accepts(S, next_float_up(c), lab)
    assert abs(c - (BIGSP - COLOR_MAX) / (4.0 if lab else 2.0)) < 0.01
    lut = port.spatial_lut(S, c, 1 if lab else 0)
    assert 64000 <= int(lut.max()) < BIGSP - COLOR_MAX
    assert int(lut.max()) + COLOR_MAX - 1 >= BIGSP - 3
    assert (port.spatial_lut(S, 0.0, 1 if lab else 0) == 0).all()


def test_limit_cases_use_the_limit():
    for c in LIMIT_CASES:
        _, _, H, W, K, kw = c
        S = sweep_S(H, W, K)
        if kw["compactness"]:
            assert kw["compactness"] == compactness_limit(S, kw["convert_to_lab"])
            assert int(np.float32(kw["compactness"]).view(np.uint32)) > 0
