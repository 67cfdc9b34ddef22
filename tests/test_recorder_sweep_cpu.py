"""The debug_mode recorder sweep without a GPU: its cases (tests/recorder_sweep_cases.py) against their pinned
reference digests (tests/golden/recorder_sweep_reference_digests.npz), their coverage of the parameter space, and the
compiled reference where oracle/_ref holds it."""
import hashlib
import os

import numpy as np
import pytest

from cases import SWEEP_REGIONS
from recorder_sweep_cases import (CASES, FAMILIES, LIMIT_RECORDER_CASES, REF_KIND, SWEEP_CASES, accepted, regions,
                                  reference_report)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "recorder_sweep_reference_digests.npz")


@pytest.fixture(scope="module")
def golden():
    g = np.load(GOLDEN)
    return {n: (s, int(l)) for n, s, l in zip(g["names"].tolist(), g["sha256"].tolist(), g["length"].tolist())}


def test_digests_cover_every_case(golden):
    """The file holds one digest per case and nothing else (a dropped case or a stale file fails here)."""
    names = [c.name for c in CASES]
    assert len(set(names)) == len(names)
    assert sorted(golden) == sorted(names)
    assert all(len(s) == 64 and n > 0 for s, n in golden.values())


@pytest.mark.parametrize("family", FAMILIES)
def test_family_reaches_every_region(family):
    """Each family's sweep has a case in every region of SWEEP_REGIONS, every start, and (real family) every class."""
    cases = [c for c in SWEEP_CASES if c.family == family]
    assert len(cases) == 16
    reached = set().union(*[regions(c) for c in cases])
    assert not set(SWEEP_REGIONS) - reached, sorted(set(SWEEP_REGIONS) - reached)
    assert {c.start for c in cases} == {"cold", "warm", "setter"}
    if family == "real":
        assert {(c.cls, c.manhattan) for c in cases} == {(k, m) for k in REF_KIND if k.startswith("SlicReal")
                                                        for m in (True, False)}
    if family == "preemptive":
        assert {c.manhattan for c in cases} == {True, False} and len({c.thres for c in cases}) >= 4


def test_limit_cases_cover_both_ends_and_distances():
    assert {(c.manhattan, c.compactness == 0, c.lab) for c in LIMIT_RECORDER_CASES} == \
        {(m, z, lab) for m in (True, False) for z in (True, False) for lab in (True, False)}


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_every_case_is_accepted(case):
    assert accepted(case), case


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_reference_reproduces_digest_where_built(golden, case):
    """The compiled reference (where oracle/_ref holds it) still gives the pinned bytes."""
    from oracle.recorder import RecorderRef
    if not RecorderRef.available():
        pytest.skip("oracle/_ref/libfslic_ref_recorder.so is not built (make -C oracle -f recorder.mk ref)")
    rep = reference_report(case, RecorderRef())
    assert (hashlib.sha256(rep).hexdigest(), len(rep)) == golden[case.name]
