"""SimpleCRFGroup without a GPU: the ABI declarations of the group entry points and the checks that come before any
device work."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GROUP_SYMBOLS = ("fslic_b200_crfgroup_inference", "fslic_b200_crfdev_group_push_label_frames",
                 "fslic_b200_crfdev_group_set_proba", "fslic_b200_crfdev_group_reset_inferred",
                 "fslic_b200_crfdev_group_get_inferred", "fslic_b200_crfgroup_pop_frame")


def test_abi_declares_and_binds_the_group_entry_points():
    from fast_slic_b200 import _lib, crf
    L = crf._L()
    header = open(os.path.join(ROOT, "include", "fslic_b200.h")).read()
    declared = set(re.findall(r"\b(fslic_b200_\w+)\s*\(", header))
    for sym in GROUP_SYMBOLS:
        assert sym in declared and sym in _lib.EXPORTED_SYMBOLS, sym
        assert getattr(L, sym).argtypes is not None, sym


def test_null_and_negative_groups_are_refused():
    from fast_slic_b200 import crf
    L = crf._L()
    null_member = (C.c_void_p * 2)(None, None)
    for crfs, n in ((None, 1), (null_member, 2), (null_member, -1)):
        assert L.fslic_b200_crfgroup_inference(crfs, n, 1, None) != 0
        assert L.fslic_b200_crfdev_group_set_proba(crfs, n, None, None) != 0
        assert L.fslic_b200_crfdev_group_reset_inferred(crfs, n, None) != 0
        assert L.fslic_b200_crfdev_group_get_inferred(crfs, n, None, None) != 0
        assert L.fslic_b200_crfgroup_pop_frame(crfs, n, None) != 0
        assert L.fslic_b200_crfdev_group_push_label_frames(crfs, n, 2, 2, 1, None, None, None, 0, None, None) != 0
    assert L.fslic_b200_crfgroup_pop_frame(None, 0, None) == 0


def test_group_needs_simple_crf_members():
    from fast_slic_b200.crf import SimpleCRFGroup
    with pytest.raises(ValueError):
        SimpleCRFGroup([])
    for bad in ([object()], [1, 2], [None]):
        with pytest.raises(ValueError):
            SimpleCRFGroup(bad)
