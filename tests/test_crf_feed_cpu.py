"""The CRF's device feed without a GPU: the logf clone's host compile against glibc on every input and against the
pinned digest, the ABI declarations, and the argument checks that come before any device work."""
import ctypes as C
import hashlib
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOGF_DIGESTS = os.path.join(ROOT, "tests", "golden", "logf_reference_digests.npz")
NEW_SYMBOLS = ("fslic_b200_crfdev_push_scratch_bytes", "fslic_b200_crfdev_push_label_frames",
               "fslic_b200_crfdev_set_unary", "fslic_b200_crfdev_set_proba", "fslic_b200_crfdev_set_mask",
               "fslic_b200_crfdev_get_inferred", "fslic_b200_debug_logf_host", "fslic_b200_debug_logf_device")


def test_host_logf_clone_equals_glibc_on_every_input():
    """The host compile of glibc_logf.cuh equals glibc's logf on all 2^32 bit patterns (NaN sign and payload
    included), and the stream of outputs hashes to the pinned digest.  About half a minute."""
    from fast_slic_b200 import crf
    from oracle_crf.crf import glibc_logf_range
    L = crf._L()
    z = np.load(LOGF_DIGESTS)
    want_sha = bytes(z["sha"][z["keys"].tolist().index("logf/all")])
    h = hashlib.sha256()
    chunk = 1 << 26
    out = np.empty(chunk, np.float32)
    for first in range(0, 1 << 32, chunk):
        assert L.fslic_b200_debug_logf_host(first, chunk, out.ctypes.data_as(C.c_void_p)) == 0
        want = glibc_logf_range(first, chunk)
        bad = np.flatnonzero(out.view(np.uint32) != want.view(np.uint32))
        assert not len(bad), "logf clone differs at %d inputs, first 0x%08x" % (len(bad), first + int(bad[0]))
        h.update(out.tobytes())
    assert h.digest() == want_sha


def test_logf_special_cases():
    from fast_slic_b200 import crf
    L = crf._L()
    cases = {0x00000000: 0xff800000, 0x80000000: 0xff800000, 0x3f800000: 0x00000000, 0x7f800000: 0x7f800000,
             0xff800000: 0xffc00000, 0xbf800000: 0xffc00000, 0x80000001: 0xffc00000, 0x7f800001: 0x7fc00001,
             0xffa12345: 0xffe12345, 0x7fc00000: 0x7fc00000}
    out = np.empty(1, np.float32)
    for x, want in cases.items():
        assert L.fslic_b200_debug_logf_host(x, 1, out.ctypes.data_as(C.c_void_p)) == 0
        assert int(out.view(np.uint32)[0]) == want, hex(x)
    assert L.fslic_b200_debug_logf_host(0, -1, None) != 0


def test_abi_declares_and_binds_the_feed_entry_points():
    from fast_slic_b200 import _lib, crf
    L = crf._L()
    header = open(os.path.join(ROOT, "include", "fslic_b200.h")).read()
    declared = set(re.findall(r"\b(fslic_b200_\w+)\s*\(", header))
    for sym in NEW_SYMBOLS:
        assert sym in declared and sym in _lib.EXPORTED_SYMBOLS, sym
        assert getattr(L, sym).argtypes is not None, sym  # bound: pointers and size_t must not pass as C ints
    assert L.fslic_b200_crfdev_push_scratch_bytes.restype is not None


def test_push_scratch_covers_the_graph_and_the_lists():
    from fast_slic_b200 import _lib, crf
    L = crf._L()
    g = _lib.lib().fslic_b200_connectivity_batch_scratch_bytes
    f = L.fslic_b200_crfdev_push_scratch_bytes
    for K in (1, 1600, 65535):
        for B in (1, 8):
            assert f(K, B) >= g(K, B) + B * K * 4 * 13, (K, B)
    assert f(65535, 1024) == 2 ** 64 - 1


def test_null_crf_is_refused():
    from fast_slic_b200 import crf
    L = crf._L()
    assert L.fslic_b200_crfdev_push_label_frames(None, 1, 2, 2, 1, None, None, None, 0, None, None) != 0
    for name in ("set_unary", "set_proba", "get_inferred"):
        assert getattr(L, "fslic_b200_crfdev_" + name)(None, 0, None, None) != 0
    assert L.fslic_b200_crfdev_set_mask(None, 0, None, C.c_float(1.0), None) != 0


def _unbound_crf(C_=3, N=4):
    """A SimpleCRF object without a device CRF behind it: enough to reach the argument checks, which come first."""
    from fast_slic_b200.crf import SimpleCRF
    import threading
    crf = SimpleCRF.__new__(SimpleCRF)
    crf._C, crf._N, crf.device, crf._h = C_, N, 0, None
    crf.lock = threading.RLock()
    return crf


def test_push_label_frames_refuses_host_inputs():
    crf = _unbound_crf()
    lab = np.zeros((2, 5, 6), np.int16)
    cl = np.zeros((2, 4, 32), np.uint8)
    for labels, clusters in ((lab, cl), (torch.from_numpy(lab), torch.from_numpy(cl)), (lab[0], cl[0]),
                             (lab.tolist(), cl)):
        with pytest.raises(ValueError):
            crf.push_label_frames(labels, clusters)


def test_get_inferred_out_must_be_a_cuda_tensor():
    from fast_slic_b200.crf import SimpleCRFFrame
    frame = SimpleCRFFrame(_unbound_crf(), 0)
    for out in (np.zeros((3, 4), np.float32), torch.zeros(3, 4)):
        with pytest.raises(ValueError):
            frame.get_inferred(out=out)
